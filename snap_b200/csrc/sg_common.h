// sg_common.h -- shared POD types of the device engine (index view, parameters, probability tables,
// per-worker scratch).  Plain structs: usable from nvcc device code and from host C++.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include "../../include/snapgpu.h"

#if defined(__CUDACC__)
#define SG_HD __host__ __device__ __forceinline__
#define SG_HDN __host__ __device__ __noinline__
#else
#define SG_HD inline
#define SG_HDN inline
#endif

// Lane of the calling thread within its warp on the device (all 32 lanes of a warp run one read's state machine uniformly and
// split the work inside the leaves); -1 in a host build, where the scalar forms of the leaves are used.  The aligner state
// itself is shared by the warp's lanes (one copy per warp), so the lane cannot be a member of it.
SG_HD int sg_lane()
{
#if defined(__CUDA_ARCH__)
    return (int)(threadIdx.x & 31u);
#else
    return -1;
#endif
}

#define SG_MAX_K 127                 // reference LandauVishkin.h:11
#define SG_N_PADDING 1000            // reference Genome.h:446
#define SG_MAX_MERGE_DIST 48         // reference BaseAligner.h:177 (also hashTableElementSize, :213)
#define SG_ELEM_SIZE 48
#define SG_UNUSED_SCORE 0xffffu      // BaseAligner.h:141
#define SG_SCORE_ABOVE_LIMIT (-1)    // LandauVishkin.h:14
#define SG_TOO_BIG_SCORE 65536       // LandauVishkin.h:15
#define SG_MAX_INDEL_TABLE 1200
#define SG_MAX_PERFECT_TABLE 1001
#define SG_MAPQ_LIMIT_FOR_SINGLE_HIT 10   // AlignerOptions.h:49
#define SG_VEC 8                     // AffineGapVectorized.h:18 VEC_SIZE

// The index as it lives in HBM.
struct SgIndexView {
    const uint8_t  *tables;          // all hash tables, entries back to back; table t starts at entry tableStart[t]
    const uint64_t *tableStart;      // [nTables]
    const uint64_t *tableSize;       // [nTables] slots
    const uint64_t *tableMagic;      // [nTables] floor((2^64-1)/tableSize): h % size by multiply-high (device probe path)
    const uint32_t *overflow;        // overflow table (count, hits descending ...)
    const uint8_t  *bases;           // pointer to genome location 0; [-SG_N_PADDING, nBases+SG_N_PADDING) is readable, padding is 'n'
    const int64_t  *contigStart;     // [nContigs] beginningLocation, ascending
    int64_t  nBases;                 // Genome::getCountOfBases()
    int64_t  altFirstLocation;       // genomeLocationOfFirstALTContig (LLONG_MAX if none), Genome.cpp:460-476
    uint64_t overflowSize;
    uint32_t nContigs;
    uint32_t seedLen;
    uint32_t keyBytes;               // hashTableKeySize
    uint32_t nTables;
    uint32_t large;                  // 1: two values per entry (-large)
    uint32_t entryBytes;             // 4*valueCount + keyBytes
    uint32_t chromosomePadding;
    uint32_t invalidValue;           // 0xffffffff
    // layout 1 (sg_bucket.h): sector buckets keyed by the canonical seed; `tables` etc. are then unused (NULL)
    uint32_t layout;                 // 0: the reference's tables (8 / 12-byte entries, quadratic probing); 1: 32-byte sector buckets
    uint32_t pad0;
    const uint64_t *buckets;         // [nBuckets * 4]
    uint64_t nBuckets;
    // ALT liftover (Genome::Contig::projBeginningLocation / isProjRC / projCigarOps, Genome.cpp:348-403), NULL for an index
    // without ALT contigs: projStart[c] as the Genome file gives it; projRC[c]; projOps[0, nContigs] = where contig c's ops
    // begin in projOps (absolute index; c's ops end where c+1's begin), followed by the ops, each count << 8 | action character
    const int64_t  *projStart;
    const uint8_t  *projRC;
    const uint32_t *projOps;
};
#define SG_LAYOUT_SNAP 0
#define SG_LAYOUT_BUCKET 1

// Probability / schedule tables (host-computed with the host libm so doubles are bit-identical to the reference's).
struct SgTables {
    double phred[256];                         // lv_phredToProbability, LandauVishkin.cpp:745-753
    double indel[SG_MAX_INDEL_TABLE];          // lv_indelProbabilities, :735-740
    double perfect[SG_MAX_PERFECT_TABLE];      // lv_perfectMatchProbability, :757-760
    double mapqThreshold[72];                  // mapqThreshold[m] = largest x with (int)(-10*log10(x)) >= m   (mapq.h:54)
    double snpPowSeedLen;                      // pow(1 - SNP_PROB, seedLen), BaseAligner.cpp:1314
    uint32_t wrapSeed[33];                     // GetWrappedNextSeedToTest(seedLen, w), SeedSequencer.cpp:105
};

struct SgParams {
    uint32_t maxHits, maxK, numSeedsFromCommandLine;
    double   seedCoverage;
    uint32_t minWeightToCheck, extraSearchDepth, minReadLength;
    int32_t  useAffineGap, matchReward, subPenalty, gapOpenPenalty, gapExtendPenalty, fivePrimeEndBonus, threePrimeEndBonus;
    int32_t  noUkkonen, noOrderedEvaluation, noTruncation, noEditDistance, noBandedAffineGap;
    int32_t  altAwareness, maxScoreGapToPreferNonAltAlignment, explorePopularSeeds, stopOnFirstHit;
    // derived on the host
    uint32_t numWeightLists;         // BaseAligner.cpp:173-180
    uint32_t poolSize;               // hashTableElementPoolSize, BaseAligner.cpp:183
    uint32_t tableSlots;             // power of two >= 2*poolSize (our candidate lookup table)
    uint32_t maxReadLen;             // scratch sizing bound
    int32_t  agSpecialised;          // device tuning knob (no effect on results): SgAgParams.usePacked of the single-end kernel's second pass
                                     // (+ 4: its bands of up to 32 columns take the two-unit form, SNAPGPU_SINGLE_AG_NARROW)
    uint32_t tmaMinHits;             // device tuning knob (no effect on results): hit lists of at least this many locations are staged through shared memory with bulk copies; 0 = never
};

// One candidate-table element: reference BaseAligner::HashTableElement (BaseAligner.h:223-258), compacted.
struct SgElem {
    uint64_t candidatesUsed;
    uint64_t candidatesScored;
    double   matchProbabilityForBestScore;
    int64_t  bestScoreGenomeLocation;
    uint32_t baseGenomeLocation;     // 32-bit index path: location - location % 48
    uint32_t weightNext, weightPrev; // element index, or SG_SENTINEL + weight for the list head
    uint32_t slot;                   // where this element sits in the lookup table (for O(1) clearing)
    uint32_t weight;
    uint32_t lowestPossibleScore;
    uint32_t bestScore;
    int32_t  basesClippedBefore, basesClippedAfter, agScore, seedOffset;
    uint8_t  direction, allExtantCandidatesScored, usedAffineGapScoring, pad;
    uint16_t candSeedOffset[SG_ELEM_SIZE];   // Candidate::seedOffset
};
#define SG_SENTINEL 0x80000000u

// Per-worker (per-warp) scratch arena; all pointers are device global (or host in the test build).
struct SgScratch {
    SgElem   *pool;                  // [poolSize]
    uint32_t *table;                 // [tableSlots]  element index + 1, 0 = empty
    uint32_t *listNext, *listPrev;   // [numWeightLists] list heads
    uint8_t  *rcRead, *rcQual;       // [maxReadLen]  reverse complement read / reversed quality
    uint8_t  *revRead[2];            // [maxReadLen]  reversedRead[FORWARD], reversedRead[RC]
    uint8_t  *seedUsed;              // [(maxReadLen+7)/8]
    // Landau-Vishkin
    int16_t  *lvL;                   // [(MAX_K+1)*(2*MAX_K+1)]
    uint8_t  *lvA;
    int16_t  *lvBtMatched, *lvBtD;   // [MAX_K+1]
    uint8_t  *lvBtAction;
    // affine gap
    int16_t  *agH, *agHm1, *agE;     // [agCols]
    uint8_t  *agBt[2];               // [agRows*agCols] traceback bits; [0] forward object, [1] reverse object; PERSISTENT across calls
    int16_t  *agProf;                // [5*agCols] striped query profile of the current affine-gap call (device warp forms): int16 per cell in
                                     // every form, as the reference keeps it (the packed forms pair two cells as s16x2)
    uint32_t agCols, agRows;
    uint32_t *agSnap;                // unused: an earlier narrow-band form kept its per-round H here; the SIMT emulator of the CPU suite still sets it
    // Small copies in SHARED memory (the alignment kernels set them per warp; NULL / 0 elsewhere): Landau-Vishkin needs (k+1)(2k+1)
    // cells of L and A for the k it is called with and k+1 backtrace entries -- a few hundred bytes at the usual k <= 15 -- and
    // arrays that small must not live in (and be written back to) HBM.
    int16_t  *lvLs;  uint8_t *lvAs;  uint32_t lvSmallCells;
    int16_t  *lvBtMatchedS, *lvBtDS; uint8_t *lvBtActionS; uint32_t lvBtSmall;
    // Hit-list staging (device): long overflow lists are copied into shared memory with one bulk asynchronous copy (TMA,
    // cp.async.bulk + mbarrier) per chunk instead of being read word by word from HBM.  hitStage: 16-byte aligned, hitStageWords
    // words (it is the Landau-Vishkin cell block, idle while hits are filed); hitBar: the warp's mbarrier; 0 words = off.
    uint32_t *hitStage; uint32_t hitStageWords; unsigned long long *hitBar; uint32_t hitPhase;
};

SG_HD size_t sg_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bytes of scratch one worker needs, and the carving of it.  agCols: padded pattern length; agRows: text rows.
SG_HD size_t sg_scratch_bytes(const SgParams &p)
{
    size_t agCols = sg_align_up((size_t)p.maxReadLen * 3 / 2 + 64, 64);   // banded layout needs numSeg*segLen <= 4/3*P + 7 columns
    size_t agRows = (size_t)p.maxReadLen + SG_MAX_K + 1;
    size_t b = 0;
    b += sg_align_up(sizeof(SgElem) * (size_t)p.poolSize, 256);
    b += sg_align_up(sizeof(uint32_t) * (size_t)p.tableSlots, 256);
    b += sg_align_up(sizeof(uint32_t) * 2 * (size_t)p.numWeightLists, 256);
    b += sg_align_up((size_t)p.maxReadLen + 16, 256) * 4;                 // rcRead, rcQual, revRead x2
    b += sg_align_up(((size_t)p.maxReadLen + 7) / 8 + 16, 256);
    b += sg_align_up(sizeof(int16_t) * (SG_MAX_K + 1) * (2 * SG_MAX_K + 3), 256);
    b += sg_align_up((SG_MAX_K + 1) * (2 * SG_MAX_K + 3), 256);
    b += sg_align_up(sizeof(int16_t) * (SG_MAX_K + 2), 256) * 2;
    b += sg_align_up(SG_MAX_K + 2, 256);
    b += sg_align_up(sizeof(int16_t) * agCols, 256) * 3;
    b += sg_align_up(agRows * agCols, 256) * 2;
    b += sg_align_up(10 * agCols, 256);               // agProf: five int16 rows of up to agCols cells
    return b;
}

SG_HD void sg_scratch_carve(const SgParams &p, uint8_t *base, SgScratch *s)
{
    size_t agCols = sg_align_up((size_t)p.maxReadLen * 3 / 2 + 64, 64);   // banded layout needs numSeg*segLen <= 4/3*P + 7 columns
    size_t agRows = (size_t)p.maxReadLen + SG_MAX_K + 1;
    uint8_t *q = base;
    s->pool = (SgElem *)q;            q += sg_align_up(sizeof(SgElem) * (size_t)p.poolSize, 256);
    s->table = (uint32_t *)q;         q += sg_align_up(sizeof(uint32_t) * (size_t)p.tableSlots, 256);
    s->listNext = (uint32_t *)q;      s->listPrev = s->listNext + p.numWeightLists;
                                      q += sg_align_up(sizeof(uint32_t) * 2 * (size_t)p.numWeightLists, 256);
    size_t rl = sg_align_up((size_t)p.maxReadLen + 16, 256);
    s->rcRead = q; q += rl; s->rcQual = q; q += rl; s->revRead[0] = q; q += rl; s->revRead[1] = q; q += rl;
    s->seedUsed = q;                  q += sg_align_up(((size_t)p.maxReadLen + 7) / 8 + 16, 256);
    s->lvL = (int16_t *)q;            q += sg_align_up(sizeof(int16_t) * (SG_MAX_K + 1) * (2 * SG_MAX_K + 3), 256);
    s->lvA = q;                       q += sg_align_up((SG_MAX_K + 1) * (2 * SG_MAX_K + 3), 256);
    s->lvBtMatched = (int16_t *)q;    q += sg_align_up(sizeof(int16_t) * (SG_MAX_K + 2), 256);
    s->lvBtD = (int16_t *)q;          q += sg_align_up(sizeof(int16_t) * (SG_MAX_K + 2), 256);
    s->lvBtAction = q;                q += sg_align_up(SG_MAX_K + 2, 256);
    s->agH = (int16_t *)q;            q += sg_align_up(sizeof(int16_t) * agCols, 256);
    s->agHm1 = (int16_t *)q;          q += sg_align_up(sizeof(int16_t) * agCols, 256);
    s->agE = (int16_t *)q;            q += sg_align_up(sizeof(int16_t) * agCols, 256);
    s->agBt[0] = q;                   q += sg_align_up(agRows * agCols, 256);
    s->agBt[1] = q;                   q += sg_align_up(agRows * agCols, 256);
    s->agProf = (int16_t *)q;         q += sg_align_up(10 * agCols, 256);
    s->agCols = (uint32_t)agCols;
    s->agRows = (uint32_t)agRows;
    s->agSnap = (uint32_t *)0;
    s->lvLs = (int16_t *)0; s->lvAs = (uint8_t *)0; s->lvSmallCells = 0;
    s->lvBtMatchedS = (int16_t *)0; s->lvBtDS = (int16_t *)0; s->lvBtActionS = (uint8_t *)0; s->lvBtSmall = 0;
    s->hitStage = (uint32_t *)0; s->hitStageWords = 0; s->hitBar = (unsigned long long *)0; s->hitPhase = 0;
}

// The per-warp block of shared memory behind those small copies and the four derived strings of a short read.
#ifndef SG_SMALL_LV_CELLS
#define SG_SMALL_LV_CELLS 512        // (k+1)(2k+1) <= 512  <=>  k <= 15
#endif
#define SG_SMALL_BT 32
#define SG_SMALL_READ_LEN 152
struct
#if defined(__CUDACC__)
__align__(16)
#endif
SgWarpSmall {
    int16_t lvL[SG_SMALL_LV_CELLS];      // (doubles as the hit-list staging buffer: 1024 bytes, 16-byte aligned)
    uint8_t lvA[SG_SMALL_LV_CELLS];
    int16_t btMatched[SG_SMALL_BT], btD[SG_SMALL_BT];
    uint8_t btAction[SG_SMALL_BT];
    uint8_t str[4][SG_SMALL_READ_LEN + 16];  // rcRead, rcQual, revRead[0], revRead[1] (16 bytes of slack each, like the arena's)
    uint8_t seedUsed[32];
    unsigned long long hitBar;           // mbarrier of the warp's bulk copies
};

// Per-read work counters accumulated by a worker (flushed with atomics at the end).
struct SgWork {
    uint32_t lookups, entriesProbed, overflowWords, lvCalls, agCalls, popularIgnored;
};
