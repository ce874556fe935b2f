// snapgpu.cu -- the CUDA library behind include/snapgpu.h (sm_90a).
//
// Index image in HBM, per-warp scratch arenas, the alignment kernels and the C ABI.  There is no CPU
// fallback anywhere in this file: every entry point that needs the device fails with an error when no
// usable CUDA device / kernel image is present.
#include <cuda_runtime.h>
#include <nccl.h>                    // types only: NCCL is dlopen'ed, never linked (see snapgpu_group_create)
#include <dlfcn.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <errno.h>
#include <sys/stat.h>
#include <sys/types.h>
#include <string>
#include <vector>
#include <chrono>
#include <algorithm>
#include <functional>
#include <new>

#define SG_WITH_PAIRED 1
#include "sg_align.h"
#include "sg_paired.h"
#include "sg_host.h"
#include "sg_build.cuh"
#include "sg_fastq.cuh"
#include "sg_sam.h"
#include "sg_bam.h"
#include "sg_bampost.h"
#include "sg_deflate.h"
#include "sg_samheader.h"
#include "sg_spacing.h"

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_lastError = "";

static int sg_fail(const std::string &msg)
{
    g_lastError = msg;
    return 1;
}

#define SG_CUDA(call)                                                                                     \
    do {                                                                                                  \
        cudaError_t e__ = (call);                                                                         \
        if (e__ != cudaSuccess) {                                                                         \
            return sg_fail(std::string(#call) + ": " + cudaGetErrorString(e__));                          \
        }                                                                                                 \
    } while (0)

// Multiprocessors of the current device: the grid-stride kernels get a whole number of CTAs per SM.
static int sg_sms()
{
    int device = 0, n = 0;
    if (cudaGetDevice(&device) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n < 1) {
        cudaGetLastError();
        return 1;
    }
    return n;
}

struct snapgpu_index {
    int device = 0;
    SgIndexView view;                    // device pointers
    snapgpu_index_info info;
    uint8_t  *d_tables = nullptr;        // the reference's table layout (SG_LAYOUT_SNAP); NULL for a sector-bucket index
    uint64_t *d_buckets = nullptr;       // sector buckets (SG_LAYOUT_BUCKET, sg_bucket.h)
    bool builtOnDevice = false;          // bases -> index on the device (its buckets are re-laid into the reference's tables for saving)
    uint64_t *d_tableStart = nullptr, *d_tableSize = nullptr, *d_tableMagic = nullptr;
    uint32_t *d_overflow = nullptr;
    uint8_t  *d_basesPadded = nullptr;
    int64_t  *d_contigStart = nullptr;
    int64_t  *d_projStart = nullptr;     // ALT liftover data (SgIndexView::projStart / projRC / projOps); NULL without ALT contigs
    uint8_t  *d_projRC = nullptr;
    uint32_t *d_projOps = nullptr;
    SgTables *d_tables_prob = nullptr;   // probability / schedule tables
    SgTables  h_tables_prob;
    // host-side metadata (needed to write the index back out in the reference's directory format)
    std::vector<uint64_t> h_tableStart, h_tableSize, h_tableUsed;
    std::vector<int64_t> h_contigStart;
    std::vector<std::string> h_contigName;
    std::vector<uint8_t> h_contigIsAlt;
    std::vector<int32_t> h_contigOriginal;   // originalContigNumber of each contig (Genome.h:470)
    std::vector<int64_t> h_projStart;
    std::vector<uint8_t> h_projRC;
    std::vector<uint32_t> h_projOps;
    std::vector<SgContigLine> h_contigLines; // the Genome file's contig lines (written back by snapgpu_index_save_ex)
};

struct snapgpu_aligner {
    const snapgpu_index *index = nullptr;
    SgParams params;
    snapgpu_params userParams;
    // paired-end handle (snapgpu_paired_aligner_create): `params` drives the intersecting aligner, `paramsSingle` the
    // single-end fallback aligner; a worker's arena = [single scratch | paired scratch]
    bool paired = false;
    bool twoPass = false;                // single-end: MODE 1 + MODE 2 launches of sg_align_kernel instead of one MODE 0
    SgParams paramsSingle;
    SgPairedParams pparams;
    size_t singleScratchBytes = 0;
    int *d_error = nullptr;              // latched kernel-side error code (0 = none)
    // Pairs whose candidate pools outgrow the (small) per-worker caps are queued and re-aligned from scratch by a few
    // workers that own full-size pools: second launch of the same kernel over the retry list.
    SgPairedParams pparamsBig;
    int nBigWorkers = 0;
    size_t bigScratchBytesPerWorker = 0;
    uint8_t *d_bigScratch = nullptr;
    uint32_t *d_retryList = nullptr;     // [maxUnits]
    unsigned long long *d_retryCount = nullptr, *d_next2 = nullptr;
    // staged paired launch (sg_align_paired_kernel STAGE 1 + STAGE 2): per-pair hand-off records and the pool of phase-4 candidates
    bool staged = false;
    void *d_handoff = nullptr;           // SgPairHandoff[maxUnits]
    snapgpu_paired_result *d_candPool = nullptr;
    unsigned long long candPoolCap = 0;
    unsigned long long *d_candPoolUsed = nullptr, *d_next3 = nullptr;
    int device = 0;
    int numSMs = 0;
    int warpsPerBlock = 8, blocksPerSM = 4;
    int pass1BlocksPerSM = 4;            // resident CTAs per SM of the first (no affine gap) pass of the two-pass single-end launch
    int stageBlocks[4] = {4, 8, 4, 8};   // paired staged launch: resident CTAs per SM of stage 1, 2, 3 ([0] unused)
    int nWorkers = 0;
    size_t scratchBytesPerWorker = 0;
    uint8_t *d_scratch = nullptr;
    unsigned long long *d_next = nullptr;
    cudaStream_t stream = nullptr;       // compute stream (all kernels of this aligner are serialised on it: they share the arenas)
    cudaStream_t streamIn = nullptr, streamOut = nullptr;   // H2D / D2H copy streams of the host-buffer path
    // overlapped two-pass launch (single-end): the second pass runs on stream2 while the first still produces its list
    bool overlap = false;
    int overlapPass1Blocks = 2;          // CTAs per SM of the first pass while the two run together (its 32-register build)
    int64_t overlapMinReads = 0;         // smaller batches take the sequential two-pass form (three launches and a list fill do not pay)
    cudaStream_t stream2 = nullptr;
    cudaEvent_t evFork = nullptr, evJoin = nullptr;
    unsigned int *d_producersDone = nullptr;
    int64_t maxBatchReads = 0;
    int64_t chunkReads = 0;              // reads per pipeline stage of snapgpu_align_single (the largest)
    int64_t firstChunkReads = 0;         // the first stage of a call is this small; the second takes the rest of one full stage
    size_t chunkBases = 0;
    // two pipeline slots: while the GPU aligns chunk c the host packs chunk c+1 into the other slot's pinned staging
    struct Slot {
        char *h_bases = nullptr, *h_quals = nullptr; uint64_t *h_offsets = nullptr; uint32_t *h_lens = nullptr;
        uint8_t *h_results = nullptr;        // snapgpu_single_result[] or snapgpu_paired_result[]
        char *d_bases = nullptr, *d_quals = nullptr; uint64_t *d_offsets = nullptr; uint32_t *d_lens = nullptr;
        uint8_t *d_results = nullptr;
        cudaEvent_t evIn = nullptr, evKernel = nullptr, evOut = nullptr;
        int64_t pendingFirst = -1, pendingCount = 0;    // results waiting in h_results for reads [pendingFirst, +pendingCount)
    } slot[2];
    snapgpu_counters *h_counters = nullptr, *d_counters = nullptr;
    int64_t launches = 0;
    // `-om` (snapgpu_align_single_secondary*): one raw secondary-result buffer of secRawCap records per worker, grown on demand
    snapgpu_single_result *d_secRaw = nullptr;
    int secRawCap = 0;
};

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------

// K1 (parity / roofline entry): batched lookupSeed32.  One seed per warp at a time (lanes probe the chains together), but
// SG_LOOKUP_BATCH seeds per warp are in flight: their 32 entry loads are all issued before the first one is resolved.
#ifndef SG_LOOKUP_BATCH
#define SG_LOOKUP_BATCH 2            // seeds in flight per warp; beyond two, the extra outstanding misses
#endif                              // thrash address translation rather than add DRAM throughput
#ifndef SG_LOOKUP_MB
#define SG_LOOKUP_MB 4
#endif
__global__ void __launch_bounds__(256, SG_LOOKUP_MB)
sg_lookup_kernel(SgIndexView ix, const uint8_t *seeds, long long nSeeds, uint32_t maxHitsPerSeed,
                 long long *nHits, uint32_t *hits, uint32_t *probes)
{
    const int lane = threadIdx.x & 31;
    long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nWarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long i0 = warp * SG_LOOKUP_BATCH; i0 < nSeeds; i0 += nWarps * SG_LOOKUP_BATCH) {
        uint64_t b[SG_LOOKUP_BATCH], rc[SG_LOOKUP_BATCH];
        bool ok[SG_LOOKUP_BATCH];
        SgProbeRound pr[SG_LOOKUP_BATCH];
        #pragma unroll
        for (int g = 0; g < SG_LOOKUP_BATCH; g++) {
            const long long i = i0 + g;
            ok[g] = false;
            if (i < nSeeds) {
                ok[g] = sg_warp_seed_pack(seeds + i * ix.seedLen, ix.seedLen, lane, &b[g], &rc[g]);
                if (ok[g]) sg_warp_probe_issue(ix, b[g], rc[g], lane, pr[g]);
            }
        }
        #pragma unroll
        for (int g = 0; g < SG_LOOKUP_BATCH; g++) {
            const long long i = i0 + g;
            if (i >= nSeeds) break;
            SgHits h;
            uint32_t examined = 0, ow = 0;
            h.nHits[0] = h.nHits[1] = 0; h.hits[0] = h.hits[1] = ix.overflow;
            if (ok[g]) {
                if (!sg_warp_probe_finish(ix, pr[g], b[g], rc[g], lane, &h, &examined, &ow)) {
                    examined = 0; ow = 0;
                    sg_warp_lookup_seed32(ix, b[g], rc[g], lane, &h, &examined, &ow);       // a chain longer than one round: exact slow path
                }
            }
            if (lane == 0) {
                nHits[2 * i] = h.nHits[0];
                nHits[2 * i + 1] = h.nHits[1];
                if (probes) probes[i] = examined;
            }
            if (hits) {
                for (int d = 0; d < 2; d++) {
                    uint32_t n = h.nHits[d] < maxHitsPerSeed ? h.nHits[d] : maxHitsPerSeed;
                    for (uint32_t k = lane; k < n; k += 32) hits[(2 * i + d) * (long long)maxHitsPerSeed + k] = h.hits[d][k];
                }
            }
        }
    }
}

// The same entry on a sector-bucket index (sg_bucket.h): ONE THREAD per seed -- a lookup is one 32-byte sector (two 16-byte loads of
// the same sector), there is nothing for a warp to share, and what the phase needs is as many independent sector requests in flight as
// the memory system takes (2048 threads per SM, one request each; snapgpu_measure_random_sector_rate measures the ceiling at that depth).
__global__ void __launch_bounds__(256, 8)
sg_lookup_bucket_kernel(const __grid_constant__ SgIndexView ix, const uint8_t *seeds, long long nSeeds, uint32_t maxHitsPerSeed,
                        long long *nHits, uint32_t *hits, uint32_t *probes)
{
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nSeeds; i += stride) {
        uint64_t b, rc;
        SgHits h;
        uint32_t examined = 0, ow = 0;
        h.nHits[0] = h.nHits[1] = 0; h.hits[0] = h.hits[1] = ix.overflow;
        if (sg_seed_pack(seeds + i * ix.seedLen, ix.seedLen, &b, &rc)) sg_bucket_lookup_seed32(ix, b, rc, h.nHits, h.hits, &examined, &ow);
        nHits[2 * i] = h.nHits[0];
        nHits[2 * i + 1] = h.nHits[1];
        if (probes) probes[i] = examined;
        if (hits) {
            for (int d = 0; d < 2; d++) {
                const uint32_t n = h.nHits[d] < maxHitsPerSeed ? h.nHits[d] : maxHitsPerSeed;
                for (uint32_t k = 0; k < n; k++) hits[(2 * i + d) * (long long)maxHitsPerSeed + k] = h.hits[d][k];
            }
        }
    }
}

// The alignment kernel: persistent grid, one warp per read at a time, reads handed out by an atomic counter.
// The BaseAligner state machine is inherently sequential, so all 32 lanes execute it uniformly (see sg_warp.cuh)
// and split the work inside the data-parallel leaves (hash-chain probing of both strands, ...).
// The register budget (and with it the number of resident warps per SM) is a template parameter so that the host can
// pick the occupancy that measures best: MB CTAs of 8 warps per SM.
//
// MODE 0: the whole of AlignRead for reads [0, n).
// MODE 1 / MODE 2, the two-pass form used when affine gap is on: only ~1 read in 4 ever reaches the affine-gap rescoring, yet
//   that code is most of the kernel's instruction footprint, and the kernel is bound by instruction supply (DESIGN.md).
//   MODE 1 is an instantiation without the affine-gap code: it finishes the reads that never need it and appends the others,
//   at the moment they first would, to deferList.  MODE 2 (full code) then aligns deferList[0, *deferCount) from scratch.
//   Results are those of MODE 0 by construction (a deferred read's partial work is discarded, counters included).
#define SG_DEFER_EMPTY 0xffffffffu
#define SG_OVERLAP_STARVE_NS 2000000ULL
template <int MB, int MODE>
__global__ void __launch_bounds__(256, MB)
sg_align_kernel(const __grid_constant__ SgIndexView ixParam, const __grid_constant__ SgParams prParam, const SgTables *tb, uint8_t *scratchBase,
                size_t scratchBytesPerWorker, long long n, const uint8_t *bases, const uint8_t *quals, const unsigned long long *offsets, const uint32_t *lens,
                snapgpu_single_result *results, snapgpu_counters *counters, unsigned long long *next, unsigned long long *deferCount, uint32_t *deferList,
                unsigned int *producersDone, unsigned int producerCtas, unsigned int workerBase)
{
    // Overlapped form (producerCtas != 0): the two passes run at the same time on disjoint arenas.  The first pass publishes every
    // deferred read by writing its index into a list pre-filled with SG_DEFER_EMPTY, and each of its CTAs counts itself in
    // *producersDone on exit; a warp of the second pass takes the next list position and polls it until it holds an index or every
    // producer CTA has left (then an empty position means the list ends before it).
    // producersDone[1] counts producer CTAs that have STARTED.  A consumer CTA that finds none after SG_OVERLAP_STARVE_NS leaves without
    // having taken a list position: if consumers ever filled the machine before a single producer CTA was placed, waiting would never end;
    // the consumer launch that follows the producers in stream order finishes whatever such CTAs left.
    const bool overlapped = producerCtas != 0;
    if (MODE == 1 && overlapped && threadIdx.x == 0) atomicAdd(producersDone + 1, 1u);
    if (MODE == 2 && overlapped) {
        __shared__ int sGiveUp;
        if (threadIdx.x == 0) {
            int giveUp = 0;
            unsigned long long t0 = 0, t1 = 0;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
            while (((const volatile unsigned int *)producersDone)[1] == 0u && ((const volatile unsigned int *)producersDone)[0] < producerCtas) {
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                if (t1 - t0 > SG_OVERLAP_STARVE_NS) { giveUp = 1; break; }
                __nanosleep(1000);
            }
            sGiveUp = giveUp;
            if (giveUp) atomicAdd(producersDone + 2, 1u);
        }
        __syncthreads();
        if (sGiveUp) return;
    }
    if (MODE == 2 && !overlapped) n = (long long)*deferCount;
    const int lane = threadIdx.x & 31;
    const long long worker = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) + workerBase;

    // The aligner state is the same in all 32 lanes of a warp (they run the state machine uniformly), so it lives ONCE per warp in
    // shared memory rather than 32 times in local memory: as per-thread stack it was 95 % of the kernel's L2 traffic and, with
    // tens of KB of stack per warp times thousands of resident warps, most of its DRAM traffic.
    // Every lane stores the same value to the same word; the warp is converged wherever this state is updated.
    __shared__ SgIndexView sIx;
    __shared__ SgParams sPr;
    __shared__ SgAligner sA[8];
    __shared__ snapgpu_single_result sR[8];
    __shared__ SgWarpSmall sW[8];        // small hot arrays of the warp: Landau-Vishkin cells, the derived strings of a short read
    if (threadIdx.x == 0) { sIx = ixParam; sPr = prParam; }
    __syncthreads();
    const SgIndexView &ix = sIx; const SgParams &pr = sPr;
    SgAligner &A = sA[threadIdx.x >> 5];
    snapgpu_single_result &r = sR[threadIdx.x >> 5];
    SgWarpSmall &W = sW[threadIdx.x >> 5];
    A.ix = &ix; A.pr = &pr; A.tb = tb;
    A.maxK = pr.maxK;
    A.agCands = nullptr; A.nAgCands = 0; A.maxAgCands = 0; A.agCandsOverflow = 0;
    sg_scratch_carve(pr, scratchBase + (size_t)worker * scratchBytesPerWorker, &A.sc);
    A.sc.lvLs = W.lvL; A.sc.lvAs = W.lvA; A.sc.lvSmallCells = SG_SMALL_LV_CELLS;
    A.sc.lvBtMatchedS = W.btMatched; A.sc.lvBtDS = W.btD; A.sc.lvBtActionS = W.btAction; A.sc.lvBtSmall = SG_SMALL_BT;
    A.sc.hitStage = (uint32_t *)W.lvL; A.sc.hitStageWords = SG_SMALL_LV_CELLS * 2 / 4; A.sc.hitBar = &W.hitBar; A.sc.hitPhase = 0;
    __syncwarp();
    sg_warp_hits_barrier_init(A.sc, lane);
    uint8_t *const arenaStr[5] = {A.sc.rcRead, A.sc.rcQual, A.sc.revRead[0], A.sc.revRead[1], A.sc.seedUsed};
    A.ag = sg_ag_params(pr.matchReward, pr.subPenalty, pr.gapOpenPenalty, pr.gapExtendPenalty, pr.fivePrimeEndBonus, pr.threePrimeEndBonus);
    if (MODE == 2) A.ag.usePacked = sg_ag_small_scores(A.ag, pr.maxReadLen) ? pr.agSpecialised : 0;
    A.invalidLocation = SNAPGPU_INVALID_LOCATION_32;
    A.nUsedElements = 0;         // the scratch lookup table is all-zero at creation and left clean after every read
    A.work.lookups = A.work.entriesProbed = A.work.overflowWords = A.work.lvCalls = A.work.agCalls = A.work.popularIgnored = 0;
    __syncwarp();
    unsigned long long cTotal = 0, cUseless = 0, cSingle = 0, cMulti = 0, cNotFound = 0;

    for (;;) {
        unsigned long long i = 0;
        if (lane == 0) i = atomicAdd(next, 1ULL);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (MODE == 2 && overlapped) {
            if (i >= (unsigned long long)n) break;           // (n = the batch size here: the list cannot be longer)
            // every lane polls (one broadcast transaction per load): the loop is warp-uniform, so the warp stays converged -- the state machine
            // below updates its per-warp state from all lanes at once and must never run as two groups of lanes
            unsigned int v;
            {
                const volatile uint32_t *slot = deferList + i;
                for (;;) {
                    v = *slot;
                    v = __shfl_sync(0xffffffffu, v, 0);
                    if (v != SG_DEFER_EMPTY) break;
                    unsigned int done = *(const volatile unsigned int *)producersDone;
                    done = __shfl_sync(0xffffffffu, done, 0);
                    if (done >= producerCtas) { __threadfence(); v = *slot; v = __shfl_sync(0xffffffffu, v, 0); break; }
                    __nanosleep(500);
                }
            }
            __syncwarp();
            if (v == SG_DEFER_EMPTY) break;
            i = v;
        } else {
            if (i >= (unsigned long long)n) break;
            if (MODE == 2) i = deferList[i];
        }
        const uint8_t *rd = bases + offsets[i];
        const uint8_t *rq = quals + offsets[i];
        const uint32_t len = lens[i];
        memset(&r, 0, sizeof(r));
        if (MODE != 2) cTotal++;
        uint32_t countOfNs = 0;
        #pragma unroll 1
        for (uint32_t k = lane; k < len; k += 32) countOfNs += (rd[k] == 'N');
        countOfNs = __reduce_add_sync(0xffffffffu, countOfNs);
        if (len < pr.minReadLength || countOfNs > pr.maxK || len > pr.maxReadLen) {
            // SingleAligner.cpp:213-233 (reads longer than the configured scratch bound are reported NotFound
            // with reserved = 1 so the host wrapper can raise an error)
            r.status = SNAPGPU_NOT_FOUND; r.location = A.invalidLocation; r.mapq = 0; r.direction = SNAPGPU_FORWARD;
            r.reserved = (len > pr.maxReadLen) ? 1u : 0u;
            cUseless++;
            if (lane == 0) results[i] = r;
            continue;
        }
        {
            // the four derived strings (and the seed-used bits) of a short read live in shared memory, of a longer one in the arena
            const bool shortRead = len <= SG_SMALL_READ_LEN;
            A.sc.rcRead = shortRead ? W.str[0] : arenaStr[0]; A.sc.rcQual = shortRead ? W.str[1] : arenaStr[1];
            A.sc.revRead[0] = shortRead ? W.str[2] : arenaStr[2]; A.sc.revRead[1] = shortRead ? W.str[3] : arenaStr[3];
            A.sc.seedUsed = shortRead ? W.seedUsed : arenaStr[4];
            __syncwarp();
        }
        if (MODE == 1) {
            const SgWork workBefore = A.work;
            sg_align_read_t<false, true>(A, rd, rq, len, &r);
            if (A.deferred) {
                if (lane == 0) deferList[atomicAdd(deferCount, 1ULL)] = (uint32_t)i;
                A.work = workBefore;
                continue;
            }
        } else if (MODE == 2) {
            sg_align_read_t<false, false, false, 1>(A, rd, rq, len, &r);     // (AGM 1: with the two-unit narrow-band form)
        } else {
            sg_align_read(A, rd, rq, len, &r);
        }
        if (lane == 0) results[i] = r;
        if (r.status == SNAPGPU_SINGLE_HIT) cSingle++;
        else if (r.status == SNAPGPU_MULTIPLE_HITS) cMulti++;
        else cNotFound++;
        if (lane == 0 && counters && r.status != SNAPGPU_NOT_FOUND && r.mapq >= 0 && r.mapq <= 70) {
            atomicAdd((unsigned long long *)&counters->mapqHistogram[r.mapq], 1ULL);
        }
    }
    // leave the scratch lookup table clean for the next launch
    A.clearCandidates();
    if (MODE == 1 && overlapped) {
        __threadfence();                 // this warp's list entries before its CTA's count
        __syncthreads();
        if (threadIdx.x == 0) atomicAdd(producersDone, 1u);
    }
    if (counters && lane == 0) {
        atomicAdd((unsigned long long *)&counters->totalReads, cTotal);
        atomicAdd((unsigned long long *)&counters->uselessReads, cUseless);
        atomicAdd((unsigned long long *)&counters->singleHits, cSingle);
        atomicAdd((unsigned long long *)&counters->multiHits, cMulti);
        atomicAdd((unsigned long long *)&counters->notFound, cNotFound);
        atomicAdd((unsigned long long *)&counters->nHashTableLookups, (unsigned long long)A.work.lookups);
        atomicAdd((unsigned long long *)&counters->nHashEntriesProbed, (unsigned long long)A.work.entriesProbed);
        atomicAdd((unsigned long long *)&counters->nOverflowWordsRead, (unsigned long long)A.work.overflowWords);
        atomicAdd((unsigned long long *)&counters->lvCalls, (unsigned long long)A.work.lvCalls);
        atomicAdd((unsigned long long *)&counters->affineGapCalls, (unsigned long long)A.work.agCalls);
        atomicAdd((unsigned long long *)&counters->nHitsIgnoredBecauseOfTooHighPopularity, (unsigned long long)A.work.popularIgnored);
    }
}


// `-om`: sg_align_kernel's one-launch form with the SEC instantiation of the aligner (sg_align.h): every read also leaves its secondary
// alignments.  A warp records them in its own raw buffer of secRawCap records (the reference's secondaryResults buffer) and, once
// finalizeSecondaryResults has pruned them, copies the survivors to secondary[i * secCap ...): nSecondary[i] = their number, or minus their
// number when they do not fit secCap (none copied: the caller asks again with more room).  A raw buffer that fills up latches error 4
// (the reference's AlignRead returns false there and SingleAligner.cpp:250-263 doubles the buffer; the host entry point does the same).
__global__ void __launch_bounds__(256, 4)
sg_align_secondary_kernel(const __grid_constant__ SgIndexView ixParam, const __grid_constant__ SgParams prParam, const SgTables *tb, uint8_t *scratchBase,
                          size_t scratchBytesPerWorker, long long n, const uint8_t *bases, const uint8_t *quals, const unsigned long long *offsets, const uint32_t *lens,
                          snapgpu_single_result *results, snapgpu_counters *counters, unsigned long long *next, int *error,
                          snapgpu_single_result *secRaw, int secRawCap, int secMaxEditDist, int secMaxResults, int secMaxPerContig,
                          snapgpu_single_result *secondary, long long secCap, int32_t *nSecondary)
{
    const int lane = threadIdx.x & 31;
    const long long worker = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    __shared__ SgIndexView sIx;
    __shared__ SgParams sPr;
    __shared__ SgAligner sA[8];
    __shared__ snapgpu_single_result sR[8];
    __shared__ SgWarpSmall sW[8];
    if (threadIdx.x == 0) { sIx = ixParam; sPr = prParam; }
    __syncthreads();
    const SgIndexView &ix = sIx; const SgParams &pr = sPr;
    SgAligner &A = sA[threadIdx.x >> 5];
    snapgpu_single_result &r = sR[threadIdx.x >> 5];
    SgWarpSmall &W = sW[threadIdx.x >> 5];
    A.ix = &ix; A.pr = &pr; A.tb = tb;
    A.maxK = pr.maxK;
    A.agCands = nullptr; A.nAgCands = 0; A.maxAgCands = 0; A.agCandsOverflow = 0;
    A.secResults = secRaw + (size_t)worker * (size_t)secRawCap; A.nSec = 0; A.maxSec = secRawCap; A.secOverflow = 0;
    A.secMaxEditDist = secMaxEditDist; A.secMaxResults = secMaxResults; A.secMaxPerContig = secMaxPerContig;
    sg_scratch_carve(pr, scratchBase + (size_t)worker * scratchBytesPerWorker, &A.sc);
    A.sc.lvLs = W.lvL; A.sc.lvAs = W.lvA; A.sc.lvSmallCells = SG_SMALL_LV_CELLS;
    A.sc.lvBtMatchedS = W.btMatched; A.sc.lvBtDS = W.btD; A.sc.lvBtActionS = W.btAction; A.sc.lvBtSmall = SG_SMALL_BT;
    A.sc.hitStage = (uint32_t *)W.lvL; A.sc.hitStageWords = SG_SMALL_LV_CELLS * 2 / 4; A.sc.hitBar = &W.hitBar; A.sc.hitPhase = 0;
    __syncwarp();
    sg_warp_hits_barrier_init(A.sc, lane);
    uint8_t *const arenaStr[5] = {A.sc.rcRead, A.sc.rcQual, A.sc.revRead[0], A.sc.revRead[1], A.sc.seedUsed};
    A.ag = sg_ag_params(pr.matchReward, pr.subPenalty, pr.gapOpenPenalty, pr.gapExtendPenalty, pr.fivePrimeEndBonus, pr.threePrimeEndBonus);
    A.invalidLocation = SNAPGPU_INVALID_LOCATION_32;
    A.nUsedElements = 0;
    A.work.lookups = A.work.entriesProbed = A.work.overflowWords = A.work.lvCalls = A.work.agCalls = A.work.popularIgnored = 0;
    __syncwarp();
    unsigned long long cTotal = 0, cUseless = 0, cSingle = 0, cMulti = 0, cNotFound = 0;

    for (;;) {
        unsigned long long i = 0;
        if (lane == 0) i = atomicAdd(next, 1ULL);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= (unsigned long long)n) break;
        const uint8_t *rd = bases + offsets[i];
        const uint8_t *rq = quals + offsets[i];
        const uint32_t len = lens[i];
        memset(&r, 0, sizeof(r));
        cTotal++;
        uint32_t countOfNs = 0;
        #pragma unroll 1
        for (uint32_t k = lane; k < len; k += 32) countOfNs += (rd[k] == 'N');
        countOfNs = __reduce_add_sync(0xffffffffu, countOfNs);
        if (len < pr.minReadLength || countOfNs > pr.maxK || len > pr.maxReadLen) {
            r.status = SNAPGPU_NOT_FOUND; r.location = A.invalidLocation; r.mapq = 0; r.direction = SNAPGPU_FORWARD;
            r.reserved = (len > pr.maxReadLen) ? 1u : 0u;
            cUseless++;
            if (lane == 0) { results[i] = r; nSecondary[i] = 0; }
            continue;
        }
        {
            const bool shortRead = len <= SG_SMALL_READ_LEN;
            A.sc.rcRead = shortRead ? W.str[0] : arenaStr[0]; A.sc.rcQual = shortRead ? W.str[1] : arenaStr[1];
            A.sc.revRead[0] = shortRead ? W.str[2] : arenaStr[2]; A.sc.revRead[1] = shortRead ? W.str[3] : arenaStr[3];
            A.sc.seedUsed = shortRead ? W.seedUsed : arenaStr[4];
            __syncwarp();
        }
        sg_align_read_t<false, false, true>(A, rd, rq, len, &r);
        __syncwarp();
        if (A.secOverflow) {
            if (lane == 0) { atomicCAS(error, 0, 4); results[i] = r; nSecondary[i] = 0; }
            continue;
        }
        const int nSec = A.nSec;
        if ((long long)nSec <= secCap) {
            // 88-byte records, word by word across the lanes
            const uint32_t *src = (const uint32_t *)A.secResults;
            uint32_t *dst = (uint32_t *)(secondary + (size_t)i * (size_t)secCap);
            const int words = nSec * (int)(sizeof(snapgpu_single_result) / 4);
            for (int w = lane; w < words; w += 32) dst[w] = src[w];
        }
        if (lane == 0) { results[i] = r; nSecondary[i] = ((long long)nSec <= secCap) ? nSec : -nSec; }
        __syncwarp();
        if (r.status == SNAPGPU_SINGLE_HIT) cSingle++;
        else if (r.status == SNAPGPU_MULTIPLE_HITS) cMulti++;
        else cNotFound++;
        if (lane == 0 && counters && r.status != SNAPGPU_NOT_FOUND && r.mapq >= 0 && r.mapq <= 70) {
            atomicAdd((unsigned long long *)&counters->mapqHistogram[r.mapq], 1ULL);
        }
    }
    A.clearCandidates();
    if (counters && lane == 0) {
        atomicAdd((unsigned long long *)&counters->totalReads, cTotal);
        atomicAdd((unsigned long long *)&counters->uselessReads, cUseless);
        atomicAdd((unsigned long long *)&counters->singleHits, cSingle);
        atomicAdd((unsigned long long *)&counters->multiHits, cMulti);
        atomicAdd((unsigned long long *)&counters->notFound, cNotFound);
        atomicAdd((unsigned long long *)&counters->nHashTableLookups, (unsigned long long)A.work.lookups);
        atomicAdd((unsigned long long *)&counters->nHashEntriesProbed, (unsigned long long)A.work.entriesProbed);
        atomicAdd((unsigned long long *)&counters->nOverflowWordsRead, (unsigned long long)A.work.overflowWords);
        atomicAdd((unsigned long long *)&counters->lvCalls, (unsigned long long)A.work.lvCalls);
        atomicAdd((unsigned long long *)&counters->affineGapCalls, (unsigned long long)A.work.agCalls);
        atomicAdd((unsigned long long *)&counters->nHitsIgnoredBecauseOfTooHighPopularity, (unsigned long long)A.work.popularIgnored);
    }
}


// The paired-end kernel: same execution model, one warp per PAIR.  Worker arena = single-end scratch followed by the
// paired scratch (hit sets, candidate pools, merge anchors, phase-4 candidate buffer, the second pair of affine-gap
// traceback arrays).
//
// STAGE 0: sg_paired_align() whole (also the retry pass over workList with full-size pools).
// STAGE 1 / STAGE 2, the staged launch: stage 1 runs the seed / Landau-Vishkin phases of every pair (sg_paired_align_stage1) and
//   leaves `results[i]`, the phase-4 candidate list (copied to candPool) and an SgPairHandoff record; stage 2, another launch
//   with its own instantiation, takes every unfinished pair over from there (affine-gap phase, single-end fallback).  Each
//   kernel carries only its own phases' code -- the kernels are bound by instruction supply (DESIGN.md) -- and the work of a
//   pair stays attributed to the pair (SgPairHandoff::work) so that the counters do not depend on the launch form.
struct SgPairHandoff {
    int32_t stage;                   // 0: nothing left to do (final result written, or queued for the retry pass); else sg_paired_align_stage1's return value
    int32_t nLVCand;                 // phase-4 candidates at candPool[candBase, +nLVCand)
    unsigned long long candBase;
    uint32_t work[8];                // stage 1's counters for this pair: lookups, entriesProbed, overflowWords, lvCalls, agCalls, popularIgnored, P.lvCalls, P.agCalls
};

template <int MB, int STAGE>
__global__ void __launch_bounds__(256, MB)
sg_align_paired_kernel(const __grid_constant__ SgIndexView ixParam, const __grid_constant__ SgParams prParam, const __grid_constant__ SgParams prSingleParam,
                       const __grid_constant__ SgPairedParams ppParam, const SgTables *tb, uint8_t *scratchBase,
                       size_t scratchBytesPerWorker, size_t singleScratchBytes, long long nPairs, const uint8_t *bases, const uint8_t *quals,
                       const unsigned long long *offsets, const uint32_t *lens, snapgpu_paired_result *results, snapgpu_counters *counters,
                       unsigned long long *next, int *errorWord, const uint32_t *workList, unsigned long long *retryCount, uint32_t *retryList,
                       SgPairHandoff *handoff, snapgpu_paired_result *candPool, unsigned long long candPoolCap, unsigned long long *candPoolUsed)
{
    // workList == NULL: first pass over pairs [0, nPairs), pairs that outgrow this arena's caps go to retryList.
    // workList != NULL: retry pass over workList[0, *retryCount) with full-size pools.
    if (workList) nPairs = (long long)*retryCount;
    const int lane = threadIdx.x & 31;
    const long long worker = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint8_t *arena = scratchBase + (size_t)worker * scratchBytesPerWorker;

    // warp-uniform state: one copy per warp in shared memory (see sg_align_kernel)
    __shared__ SgIndexView sIx;
    __shared__ SgParams sPr, sPrSingle;
    __shared__ SgPairedParams sPp;
    __shared__ SgAligner sS[8];
    __shared__ SgPairedAligner sP[8];
    __shared__ snapgpu_paired_result sR[8];
    if (threadIdx.x == 0) { sIx = ixParam; sPr = prParam; sPrSingle = prSingleParam; sPp = ppParam; }
    __syncthreads();
    const SgIndexView &ix = sIx; const SgParams &pr = sPr; const SgParams &prSingle = sPrSingle; const SgPairedParams &pp = sPp;
    SgAligner &S = sS[threadIdx.x >> 5];
    SgPairedAligner &P = sP[threadIdx.x >> 5];
    snapgpu_paired_result &r = sR[threadIdx.x >> 5];
    S.ix = &ix; S.pr = &prSingle; S.tb = tb;
    S.maxK = prSingle.maxK;
    S.agCands = nullptr; S.nAgCands = 0; S.maxAgCands = 0; S.agCandsOverflow = 0;
    sg_scratch_carve(prSingle, arena, &S.sc);
    S.ag = sg_ag_params(pr.matchReward, pr.subPenalty, pr.gapOpenPenalty, pr.gapExtendPenalty, pr.fivePrimeEndBonus, pr.threePrimeEndBonus);
    S.ag.usePacked = !sg_ag_small_scores(S.ag, pr.maxReadLen) ? 0 : (STAGE == 2) ? pp.stage2Packed : 1;      // `snap paired` rescoring is mostly unbanded (wide score limits): the packed form pays here
    S.invalidLocation = SNAPGPU_INVALID_LOCATION_32;
    S.nUsedElements = 0;
    S.work.lookups = S.work.entriesProbed = S.work.overflowWords = S.work.lvCalls = S.work.agCalls = S.work.popularIgnored = 0;

    P.single = &S; P.ix = &ix; P.pr = &pr; P.pp = &pp; P.tb = tb;
    sg_paired_scratch_carve(pr, pp, arena + singleScratchBytes, &P.ps);
    P.ag = S.ag; P.invalidLocation = SNAPGPU_INVALID_LOCATION_32;
    P.lvCalls = P.agCalls = 0; P.error = 0; P.maxK = (int)pr.maxK;
    unsigned long long cTotal = 0, cUseless = 0, cSingle = 0, cMulti = 0, cNotFound = 0;

    for (;;) {
        unsigned long long i = 0;
        if (lane == 0) i = atomicAdd(next, 1ULL);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= (unsigned long long)nPairs) break;
        const bool firstPass = workList == (const uint32_t *)0;
        if (!firstPass) i = workList[i];
        SgPairHandoff h;
        if (STAGE >= 2) {
            h = handoff[i];
            if (h.stage == 0) continue;
        }
        const uint8_t *rb[2], *rq[2]; uint32_t ln[2]; bool useful[2]; bool tooLong = false;
        for (int w = 0; w < 2; w++) {
            rb[w] = bases + offsets[2 * i + w]; rq[w] = quals + offsets[2 * i + w]; ln[w] = lens[2 * i + w];
            if (STAGE >= 2) continue;
            uint32_t countOfNs = 0;
            #pragma unroll 1
            for (uint32_t k = lane; k < ln[w]; k += 32) countOfNs += (rb[w][k] == 'N');
            countOfNs = __reduce_add_sync(0xffffffffu, countOfNs);
            useful[w] = ln[w] >= pr.minReadLength && countOfNs <= pr.maxK;       // PairedAligner.cpp:669-676
            tooLong = tooLong || ln[w] > pr.maxReadLen;
        }
        P.error = 0;
        const SgWork workBefore = S.work; const uint32_t lvBefore = P.lvCalls, agBefore = P.agCalls;
        int nextStage = 0;               // staged launch: the pair goes on to the next kernel with this stage value
        int nLV = 0;
        if (STAGE >= 2) {
            // take the pair over: the result so far (+ for stage 2 the derived strings and the phase-4 candidates)
            __syncwarp();
            for (uint32_t k = lane; k < sizeof(r) / 4; k += 32) ((uint32_t *)&r)[k] = ((const uint32_t *)&results[i])[k];
            if (STAGE == 2) {
                for (uint32_t k = lane; k < (uint32_t)h.nLVCand * (sizeof(r) / 4); k += 32) ((uint32_t *)P.ps.lvCandidates)[k] = ((const uint32_t *)(candPool + h.candBase))[k];
                __syncwarp();
                sg_paired_restore_reads(P, rb, rq, ln);
                nextStage = sg_paired_align_stage2<2>(P, &r, h.stage, h.nLVCand);
            } else {
                __syncwarp();
                sg_paired_align_stage3(P, rb, rq, ln, &r, h.stage);
            }
        } else {
            memset(&r, 0, sizeof(r));
            if (firstPass) cTotal += 2;
            if (tooLong) { if (lane == 0) atomicMax(errorWord, 3); useful[0] = useful[1] = false; }
            if (!useful[0] && !useful[1]) {
                r.status[0] = r.status[1] = SNAPGPU_NOT_FOUND; r.location[0] = r.location[1] = P.invalidLocation;
                cUseless += 2;
                if (lane == 0) { results[i] = r; if (STAGE == 1) handoff[i].stage = 0; }
                continue;
            }
            if (STAGE == 1) {
                nextStage = sg_paired_align_stage1(P, rb, rq, ln, &r, &nLV);
                if (STAGE == 1) { h.candBase = 0; for (int k = 0; k < 8; k++) h.work[k] = 0; }
            } else {
                sg_paired_align(P, rb, rq, ln, &r);
            }
        }
        if ((STAGE == 1 || STAGE == 2) && nextStage != 0 && !P.error) {
            // hand the pair over to the next stage's kernel; its work so far travels with it
            if (STAGE == 1 && nLV > 0) {
                unsigned long long base = 0;
                if (lane == 0) base = atomicAdd(candPoolUsed, (unsigned long long)nLV);
                base = __shfl_sync(0xffffffffu, base, 0);
                if (base + (unsigned long long)nLV > candPoolCap) P.error = 4;       // hand-off pool exhausted: the retry pass does the pair whole
                h.candBase = base;
            }
            if (!P.error) {
                __syncwarp();
                if (STAGE == 1) {
                    for (uint32_t k = lane; k < (uint32_t)nLV * (sizeof(r) / 4); k += 32) ((uint32_t *)(candPool + h.candBase))[k] = ((const uint32_t *)P.ps.lvCandidates)[k];
                }
                for (uint32_t k = lane; k < sizeof(r) / 4; k += 32) ((uint32_t *)&results[i])[k] = ((const uint32_t *)&r)[k];
                if (lane == 0) {
                    SgPairHandoff o;
                    o.stage = nextStage; o.nLVCand = nLV; o.candBase = h.candBase;
                    o.work[0] = h.work[0] + (S.work.lookups - workBefore.lookups); o.work[1] = h.work[1] + (S.work.entriesProbed - workBefore.entriesProbed);
                    o.work[2] = h.work[2] + (S.work.overflowWords - workBefore.overflowWords); o.work[3] = h.work[3] + (S.work.lvCalls - workBefore.lvCalls);
                    o.work[4] = h.work[4] + (S.work.agCalls - workBefore.agCalls); o.work[5] = h.work[5] + (S.work.popularIgnored - workBefore.popularIgnored);
                    o.work[6] = h.work[6] + (P.lvCalls - lvBefore); o.work[7] = h.work[7] + (P.agCalls - agBefore);
                    handoff[i] = o;
                }
                __syncwarp();
                S.work = workBefore; P.lvCalls = lvBefore; P.agCalls = agBefore;
                continue;
            }
        }
        if (STAGE == 1 || STAGE == 2) { if (lane == 0) handoff[i].stage = 0; }      // final here (or queued for the retry pass)
        if (P.error == 4 && firstPass) {
            // this arena's pools are too small for the pair: hand it to the retry pass (and do not count the aborted work)
            if (lane == 0) retryList[atomicAdd(retryCount, 1ULL)] = (uint32_t)i;
            S.work = workBefore; P.lvCalls = lvBefore; P.agCalls = agBefore;
            continue;
        }
        if (STAGE >= 2) {
            S.work.lookups += h.work[0]; S.work.entriesProbed += h.work[1]; S.work.overflowWords += h.work[2]; S.work.lvCalls += h.work[3];
            S.work.agCalls += h.work[4]; S.work.popularIgnored += h.work[5]; P.lvCalls += h.work[6]; P.agCalls += h.work[7];
        }
        if (P.error) {
            if (lane == 0) atomicMax(errorWord, P.error);
            memset(&r, 0, sizeof(r));
            r.status[0] = r.status[1] = SNAPGPU_NOT_FOUND; r.location[0] = r.location[1] = P.invalidLocation;
        }
        if (lane == 0) results[i] = r;
        for (int w = 0; w < 2; w++) {
            if (r.status[w] == SNAPGPU_SINGLE_HIT) cSingle++;
            else if (r.status[w] == SNAPGPU_MULTIPLE_HITS) cMulti++;
            else cNotFound++;
            if (lane == 0 && counters && r.status[w] != SNAPGPU_NOT_FOUND && r.mapq[w] >= 0 && r.mapq[w] <= 70) {
                atomicAdd((unsigned long long *)&counters->mapqHistogram[r.mapq[w]], 1ULL);
            }
        }
    }
    S.clearCandidates();
    if (counters && lane == 0) {
        atomicAdd((unsigned long long *)&counters->totalReads, cTotal);
        atomicAdd((unsigned long long *)&counters->uselessReads, cUseless);
        atomicAdd((unsigned long long *)&counters->singleHits, cSingle);
        atomicAdd((unsigned long long *)&counters->multiHits, cMulti);
        atomicAdd((unsigned long long *)&counters->notFound, cNotFound);
        atomicAdd((unsigned long long *)&counters->nHashTableLookups, (unsigned long long)S.work.lookups);
        atomicAdd((unsigned long long *)&counters->nHashEntriesProbed, (unsigned long long)S.work.entriesProbed);
        atomicAdd((unsigned long long *)&counters->nOverflowWordsRead, (unsigned long long)S.work.overflowWords);
        atomicAdd((unsigned long long *)&counters->lvCalls, (unsigned long long)S.work.lvCalls + P.lvCalls);
        atomicAdd((unsigned long long *)&counters->affineGapCalls, (unsigned long long)S.work.agCalls + P.agCalls);
        atomicAdd((unsigned long long *)&counters->nHitsIgnoredBecauseOfTooHighPopularity, (unsigned long long)S.work.popularIgnored);
    }
}

// leaf-test kernels: one job per thread, scalar leaves (the warp-cooperative forms are exercised through the
// alignment kernel and compared against these on the same inputs by the tests)
__global__ void sg_test_lv_kernel(const SgTables *tb, SgParams pr, uint8_t *scratchBase, size_t scratchBytes,
                                  const uint8_t *textBuf, const uint8_t *patBuf, const uint8_t *qualBuf,
                                  const snapgpu_lv_job *jobs, long long nJobs, snapgpu_lv_out *out)
{
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long nT = (long long)gridDim.x * blockDim.x;
    SgScratch s;
    sg_scratch_carve(pr, scratchBase + (size_t)t * scratchBytes, &s);
    for (long long j = t; j < nJobs; j += nT) {
        SgLvResult r;
        sg_lv_compute(*tb, s, jobs[j].dir, textBuf + jobs[j].textOff, jobs[j].textLen, patBuf + jobs[j].patOff, qualBuf + jobs[j].patOff,
                      jobs[j].patternLen, jobs[j].k, &r);
        out[j].score = r.score; out[j].netIndel = r.netIndel; out[j].totalIndels = r.totalIndels; out[j].textSpan = r.textSpan;
        out[j].matchProbability = r.matchProbability;
    }
}

__global__ void sg_test_ag_kernel(const SgTables *tb, SgParams pr, SgAgParams P, uint8_t *scratchBase, size_t scratchBytes,
                                  const uint8_t *textBuf, const uint8_t *patBuf, const uint8_t *qualBuf,
                                  const snapgpu_ag_job *jobs, long long nJobs, snapgpu_ag_out *out)
{
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long nT = (long long)gridDim.x * blockDim.x;
    SgScratch s;
    sg_scratch_carve(pr, scratchBase + (size_t)t * scratchBytes, &s);
    for (long long j = t; j < nJobs; j += nT) {
        SgAgResult r;
        r.agScore = -1; r.textOffset = 0; r.patternOffset = 0; r.nEdits = 0; r.matchProbability = 0.0;
        sg_ag_compute(*tb, s, P, jobs[j].dir, jobs[j].banded != 0, textBuf + jobs[j].textOff, jobs[j].textLen, patBuf + jobs[j].patOff,
                      qualBuf + jobs[j].patOff, jobs[j].patternLen, jobs[j].w, jobs[j].scoreInit, jobs[j].isRC != 0,
                      jobs[j].useClippingOptimizations != 0, &r);
        out[j].agScore = r.agScore; out[j].textOffset = r.textOffset; out[j].patternOffset = r.patternOffset; out[j].nEdits = r.nEdits;
        out[j].matchProbability = r.matchProbability;
    }
}

// warp-cooperative leaves, one job per warp; with a single warp the jobs run in order on one scratch arena, i.e. with the
// same call history as a sequential CPU run (matters for the affine-gap traceback array, see sg_ag.h)
__global__ void sg_test_lv_warp_kernel(const SgTables *tb, SgParams pr, uint8_t *scratchBase, size_t scratchBytes,
                                       const uint8_t *textBuf, const uint8_t *patBuf, const uint8_t *qualBuf,
                                       const snapgpu_lv_job *jobs, long long nJobs, snapgpu_lv_out *out)
{
    const int lane = threadIdx.x & 31;
    long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    long long nW = ((long long)gridDim.x * blockDim.x) >> 5;
    SgScratch s;
    sg_scratch_carve(pr, scratchBase + (size_t)wid * scratchBytes, &s);
    for (long long j = wid; j < nJobs; j += nW) {
        SgLvResult r;
        sg_lv_compute(*tb, s, jobs[j].dir, textBuf + jobs[j].textOff, jobs[j].textLen, patBuf + jobs[j].patOff, qualBuf + jobs[j].patOff,
                      jobs[j].patternLen, jobs[j].k, &r, lane);
        __syncwarp();
        if (lane == 0) {
            out[j].score = r.score; out[j].netIndel = r.netIndel; out[j].totalIndels = r.totalIndels; out[j].textSpan = r.textSpan;
            out[j].matchProbability = r.matchProbability;
        }
    }
}

__global__ void sg_test_ag_warp_kernel(const SgTables *tb, SgParams pr, SgAgParams P, uint8_t *scratchBase, size_t scratchBytes,
                                       const uint8_t *textBuf, const uint8_t *patBuf, const uint8_t *qualBuf,
                                       const snapgpu_ag_job *jobs, long long nJobs, snapgpu_ag_out *out)
{
    const int lane = threadIdx.x & 31;
    long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    long long nW = ((long long)gridDim.x * blockDim.x) >> 5;
    SgScratch s;
    sg_scratch_carve(pr, scratchBase + (size_t)wid * scratchBytes, &s);
    // usePacked & 4: the two-unit narrow-band form.  & 8 once put that form's per-round H in the arena instead of shared memory; the
    // looped form keeps no per-round H, so 8 now runs the same form (the tests still name both)
    for (long long j = wid; j < nJobs; j += nW) {
        SgAgResult r;
        r.agScore = -1; r.textOffset = 0; r.patternOffset = 0; r.nEdits = 0; r.matchProbability = 0.0;
        sg_warp_ag_compute<3>(*tb, s, P, jobs[j].dir, jobs[j].banded != 0, textBuf + jobs[j].textOff, jobs[j].textLen, patBuf + jobs[j].patOff,
                           qualBuf + jobs[j].patOff, jobs[j].patternLen, jobs[j].w, jobs[j].scoreInit, jobs[j].isRC != 0,
                           jobs[j].useClippingOptimizations != 0, &r, lane);
        __syncwarp();
        if (lane == 0) {
            out[j].agScore = r.agScore; out[j].textOffset = r.textOffset; out[j].patternOffset = r.patternOffset; out[j].nEdits = r.nEdits;
            out[j].matchProbability = r.matchProbability;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

const char *snapgpu_last_error(void) { return g_lastError.c_str(); }
int snapgpu_abi_version(void) { return SNAPGPU_ABI_VERSION; }

void *snapgpu_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 16) != cudaSuccess) { cudaGetLastError(); g_lastError = "snapgpu_host_alloc: cudaMallocHost failed"; return nullptr; }
    return p;
}

void snapgpu_host_free(void *p) { if (p) cudaFreeHost(p); }

int snapgpu_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

void snapgpu_params_default(snapgpu_params *p)
{
    memset(p, 0, sizeof(*p));
    p->struct_size = sizeof(*p);
    p->maxHits = 300; p->maxDist = 14; p->numSeedsFromCommandLine = 25; p->seedCoverage = 0.0;
    p->minWeightToCheck = 1; p->extraSearchDepth = 1; p->minReadLength = 50; p->useAffineGap = 1;
    p->matchReward = 1; p->subPenalty = 4; p->gapOpenPenalty = 6; p->gapExtendPenalty = 1;
    p->fivePrimeEndBonus = 10; p->threePrimeEndBonus = 7;
    p->altAwareness = 1; p->maxScoreGapToPreferNonAltAlignment = 64;
    p->maxSecondaryAlignmentAdditionalEditDistance = -1; p->ignoreAlignmentAdjustmentsForOm = 1;
}

static int require_device(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return sg_fail("no usable CUDA device: this library has no CPU fallback");
    }
    if (device < 0 || device >= n) return sg_fail("CUDA device ordinal out of range");
    SG_CUDA(cudaSetDevice(device));
    cudaFuncAttributes fa;
    e = cudaFuncGetAttributes(&fa, sg_align_kernel<2, 0>);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return sg_fail(std::string("no sm_90a kernel image usable on this device: ") + cudaGetErrorString(e));
    }
    return 0;
}

// Which layout the lookup structure gets in HBM: sector buckets (default) or the reference's own tables (SNAPGPU_INDEX_LAYOUT=snap;
// kept for probe-for-probe parity tests of GetFirstValueForKey and as the form an index is written out in).
static uint32_t wanted_layout()
{
    if (const char *e = getenv("SNAPGPU_INDEX_LAYOUT")) { if (!strcmp(e, "snap") || !strcmp(e, "0")) return SG_LAYOUT_SNAP; }
    return SG_LAYOUT_BUCKET;
}

// Sector buckets from the reference-layout tables already in HBM (ix->d_tables ...); frees those tables on success.
static int relayout_on_device(snapgpu_index *ix, size_t *hbm)
{
    SgIndexView &v = ix->view;
    if (v.keyBytes != 4 || v.seedLen < 16 || v.seedLen > 24) return 0;          // other key geometries keep the reference layout
    unsigned long long *d_count = nullptr; int *d_failed = nullptr;
    SG_CUDA(cudaMalloc((void **)&d_count, 8)); SG_CUDA(cudaMemset(d_count, 0, 8));
    SG_CUDA(cudaMalloc((void **)&d_failed, 4));
    sg_build_count_values_kernel<<<sg_sms() * 8, 256>>>(v.tables, (unsigned long long)ix->info.hashTableSlots, v.entryBytes, v.large, v.invalidValue, d_count);
    unsigned long long nEntries = 0;
    SG_CUDA(cudaMemcpy(&nEntries, d_count, 8, cudaMemcpyDeviceToHost));
    double load = sg_bucket_default_load();
    bool done = false;
    for (int attempt = 0; attempt < 4 && !done; attempt++, load *= 0.7) {
        const uint64_t nBuckets = sg_bucket_count_for(nEntries, v.seedLen, load);
        if (ix->d_buckets) { cudaFree(ix->d_buckets); ix->d_buckets = nullptr; }
        SG_CUDA(cudaMalloc((void **)&ix->d_buckets, (size_t)nBuckets * 32 + 64));
        sg_build_fill_kernel<<<sg_sms() * 8, 256>>>((unsigned long long *)ix->d_buckets, (long long)nBuckets * SG_BUCKET_SLOTS + 8, SG_BUCKET_EMPTY);
        SG_CUDA(cudaMemset(d_failed, 0, 4));
        dim3 grid(sg_sms() * 4, v.nTables < 64 ? v.nTables : 64);
        sg_build_relayout_kernel<<<grid, 256>>>(v.tables, v.tableStart, v.tableSize, v.nTables, v.entryBytes, v.large, v.keyBytes * 8, v.seedLen, v.invalidValue,
                                                (unsigned long long *)ix->d_buckets, nBuckets, d_failed);
        SG_CUDA(cudaGetLastError());
        int failed = 0;
        SG_CUDA(cudaMemcpy(&failed, d_failed, 4, cudaMemcpyDeviceToHost));
        if (!failed) { v.nBuckets = nBuckets; done = true; }
    }
    cudaFree(d_count); cudaFree(d_failed);
    if (!done) return sg_fail("bucket layout: a key landed too far from its home bucket even at low load");
    *hbm -= (size_t)ix->info.hashTableSlots * v.entryBytes;
    cudaFree(ix->d_tables); ix->d_tables = nullptr;
    v.tables = nullptr; v.layout = SG_LAYOUT_BUCKET; v.buckets = ix->d_buckets;
    *hbm += (size_t)v.nBuckets * 32;
    ix->info.hashTableSlots = v.nBuckets * SG_BUCKET_SLOTS;
    ix->info.reserved = SG_LAYOUT_BUCKET;
    return 0;
}

static int upload_index(const SgHostIndex &h, int device, snapgpu_index **out)
{
    if (require_device(device)) return 1;
    snapgpu_index *ix = new (std::nothrow) snapgpu_index;
    if (!ix) return sg_fail("out of memory");
    ix->device = device;
    size_t hbm = 0;
    #define UP(dst, src, bytes) do { size_t b__ = (bytes); if (b__ == 0) b__ = 16; SG_CUDA(cudaMalloc((void **)&(dst), b__)); \
        if ((bytes) > 0) SG_CUDA(cudaMemcpy((dst), (src), (bytes), cudaMemcpyHostToDevice)); hbm += b__; } while (0)
    UP(ix->d_tables, h.tables.data(), h.tables.size());
    UP(ix->d_tableStart, h.tableStart.data(), h.tableStart.size() * 8);
    UP(ix->d_tableSize, h.tableSize.data(), h.tableSize.size() * 8);
    UP(ix->d_tableMagic, h.tableMagic.data(), h.tableMagic.size() * 8);
    UP(ix->d_overflow, h.overflow.data(), h.overflow.size() * 4);          // (sg_load_index_directory leaves 8 words of slack: bulk copies round up to 16 bytes)
    UP(ix->d_basesPadded, h.basesPadded.data(), h.basesPadded.size());
    UP(ix->d_contigStart, h.contigStart.data(), h.contigStart.size() * 8);
    if (!h.projStart.empty()) {
        UP(ix->d_projStart, h.projStart.data(), h.projStart.size() * 8);
        UP(ix->d_projRC, h.projRC.data(), h.projRC.size());
        UP(ix->d_projOps, h.projOps.data(), h.projOps.size() * 4);
        ix->h_projStart = h.projStart; ix->h_projRC = h.projRC; ix->h_projOps = h.projOps;
    }
    sg_init_tables(ix->h_tables_prob, h.seedLen);
    UP(ix->d_tables_prob, &ix->h_tables_prob, sizeof(SgTables));
    #undef UP
    SgIndexView v = h.view();
    v.tables = ix->d_tables; v.tableStart = ix->d_tableStart; v.tableSize = ix->d_tableSize; v.tableMagic = ix->d_tableMagic; v.overflow = ix->d_overflow;
    v.bases = ix->d_basesPadded + SG_N_PADDING; v.contigStart = ix->d_contigStart;
    v.projStart = ix->d_projStart; v.projRC = ix->d_projRC; v.projOps = ix->d_projOps;
    ix->view = v;
    memset(&ix->info, 0, sizeof(ix->info));
    ix->info.countOfBases = h.nBases; ix->info.seedLen = h.seedLen; ix->info.hashTableKeySize = h.keyBytes;
    ix->info.nHashTables = h.nTables; ix->info.locationSize = 4; ix->info.largeHashTable = h.large;
    ix->info.chromosomePadding = h.chromosomePadding; ix->info.nContigs = (uint32_t)h.contigStart.size();
    ix->info.overflowTableSize = h.overflowSize; ix->info.hashTableSlots = h.totalSlots; ix->info.hbmBytes = hbm;
    ix->h_tableStart = h.tableStart; ix->h_tableSize = h.tableSize; ix->h_tableUsed = h.tableUsed;
    ix->h_contigStart = h.contigStart; ix->h_contigName = h.contigName; ix->h_contigIsAlt = h.contigIsAlt; ix->h_contigOriginal = h.contigOriginal;
    ix->h_contigLines = h.contigLines;
    ix->view.layout = SG_LAYOUT_SNAP; ix->view.pad0 = 0; ix->view.buckets = nullptr; ix->view.nBuckets = 0;
    if (wanted_layout() == SG_LAYOUT_BUCKET) {
        if (relayout_on_device(ix, &hbm)) { snapgpu_index_close(ix); return 1; }
        ix->info.hbmBytes = hbm;
    }
    *out = ix;
    return 0;
}

int snapgpu_index_open(const char *directory, int device, snapgpu_index **out)
{
    if (!directory || !out) return sg_fail("null argument");
    *out = nullptr;
    if (require_device(device)) return 1;
    SgHostIndex h;
    std::string err;
    if (!sg_load_index_directory(directory, h, err)) return sg_fail("snapgpu_index_open: " + err);
    return upload_index(h, device, out);
}

// Device memory a build or save may plan with: what cudaMemGetInfo reports as free, less a margin for the allocator and the
// driver (256 MiB + 1/64 of the device).
static int sg_usable_bytes(size_t *out)
{
    size_t freeBytes = 0, totalBytes = 0;
    SG_CUDA(cudaMemGetInfo(&freeBytes, &totalBytes));
    const size_t margin = ((size_t)256 << 20) + totalBytes / 64;
    *out = freeBytes > margin ? freeBytes - margin : 0;
    return 0;
}

// SNAPGPU_BUILD_PASSES=n: the device build and the save use at least n passes (default: as few as the free memory allows).
static uint32_t sg_min_passes()
{
    if (const char *e = getenv("SNAPGPU_BUILD_PASSES")) {
        const long long v = atoll(e);
        if (v > 1) return v > (long long)SG_BUILD_BINS ? SG_BUILD_BINS : (uint32_t)v;
    }
    return 1;
}

// Scratch of the key-range passes: keys and locations, double-buffered for the radix sort, and cub's storage.
struct SgPassScratch {
    unsigned long long *keys[2] = {nullptr, nullptr};
    uint32_t *locs[2] = {nullptr, nullptr};
    void *temp = nullptr;
    long long *nSel = nullptr;
    ~SgPassScratch() { cudaFree(keys[0]); cudaFree(keys[1]); cudaFree(locs[0]); cudaFree(locs[1]); cudaFree(temp); cudaFree(nSel); }
};

// cub storage of a pass over up to n positions (the selection runs over all nPos positions)
static int sg_pass_temp_bytes(long long nPos, long long n, uint32_t seedLen, size_t *bytes)
{
    size_t sel = 0, sort = 0;
    SgBuildPassSelect pred = {nullptr, nPos, seedLen, 0, 0};
    SG_CUDA(cub::DeviceSelect::If(nullptr, sel, thrust::make_counting_iterator<long long>(0), (uint32_t *)nullptr, (long long *)nullptr, nPos, pred));
    cub::DoubleBuffer<unsigned long long> kb(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> vb(nullptr, nullptr);
    SG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort, kb, vb, n, 0, (int)(2 * seedLen)));
    *bytes = std::max(sel, sort) + 16;
    return 0;
}

// Plans the key-range passes from the valid seeds per bin: 24 bytes per position of a pass, plus cub's storage, must fit the memory
// free now.  bounds: bin edges of the passes; *maxN: positions of the largest pass.
static int sg_plan_key_passes(const std::vector<unsigned long long> &bins, long long nPos, uint32_t seedLen, uint32_t minPasses,
                              std::vector<uint32_t> &bounds, long long *maxN)
{
    size_t usable = 0, temp = 0;
    if (sg_usable_bytes(&usable) || sg_pass_temp_bytes(nPos, nPos, seedLen, &temp)) return 1;
    std::vector<uint64_t> bytes(SG_BUILD_BINS);
    for (uint32_t b = 0; b < SG_BUILD_BINS; b++) bytes[b] = (uint64_t)bins[b] * 24;
    uint32_t bad = 0;
    if (!sg_plan_passes(bytes.data(), SG_BUILD_BINS, usable > temp ? usable - temp : 0, minPasses, bounds, &bad))
        return sg_fail("snapgpu_index_build: the seeds whose top 16 bits are " + std::to_string(bad) + " alone need " + std::to_string(bytes[bad] + temp) +
                       " bytes of sort scratch; " + std::to_string(usable) + " bytes of device memory are free");
    *maxN = 0;
    for (size_t p = 0; p + 1 < bounds.size(); p++) {
        long long n = 0;
        for (uint32_t b = bounds[p]; b < bounds[p + 1]; b++) n += (long long)bins[b];
        *maxN = std::max(*maxN, n);
    }
    return 0;
}

// Runs fn(sortedKeys, sortedLocs, n) on the positions of each key-range pass: selected in descending location order, then
// stable-sorted on the seed, so that equal seeds keep descending locations (as the single sweep leaves them).
static int sg_key_pass_sweep(const uint8_t *d_bases, long long nPos, uint32_t seedLen, const std::vector<uint32_t> &bounds, long long maxN,
                             const std::function<int(const unsigned long long *, const uint32_t *, long long)> &fn)
{
    SgPassScratch s;
    size_t tempBytes = 0;
    if (sg_pass_temp_bytes(nPos, maxN, seedLen, &tempBytes)) return 1;
    const size_t n8 = (size_t)maxN * 8 + 16, n4 = (size_t)maxN * 4 + 16;
    SG_CUDA(cudaMalloc((void **)&s.keys[0], n8)); SG_CUDA(cudaMalloc((void **)&s.keys[1], n8));
    SG_CUDA(cudaMalloc((void **)&s.locs[0], n4)); SG_CUDA(cudaMalloc((void **)&s.locs[1], n4));
    SG_CUDA(cudaMalloc(&s.temp, tempBytes)); SG_CUDA(cudaMalloc((void **)&s.nSel, 8));
    const int grid = sg_sms() * 8;
    for (size_t p = 0; p + 1 < bounds.size(); p++) {
        SgBuildPassSelect pred = {d_bases, nPos, seedLen, bounds[p], bounds[p + 1]};
        size_t tb = tempBytes;
        SG_CUDA(cub::DeviceSelect::If(s.temp, tb, thrust::make_counting_iterator<long long>(0), s.locs[0], s.nSel, nPos, pred));
        long long n = 0;
        SG_CUDA(cudaMemcpy(&n, s.nSel, 8, cudaMemcpyDeviceToHost));
        if (n > maxN) return sg_fail("snapgpu_index_build: a key-range pass selected more positions than its seeds counted");
        if (n == 0) continue;
        sg_build_pass_keys_kernel<<<grid, 256>>>(d_bases, nPos, seedLen, n, s.locs[0], s.keys[0]);
        SG_CUDA(cudaGetLastError());
        cub::DoubleBuffer<unsigned long long> kb(s.keys[0], s.keys[1]);
        cub::DoubleBuffer<uint32_t> vb(s.locs[0], s.locs[1]);
        tb = 0;
        SG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, n, 0, (int)(2 * seedLen)));
        if (tb > tempBytes) return sg_fail("snapgpu_index_build: sort storage larger than planned");
        SG_CUDA(cub::DeviceRadixSort::SortPairs(s.temp, tb, kb, vb, n, 0, (int)(2 * seedLen)));
        if (fn((const unsigned long long *)kb.Current(), (const uint32_t *)vb.Current(), n)) return 1;
    }
    SG_CUDA(cudaDeviceSynchronize());
    return 0;
}

// Device-side index construction (kernels in sg_build.cuh).  d_basesPadded: SG_N_PADDING 'n', the nBases bases,
// SG_N_PADDING 'n' -- ownership passes to the index on success.
//
// Memory: one sweep sorts every position at once, 24 bytes each, and keeps 12 of them while the final structures are allocated.
// When that does not fit the free device memory (or SNAPGPU_BUILD_PASSES asks for passes), the positions are taken in key-range
// passes (sg_build.cuh): a count sweep sizes the tables, buckets and overflow table from the exact distinct-seed counts, they are
// allocated, and an insert sweep, planned against the memory then left, fills them.  The result is the same index either way.
// `contigs`: the Genome file's contig lines; the index keeps their names, ALT flags and liftover data as snapgpu_index_open does.
static int build_index_on_device(uint8_t *d_basesPadded, int64_t nBases, const std::vector<SgContigLine> &contigs,
                                 uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out, uint32_t layout)
{
    if (seedLen < 16 || seedLen > 24) return sg_fail("snapgpu_index_build: seed length must be in [16, 24]");
    if (nBases <= (int64_t)seedLen + 2 || nBases > 0xffffffffLL - 16) return sg_fail("snapgpu_index_build: genome size unsupported for 4-byte locations");
    SgHostIndex meta;
    std::string metaErr;
    if (!sg_set_contigs(meta, contigs, metaErr)) return sg_fail("snapgpu_index_build: " + metaErr);
    for (size_t c = 0; c < contigs.size(); c++)
        if (contigs[c].start < 0 || contigs[c].start >= nBases || (c > 0 && contigs[c].start <= contigs[c - 1].start))
            return sg_fail("snapgpu_index_build: contig beginning locations must ascend within the genome");
    const uint32_t nContigs = (uint32_t)contigs.size();
    const uint32_t keyBytes = 4, keyBits = 32;
    const uint32_t nTables = 1u << ((seedLen - 16) * 2);
    const long long nPos = nBases - seedLen - 1;          // GenomeIndex.cpp:645-652: locations [0, countOfBases - seedLen - 1)
    snapgpu_index *ix = new (std::nothrow) snapgpu_index;
    if (!ix) return sg_fail("out of memory");
    ix->device = device;
    ix->d_basesPadded = d_basesPadded;
    const uint8_t *d_bases = d_basesPadded + SG_N_PADDING;

    unsigned long long *d_keys = nullptr, *d_keys2 = nullptr; uint32_t *d_locs = nullptr, *d_locs2 = nullptr;
    void *d_temp = nullptr; size_t tempBytes = 0;
    unsigned long long *d_stats = nullptr;       // [nTables] used, then overflowWords, nValid, cursor
    int *d_failed = nullptr;
    const int grid = sg_sms() * 8;
    int hist = nTables <= 4096 ? 1 : 0;
    if (const char *e = getenv("SNAPGPU_BUILD_SHARED_HIST")) hist = (atoi(e) != 0 && nTables <= 4096) ? 1 : 0;      // (test hook for the many-tables form)
    auto count = [&](const unsigned long long *k, long long n) -> int {
        sg_build_count_kernel<<<grid, 256, (size_t)((hist ? nTables : 0) + 2) * 8>>>(k, n, keyBits, seedLen, nTables, hist, d_stats, d_stats + nTables, d_stats + nTables + 1);
        SG_CUDA(cudaGetLastError());
        return 0;
    };

    // One sweep when its sort (24 bytes per position) fits, and so do the 12 bytes per position it keeps beside the final structures
    // (sized here for every position a distinct seed, at the default bucket load; the overflow table takes at most 1.5 words each).
    const uint32_t minPasses = sg_min_passes();
    bool onePass = minPasses == 1;
    if (onePass) {
        size_t usable = 0;
        if (sg_usable_bytes(&usable)) return 1;
        cub::DoubleBuffer<unsigned long long> kq(nullptr, nullptr);
        cub::DoubleBuffer<uint32_t> vq(nullptr, nullptr);
        SG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tempBytes, kq, vq, (long long)nPos, 0, (int)(2 * seedLen + 1)));
        const double finals = layout == SG_LAYOUT_BUCKET ? (double)sg_bucket_count_for((uint64_t)nPos, seedLen, sg_bucket_default_load()) * 32
                                                         : ((double)nPos * 1.3 + 101.0 * nTables) * 8;
        onePass = (double)nPos * 24 + tempBytes <= (double)usable && (double)nPos * 12 + finals + (double)nPos * 6 <= (double)usable;
    }
    std::vector<unsigned long long> bins;        // key-range passes: valid seeds per bin
    size_t countPasses = 1;
    const unsigned long long *sk = nullptr; const uint32_t *sv = nullptr;
    if (onePass) {
        SG_CUDA(cudaMalloc((void **)&d_keys, (size_t)nPos * 8)); SG_CUDA(cudaMalloc((void **)&d_keys2, (size_t)nPos * 8));
        SG_CUDA(cudaMalloc((void **)&d_locs, (size_t)nPos * 4)); SG_CUDA(cudaMalloc((void **)&d_locs2, (size_t)nPos * 4));
        sg_build_emit_kernel<<<grid, 256>>>(d_bases, nPos, seedLen, d_keys, d_locs);
        SG_CUDA(cudaGetLastError());
        cub::DoubleBuffer<unsigned long long> kb(d_keys, d_keys2);
        cub::DoubleBuffer<uint32_t> vb(d_locs, d_locs2);
        SG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tempBytes, kb, vb, (long long)nPos, 0, (int)(2 * seedLen + 1)));
        SG_CUDA(cudaMalloc(&d_temp, tempBytes + 16));
        SG_CUDA(cub::DeviceRadixSort::SortPairs(d_temp, tempBytes, kb, vb, (long long)nPos, 0, (int)(2 * seedLen + 1)));
        SG_CUDA(cudaDeviceSynchronize());
        cudaFree(d_temp);
        sk = kb.Current(); sv = vb.Current();
        cudaFree(kb.Alternate()); cudaFree(vb.Alternate());

        SG_CUDA(cudaMalloc((void **)&d_stats, (size_t)(nTables + 3) * 8));
        SG_CUDA(cudaMemset(d_stats, 0, (size_t)(nTables + 3) * 8));
        if (count(sk, nPos)) return 1;
    } else {
        // count sweep: valid seeds per bin, the passes they allow, then per pass the tables' distinct seeds and overflow words
        bins.resize(SG_BUILD_BINS);
        unsigned long long *d_bins = nullptr;
        SG_CUDA(cudaMalloc((void **)&d_bins, (size_t)SG_BUILD_BINS * 8));
        SG_CUDA(cudaMemset(d_bins, 0, (size_t)SG_BUILD_BINS * 8));
        sg_build_histogram_kernel<<<grid, 256>>>(d_bases, nPos, seedLen, d_bins);
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cudaMemcpy(bins.data(), d_bins, (size_t)SG_BUILD_BINS * 8, cudaMemcpyDeviceToHost));
        cudaFree(d_bins);
        SG_CUDA(cudaMalloc((void **)&d_stats, (size_t)(nTables + 3) * 8));
        SG_CUDA(cudaMemset(d_stats, 0, (size_t)(nTables + 3) * 8));
        std::vector<uint32_t> bounds;
        long long maxN = 0;
        if (sg_plan_key_passes(bins, nPos, seedLen, minPasses, bounds, &maxN)) { cudaFree(d_stats); return 1; }
        countPasses = bounds.size() - 1;
        if (sg_key_pass_sweep(d_bases, nPos, seedLen, bounds, maxN, [&](const unsigned long long *k, const uint32_t *, long long n) { return count(k, n); })) {
            cudaFree(d_stats); return 1;
        }
    }
    // insert sweep: the one sorted array, or key-range passes planned against the memory left once the final structures exist
    size_t insertPasses = 1;
    auto insertAll = [&](unsigned long long *tables, unsigned long long *buckets, unsigned long long nB) -> int {
        if (onePass) {
            sg_build_insert_kernel<<<grid, 256>>>(sk, sv, nPos, keyBits, seedLen, ix->d_tableStart, ix->d_tableSize, tables, ix->d_overflow, d_stats + nTables + 2,
                                                  nBases, d_failed, buckets, nB);
            SG_CUDA(cudaGetLastError());
            return 0;
        }
        std::vector<uint32_t> bounds;
        long long maxN = 0;
        if (sg_plan_key_passes(bins, nPos, seedLen, minPasses, bounds, &maxN)) return 1;
        insertPasses = bounds.size() - 1;
        return sg_key_pass_sweep(d_bases, nPos, seedLen, bounds, maxN, [&](const unsigned long long *k, const uint32_t *l, long long n) -> int {
            sg_build_insert_kernel<<<grid, 256>>>(k, l, n, keyBits, seedLen, ix->d_tableStart, ix->d_tableSize, tables, ix->d_overflow, d_stats + nTables + 2,
                                                  nBases, d_failed, buckets, nB);
            SG_CUDA(cudaGetLastError());
            return 0;
        });
    };
    std::vector<unsigned long long> stats(nTables + 3);
    SG_CUDA(cudaMemcpy(stats.data(), d_stats, (size_t)(nTables + 3) * 8, cudaMemcpyDeviceToHost));
    const unsigned long long overflowWords = stats[nTables];
    if ((unsigned long long)nBases + overflowWords > 0xfffffff0ULL) return sg_fail("snapgpu_index_build: ran out of overflow table namespace (GenomeIndex.cpp:688)");

    // table sizes: the reference sizes tables at (1 + slack) x expected content with slack 0.3 (GenomeIndex.cpp:1084-1100)
    std::vector<uint64_t> tstart(nTables), tsize(nTables), tmagic(nTables);
    uint64_t slots = 0, distinct = 0;
    for (uint32_t t = 0; t < nTables; t++) {
        const uint64_t sz = sg_table_slots(stats[t], 0.3);
        tstart[t] = slots; tsize[t] = sz; tmagic[t] = ~0ULL / sz; slots += sz;
        distinct += stats[t];
    }
    size_t hbm = 0;
    SG_CUDA(cudaMalloc((void **)&ix->d_tableStart, nTables * 8)); SG_CUDA(cudaMalloc((void **)&ix->d_tableSize, nTables * 8));
    SG_CUDA(cudaMalloc((void **)&ix->d_tableMagic, nTables * 8));
    SG_CUDA(cudaMemcpy(ix->d_tableMagic, tmagic.data(), nTables * 8, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(ix->d_tableStart, tstart.data(), nTables * 8, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(ix->d_tableSize, tsize.data(), nTables * 8, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMalloc((void **)&ix->d_overflow, (size_t)(overflowWords + 4) * 4)); hbm += (size_t)(overflowWords + 4) * 4;
    SG_CUDA(cudaMalloc((void **)&d_failed, 4));
    uint64_t nBuckets = 0;
    if (layout == SG_LAYOUT_BUCKET) {
        // sector buckets keyed by the canonical seed (sg_bucket.h): every distinct seed is one slot
        double load = sg_bucket_default_load();
        bool done = false;
        for (int attempt = 0; attempt < 4 && !done; attempt++, load *= 0.7) {
            nBuckets = sg_bucket_count_for(distinct, seedLen, load);
            if (ix->d_buckets) { cudaFree(ix->d_buckets); ix->d_buckets = nullptr; }
            SG_CUDA(cudaMalloc((void **)&ix->d_buckets, (size_t)nBuckets * 32 + 64));
            sg_build_fill_kernel<<<grid, 256>>>((unsigned long long *)ix->d_buckets, (long long)nBuckets * SG_BUCKET_SLOTS + 8, SG_BUCKET_EMPTY);
            SG_CUDA(cudaMemset(ix->d_overflow, 0, (size_t)(overflowWords + 4) * 4));
            SG_CUDA(cudaMemset(d_failed, 0, 4));
            SG_CUDA(cudaMemset(d_stats + nTables + 2, 0, 8));
            if (insertAll(nullptr, (unsigned long long *)ix->d_buckets, nBuckets)) return 1;
            int failed = 0;
            SG_CUDA(cudaMemcpy(&failed, d_failed, 4, cudaMemcpyDeviceToHost));
            done = !failed;
        }
        cudaFree((void *)sk); cudaFree((void *)sv); cudaFree(d_stats); cudaFree(d_failed);
        if (!done) return sg_fail("snapgpu_index_build: bucket layout: a key landed too far from its home bucket even at low load");
        hbm += (size_t)nBuckets * 32 + 64;
    } else {
        SG_CUDA(cudaMalloc((void **)&ix->d_tables, slots * 8 + 16)); hbm += slots * 8 + 16;
        sg_build_fill_kernel<<<grid, 256>>>((unsigned long long *)ix->d_tables, (long long)slots + 2, 0x00000000ffffffffULL);
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cudaMemset(ix->d_overflow, 0, (size_t)(overflowWords + 4) * 4));
        SG_CUDA(cudaMemset(d_failed, 0, 4));
        if (insertAll((unsigned long long *)ix->d_tables, nullptr, 0)) return 1;
        int failed = 0;
        SG_CUDA(cudaMemcpy(&failed, d_failed, 4, cudaMemcpyDeviceToHost));
        cudaFree((void *)sk); cudaFree((void *)sv); cudaFree(d_stats); cudaFree(d_failed);
        if (failed) return sg_fail("snapgpu_index_build: hash table overflow during insertion");
    }
    if (!onePass && minPasses == 1)            // passes the free memory called for (not asked for): say so once
        fprintf(stderr, "snapgpu_index_build: the sort did not fit the free device memory at once: %zu key-range passes to count, %zu to insert\n",
                countPasses, insertPasses);

    SG_CUDA(cudaMalloc((void **)&ix->d_contigStart, (size_t)nContigs * 8 + 16));
    SG_CUDA(cudaMemcpy(ix->d_contigStart, meta.contigStart.data(), (size_t)nContigs * 8, cudaMemcpyHostToDevice));
    if (!meta.projStart.empty()) {             // ALT liftover arrays, as upload_index places them
        SG_CUDA(cudaMalloc((void **)&ix->d_projStart, meta.projStart.size() * 8));
        SG_CUDA(cudaMemcpy(ix->d_projStart, meta.projStart.data(), meta.projStart.size() * 8, cudaMemcpyHostToDevice));
        SG_CUDA(cudaMalloc((void **)&ix->d_projRC, meta.projRC.size() + 16));
        SG_CUDA(cudaMemcpy(ix->d_projRC, meta.projRC.data(), meta.projRC.size(), cudaMemcpyHostToDevice));
        SG_CUDA(cudaMalloc((void **)&ix->d_projOps, meta.projOps.size() * 4));
        SG_CUDA(cudaMemcpy(ix->d_projOps, meta.projOps.data(), meta.projOps.size() * 4, cudaMemcpyHostToDevice));
        hbm += meta.projStart.size() * 8 + meta.projRC.size() + 16 + meta.projOps.size() * 4;
    }
    sg_init_tables(ix->h_tables_prob, seedLen);
    SG_CUDA(cudaMalloc((void **)&ix->d_tables_prob, sizeof(SgTables)));
    SG_CUDA(cudaMemcpy(ix->d_tables_prob, &ix->h_tables_prob, sizeof(SgTables), cudaMemcpyHostToDevice));
    hbm += (size_t)nBases + 2 * SG_N_PADDING;

    SgIndexView v;
    memset(&v, 0, sizeof(v));
    v.tables = ix->d_tables; v.tableStart = ix->d_tableStart; v.tableSize = ix->d_tableSize; v.tableMagic = ix->d_tableMagic; v.overflow = ix->d_overflow;
    v.bases = d_bases; v.contigStart = ix->d_contigStart; v.nBases = nBases; v.altFirstLocation = meta.altFirstLocation;
    v.projStart = ix->d_projStart; v.projRC = ix->d_projRC; v.projOps = ix->d_projOps;
    v.overflowSize = overflowWords; v.nContigs = nContigs; v.seedLen = seedLen; v.keyBytes = keyBytes; v.nTables = nTables;
    v.large = 0; v.entryBytes = 8; v.chromosomePadding = chromosomePadding; v.invalidValue = 0xffffffffu;
    v.layout = layout; v.pad0 = 0; v.buckets = ix->d_buckets; v.nBuckets = nBuckets;
    ix->view = v;
    ix->builtOnDevice = true;
    memset(&ix->info, 0, sizeof(ix->info));
    ix->info.countOfBases = nBases; ix->info.seedLen = seedLen; ix->info.hashTableKeySize = keyBytes; ix->info.nHashTables = nTables;
    ix->info.locationSize = 4; ix->info.largeHashTable = 0; ix->info.chromosomePadding = chromosomePadding; ix->info.nContigs = nContigs;
    ix->info.overflowTableSize = overflowWords; ix->info.hashTableSlots = layout == SG_LAYOUT_BUCKET ? nBuckets * SG_BUCKET_SLOTS : slots; ix->info.hbmBytes = hbm;
    ix->info.reserved = layout;
    ix->h_tableStart = tstart; ix->h_tableSize = tsize;
    ix->h_tableUsed.assign(stats.begin(), stats.begin() + nTables);
    ix->h_contigStart = meta.contigStart; ix->h_contigName = meta.contigName; ix->h_contigIsAlt = meta.contigIsAlt; ix->h_contigOriginal = meta.contigOriginal;
    ix->h_projStart = meta.projStart; ix->h_projRC = meta.projRC; ix->h_projOps = meta.projOps;
    ix->h_contigLines = contigs;
    *out = ix;
    return 0;
}

// The contig lines an index built from bases and contig starts alone gets: contigs chr1..chrN, none ALT, no liftover.
static std::vector<SgContigLine> plain_contigs(const int64_t *contigStarts, uint32_t nContigs)
{
    std::vector<SgContigLine> lines(nContigs);
    for (uint32_t c = 0; c < nContigs; c++) { lines[c].start = contigStarts[c]; lines[c].original = (int32_t)c; lines[c].name = "chr" + std::to_string(c + 1); }
    return lines;
}

// snapgpu_contig descriptors -> the Genome file's contig lines, checked: names present, beginning locations ascending inside the genome
static int described_contigs(const snapgpu_contig *contigs, uint32_t nContigs, int64_t nBases, std::vector<SgContigLine> &lines)
{
    lines.assign(nContigs, SgContigLine());
    for (uint32_t c = 0; c < nContigs; c++) {
        const snapgpu_contig &d = contigs[c];
        if (!d.name) return sg_fail("snapgpu_index_build_genome: contig " + std::to_string(c) + " has no name");
        if (d.beginningLocation < 0 || d.beginningLocation >= nBases || (c > 0 && d.beginningLocation <= contigs[c - 1].beginningLocation))
            return sg_fail("snapgpu_index_build_genome: contig beginning locations must ascend within the genome (contig " + std::to_string(c) + ")");
        SgContigLine &L = lines[c];
        L.start = d.beginningLocation; L.flags = d.isAlt ? 1u : 0u; L.original = d.originalContigNumber;
        L.projStart = d.projBeginningLocation; L.projFlags = d.projIsRC ? 1u : 0u;
        L.name = d.name;
        L.projCigar = d.projCigar ? d.projCigar : "*";
    }
    return 0;
}

// Copies the nBases bases (host or device memory) between SG_N_PADDING 'n' on each side, then builds; the padded copy passes to
// the index.
static int build_from(const char *bases, bool onDevice, int64_t nBases, const std::vector<SgContigLine> &contigs, uint32_t seedLen,
                      uint32_t chromosomePadding, int device, snapgpu_index **out)
{
    if (require_device(device)) return 1;
    if (nBases <= 0) return sg_fail("snapgpu_index_build: empty genome");
    uint8_t *d_padded = nullptr;
    SG_CUDA(cudaMalloc((void **)&d_padded, (size_t)nBases + 2 * SG_N_PADDING));
    SG_CUDA(cudaMemset(d_padded, 'n', (size_t)nBases + 2 * SG_N_PADDING));
    SG_CUDA(cudaMemcpy(d_padded + SG_N_PADDING, bases, (size_t)nBases, onDevice ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    int rc = build_index_on_device(d_padded, nBases, contigs, seedLen, chromosomePadding, device, out, wanted_layout());
    if (rc) cudaFree(d_padded);
    return rc;
}

int snapgpu_index_build(const char *bases, int64_t nBases, const int64_t *contigStarts, uint32_t nContigs,
                        uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out)
{
    if (!bases || !contigStarts || !out || nContigs == 0) return sg_fail("null argument");
    *out = nullptr;
    return build_from(bases, false, nBases, plain_contigs(contigStarts, nContigs), seedLen, chromosomePadding, device, out);
}

// Same, from bases already in HBM (d_bases: nBases bytes, device pointer); copies them into the index image.
int snapgpu_index_build_device(const char *d_bases, int64_t nBases, const int64_t *contigStarts, uint32_t nContigs,
                               uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out)
{
    if (!d_bases || !contigStarts || !out || nContigs == 0) return sg_fail("null argument");
    *out = nullptr;
    return build_from(d_bases, true, nBases, plain_contigs(contigStarts, nContigs), seedLen, chromosomePadding, device, out);
}

int snapgpu_index_build_genome(const char *bases, int64_t nBases, const snapgpu_contig *contigs, uint32_t nContigs,
                               uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out)
{
    if (!bases || !contigs || !out || nContigs == 0) return sg_fail("null argument");
    *out = nullptr;
    std::vector<SgContigLine> lines;
    if (described_contigs(contigs, nContigs, nBases, lines)) return 1;
    return build_from(bases, false, nBases, lines, seedLen, chromosomePadding, device, out);
}

int snapgpu_index_build_genome_device(const char *d_bases, int64_t nBases, const snapgpu_contig *contigs, uint32_t nContigs,
                                      uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out)
{
    if (!d_bases || !contigs || !out || nContigs == 0) return sg_fail("null argument");
    *out = nullptr;
    std::vector<SgContigLine> lines;
    if (described_contigs(contigs, nContigs, nBases, lines)) return 1;
    return build_from(d_bases, true, nBases, lines, seedLen, chromosomePadding, device, out);
}

// Writes the index out in the reference's own 4-file directory format (v7.1: GenomeIndex.cpp:1007-1008 header,
// HashTable.cpp:199-260 table headers, GenomeIndex.cpp:964-988 overflow, Genome.cpp:203-253 genome), so that the
// stock `snap-aligner` can load an index built by snapgpu_index_build, in the table geometry `o` asks for.
int snapgpu_index_save_ex(const snapgpu_index *ix, const char *directory, const snapgpu_save_options *o)
{
    if (!ix || !directory || !o) return sg_fail("null argument");
    if (o->struct_size != sizeof(snapgpu_save_options)) return sg_fail("snapgpu_save_options.struct_size mismatch (ABI)");
    const uint32_t seedLen = ix->view.seedLen, kb = o->keyBytes, large = o->large ? 1u : 0u;
    const double slack = o->slack;
    const bool relay = ix->view.layout == SG_LAYOUT_BUCKET;
    if ((relay || !(kb == 4 && !large && slack == 0.3)) && !sg_relay_geometry_ok(seedLen, kb))
        return sg_fail("snapgpu_index_save_ex: a " + std::to_string(kb) + "-byte key does not suit seed length " + std::to_string(seedLen) +
                       " (the seed must fill the key and leave at most 16 bits of table number: 2*seedLen >= 8*keyBytes and 2*seedLen - 8*keyBytes <= 16)");
    if (!(slack > 0.0 && slack <= 100.0)) return sg_fail("snapgpu_index_save_ex: slack must be positive (the reference's default is 0.3)");
    const bool defaults = kb == 4 && !large && slack == 0.3;
    SG_CUDA(cudaSetDevice(ix->device));
    // The reference's directory format holds the reference's tables.  An index built on the device in sector buckets has them
    // re-laid from its buckets in the requested geometry: entries per table counted (sg_relay_count_kernel) and tables sized from
    // the counts, then one range of tables at a time, in staging buffers that fit the free device memory, inserted
    // (sg_relay_insert_kernel), packed to the file's entry stride and written out in table order; its overflow table is written as it
    // is.  An index in the reference's layout writes its own tables.
    uint32_t nT = ix->view.nTables, keyBytes = ix->view.keyBytes, isLarge = ix->view.large;
    std::vector<uint64_t> tstart = ix->h_tableStart, tsize = ix->h_tableSize, tused = ix->h_tableUsed;
    std::vector<uint32_t> ranges = {0, nT};
    uint64_t rangeSlots = 0;
    uint32_t stageBytes = 0, fileBytes = 0;
    struct DeviceBuffers {
        uint8_t *stage = nullptr, *packed = nullptr; uint64_t *tableStart = nullptr, *tableSize = nullptr; unsigned long long *used = nullptr; int *failed = nullptr;
        ~DeviceBuffers() { cudaFree(stage); cudaFree(packed); cudaFree(tableStart); cudaFree(tableSize); cudaFree(used); cudaFree(failed); }
    } dev;
    if (relay) {
        if (!ix->builtOnDevice) return sg_fail("snapgpu_index_save: this index was loaded from a reference-format directory (copy that), or open it with SNAPGPU_INDEX_LAYOUT=snap");
        nT = 1u << (2 * seedLen - 8 * kb); keyBytes = kb; isLarge = large;
        stageBytes = sg_relay_stage_bytes(kb, large); fileBytes = sg_relay_file_bytes(kb, large);
        const int grid = sg_sms() * 8;
        SG_CUDA(cudaMalloc((void **)&dev.used, (size_t)nT * 8)); SG_CUDA(cudaMemset(dev.used, 0, (size_t)nT * 8));
        SG_CUDA(cudaMalloc((void **)&dev.failed, 4)); SG_CUDA(cudaMemset(dev.failed, 0, 4));
        sg_relay_count_kernel<<<grid, 256>>>((const unsigned long long *)ix->d_buckets, ix->view.nBuckets, seedLen, kb, large, nT, dev.used, dev.failed);
        SG_CUDA(cudaGetLastError());
        tused.assign(nT, 0);
        int failed = 0;
        SG_CUDA(cudaMemcpy(tused.data(), dev.used, (size_t)nT * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(&failed, dev.failed, 4, cudaMemcpyDeviceToHost));
        if (failed) return sg_fail("snapgpu_index_save: a bucket slot is out of reach of its home bucket");
        tstart.assign(nT, 0); tsize.assign(nT, 0);
        uint64_t slots = 0;
        for (uint32_t t = 0; t < nT; t++) { tsize[t] = sg_table_slots(tused[t], slack); tstart[t] = slots; slots += tsize[t]; }
        SG_CUDA(cudaMalloc((void **)&dev.tableStart, (size_t)nT * 8)); SG_CUDA(cudaMalloc((void **)&dev.tableSize, (size_t)nT * 8));
        SG_CUDA(cudaMemcpy(dev.tableStart, tstart.data(), (size_t)nT * 8, cudaMemcpyHostToDevice));
        SG_CUDA(cudaMemcpy(dev.tableSize, tsize.data(), (size_t)nT * 8, cudaMemcpyHostToDevice));
        // a range's device bytes per slot: the staging form, and the packed entries when their stride differs from it
        const uint32_t perSlot = stageBytes + (fileBytes != stageBytes ? fileBytes : 0);
        const uint32_t minPasses = sg_min_passes();
        size_t usable = 0;
        if (sg_usable_bytes(&usable)) return 1;
        std::vector<uint64_t> bytes(nT);
        for (uint32_t t = 0; t < nT; t++) bytes[t] = tsize[t] * perSlot;
        uint32_t bad = 0;
        if (!sg_plan_passes(bytes.data(), nT, usable > 64 ? usable - 64 : 0, minPasses, ranges, &bad))
            return sg_fail("snapgpu_index_save: hash table " + std::to_string(bad) + " alone needs " + std::to_string(bytes[bad]) + " bytes of device memory to be re-laid; " +
                           std::to_string(usable) + " bytes are free" + (nT == 1 ? " (this geometry has a single table)" : ""));
        for (size_t p = 0; p + 1 < ranges.size(); p++)
            rangeSlots = std::max<uint64_t>(rangeSlots, tstart[ranges[p + 1] - 1] + tsize[ranges[p + 1] - 1] - tstart[ranges[p]]);
        SG_CUDA(cudaMalloc((void **)&dev.stage, (size_t)rangeSlots * stageBytes + 16));
        if (fileBytes != stageBytes) SG_CUDA(cudaMalloc((void **)&dev.packed, (size_t)rangeSlots * fileBytes + 16));
        if (ranges.size() > 2 && minPasses == 1)
            fprintf(stderr, "snapgpu_index_save: the tables did not fit the free device memory at once: %zu table-range passes\n", ranges.size() - 1);
    } else {
        if (!defaults)
            return sg_fail(std::string("snapgpu_index_save_ex: an index in the reference's table layout (") +
                           (ix->builtOnDevice ? "built on the device with SNAPGPU_INDEX_LAYOUT=snap" : "opened from a directory") +
                           ") saves only with the default options: 4-byte keys, default tables, slack 0.3");
        if (ix->view.keyBytes != 4 || (ix->view.entryBytes != 8 && ix->view.entryBytes != 12))
            return sg_fail("snapgpu_index_save: unsupported entry geometry (only 4-byte keys: the image of other seed lengths is re-strided, see sg_load_index_directory)");
    }
    std::string dir(directory);
    {
        // mkdir -p without a shell (a directory name is data, not a command line)
        for (size_t p = 1; p <= dir.size(); p++) {
            if (p == dir.size() || dir[p] == '/') {
                const std::string part = dir.substr(0, p);
                if (mkdir(part.c_str(), 0777) != 0 && errno != EEXIST) return sg_fail("snapgpu_index_save: cannot create directory " + part);
            }
        }
        struct stat sb;
        if (stat(dir.c_str(), &sb) != 0 || !S_ISDIR(sb.st_mode)) return sg_fail("snapgpu_index_save: not a directory: " + dir);
    }
    const size_t CH = (size_t)256 << 20;
    std::vector<uint8_t> buf(CH);
    // Genome
    {
        FILE *f = fopen((dir + "/Genome").c_str(), "wb");
        if (!f) return sg_fail("snapgpu_index_save: cannot write Genome");
        const std::string head = sg_genome_file_header(ix->view.nBases, ix->h_contigLines);
        if (fwrite(head.data(), 1, head.size(), f) != head.size()) { fclose(f); return sg_fail("snapgpu_index_save: short write"); }
        for (size_t off = 0; off < (size_t)ix->view.nBases; off += CH) {
            size_t m = (size_t)ix->view.nBases - off < CH ? (size_t)ix->view.nBases - off : CH;
            SG_CUDA(cudaMemcpy(buf.data(), ix->view.bases + off, m, cudaMemcpyDeviceToHost));
            if (fwrite(buf.data(), 1, m, f) != m) { fclose(f); return sg_fail("snapgpu_index_save: short write"); }
        }
        fclose(f);
    }
    // OverflowTable
    {
        FILE *f = fopen((dir + "/OverflowTable").c_str(), "wb");
        if (!f) return sg_fail("snapgpu_index_save: cannot write OverflowTable");
        size_t total = (size_t)ix->view.overflowSize * 4;
        for (size_t off = 0; off < total; off += CH) {
            size_t m = total - off < CH ? total - off : CH;
            SG_CUDA(cudaMemcpy(buf.data(), (const uint8_t *)ix->view.overflow + off, m, cudaMemcpyDeviceToHost));
            if (fwrite(buf.data(), 1, m, f) != m) { fclose(f); return sg_fail("snapgpu_index_save: short write"); }
        }
        fclose(f);
    }
    // GenomeIndexHash
    size_t hashBytes = 0;
    {
        FILE *f = fopen((dir + "/GenomeIndexHash").c_str(), "wb");
        if (!f) return sg_fail("snapgpu_index_save: cannot write GenomeIndexHash");
        const uint32_t eb = relay ? fileBytes : ix->view.entryBytes;
        for (size_t p = 0; p + 1 < ranges.size(); p++) {
            const uint64_t rangeBase = tstart[ranges[p]];
            const uint8_t *out = nullptr;
            if (relay) {
                const uint64_t n = tstart[ranges[p + 1] - 1] + tsize[ranges[p + 1] - 1] - rangeBase;
                const int grid = sg_sms() * 8;
                sg_relay_stage_clear_kernel<<<grid, 256>>>(dev.stage, stageBytes, n);
                SG_CUDA(cudaMemset(dev.failed, 0, 4));
                sg_relay_insert_kernel<<<grid, 256>>>((const unsigned long long *)ix->d_buckets, ix->view.nBuckets, seedLen, kb, large, ranges[p], ranges[p + 1],
                                                      dev.tableStart, dev.tableSize, rangeBase, dev.stage, stageBytes, dev.failed);
                SG_CUDA(cudaGetLastError());
                int failed = 0;
                SG_CUDA(cudaMemcpy(&failed, dev.failed, 4, cudaMemcpyDeviceToHost));
                if (failed) { fclose(f); return sg_fail("snapgpu_index_save: a bucket slot could not be placed in the reference's tables"); }
                out = dev.stage;
                if (dev.packed) {
                    sg_relay_pack_kernel<<<grid, 256>>>(dev.stage, stageBytes, n, dev.packed, kb, large);
                    SG_CUDA(cudaGetLastError());
                    out = dev.packed;
                }
            }
            for (uint32_t t = ranges[p]; t < ranges[p + 1]; t++) {
                uint8_t head[36];
                sg_table_header(head, tsize[t], t < tused.size() ? tused[t] : 0, keyBytes, isLarge, ix->view.invalidValue);
                if (fwrite(head, 1, 36, f) != 36) { fclose(f); return sg_fail("snapgpu_index_save: short write"); }
                hashBytes += 36;
                size_t total = (size_t)tsize[t] * eb;
                const uint8_t *src = relay ? out + (size_t)(tstart[t] - rangeBase) * eb : ix->view.tables + (size_t)tstart[t] * eb;
                for (size_t off = 0; off < total; off += CH) {
                    size_t m = total - off < CH ? total - off : CH;
                    SG_CUDA(cudaMemcpy(buf.data(), src + off, m, cudaMemcpyDeviceToHost));
                    if (fwrite(buf.data(), 1, m, f) != m) { fclose(f); return sg_fail("snapgpu_index_save: short write"); }
                }
                hashBytes += total;
            }
        }
        if (fclose(f) != 0) return sg_fail("snapgpu_index_save: cannot write GenomeIndexHash");
    }
    {
        FILE *f = fopen((dir + "/GenomeIndex").c_str(), "w");
        if (!f) return sg_fail("snapgpu_index_save: cannot write GenomeIndex");
        const std::string text = sg_genome_index_text(nT, ix->view.overflowSize, seedLen, ix->view.chromosomePadding, keyBytes, hashBytes, isLarge);
        fputs(text.c_str(), f);
        fclose(f);
    }
    return 0;
}

int snapgpu_index_save(const snapgpu_index *ix, const char *directory)
{
    snapgpu_save_options o;
    memset(&o, 0, sizeof(o));
    o.struct_size = sizeof(o); o.keyBytes = 4; o.large = 0; o.slack = 0.3;
    return snapgpu_index_save_ex(ix, directory, &o);
}

// ---- copies of an index on other devices of the same process (SURVEY 8e) ----
struct SgCloneCopy { void *dst; const void *src; size_t bytes; };

// Allocates, on `device`, every array of `src`'s image and lists the copies that fill them; the caller performs the copies
// (cudaMemcpyPeer, or one ncclBroadcast per array) and then calls clone_finish().
static int clone_alloc(const snapgpu_index *src, int device, snapgpu_index **out, std::vector<SgCloneCopy> &copies)
{
    if (require_device(device)) return 1;
    snapgpu_index *ix = new (std::nothrow) snapgpu_index;
    if (!ix) return sg_fail("out of memory");
    ix->device = device;
    const SgIndexView &sv = src->view;
    const size_t tableBytes = sv.layout == SG_LAYOUT_BUCKET ? 0 : (size_t)src->info.hashTableSlots * sv.entryBytes + 16;
    const size_t nT = sv.nTables;
    size_t hbm = 0;
    #define DUP(dst, srcp, bytes) do { size_t b__ = (bytes); if (b__ == 0) b__ = 16; SG_CUDA(cudaMalloc((void **)&(dst), b__)); \
        if ((bytes) > 0) { SgCloneCopy c__ = {(void *)(dst), (const void *)(srcp), (size_t)(bytes)}; copies.push_back(c__); } hbm += b__; } while (0)
    if (sv.layout == SG_LAYOUT_BUCKET) { DUP(ix->d_buckets, src->d_buckets, (size_t)sv.nBuckets * 32 + 64); }
    else { DUP(ix->d_tables, src->d_tables, tableBytes); }
    DUP(ix->d_tableStart, src->d_tableStart, nT * 8);
    DUP(ix->d_tableSize, src->d_tableSize, nT * 8);
    DUP(ix->d_tableMagic, src->d_tableMagic, nT * 8);
    DUP(ix->d_overflow, src->d_overflow, (size_t)(sv.overflowSize + 4) * 4);
    DUP(ix->d_basesPadded, src->d_basesPadded, (size_t)sv.nBases + 2 * SG_N_PADDING);
    DUP(ix->d_contigStart, src->d_contigStart, (size_t)sv.nContigs * 8);
    DUP(ix->d_tables_prob, src->d_tables_prob, sizeof(SgTables));
    if (src->d_projStart) {
        DUP(ix->d_projStart, src->d_projStart, src->h_projStart.size() * 8);
        DUP(ix->d_projRC, src->d_projRC, src->h_projRC.size());
        DUP(ix->d_projOps, src->d_projOps, src->h_projOps.size() * 4);
    }
    #undef DUP
    SgIndexView v = sv;
    v.tables = ix->d_tables; v.tableStart = ix->d_tableStart; v.tableSize = ix->d_tableSize; v.tableMagic = ix->d_tableMagic; v.overflow = ix->d_overflow;
    v.bases = ix->d_basesPadded + SG_N_PADDING; v.contigStart = ix->d_contigStart; v.buckets = ix->d_buckets;
    v.projStart = ix->d_projStart; v.projRC = ix->d_projRC; v.projOps = ix->d_projOps;
    ix->h_projStart = src->h_projStart; ix->h_projRC = src->h_projRC; ix->h_projOps = src->h_projOps;
    ix->view = v;
    ix->builtOnDevice = src->builtOnDevice;
    ix->info = src->info; ix->info.hbmBytes = hbm;
    ix->h_tables_prob = src->h_tables_prob;
    ix->h_tableStart = src->h_tableStart; ix->h_tableSize = src->h_tableSize; ix->h_tableUsed = src->h_tableUsed;
    ix->h_contigStart = src->h_contigStart; ix->h_contigName = src->h_contigName; ix->h_contigIsAlt = src->h_contigIsAlt; ix->h_contigOriginal = src->h_contigOriginal;
    ix->h_contigLines = src->h_contigLines;
    *out = ix;
    return 0;
}

// A copy of `src` on `device`: every array of the image is copied device to device (cudaMemcpyPeer: NVLink / NVSwitch when peer
// access is possible, staged through the host by the driver otherwise).
int snapgpu_index_replicate(const snapgpu_index *src, int device, snapgpu_index **out)
{
    if (!src || !out) return sg_fail("null argument");
    *out = nullptr;
    if (require_device(device)) return 1;
    if (device != src->device) {
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, device, src->device) == cudaSuccess && can) {
            cudaError_t e = cudaDeviceEnablePeerAccess(src->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            cudaGetLastError();
        }
    }
    std::vector<SgCloneCopy> copies;
    snapgpu_index *ix = nullptr;
    if (clone_alloc(src, device, &ix, copies)) { if (ix) snapgpu_index_close(ix); return 1; }
    for (size_t k = 0; k < copies.size(); k++) {
        if (cudaMemcpyPeer(copies[k].dst, device, copies[k].src, src->device, copies[k].bytes) != cudaSuccess) {
            std::string msg = std::string("snapgpu_index_replicate: cudaMemcpyPeer: ") + cudaGetErrorString(cudaGetLastError());
            snapgpu_index_close(ix);
            return sg_fail(msg);
        }
    }
    SG_CUDA(cudaDeviceSynchronize());
    *out = ix;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// A group of devices driven by ONE process (the SNAP extension: one feeder thread per device): NCCL communicators over them,
// for the two collectives the path has -- the index broadcast at start-up and the statistics all-reduce at the end (SURVEY 8e).
// NCCL is loaded at run time (dlopen), not linked: a process that already carries an NCCL (PyTorch ships its own) keeps using that
// one, and a single-device user of this library needs none.
// ------------------------------------------------------------------------------------------------
typedef ncclResult_t (*sg_ncclCommInitAll_t)(ncclComm_t *, int, const int *);
typedef ncclResult_t (*sg_ncclCommDestroy_t)(ncclComm_t);
typedef ncclResult_t (*sg_ncclGroup_t)(void);
typedef ncclResult_t (*sg_ncclBroadcast_t)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t);
typedef ncclResult_t (*sg_ncclAllReduce_t)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
typedef const char *(*sg_ncclGetErrorString_t)(ncclResult_t);

struct SgNccl {
    void *lib = nullptr;
    sg_ncclCommInitAll_t CommInitAll = nullptr; sg_ncclCommDestroy_t CommDestroy = nullptr; sg_ncclGroup_t GroupStart = nullptr, GroupEnd = nullptr;
    sg_ncclBroadcast_t Broadcast = nullptr; sg_ncclAllReduce_t AllReduce = nullptr; sg_ncclGetErrorString_t GetErrorString = nullptr;
};
static SgNccl g_nccl;

static int load_nccl()
{
    if (g_nccl.lib) return 0;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    void *h = nullptr;
    for (int k = 0; k < 2 && !h; k++) h = dlopen(names[k], RTLD_NOW | RTLD_GLOBAL);
    if (!h) return sg_fail(std::string("NCCL is not loadable (libnccl.so.2): ") + (dlerror() ? dlerror() : ""));
    SgNccl n; n.lib = h;
    n.CommInitAll = (sg_ncclCommInitAll_t)dlsym(h, "ncclCommInitAll"); n.CommDestroy = (sg_ncclCommDestroy_t)dlsym(h, "ncclCommDestroy");
    n.GroupStart = (sg_ncclGroup_t)dlsym(h, "ncclGroupStart"); n.GroupEnd = (sg_ncclGroup_t)dlsym(h, "ncclGroupEnd");
    n.Broadcast = (sg_ncclBroadcast_t)dlsym(h, "ncclBroadcast"); n.AllReduce = (sg_ncclAllReduce_t)dlsym(h, "ncclAllReduce");
    n.GetErrorString = (sg_ncclGetErrorString_t)dlsym(h, "ncclGetErrorString");
    if (!n.CommInitAll || !n.CommDestroy || !n.GroupStart || !n.GroupEnd || !n.Broadcast || !n.AllReduce || !n.GetErrorString) return sg_fail("libnccl.so.2 lacks a needed symbol");
    g_nccl = n;
    return 0;
}

#define SG_NCCL(call) do { ncclResult_t r__ = (call); if (r__ != ncclSuccess) return sg_fail(std::string(#call) + ": " + g_nccl.GetErrorString(r__)); } while (0)

struct snapgpu_group {
    std::vector<int> devices;
    std::vector<ncclComm_t> comms;
    std::vector<cudaStream_t> streams;
    std::vector<snapgpu_counters *> d_counters;
};

int snapgpu_group_create(const int *devices, int nDevices, snapgpu_group **out)
{
    if (!devices || !out || nDevices < 1) return sg_fail("bad argument");
    *out = nullptr;
    for (int k = 0; k < nDevices; k++) if (require_device(devices[k])) return 1;
    if (load_nccl()) return 1;
    snapgpu_group *g = new (std::nothrow) snapgpu_group;
    if (!g) return sg_fail("out of memory");
    g->devices.assign(devices, devices + nDevices);
    g->comms.assign(nDevices, (ncclComm_t)nullptr);
    g->streams.assign(nDevices, (cudaStream_t)nullptr);
    g->d_counters.assign(nDevices, (snapgpu_counters *)nullptr);
    ncclResult_t r = g_nccl.CommInitAll(g->comms.data(), nDevices, devices);
    if (r != ncclSuccess) { delete g; return sg_fail(std::string("ncclCommInitAll: ") + g_nccl.GetErrorString(r)); }
    for (int k = 0; k < nDevices; k++) {
        SG_CUDA(cudaSetDevice(devices[k]));
        SG_CUDA(cudaStreamCreateWithFlags(&g->streams[k], cudaStreamNonBlocking));
        SG_CUDA(cudaMalloc((void **)&g->d_counters[k], sizeof(snapgpu_counters)));
    }
    *out = g;
    return 0;
}

void snapgpu_group_destroy(snapgpu_group *g)
{
    if (!g) return;
    for (size_t k = 0; k < g->devices.size(); k++) {
        cudaSetDevice(g->devices[k]);
        if (g->comms[k]) g_nccl.CommDestroy(g->comms[k]);
        if (g->streams[k]) cudaStreamDestroy(g->streams[k]);
        cudaFree(g->d_counters[k]);
    }
    delete g;
}

int snapgpu_group_size(const snapgpu_group *g) { return g ? (int)g->devices.size() : 0; }

// One upload, then ncclBroadcast of every array of the image from the group's first device: out[0] = src, out[k] = the copy on device k.
int snapgpu_index_broadcast(snapgpu_group *g, snapgpu_index *src, snapgpu_index **out)
{
    if (!g || !src || !out) return sg_fail("null argument");
    const int n = (int)g->devices.size();
    if (src->device != g->devices[0]) return sg_fail("snapgpu_index_broadcast: the source index must live on the group's first device");
    std::vector<std::vector<SgCloneCopy> > copies(n);
    out[0] = src;
    for (int k = 1; k < n; k++) {
        out[k] = nullptr;
        if (clone_alloc(src, g->devices[k], &out[k], copies[k])) return 1;
    }
    if (n == 1) return 0;
    const size_t nArrays = copies[1].size();
    for (size_t a = 0; a < nArrays; a++) {
        SG_NCCL(g_nccl.GroupStart());
        for (int k = 0; k < n; k++) {
            const void *srcp = copies[1][a].src;
            void *dst = k == 0 ? (void *)srcp : copies[k][a].dst;
            ncclResult_t r = g_nccl.Broadcast(srcp, dst, copies[1][a].bytes, ncclUint8, 0, g->comms[k], g->streams[k]);
            if (r != ncclSuccess) { g_nccl.GroupEnd(); return sg_fail(std::string("ncclBroadcast: ") + g_nccl.GetErrorString(r)); }
        }
        SG_NCCL(g_nccl.GroupEnd());
    }
    for (int k = 0; k < n; k++) { SG_CUDA(cudaSetDevice(g->devices[k])); SG_CUDA(cudaStreamSynchronize(g->streams[k])); }
    return 0;
}

// AlignerStats reduction (AlignerStats.h:41-84, AlignerContext.cpp:241-245): counters[k] = the HOST counters of device k's feeder; each
// is replaced by the sum over the group, computed by ncclAllReduce(SUM) over the devices.
int snapgpu_counters_allreduce(snapgpu_group *g, snapgpu_counters *counters)
{
    if (!g || !counters) return sg_fail("null argument");
    const int n = (int)g->devices.size();
    const size_t words = sizeof(snapgpu_counters) / 8;
    for (int k = 0; k < n; k++) {
        SG_CUDA(cudaSetDevice(g->devices[k]));
        SG_CUDA(cudaMemcpyAsync(g->d_counters[k], &counters[k], sizeof(snapgpu_counters), cudaMemcpyHostToDevice, g->streams[k]));
    }
    SG_NCCL(g_nccl.GroupStart());
    for (int k = 0; k < n; k++) {
        ncclResult_t r = g_nccl.AllReduce(g->d_counters[k], g->d_counters[k], words, ncclInt64, ncclSum, g->comms[k], g->streams[k]);
        if (r != ncclSuccess) { g_nccl.GroupEnd(); return sg_fail(std::string("ncclAllReduce: ") + g_nccl.GetErrorString(r)); }
    }
    SG_NCCL(g_nccl.GroupEnd());
    for (int k = 0; k < n; k++) {
        SG_CUDA(cudaSetDevice(g->devices[k]));
        SG_CUDA(cudaMemcpyAsync(&counters[k], g->d_counters[k], sizeof(snapgpu_counters), cudaMemcpyDeviceToHost, g->streams[k]));
        SG_CUDA(cudaStreamSynchronize(g->streams[k]));
    }
    return 0;
}

int snapgpu_index_info_get(const snapgpu_index *idx, snapgpu_index_info *info)
{
    if (!idx || !info) return sg_fail("null argument");
    *info = idx->info;
    return 0;
}

void snapgpu_index_close(snapgpu_index *ix)
{
    if (!ix) return;
    cudaSetDevice(ix->device);
    cudaFree(ix->d_tables); cudaFree(ix->d_buckets); cudaFree(ix->d_tableStart); cudaFree(ix->d_tableSize); cudaFree(ix->d_tableMagic); cudaFree(ix->d_overflow);
    cudaFree(ix->d_basesPadded); cudaFree(ix->d_contigStart); cudaFree(ix->d_tables_prob);
    cudaFree(ix->d_projStart); cudaFree(ix->d_projRC); cudaFree(ix->d_projOps);
    delete ix;
}

int snapgpu_lookup_seeds(const snapgpu_index *idx, const char *seeds, int64_t nSeeds, uint32_t maxHitsPerSeed,
                         int64_t *nHits, uint32_t *hits, uint32_t *probes)
{
    if (!idx || !seeds || !nHits) return sg_fail("null argument");
    if (require_device(idx->device)) return 1;
    if (nSeeds <= 0) return 0;
    uint8_t *d_seeds = nullptr; long long *d_nHits = nullptr; uint32_t *d_hits = nullptr, *d_probes = nullptr;
    const size_t sb = (size_t)nSeeds * idx->view.seedLen;
    SG_CUDA(cudaMalloc((void **)&d_seeds, sb));
    SG_CUDA(cudaMalloc((void **)&d_nHits, (size_t)nSeeds * 2 * 8));
    if (hits) SG_CUDA(cudaMalloc((void **)&d_hits, (size_t)nSeeds * 2 * maxHitsPerSeed * 4 + 16));
    if (probes) SG_CUDA(cudaMalloc((void **)&d_probes, (size_t)nSeeds * 4));
    SG_CUDA(cudaMemcpy(d_seeds, seeds, sb, cudaMemcpyHostToDevice));
    int blocks = (int)((nSeeds * 32 + 255) / 256);
    if (blocks > sg_sms() * 16) blocks = sg_sms() * 16;
    if (idx->view.layout == SG_LAYOUT_BUCKET) {
        int bb = (int)((nSeeds + 255) / 256); if (bb > sg_sms() * 8) bb = sg_sms() * 8;
        sg_lookup_bucket_kernel<<<bb, 256>>>(idx->view, d_seeds, nSeeds, maxHitsPerSeed, d_nHits, d_hits, d_probes);
    } else
    sg_lookup_kernel<<<blocks, 256>>>(idx->view, d_seeds, nSeeds, maxHitsPerSeed, d_nHits, d_hits, d_probes);
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaDeviceSynchronize());
    SG_CUDA(cudaMemcpy(nHits, d_nHits, (size_t)nSeeds * 2 * 8, cudaMemcpyDeviceToHost));
    if (hits) SG_CUDA(cudaMemcpy(hits, d_hits, (size_t)nSeeds * 2 * maxHitsPerSeed * 4, cudaMemcpyDeviceToHost));
    if (probes) SG_CUDA(cudaMemcpy(probes, d_probes, (size_t)nSeeds * 4, cudaMemcpyDeviceToHost));
    cudaFree(d_seeds); cudaFree(d_nHits); cudaFree(d_hits); cudaFree(d_probes);
    return 0;
}

// Random 32-byte sector reads (see the header): the ceiling hash probing is measured against.
__global__ void __launch_bounds__(256, 8)
sg_random_sector_kernel(const uint8_t *tbl, unsigned long long nSectors, unsigned long long nAccess, unsigned long long salt, unsigned long long *sink)
{
    const unsigned long long nT = (unsigned long long)gridDim.x * blockDim.x;
    uint32_t acc = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nAccess; i += nT) {
        const unsigned long long unit = __umul64hi(sg_fmix64(i ^ salt), nSectors);
        const uint4 *p = (const uint4 *)(tbl + unit * 32);
        const uint4 a = __ldg(p), b = __ldg(p + 1);
        acc += a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w;
    }
    if (acc == 0x12345678u) atomicAdd(sink, 1ULL);
}

int snapgpu_measure_random_sector_rate(int device, uint64_t tableBytes, uint64_t nAccesses, double *sectorsPerSecond)
{
    if (!sectorsPerSecond || tableBytes < 4096 || nAccesses == 0) return sg_fail("bad argument");
    if (require_device(device)) return 1;
    uint8_t *tbl = nullptr; unsigned long long *sink = nullptr;
    tableBytes = tableBytes / 4096 * 4096;
    SG_CUDA(cudaMalloc((void **)&tbl, tableBytes));
    SG_CUDA(cudaMalloc((void **)&sink, 8));
    SG_CUDA(cudaMemset(tbl, 1, tableBytes));
    SG_CUDA(cudaMemset(sink, 0, 8));
    cudaEvent_t e0, e1;
    SG_CUDA(cudaEventCreate(&e0)); SG_CUDA(cudaEventCreate(&e1));
    sg_random_sector_kernel<<<sg_sms() * 8, 256>>>(tbl, tableBytes / 32, nAccesses / 8 + 1, 1, sink);
    SG_CUDA(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < 3; r++) {
        SG_CUDA(cudaEventRecord(e0));
        sg_random_sector_kernel<<<sg_sms() * 8, 256>>>(tbl, tableBytes / 32, nAccesses, 77 + r, sink);
        SG_CUDA(cudaEventRecord(e1));
        SG_CUDA(cudaEventSynchronize(e1));
        float ms = 0; SG_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(tbl); cudaFree(sink);
    *sectorsPerSecond = (double)nAccesses / ((double)best * 1e-3);
    return 0;
}

// Device-resident variant used by bench.py's seed-phase roofline: everything already in HBM, launched on `stream`.
int snapgpu_lookup_seeds_device(const snapgpu_index *idx, const char *d_seeds, int64_t nSeeds, uint32_t maxHitsPerSeed,
                                int64_t *d_nHits, uint32_t *d_hits, uint32_t *d_probes, void *cudaStream)
{
    if (!idx || !d_seeds || !d_nHits) return sg_fail("null argument");
    if (nSeeds <= 0) return 0;
    int blocks = (int)((nSeeds * 32 + 255) / 256);
    if (blocks > sg_sms() * 16) blocks = sg_sms() * 16;
    if (idx->view.layout == SG_LAYOUT_BUCKET) {
        int bb = (int)((nSeeds + 255) / 256); if (bb > sg_sms() * 8) bb = sg_sms() * 8;
        sg_lookup_bucket_kernel<<<bb, 256, 0, (cudaStream_t)cudaStream>>>(idx->view, (const uint8_t *)d_seeds, nSeeds, maxHitsPerSeed,
                                                                        (long long *)d_nHits, d_hits, d_probes);
    } else
    sg_lookup_kernel<<<blocks, 256, 0, (cudaStream_t)cudaStream>>>(idx->view, (const uint8_t *)d_seeds, nSeeds, maxHitsPerSeed,
                                                                   (long long *)d_nHits, d_hits, d_probes);
    SG_CUDA(cudaGetLastError());
    return 0;
}

// Shared part of the two create functions: worker arenas, streams, the two pipeline slots.
// maxBatchReads counts READS (2 per pair); resultBytesPerRead: bytes of result per read in the staging buffers.
static int aligner_init_common(snapgpu_aligner *a, int64_t maxBatchReads, int64_t maxUnits, size_t scratchBytesPerWorker, size_t resultBytesPerUnit,
                               int readsPerUnit, int defaultBlocksPerSM, const char *blocksEnv)
{
    cudaDeviceProp prop;
    SG_CUDA(cudaGetDeviceProperties(&prop, a->device));
    a->numSMs = prop.multiProcessorCount;
    a->blocksPerSM = defaultBlocksPerSM;      // resident CTAs (of 8 warps) per SM the kernel is compiled for: 2, 3 or 4
    if (const char *e = getenv(blocksEnv)) a->blocksPerSM = atoi(e) > 0 ? atoi(e) : defaultBlocksPerSM;
    if (a->blocksPerSM < 2) a->blocksPerSM = 2;
    if (a->blocksPerSM > 4) a->blocksPerSM = 4;
    a->pass1BlocksPerSM = 8;             // the fastest of 4..8 in a sweep (32 registers, no extra spills)
    if (const char *e = getenv("SNAPGPU_PASS1_BLOCKS_PER_SM")) a->pass1BlocksPerSM = atoi(e);
    if (a->pass1BlocksPerSM < 3 || a->pass1BlocksPerSM > 8 || a->pass1BlocksPerSM == 7 || readsPerUnit != 1) a->pass1BlocksPerSM = a->blocksPerSM;
    int maxBlocks = a->blocksPerSM > a->pass1BlocksPerSM ? a->blocksPerSM : a->pass1BlocksPerSM;
    if (readsPerUnit == 2) {
        // CTAs per SM of the three stages; 8,6,8 was the fastest of a sweep of stock snap paired
        if (const char *e = getenv("SNAPGPU_PAIRED_STAGE_BLOCKS")) sscanf(e, "%d,%d,%d", &a->stageBlocks[1], &a->stageBlocks[2], &a->stageBlocks[3]);
        for (int k = 1; k <= 3; k++) {
            if (a->stageBlocks[k] != 6 && a->stageBlocks[k] != 8) a->stageBlocks[k] = 4;
            if (a->stageBlocks[k] > maxBlocks) maxBlocks = a->stageBlocks[k];
        }
    }
    // The arenas of the extra (more than blocksPerSM) CTAs per SM are a throughput option, not a need: give them up when they
    // would take more than half of the free HBM (long maximum read lengths make the arenas large).
    {
        size_t freeB = 0, totalB = 0;
        SG_CUDA(cudaMemGetInfo(&freeB, &totalB));
        while (maxBlocks > a->blocksPerSM && scratchBytesPerWorker * (size_t)a->numSMs * maxBlocks * a->warpsPerBlock > freeB / 2) {
            maxBlocks -= 2;
            if (maxBlocks < a->blocksPerSM) maxBlocks = a->blocksPerSM;
            if (a->pass1BlocksPerSM > maxBlocks) a->pass1BlocksPerSM = maxBlocks == 6 ? 6 : a->blocksPerSM;
            for (int k = 1; k <= 3; k++) if (a->stageBlocks[k] > maxBlocks) a->stageBlocks[k] = maxBlocks == 6 ? 6 : 4;
        }
    }
    a->nWorkers = a->numSMs * maxBlocks * a->warpsPerBlock;
    if ((int64_t)a->nWorkers > maxUnits) {
        int blocks = (int)((maxUnits + a->warpsPerBlock - 1) / a->warpsPerBlock);
        a->nWorkers = blocks * a->warpsPerBlock;
    }
    {
        // fewer resident warps rather than a failure when even these arenas would take most of the free HBM (pools of many seeds beside a
        // large index on an 80 GB device); warps take reads from a counter, so the results do not depend on how many there are.  Every
        // launch clamps its grid to nWorkers.  SNAPGPU_MAX_WORKERS sets a lower cap (test hook for this path).
        size_t freeB = 0, totalB = 0;
        SG_CUDA(cudaMemGetInfo(&freeB, &totalB));
        size_t fit = freeB / 4 * 3 / scratchBytesPerWorker;
        if (const char *e = getenv("SNAPGPU_MAX_WORKERS")) { const long long v = atoll(e); if (v > 0 && (size_t)v < fit) fit = (size_t)v; }
        fit = fit / a->warpsPerBlock * a->warpsPerBlock;
        if (fit >= (size_t)a->warpsPerBlock && (size_t)a->nWorkers > fit) a->nWorkers = (int)fit;
    }
    a->scratchBytesPerWorker = scratchBytesPerWorker;
    SG_CUDA(cudaMalloc((void **)&a->d_scratch, a->scratchBytesPerWorker * (size_t)a->nWorkers));
    SG_CUDA(cudaMemset(a->d_scratch, 0, a->scratchBytesPerWorker * (size_t)a->nWorkers));
    SG_CUDA(cudaMalloc((void **)&a->d_next, 8));
    SG_CUDA(cudaMalloc((void **)&a->d_error, sizeof(int)));
    SG_CUDA(cudaMemset(a->d_error, 0, sizeof(int)));
    SG_CUDA(cudaStreamCreateWithFlags(&a->stream, cudaStreamNonBlocking));
    SG_CUDA(cudaStreamCreateWithFlags(&a->streamIn, cudaStreamNonBlocking));
    SG_CUDA(cudaStreamCreateWithFlags(&a->streamOut, cudaStreamNonBlocking));
    // host-buffer pipeline stages: a small first chunk (the copy nothing overlaps with), then the rest of one full-size chunk, then full-size chunks --
    // few launches, so little of the step is spent in the tails of the persistent kernels.  Equal chunks of 128 K to 512 K reads differ little.
    a->chunkReads = 524288;
    if (const char *e = getenv("SNAPGPU_CHUNK_READS")) a->chunkReads = atoll(e) > 0 ? atoll(e) : a->chunkReads;
    if (a->chunkReads > maxBatchReads) a->chunkReads = maxBatchReads;
    a->chunkReads = (a->chunkReads + readsPerUnit - 1) / readsPerUnit * readsPerUnit;
    a->firstChunkReads = a->chunkReads / 8;
    if (const char *e = getenv("SNAPGPU_FIRST_CHUNK_READS")) a->firstChunkReads = atoll(e) > 0 ? atoll(e) : a->firstChunkReads;
    if (a->firstChunkReads > a->chunkReads) a->firstChunkReads = a->chunkReads;
    a->firstChunkReads = (a->firstChunkReads + readsPerUnit - 1) / readsPerUnit * readsPerUnit;
    if (a->firstChunkReads < readsPerUnit) a->firstChunkReads = readsPerUnit;
    a->chunkBases = (size_t)a->chunkReads * (size_t)a->params.maxReadLen;
    const size_t resultBytes = (size_t)(a->chunkReads / readsPerUnit) * resultBytesPerUnit;
    for (int k = 0; k < 2; k++) {
        snapgpu_aligner::Slot &sl = a->slot[k];
        SG_CUDA(cudaMallocHost((void **)&sl.h_bases, a->chunkBases));
        SG_CUDA(cudaMallocHost((void **)&sl.h_quals, a->chunkBases));
        SG_CUDA(cudaMallocHost((void **)&sl.h_offsets, (size_t)a->chunkReads * 8));
        SG_CUDA(cudaMallocHost((void **)&sl.h_lens, (size_t)a->chunkReads * 4));
        SG_CUDA(cudaMallocHost((void **)&sl.h_results, resultBytes));
        SG_CUDA(cudaMalloc((void **)&sl.d_bases, a->chunkBases));
        SG_CUDA(cudaMalloc((void **)&sl.d_quals, a->chunkBases));
        SG_CUDA(cudaMalloc((void **)&sl.d_offsets, (size_t)a->chunkReads * 8));
        SG_CUDA(cudaMalloc((void **)&sl.d_lens, (size_t)a->chunkReads * 4));
        SG_CUDA(cudaMalloc((void **)&sl.d_results, resultBytes));
        SG_CUDA(cudaEventCreateWithFlags(&sl.evIn, cudaEventDisableTiming));
        SG_CUDA(cudaEventCreateWithFlags(&sl.evKernel, cudaEventDisableTiming));
        SG_CUDA(cudaEventCreateWithFlags(&sl.evOut, cudaEventDisableTiming));
    }
    SG_CUDA(cudaMallocHost((void **)&a->h_counters, sizeof(snapgpu_counters)));
    SG_CUDA(cudaMalloc((void **)&a->d_counters, sizeof(snapgpu_counters)));
    return 0;
}

static uint32_t env_max_read_len()
{
    uint32_t maxReadLen = 400;
    if (const char *e = getenv("SNAPGPU_MAX_READ_LEN")) maxReadLen = (uint32_t)atoi(e);
    return maxReadLen;
}

int snapgpu_aligner_create(const snapgpu_index *idx, const snapgpu_params *params, int64_t maxBatchReads, snapgpu_aligner **out)
{
    if (!idx || !params || !out) return sg_fail("null argument");
    *out = nullptr;
    if (require_device(idx->device)) return 1;
    if (maxBatchReads <= 0) return sg_fail("maxBatchReads must be positive");
    snapgpu_aligner *a = new (std::nothrow) snapgpu_aligner;
    if (!a) return sg_fail("out of memory");
    a->index = idx; a->device = idx->device; a->userParams = *params; a->maxBatchReads = maxBatchReads;
    std::string err;
    if (!sg_derive_params(*params, idx->view.seedLen, env_max_read_len(), a->params, err)) { delete a; return sg_fail("snapgpu_aligner_create: " + err); }
    if (aligner_init_common(a, maxBatchReads, maxBatchReads, sg_align_up(sg_scratch_bytes(a->params), 256), sizeof(snapgpu_single_result), 1, 4,
                            "SNAPGPU_BLOCKS_PER_SM")) { snapgpu_aligner_destroy(a); return 1; }
    // two-pass launch (see sg_align_kernel) whenever some reads can finish without affine gap: not under -ne (every
    // candidate is rescored) ; without affine gap at all the first pass simply finishes everything.  SNAPGPU_TWO_PASS=0 turns it off.
    a->params.agSpecialised = 1;         // second pass: narrow-band / packed affine-gap forms (faster there; they cost throughput in the one-launch form)
    if (const char *e = getenv("SNAPGPU_SINGLE_AG_SPECIALISED")) a->params.agSpecialised = atoi(e);       // 0 off, 1 on, 2 on with the unrolled packed form
    // bands of up to 32 columns in the second pass: `rows` (default) one (row, segment) unit per warp step (sg_warp_ag_rows_banded4),
    // `duo` two per step (sg_warp_ag_duo.cuh).  Same results; on `snap single -d 14` on an H100 the second pass takes 41.7 ms with
    // `rows` and 46.9 ms with `duo` (DESIGN.md section 6).
    {
        const char *e = getenv("SNAPGPU_SINGLE_AG_NARROW");
        const bool duo = e && strcmp(e, "duo") == 0;
        if (e && !duo && strcmp(e, "rows") != 0) { snapgpu_aligner_destroy(a); return sg_fail("SNAPGPU_SINGLE_AG_NARROW must be rows or duo"); }
        if (duo) a->params.agSpecialised |= 4;
    }
    a->params.tmaMinHits = 0;            // hit-list staging through shared memory (bulk copies): off by default, not measured on H100
    if (const char *e = getenv("SNAPGPU_TMA_MIN_HITS")) a->params.tmaMinHits = (uint32_t)atoi(e);
    a->twoPass = !a->params.noEditDistance;
    if (const char *e = getenv("SNAPGPU_TWO_PASS")) a->twoPass = atoi(e) != 0;
    if (a->twoPass) {
        // overlapped launch (SNAPGPU_OVERLAP=1; off by default): needs arenas for both passes at once.  On `snap single -d 14` it was slower than
        // the two passes one after the other, whatever the number of first-pass CTAs per SM beside the second pass: with both kernels' code
        // resident on an SM the first pass alone slows down several times -- instruction supply, the reason the passes were split in the first place.
        a->overlap = false;
        if (const char *e = getenv("SNAPGPU_OVERLAP")) a->overlap = atoi(e) != 0;
        a->overlapMinReads = 4LL * a->numSMs * a->warpsPerBlock;
        if (const char *e = getenv("SNAPGPU_OVERLAP_MIN_READS")) a->overlapMinReads = atoll(e);
        if (const char *e = getenv("SNAPGPU_OVERLAP_PASS1_BLOCKS")) { const int v = atoi(e); if (v >= 1 && v <= 4) a->overlapPass1Blocks = v; }
        if (a->blocksPerSM != 4 || a->nWorkers < a->numSMs * 8 * a->warpsPerBlock) a->overlap = false;
        if (a->overlap) {
            // both kernels ask for the same shared-memory carve-out (room for 2 + 3 or for 4 CTAs of 27 KB), so that CTAs of either fit on an SM
            // the other configured first
            int carve = 72;
            if (const char *e = getenv("SNAPGPU_OVERLAP_CARVEOUT")) carve = atoi(e);
            cudaFuncSetAttribute(sg_align_kernel<8, 1>, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
            cudaFuncSetAttribute(sg_align_kernel<4, 2>, cudaFuncAttributePreferredSharedMemoryCarveout, carve);
        }
        if (cudaMalloc((void **)&a->d_retryList, (size_t)maxBatchReads * 4) != cudaSuccess || cudaMalloc((void **)&a->d_producersDone, 16) != cudaSuccess ||
            cudaStreamCreateWithFlags(&a->stream2, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&a->evFork, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&a->evJoin, cudaEventDisableTiming) != cudaSuccess ||
            cudaMalloc((void **)&a->d_retryCount, 8) != cudaSuccess || cudaMalloc((void **)&a->d_next2, 8) != cudaSuccess) {
            std::string msg = std::string("snapgpu_aligner_create: deferred-read list: ") + cudaGetErrorString(cudaGetLastError());
            snapgpu_aligner_destroy(a);
            return sg_fail(msg);
        }
    }
    *out = a;
    return 0;
}

void snapgpu_paired_params_default(snapgpu_paired_params *pp)
{
    // PairedAligner.cpp:228-243 (PairedAlignerOptions ctor), AlignerOptions.cpp:101-111
    memset(pp, 0, sizeof(*pp));
    pp->struct_size = sizeof(*pp);
    pp->minSpacing = 0; pp->maxSpacing = 1000; pp->intersectingAlignerMaxHits = 4000; pp->maxCandidatePoolSize = 1000000;
    pp->maxSeedsSingleEnd = 25; pp->maxDistForIndels = 40; pp->forceSpacing = 0;
    pp->minScoreRealignment = 3; pp->minScoreGapRealignmentALT = 3; pp->minAGScoreImprovement = 24;
    pp->enableHammingScoringBaseAligner = 1; pp->useSoftClipping = 1; pp->flattenMAPQAtOrBelow = 3;
}

int snapgpu_paired_aligner_create(const snapgpu_index *idx, const snapgpu_params *params, const snapgpu_paired_params *pparams,
                                  int64_t maxBatchPairs, snapgpu_aligner **out)
{
    if (!idx || !params || !pparams || !out) return sg_fail("null argument");
    *out = nullptr;
    if (require_device(idx->device)) return 1;
    if (maxBatchPairs <= 0) return sg_fail("maxBatchPairs must be positive");
    snapgpu_aligner *a = new (std::nothrow) snapgpu_aligner;
    if (!a) return sg_fail("out of memory");
    a->index = idx; a->device = idx->device; a->userParams = *params; a->maxBatchReads = 2 * maxBatchPairs; a->paired = true;
    std::string err;
    if (!sg_derive_paired_params(*params, *pparams, idx->view.seedLen, env_max_read_len(), a->params, a->paramsSingle, a->pparams, err)) {
        delete a; return sg_fail("snapgpu_paired_aligner_create: " + err);
    }
    a->singleScratchBytes = sg_align_up(sg_scratch_bytes(a->paramsSingle), 256);
    // per-worker pool caps (results do not depend on them: pairs that need more are re-aligned by the full-size workers)
    a->pparamsBig = a->pparams;
    uint32_t poolCap = 4096, candCap = 512;
    if (const char *e = getenv("SNAPGPU_PAIRED_POOL_CAP")) poolCap = (uint32_t)atoi(e);
    if (const char *e = getenv("SNAPGPU_PAIRED_CAND_CAP")) candCap = (uint32_t)atoi(e);
    if (poolCap < 16) poolCap = 16;
    if (candCap < 4) candCap = 4;
    a->pparams.poolCap = poolCap < a->pparams.poolSize ? (poolCap & ~1u) : a->pparams.poolSize;
    a->pparams.agCandCap = candCap < SG_MAX_AG_CANDIDATES ? candCap : SG_MAX_AG_CANDIDATES;
    const size_t perWorker = a->singleScratchBytes + sg_align_up(sg_paired_scratch_bytes(a->params, a->pparams), 256);
    if (aligner_init_common(a, 2 * maxBatchPairs, maxBatchPairs, perWorker, sizeof(snapgpu_paired_result), 2, 4, "SNAPGPU_PAIRED_BLOCKS_PER_SM")) {
        snapgpu_aligner_destroy(a); return 1;
    }
    a->bigScratchBytesPerWorker = a->singleScratchBytes + sg_align_up(sg_paired_scratch_bytes(a->params, a->pparamsBig), 256);
    size_t budget = (size_t)4 << 30;
    int nBig = (int)(budget / a->bigScratchBytesPerWorker);
    if (nBig > 128) nBig = 128;
    if (nBig < a->warpsPerBlock) nBig = a->warpsPerBlock;
    nBig = nBig / a->warpsPerBlock * a->warpsPerBlock;
    if ((int64_t)nBig > maxBatchPairs) nBig = (int)((maxBatchPairs + a->warpsPerBlock - 1) / a->warpsPerBlock) * a->warpsPerBlock;
    a->nBigWorkers = nBig;
    if (cudaMalloc((void **)&a->d_bigScratch, a->bigScratchBytesPerWorker * (size_t)nBig) != cudaSuccess ||
        cudaMemset(a->d_bigScratch, 0, a->bigScratchBytesPerWorker * (size_t)nBig) != cudaSuccess ||
        cudaMalloc((void **)&a->d_retryList, (size_t)maxBatchPairs * 4) != cudaSuccess ||
        cudaMalloc((void **)&a->d_retryCount, 8) != cudaSuccess || cudaMalloc((void **)&a->d_next2, 8) != cudaSuccess) {
        std::string msg = std::string("snapgpu_paired_aligner_create: retry arena: ") + cudaGetErrorString(cudaGetLastError());
        snapgpu_aligner_destroy(a);
        return sg_fail(msg);
    }
    a->staged = true;
    a->pparamsBig.stage2Packed = 1;
    a->pparams.stage2Packed = 2;         // stage 2 is ~90 % this one function and issue-bound: the unrolled instantiation is faster
    if (const char *e = getenv("SNAPGPU_PAIRED_STAGE2_PACKED")) a->pparams.stage2Packed = atoi(e) == 2 ? 2 : 1;
    if (const char *e = getenv("SNAPGPU_PAIRED_STAGED")) a->staged = atoi(e) != 0;
    if (a->staged) {
        unsigned long long perPair = 4;      // hand-off candidate records per pair of the batch (a pair that finds the pool full is done whole by the retry pass)
        if (const char *e = getenv("SNAPGPU_PAIRED_HANDOFF_PER_PAIR")) perPair = atoll(e) > 0 ? (unsigned long long)atoll(e) : perPair;
        a->candPoolCap = perPair * (unsigned long long)maxBatchPairs;
        if (cudaMalloc(&a->d_handoff, (size_t)maxBatchPairs * sizeof(SgPairHandoff)) != cudaSuccess ||
            cudaMalloc((void **)&a->d_candPool, (size_t)a->candPoolCap * sizeof(snapgpu_paired_result)) != cudaSuccess ||
            cudaMalloc((void **)&a->d_candPoolUsed, 8) != cudaSuccess || cudaMalloc((void **)&a->d_next3, 16) != cudaSuccess) {
            std::string msg = std::string("snapgpu_paired_aligner_create: hand-off buffers: ") + cudaGetErrorString(cudaGetLastError());
            snapgpu_aligner_destroy(a);
            return sg_fail(msg);
        }
    }
    *out = a;
    return 0;
}

void snapgpu_aligner_destroy(snapgpu_aligner *a)
{
    if (!a) return;
    cudaSetDevice(a->device);
    cudaDeviceSynchronize();
    if (a->stream) cudaStreamDestroy(a->stream);
    if (a->streamIn) cudaStreamDestroy(a->streamIn);
    if (a->streamOut) cudaStreamDestroy(a->streamOut);
    cudaFree(a->d_scratch); cudaFree(a->d_next); cudaFree(a->d_error);
    cudaFree(a->d_bigScratch); cudaFree(a->d_retryList); cudaFree(a->d_retryCount); cudaFree(a->d_next2); cudaFree(a->d_producersDone);
    if (a->stream2) cudaStreamDestroy(a->stream2);
    if (a->evFork) cudaEventDestroy(a->evFork);
    if (a->evJoin) cudaEventDestroy(a->evJoin);
    cudaFree(a->d_handoff); cudaFree(a->d_candPool); cudaFree(a->d_candPoolUsed); cudaFree(a->d_next3);
    for (int k = 0; k < 2; k++) {
        snapgpu_aligner::Slot &sl = a->slot[k];
        cudaFreeHost(sl.h_bases); cudaFreeHost(sl.h_quals); cudaFreeHost(sl.h_offsets); cudaFreeHost(sl.h_lens); cudaFreeHost(sl.h_results);
        cudaFree(sl.d_bases); cudaFree(sl.d_quals); cudaFree(sl.d_offsets); cudaFree(sl.d_lens); cudaFree(sl.d_results);
        if (sl.evIn) cudaEventDestroy(sl.evIn);
        if (sl.evKernel) cudaEventDestroy(sl.evKernel);
        if (sl.evOut) cudaEventDestroy(sl.evOut);
    }
    cudaFreeHost(a->h_counters); cudaFree(a->d_counters);
    cudaFree(a->d_secRaw);
    delete a;
}

// n = units (reads for a single-end handle, pairs for a paired one)
static int launch_align(snapgpu_aligner *a, int64_t n, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                        const uint32_t *d_lens, void *d_results, snapgpu_counters *d_counters, cudaStream_t st)
{
    SG_CUDA(cudaMemsetAsync(a->d_next, 0, 8, st));
    int64_t workers = (int64_t)a->numSMs * a->blocksPerSM * a->warpsPerBlock;
    if (workers > a->nWorkers) workers = a->nWorkers;
    if (workers > n) workers = n;
    int blocks = (int)((workers + a->warpsPerBlock - 1) / a->warpsPerBlock);
    if (blocks < 1) blocks = 1;
    if (!a->paired) {
#define SG_LAUNCH(MB, MODE, GRID, NEXT) sg_align_kernel<MB, MODE><<<GRID, a->warpsPerBlock * 32, 0, st>>>(a->index->view, a->params, a->index->d_tables_prob, \
        a->d_scratch, a->scratchBytesPerWorker, n, (const uint8_t *)d_bases, (const uint8_t *)d_quals, (const unsigned long long *)d_offsets, \
        d_lens, (snapgpu_single_result *)d_results, d_counters, NEXT, a->d_retryCount, a->d_retryList, a->d_producersDone, 0u, 0u)
#define SG_LAUNCH_MB(MODE, GRID, NEXT) if (a->blocksPerSM >= 4) SG_LAUNCH(4, MODE, GRID, NEXT); else if (a->blocksPerSM == 3) SG_LAUNCH(3, MODE, GRID, NEXT); \
        else SG_LAUNCH(2, MODE, GRID, NEXT)      /* second pass: the same speed at 4, 5 and 6 CTAs/SM */
        if (a->twoPass && a->overlap && n >= a->overlapMinReads) {
            // Overlapped form: both passes resident at once.  The first pass (latency-bound, a third of the issue slots used) runs its
            // 32-register build at overlapPass1Blocks (2) CTAs per SM on the caller's stream; the second (affine gap, issue-bound) runs
            // beside it on stream2 at 3 CTAs per SM -- 2 x 8 K + 3 x 16 K registers = the SM's file, so neither launch can keep the other
            // off the machine whichever is placed first -- and consumes the deferred-read list while it is being produced (see
            // sg_align_kernel); more CTAs of the second pass follow the first pass on the caller's stream and take over the registers it
            // leaves.  Arenas: first pass workers [0, g1*8), then the second pass's two launches.
            const int k2a = (64 - 8 * a->overlapPass1Blocks) / 16;          // 64-register CTAs that fit beside the first pass's 32-register ones
            const int g1 = a->numSMs * a->overlapPass1Blocks, g2a = a->numSMs * k2a, g2b = a->numSMs * (8 - a->overlapPass1Blocks - k2a > 4 ? 4 : 8 - a->overlapPass1Blocks - k2a);
            static const int dbg = getenv("SNAPGPU_OVERLAP_DEBUG") ? atoi(getenv("SNAPGPU_OVERLAP_DEBUG")) : 0;
            cudaEvent_t dbgEv[4] = {nullptr, nullptr, nullptr, nullptr};
            if (dbg) for (int k = 0; k < 4; k++) cudaEventCreate(&dbgEv[k]);
            SG_CUDA(cudaMemsetAsync(a->d_retryCount, 0, 8, st));
            SG_CUDA(cudaMemsetAsync(a->d_next2, 0, 8, st));
            SG_CUDA(cudaMemsetAsync(a->d_producersDone, 0, 16, st));
            SG_CUDA(cudaMemsetAsync(a->d_retryList, 0xff, (size_t)n * 4, st));
            SG_CUDA(cudaEventRecord(a->evFork, st));
            SG_CUDA(cudaStreamWaitEvent(a->stream2, a->evFork, 0));
#define SG_LAUNCH_OV(MB, MODE, GRID, STREAM, NEXT, BASE) sg_align_kernel<MB, MODE><<<GRID, a->warpsPerBlock * 32, 0, STREAM>>>(a->index->view, a->params, \
                a->index->d_tables_prob, a->d_scratch, a->scratchBytesPerWorker, n, (const uint8_t *)d_bases, (const uint8_t *)d_quals, \
                (const unsigned long long *)d_offsets, d_lens, (snapgpu_single_result *)d_results, d_counters, NEXT, a->d_retryCount, a->d_retryList, \
                a->d_producersDone, (unsigned)g1, (unsigned)(BASE))
            if (dbg) cudaEventRecord(dbgEv[0], st);
            SG_LAUNCH_OV(8, 1, g1, st, a->d_next, 0);
            if (dbg) cudaEventRecord(dbgEv[1], st);
            SG_CUDA(cudaGetLastError());
            a->launches++;
            SG_LAUNCH_OV(4, 2, g2a, a->stream2, a->d_next2, g1 * a->warpsPerBlock);
            SG_CUDA(cudaGetLastError());
            a->launches++;
            // behind the first pass in stream order: one of its CTAs per SM fits beside the second pass's three as soon as the first pass
            // has left; the other two only find room if CTAs of the launch above gave up (see sg_align_kernel), and then do their work
            SG_LAUNCH_OV(4, 2, g2b, st, a->d_next2, (g1 + g2a) * a->warpsPerBlock);
#undef SG_LAUNCH_OV
            SG_CUDA(cudaGetLastError());
            if (dbg) cudaEventRecord(dbgEv[2], st);
            SG_CUDA(cudaEventRecord(a->evJoin, a->stream2));
            SG_CUDA(cudaStreamWaitEvent(st, a->evJoin, 0));
            if (dbg) {
                cudaEventRecord(dbgEv[3], st);
                cudaStreamSynchronize(st);
                float t1 = 0, t2 = 0, t3 = 0; unsigned int c[4] = {0, 0, 0, 0}; unsigned long long deferred = 0;
                cudaEventElapsedTime(&t1, dbgEv[0], dbgEv[1]); cudaEventElapsedTime(&t2, dbgEv[0], dbgEv[2]); cudaEventElapsedTime(&t3, dbgEv[0], dbgEv[3]);
                cudaMemcpy(c, a->d_producersDone, 16, cudaMemcpyDeviceToHost); cudaMemcpy(&deferred, a->d_retryCount, 8, cudaMemcpyDeviceToHost);
                fprintf(stderr, "[overlap] n=%lld p1=%d k2a=%d k2b=%d: first pass %.2f ms, + follow-up consumers %.2f ms, all %.2f ms; producers done %u started %u, consumer CTAs that gave up %u, deferred %llu\n",
                        (long long)n, a->overlapPass1Blocks, k2a, g2b / a->numSMs, t1, t2, t3, c[0], c[1], c[2], deferred);
                for (int k = 0; k < 4; k++) cudaEventDestroy(dbgEv[k]);
            }
        } else if (a->twoPass) {
            SG_CUDA(cudaMemsetAsync(a->d_retryCount, 0, 8, st));
            SG_CUDA(cudaMemsetAsync(a->d_next2, 0, 8, st));
            int64_t w1 = (int64_t)a->numSMs * a->pass1BlocksPerSM * a->warpsPerBlock;
            if (w1 > n) w1 = n;
            if (w1 > a->nWorkers) w1 = a->nWorkers;
            int grid1 = (int)((w1 + a->warpsPerBlock - 1) / a->warpsPerBlock);
            if (grid1 < 1) grid1 = 1;
            switch (a->pass1BlocksPerSM) {
                case 8: SG_LAUNCH(8, 1, grid1, a->d_next); break;
                case 6: SG_LAUNCH(6, 1, grid1, a->d_next); break;
                case 5: SG_LAUNCH(5, 1, grid1, a->d_next); break;
                case 3: SG_LAUNCH(3, 1, grid1, a->d_next); break;
                default: SG_LAUNCH(4, 1, grid1, a->d_next); break;
            }
            SG_CUDA(cudaGetLastError());
            a->launches++;
            int64_t w2 = (int64_t)a->numSMs * a->blocksPerSM * a->warpsPerBlock;
            if (w2 > a->nWorkers) w2 = a->nWorkers;
            if (w2 > n) w2 = n;
            int grid2 = (int)((w2 + a->warpsPerBlock - 1) / a->warpsPerBlock);
            if (grid2 < 1) grid2 = 1;
            SG_LAUNCH_MB(2, grid2, a->d_next2);
        } else {
            SG_LAUNCH_MB(0, blocks, a->d_next);
        }
#undef SG_LAUNCH_MB
#undef SG_LAUNCH
    } else {
        SG_CUDA(cudaMemsetAsync(a->d_retryCount, 0, 8, st));
        SG_CUDA(cudaMemsetAsync(a->d_next2, 0, 8, st));
#define SG_LAUNCH(MB, STAGE, GRID, PP, SCRATCH, BYTES, NEXT, LIST) sg_align_paired_kernel<MB, STAGE><<<GRID, a->warpsPerBlock * 32, 0, st>>>(a->index->view, a->params, \
        a->paramsSingle, PP, a->index->d_tables_prob, SCRATCH, BYTES, a->singleScratchBytes, n, (const uint8_t *)d_bases, (const uint8_t *)d_quals, \
        (const unsigned long long *)d_offsets, d_lens, (snapgpu_paired_result *)d_results, d_counters, NEXT, a->d_error, LIST, a->d_retryCount, a->d_retryList, \
        (SgPairHandoff *)a->d_handoff, a->d_candPool, a->candPoolCap, a->d_candPoolUsed)
#define SG_LAUNCH_MB(STAGE, GRID, PP, SCRATCH, BYTES, NEXT, LIST) \
        if (a->blocksPerSM >= 4) SG_LAUNCH(4, STAGE, GRID, PP, SCRATCH, BYTES, NEXT, LIST); else if (a->blocksPerSM == 3) SG_LAUNCH(3, STAGE, GRID, PP, SCRATCH, BYTES, NEXT, LIST); \
        else SG_LAUNCH(2, STAGE, GRID, PP, SCRATCH, BYTES, NEXT, LIST)
        if (a->staged) {
            SG_CUDA(cudaMemsetAsync(a->d_candPoolUsed, 0, 8, st));
            SG_CUDA(cudaMemsetAsync(a->d_next3, 0, 16, st));
#define SG_GRID(K) ((int)((std::min<int64_t>(std::min<int64_t>((int64_t)a->numSMs * a->stageBlocks[K] * a->warpsPerBlock, a->nWorkers), n) + a->warpsPerBlock - 1) / a->warpsPerBlock))
#define SG_LAUNCH_STAGE(K, NEXT) \
            if (a->stageBlocks[K] == 8) SG_LAUNCH(8, K, SG_GRID(K), a->pparams, a->d_scratch, a->scratchBytesPerWorker, NEXT, (const uint32_t *)nullptr); \
            else if (a->stageBlocks[K] == 6) SG_LAUNCH(6, K, SG_GRID(K), a->pparams, a->d_scratch, a->scratchBytesPerWorker, NEXT, (const uint32_t *)nullptr); \
            else SG_LAUNCH(4, K, SG_GRID(K), a->pparams, a->d_scratch, a->scratchBytesPerWorker, NEXT, (const uint32_t *)nullptr)
            SG_LAUNCH_STAGE(1, a->d_next);
            SG_CUDA(cudaGetLastError());
            a->launches++;
            SG_LAUNCH_STAGE(2, a->d_next3);
            SG_CUDA(cudaGetLastError());
            a->launches++;
            SG_LAUNCH_STAGE(3, a->d_next3 + 1);
#undef SG_LAUNCH_STAGE
#undef SG_GRID
        } else {
            SG_LAUNCH_MB(0, blocks, a->pparams, a->d_scratch, a->scratchBytesPerWorker, a->d_next, (const uint32_t *)nullptr);
        }
        SG_CUDA(cudaGetLastError());
        a->launches++;
        if (a->staged || a->pparams.poolCap < a->pparamsBig.poolCap || a->pparams.agCandCap < a->pparamsBig.agCandCap) {
            // retry pass: exits at once when the list is empty
            SG_LAUNCH_MB(0, a->nBigWorkers / a->warpsPerBlock, a->pparamsBig, a->d_bigScratch, a->bigScratchBytesPerWorker, a->d_next2, (const uint32_t *)a->d_retryList);
            SG_CUDA(cudaGetLastError());
            a->launches++;
        }
#undef SG_LAUNCH_MB
#undef SG_LAUNCH
        return 0;
    }
    SG_CUDA(cudaGetLastError());
    a->launches++;
    return 0;
}

int snapgpu_aligner_check(snapgpu_aligner *a, void *cudaStream)
{
    if (!a) return sg_fail("null argument");
    SG_CUDA(cudaSetDevice(a->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : a->stream;
    int code = 0;
    SG_CUDA(cudaMemcpyAsync(&code, a->d_error, sizeof(int), cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    if (code == 0) return 0;
    SG_CUDA(cudaMemsetAsync(a->d_error, 0, sizeof(int), st));
    SG_CUDA(cudaStreamSynchronize(st));
    if (code == 1) return sg_fail("paired aligner: a scoring candidate / mate / merge-anchor pool overflowed (the reference exits here too; raise -mcp / -H)");
    if (code == 2) return sg_fail("paired aligner: more than 4096 phase-4 affine-gap candidates for one pair (buffer growth is not implemented)");
    if (code == 3) return sg_fail("a read is longer than the aligner's configured maximum (SNAPGPU_MAX_READ_LEN)");
    if (code == 4) return sg_fail("secondary alignments: a worker's raw record buffer overflowed (SNAPGPU_SECONDARY_RAW_CAP; the host entry point grows it by itself)");
    return sg_fail("aligner kernel reported an unknown error");
}

int snapgpu_align_single_device(snapgpu_aligner *a, int64_t n, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                                const uint32_t *d_lens, snapgpu_single_result *d_results, snapgpu_counters *d_counters, void *cudaStream)
{
    if (!a || !d_bases || !d_quals || !d_offsets || !d_lens || !d_results) return sg_fail("null argument");
    if (a->paired) return sg_fail("snapgpu_align_single_device called on a paired-end aligner handle");
    if (a->userParams.maxSecondaryAlignmentAdditionalEditDistance >= 0) return sg_fail("this handle was created with -om: call snapgpu_align_single_secondary_device");
    if (n < 0) return sg_fail("negative read count");
    if (n > a->maxBatchReads) return sg_fail("read count exceeds maxBatchReads (the deferred-read list and arenas are sized from it)");
    if (n == 0) return 0;
    SG_CUDA(cudaSetDevice(a->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : a->stream;
    return launch_align(a, n, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters, st);
}

int snapgpu_align_paired_device(snapgpu_aligner *a, int64_t nPairs, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                                const uint32_t *d_lens, snapgpu_paired_result *d_results, snapgpu_counters *d_counters, void *cudaStream)
{
    if (!a || !d_bases || !d_quals || !d_offsets || !d_lens || !d_results) return sg_fail("null argument");
    if (!a->paired) return sg_fail("snapgpu_align_paired_device called on a single-end aligner handle");
    if (nPairs < 0) return sg_fail("negative pair count");
    if (2 * nPairs > a->maxBatchReads) return sg_fail("pair count exceeds maxBatchPairs (the retry list, hand-off records and candidate pool are sized from it)");
    if (nPairs == 0) return 0;
    SG_CUDA(cudaSetDevice(a->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : a->stream;
    return launch_align(a, nPairs, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters, st);
}

// Drains a pipeline slot: waits for its D2H copy and hands the results to the caller's buffer.
static int drain_slot(snapgpu_aligner *a, int k, uint8_t *results, size_t resultBytesPerUnit, bool resultsPinned)
{
    snapgpu_aligner::Slot &sl = a->slot[k];
    if (sl.pendingCount == 0) return 0;
    SG_CUDA(cudaEventSynchronize(sl.evOut));
    uint8_t *dst = results + (size_t)sl.pendingFirst * resultBytesPerUnit;
    const int64_t count = sl.pendingCount;
    sl.pendingCount = 0;             // whatever happens below, the slot is free again
    if (!resultsPinned) memcpy(dst, sl.h_results, (size_t)count * resultBytesPerUnit);      // (pinned: the DMA wrote them in place)
    if (!a->paired) {
        const snapgpu_single_result *r = (const snapgpu_single_result *)dst;
        for (int64_t i = 0; i < count; i++) {
            if (r[i].reserved == 1) return sg_fail("a read is longer than the aligner's configured maximum (SNAPGPU_MAX_READ_LEN)");
        }
    }
    return 0;
}

// Host-buffer path shared by snapgpu_align_single / snapgpu_align_paired.  nUnits units of readsPerUnit reads each.
// Software pipeline over chunks of reads, two slots: pack chunk c+1 into pinned staging on the host and copy it in
// while the GPU aligns chunk c and chunk c-1's results stream out.  Kernels stay on one stream (they share the arenas).
static int align_host_impl(snapgpu_aligner *a, int64_t nUnits, int readsPerUnit, size_t resultBytesPerUnit, const char *bases, const char *quals,
                           const uint64_t *offsets, const uint32_t *lens, uint8_t *results, snapgpu_counters *counters)
{
    const int64_t n = nUnits * readsPerUnit;
    SG_CUDA(cudaSetDevice(a->device));
    SG_CUDA(cudaMemsetAsync(a->d_counters, 0, sizeof(snapgpu_counters), a->stream));
    bool callerPinned = false, resultsPinned = false;
    {
        cudaPointerAttributes pa, pq, pr;
        if (cudaPointerGetAttributes(&pa, bases) == cudaSuccess && cudaPointerGetAttributes(&pq, quals) == cudaSuccess) {
            callerPinned = pa.type == cudaMemoryTypeHost && pq.type == cudaMemoryTypeHost;
        }
        if (cudaPointerGetAttributes(&pr, results) == cudaSuccess) resultsPinned = pr.type == cudaMemoryTypeHost;
        cudaGetLastError();          // an unregistered pointer is not an error for us
    }
    int64_t done = 0;
    int c = 0;
    while (done < n) {
        const int k = c & 1;
        snapgpu_aligner::Slot &sl = a->slot[k];
        if (drain_slot(a, k, results, resultBytesPerUnit, resultsPinned)) return 1;     // slot k was used by chunk c-2
        int64_t m = 0; size_t total = 0;
        // stage sizes: first small, second the rest of a full stage, then full stages (a batch that fits one stage and a half is not cut up further)
        int64_t want = a->chunkReads;
        if (n > a->chunkReads + a->chunkReads / 2) want = c == 0 ? a->firstChunkReads : (c == 1 ? a->chunkReads - a->firstChunkReads : a->chunkReads);
        else if (n > a->firstChunkReads * 2) want = c == 0 ? a->firstChunkReads : a->chunkReads;
        if (want < readsPerUnit) want = readsPerUnit;
        while (done + m < n && m < want) {
            size_t unitBases = 0;
            for (int w = 0; w < readsPerUnit; w++) {
                const uint32_t len = lens[done + m + w];
                if (len > SNAPGPU_MAX_READ_LENGTH) return sg_fail("read longer than MAX_READ_LENGTH");
                unitBases += len;
            }
            if (total + unitBases > a->chunkBases) break;
            for (int w = 0; w < readsPerUnit; w++) {
                sl.h_offsets[m + w] = total; sl.h_lens[m + w] = lens[done + m + w];
                total += lens[done + m + w];
            }
            m += readsPerUnit;
        }
        if (m == 0) return sg_fail("a read does not fit the aligner's staging buffers");
        // reads that are back to back in the caller's buffers (the common case) are packed with one memcpy each way
        const uint64_t first = offsets[done];
        const char *src_b = sl.h_bases, *src_q = sl.h_quals;
        bool contiguous = true;
        for (int64_t i = 0; i < m; i++) { if (offsets[done + i] != first + sl.h_offsets[i]) { contiguous = false; break; } }
        if (contiguous && callerPinned) {
            // the caller's buffers are page-locked: DMA straight out of them, no staging copy
            src_b = bases + first; src_q = quals + first;
        } else if (contiguous) {
            memcpy(sl.h_bases, bases + first, total);
            memcpy(sl.h_quals, quals + first, total);
        } else {
            for (int64_t i = 0; i < m; i++) {
                memcpy(sl.h_bases + sl.h_offsets[i], bases + offsets[done + i], sl.h_lens[i]);
                memcpy(sl.h_quals + sl.h_offsets[i], quals + offsets[done + i], sl.h_lens[i]);
            }
        }
        SG_CUDA(cudaMemcpyAsync(sl.d_bases, src_b, total, cudaMemcpyHostToDevice, a->streamIn));
        SG_CUDA(cudaMemcpyAsync(sl.d_quals, src_q, total, cudaMemcpyHostToDevice, a->streamIn));
        SG_CUDA(cudaMemcpyAsync(sl.d_offsets, sl.h_offsets, (size_t)m * 8, cudaMemcpyHostToDevice, a->streamIn));
        SG_CUDA(cudaMemcpyAsync(sl.d_lens, sl.h_lens, (size_t)m * 4, cudaMemcpyHostToDevice, a->streamIn));
        SG_CUDA(cudaEventRecord(sl.evIn, a->streamIn));
        SG_CUDA(cudaStreamWaitEvent(a->stream, sl.evIn, 0));
        const int64_t units = m / readsPerUnit;
        if (launch_align(a, units, sl.d_bases, sl.d_quals, sl.d_offsets, sl.d_lens, sl.d_results, a->d_counters, a->stream)) return 1;
        SG_CUDA(cudaEventRecord(sl.evKernel, a->stream));
        SG_CUDA(cudaStreamWaitEvent(a->streamOut, sl.evKernel, 0));
        SG_CUDA(cudaMemcpyAsync(resultsPinned ? (void *)(results + (size_t)(done / readsPerUnit) * resultBytesPerUnit) : (void *)sl.h_results, sl.d_results,
                                (size_t)units * resultBytesPerUnit, cudaMemcpyDeviceToHost, a->streamOut));
        SG_CUDA(cudaEventRecord(sl.evOut, a->streamOut));
        sl.pendingFirst = done / readsPerUnit; sl.pendingCount = units;
        done += m;
        c++;
    }
    if (drain_slot(a, c & 1, results, resultBytesPerUnit, resultsPinned)) return 1;
    if (drain_slot(a, (c + 1) & 1, results, resultBytesPerUnit, resultsPinned)) return 1;
    SG_CUDA(cudaMemcpyAsync(a->h_counters, a->d_counters, sizeof(snapgpu_counters), cudaMemcpyDeviceToHost, a->stream));
    SG_CUDA(cudaStreamSynchronize(a->stream));
    if (a->paired && snapgpu_aligner_check(a, nullptr)) return 1;
    if (counters) {
        int64_t *dst = (int64_t *)counters; const int64_t *src = (const int64_t *)a->h_counters;
        for (size_t k2 = 0; k2 < sizeof(snapgpu_counters) / 8; k2++) dst[k2] += src[k2];
    }
    return 0;
}

// A call that fails part-way (an over-long read, a CUDA error) must not leave work of its own behind: the slots' pending results
// belong to THIS call's buffers, and a D2H copy may still be in flight into them.  Quiesce the three streams and free both slots,
// so the next call on the handle starts clean (it would otherwise drain the stale slot into its own, possibly smaller, buffer).
static int align_host(snapgpu_aligner *a, int64_t nUnits, int readsPerUnit, size_t resultBytesPerUnit, const char *bases, const char *quals,
                      const uint64_t *offsets, const uint32_t *lens, uint8_t *results, snapgpu_counters *counters)
{
    a->slot[0].pendingCount = a->slot[1].pendingCount = 0;
    const int rc = align_host_impl(a, nUnits, readsPerUnit, resultBytesPerUnit, bases, quals, offsets, lens, results, counters);
    if (rc) {
        const std::string keep = g_lastError;
        cudaStreamSynchronize(a->streamIn); cudaStreamSynchronize(a->stream); cudaStreamSynchronize(a->streamOut);
        cudaGetLastError();
        a->slot[0].pendingCount = a->slot[1].pendingCount = 0;
        g_lastError = keep;
    }
    return rc;
}

int snapgpu_align_single(snapgpu_aligner *a, int64_t n, const char *bases, const char *quals, const uint64_t *offsets,
                         const uint32_t *lens, snapgpu_single_result *results, snapgpu_counters *counters)
{
    if (!a || !bases || !quals || !offsets || !lens || !results) return sg_fail("null argument");
    if (a->paired) return sg_fail("snapgpu_align_single called on a paired-end aligner handle");
    if (a->userParams.maxSecondaryAlignmentAdditionalEditDistance >= 0) return sg_fail("this handle was created with -om: call snapgpu_align_single_secondary");
    if (n < 0 || n > a->maxBatchReads) return sg_fail("read count exceeds maxBatchReads");
    if (n == 0) return 0;
    return align_host(a, n, 1, sizeof(snapgpu_single_result), bases, quals, offsets, lens, (uint8_t *)results, counters);
}

// ---- secondary alignments (`-om`) ----
static int secondary_check(snapgpu_aligner *a, int64_t n, int32_t maxSecondaryAlignments, int64_t secondaryCapacityPerRead, const char *who)
{
    if (a->paired) return sg_fail(std::string(who) + " called on a paired-end aligner handle");
    if (a->userParams.maxSecondaryAlignmentAdditionalEditDistance < 0) return sg_fail(std::string(who) + ": the handle was created without -om (maxSecondaryAlignmentAdditionalEditDistance < 0)");
    if (n < 0 || n > a->maxBatchReads) return sg_fail("read count exceeds maxBatchReads");
    if (maxSecondaryAlignments <= 0) return sg_fail("maxSecondaryAlignments (-omax) must be positive");       // AlignerOptions.cpp:619-624
    if (secondaryCapacityPerRead < 0) return sg_fail("negative secondaryCapacityPerRead");
    return 0;
}

static int secondary_reserve(snapgpu_aligner *a, int cap)
{
    if (a->d_secRaw && a->secRawCap >= cap) return 0;
    SG_CUDA(cudaStreamSynchronize(a->stream));
    if (a->d_secRaw) { cudaFree(a->d_secRaw); a->d_secRaw = nullptr; a->secRawCap = 0; }
    SG_CUDA(cudaMalloc((void **)&a->d_secRaw, (size_t)a->nWorkers * (size_t)cap * sizeof(snapgpu_single_result)));
    a->secRawCap = cap;
    return 0;
}

static int launch_align_secondary(snapgpu_aligner *a, int64_t n, const char *d_bases, const char *d_quals, const uint64_t *d_offsets, const uint32_t *d_lens,
                                  snapgpu_single_result *d_results, int32_t maxSecondaryAlignments, int32_t maxSecondaryAlignmentsPerContig,
                                  int64_t secondaryCapacityPerRead, snapgpu_single_result *d_secondary, int32_t *d_nSecondary, snapgpu_counters *d_counters, cudaStream_t st)
{
    if (!a->d_secRaw) {
        int cap = 256;                   // records per worker; the reference starts at 32 per thread and doubles (SingleAligner.cpp:137-142, :259)
        if (const char *e = getenv("SNAPGPU_SECONDARY_RAW_CAP")) cap = atoi(e) > 0 ? atoi(e) : cap;
        if (secondary_reserve(a, cap)) return 1;
    }
    SG_CUDA(cudaMemsetAsync(a->d_next, 0, 8, st));
    int64_t workers = (int64_t)a->numSMs * 4 * a->warpsPerBlock;
    if (workers > a->nWorkers) workers = a->nWorkers;
    if (workers > n) workers = n;
    int blocks = (int)((workers + a->warpsPerBlock - 1) / a->warpsPerBlock);
    if (blocks < 1) blocks = 1;
    sg_align_secondary_kernel<<<blocks, a->warpsPerBlock * 32, 0, st>>>(a->index->view, a->params, a->index->d_tables_prob, a->d_scratch, a->scratchBytesPerWorker,
        n, (const uint8_t *)d_bases, (const uint8_t *)d_quals, (const unsigned long long *)d_offsets, d_lens, d_results, d_counters, a->d_next, a->d_error,
        a->d_secRaw, a->secRawCap, a->userParams.maxSecondaryAlignmentAdditionalEditDistance, maxSecondaryAlignments, maxSecondaryAlignmentsPerContig,
        d_secondary, (long long)secondaryCapacityPerRead, d_nSecondary);
    SG_CUDA(cudaGetLastError());
    a->launches++;
    return 0;
}

int snapgpu_align_single_secondary_device(snapgpu_aligner *a, int64_t n, const char *d_bases, const char *d_quals, const uint64_t *d_offsets, const uint32_t *d_lens,
                                          snapgpu_single_result *d_results, int32_t maxSecondaryAlignments, int32_t maxSecondaryAlignmentsPerContig,
                                          int64_t secondaryCapacityPerRead, snapgpu_single_result *d_secondary, int32_t *d_nSecondary,
                                          snapgpu_counters *d_counters, void *cudaStream)
{
    if (!a || !d_bases || !d_quals || !d_offsets || !d_lens || !d_results || !d_nSecondary || (!d_secondary && secondaryCapacityPerRead > 0)) return sg_fail("null argument");
    if (secondary_check(a, n, maxSecondaryAlignments, secondaryCapacityPerRead, "snapgpu_align_single_secondary_device")) return 1;
    if (n == 0) return 0;
    SG_CUDA(cudaSetDevice(a->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : a->stream;
    return launch_align_secondary(a, n, d_bases, d_quals, d_offsets, d_lens, d_results, maxSecondaryAlignments, maxSecondaryAlignmentsPerContig,
                                  secondaryCapacityPerRead, d_secondary, d_nSecondary, d_counters, st);
}

int snapgpu_align_single_secondary(snapgpu_aligner *a, int64_t n, const char *bases, const char *quals, const uint64_t *offsets, const uint32_t *lens,
                                   snapgpu_single_result *results, int32_t maxSecondaryAlignments, int32_t maxSecondaryAlignmentsPerContig,
                                   int64_t secondaryCapacityPerRead, snapgpu_single_result *secondary, int32_t *nSecondary, snapgpu_counters *counters)
{
    if (!a || !bases || !quals || !offsets || !lens || !results || !nSecondary || (!secondary && secondaryCapacityPerRead > 0)) return sg_fail("null argument");
    if (secondary_check(a, n, maxSecondaryAlignments, secondaryCapacityPerRead, "snapgpu_align_single_secondary")) return 1;
    if (n == 0) return 0;
    SG_CUDA(cudaSetDevice(a->device));
    // a cold path: plain staging, no pipeline.  Reads are packed back to back.
    std::vector<uint64_t> off;
    std::vector<char> hb, hq;
    uint64_t total = 0;
    try {
        off.resize((size_t)n);
        for (int64_t i = 0; i < n; i++) {
            if (lens[i] > a->params.maxReadLen) return sg_fail("a read is longer than the aligner's configured maximum (SNAPGPU_MAX_READ_LEN)");
            off[(size_t)i] = total; total += lens[i];
        }
        hb.resize((size_t)total + 1); hq.resize((size_t)total + 1);
    } catch (const std::bad_alloc &) {
        return sg_fail("snapgpu_align_single_secondary: out of host memory");
    }
    for (int64_t i = 0; i < n; i++) {
        memcpy(hb.data() + off[(size_t)i], bases + offsets[i], lens[i]);
        memcpy(hq.data() + off[(size_t)i], quals + offsets[i], lens[i]);
    }
    char *d_b = nullptr, *d_q = nullptr; uint64_t *d_o = nullptr; uint32_t *d_l = nullptr; snapgpu_single_result *d_r = nullptr, *d_s = nullptr; int32_t *d_n = nullptr;
    const size_t secBytes = (size_t)n * (size_t)secondaryCapacityPerRead * sizeof(snapgpu_single_result);
    int rc = 0;
    auto fail = [&](const std::string &m) { rc = sg_fail(m); };
#define SG_TRY(call) do { if (!rc) { cudaError_t e_ = (call); if (e_ != cudaSuccess) fail(std::string(#call) + ": " + cudaGetErrorString(e_)); } } while (0)
    SG_TRY(cudaMalloc((void **)&d_b, (size_t)total + 1)); SG_TRY(cudaMalloc((void **)&d_q, (size_t)total + 1));
    SG_TRY(cudaMalloc((void **)&d_o, (size_t)n * 8)); SG_TRY(cudaMalloc((void **)&d_l, (size_t)n * 4));
    SG_TRY(cudaMalloc((void **)&d_r, (size_t)n * sizeof(snapgpu_single_result))); SG_TRY(cudaMalloc((void **)&d_n, (size_t)n * 4));
    if (secBytes) SG_TRY(cudaMalloc((void **)&d_s, secBytes));
    cudaStream_t st = a->stream;
    SG_TRY(cudaMemcpyAsync(d_b, hb.data(), (size_t)total, cudaMemcpyHostToDevice, st));
    SG_TRY(cudaMemcpyAsync(d_q, hq.data(), (size_t)total, cudaMemcpyHostToDevice, st));
    SG_TRY(cudaMemcpyAsync(d_o, off.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    SG_TRY(cudaMemcpyAsync(d_l, lens, (size_t)n * 4, cudaMemcpyHostToDevice, st));
    while (!rc) {
        SG_TRY(cudaMemsetAsync(a->d_counters, 0, sizeof(snapgpu_counters), st));
        if (!rc && launch_align_secondary(a, n, d_b, d_q, d_o, d_l, d_r, maxSecondaryAlignments, maxSecondaryAlignmentsPerContig, secondaryCapacityPerRead, d_s, d_n,
                                          a->d_counters, st)) { rc = 1; break; }
        int code = 0;
        SG_TRY(cudaMemcpyAsync(&code, a->d_error, sizeof(int), cudaMemcpyDeviceToHost, st));
        SG_TRY(cudaStreamSynchronize(st));
        if (rc || code == 0) break;
        SG_TRY(cudaMemsetAsync(a->d_error, 0, sizeof(int), st));
        if (code != 4) { fail("aligner kernel reported an error"); break; }
        // a worker's raw buffer filled up: double it and align the batch again (SingleAligner.cpp:250-263 does this per read)
        if (a->secRawCap >= (1 << 16)) { fail("secondary alignments: more than 65536 candidate records for one read"); break; }
        if (secondary_reserve(a, a->secRawCap * 2)) { rc = 1; break; }
    }
    SG_TRY(cudaMemcpyAsync(results, d_r, (size_t)n * sizeof(snapgpu_single_result), cudaMemcpyDeviceToHost, st));
    SG_TRY(cudaMemcpyAsync(nSecondary, d_n, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    if (secBytes) SG_TRY(cudaMemcpyAsync(secondary, d_s, secBytes, cudaMemcpyDeviceToHost, st));
    SG_TRY(cudaMemcpyAsync(a->h_counters, a->d_counters, sizeof(snapgpu_counters), cudaMemcpyDeviceToHost, st));
    SG_TRY(cudaStreamSynchronize(st));
#undef SG_TRY
    cudaFree(d_b); cudaFree(d_q); cudaFree(d_o); cudaFree(d_l); cudaFree(d_r); cudaFree(d_s); cudaFree(d_n);
    if (rc) { const std::string keep = g_lastError; cudaStreamSynchronize(st); cudaGetLastError(); g_lastError = keep; return rc; }
    if (counters) {
        int64_t *dst = (int64_t *)counters; const int64_t *src = (const int64_t *)a->h_counters;
        for (size_t k = 0; k < sizeof(snapgpu_counters) / sizeof(int64_t); k++) dst[k] += src[k];
    }
    return 0;
}

int snapgpu_align_paired(snapgpu_aligner *a, int64_t nPairs, const char *bases, const char *quals, const uint64_t *offsets,
                         const uint32_t *lens, snapgpu_paired_result *results, snapgpu_counters *counters)
{
    if (!a || !bases || !quals || !offsets || !lens || !results) return sg_fail("null argument");
    if (!a->paired) return sg_fail("snapgpu_align_paired called on a single-end aligner handle");
    if (nPairs < 0 || 2 * nPairs > a->maxBatchReads) return sg_fail("pair count exceeds maxBatchPairs");
    if (nPairs == 0) return 0;
    return align_host(a, nPairs, 2, sizeof(snapgpu_paired_result), bases, quals, offsets, lens, (uint8_t *)results, counters);
}

// ------------------------------------------------------------------------------------------------
// Insert-size inference (`snap paired -ins`, sg_spacing.h)
//
// A call aligns its pairs in sub-launches and keeps every pair under the range stock would use for it.  A pair adds at most one
// sample, so a sub-launch of at most d = W - count pairs cannot hold a cut before its last pair ("safe").  A longer one is
// speculative: if the window fills at pair j before its end, the launch's counters are put back, [p, j] is aligned again under
// the same range (for its counters; the records are the same), and the pairs after j go on under the new range.
// Per window update a call makes: two safe sub-launches, then a speculative one of about twice the pairs the window's sample rate
// says are needed, then one of all the pairs left, then the realignment: SG_SPACING_LAUNCHES_PER_UPDATE in all.
// ------------------------------------------------------------------------------------------------
#define SG_SPACING_LAUNCHES_PER_UPDATE 5

static double sg_now_seconds()
{
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct snapgpu_spacing {
    int device = 0;
    int32_t filterFlags = 0;
    int32_t forceSpacing = 0;
    int64_t window = SG_SPACING_WINDOW;
    int32_t minSpacing = 0;
    uint32_t maxSpacing = 0;
    int64_t count = 0, samples = 0, updates = 0;
    int64_t windowPairs = 0, windowSamples = 0;      // pairs aligned and samples taken since the last update: the sample rate
    int64_t subLaunches = 0;
    double statSeconds = 0;
    int64_t *d_window = nullptr, *d_sorted = nullptr, *h_sorted = nullptr;
    void *d_sortTemp = nullptr; size_t sortTempBytes = 0;
    // per-pair scratch of one sub-launch, grown on demand
    int64_t pairCap = 0;
    int64_t *d_dist = nullptr; int32_t *d_flag = nullptr, *d_pos = nullptr;
    void *d_scanTemp = nullptr; size_t scanTempBytes = 0;
    int64_t *d_io = nullptr, *h_io = nullptr;         // [0] inclusive sample count of the sub-launch, [1] the pair that fills the window,
                                                      // [2] the aligner's latched error code
    snapgpu_counters *d_ctrSave = nullptr, *d_ctr = nullptr, *h_ctr = nullptr;
    // staging of the host-buffer entry, grown on demand
    int64_t stagePairs = 0; size_t stageBases = 0;
    char *d_bases = nullptr, *d_quals = nullptr; uint64_t *d_offsets = nullptr; uint32_t *d_lens = nullptr;
    snapgpu_paired_result *d_results = nullptr;
};

__global__ void __launch_bounds__(256) sg_spacing_sample_kernel(int64_t n, const snapgpu_paired_result *results, const uint8_t *bases,
                                                                const unsigned long long *offsets, const uint32_t *lens, uint32_t minReadLength,
                                                                int maxK, uint32_t maxReadLen, int32_t filterFlags, int32_t forceSpacing,
                                                                int64_t *dist, int32_t *flag)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool useful[2], tooLong = false;
    for (int w = 0; w < 2; w++) {
        const uint8_t *b = bases + offsets[2 * i + w];
        const uint32_t len = lens[2 * i + w];
        int countOfNs = 0;
        for (uint32_t k = 0; k < len; k++) countOfNs += b[k] == 'N';
        useful[w] = len >= minReadLength && countOfNs <= maxK;         // as the paired kernel decides it
        tooLong = tooLong || len > maxReadLen;
    }
    if (tooLong) useful[0] = useful[1] = false;
    const int64_t s = sg_spacing_sample(results[i], useful, filterFlags, forceSpacing != 0, SNAPGPU_INVALID_LOCATION_32);
    dist[i] = s;
    flag[i] = s >= 0;
}

// Appends the sub-launch's samples in pair order at `count`; io[1] = the pair whose sample fills the window.
__global__ void __launch_bounds__(256) sg_spacing_append_kernel(int64_t n, const int64_t *dist, const int32_t *pos, int64_t count, int64_t window,
                                                                int64_t *out, int64_t *io)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (i == n - 1) io[0] = pos[i];
    if (dist[i] < 0) return;
    const int64_t k = count + pos[i] - 1;
    if (k < window) out[k] = dist[i];
    if (k == window - 1) io[1] = i;
}

static void spacing_free(snapgpu_spacing *e)
{
    cudaFree(e->d_window); cudaFree(e->d_sorted); cudaFreeHost(e->h_sorted); cudaFree(e->d_sortTemp);
    cudaFree(e->d_dist); cudaFree(e->d_flag); cudaFree(e->d_pos); cudaFree(e->d_scanTemp);
    cudaFree(e->d_io); cudaFreeHost(e->h_io); cudaFree(e->d_ctrSave); cudaFree(e->d_ctr); cudaFreeHost(e->h_ctr);
    cudaFree(e->d_bases); cudaFree(e->d_quals); cudaFree(e->d_offsets); cudaFree(e->d_lens); cudaFree(e->d_results);
}

int snapgpu_spacing_create(const snapgpu_aligner *a, int32_t filterFlags, int64_t window, snapgpu_spacing **out)
{
    if (!a || !out) return sg_fail("null argument");
    *out = nullptr;
    if (!a->paired) return sg_fail("snapgpu_spacing_create: the aligner is not a paired-end one");
    if (window < 0 || window > SG_SPACING_WINDOW) return sg_fail("snapgpu_spacing_create: window must be 0 (262144) or 4..262144");
    if (window == 0) window = SG_SPACING_WINDOW;
    if (window < 4) return sg_fail("snapgpu_spacing_create: window must be 0 (262144) or 4..262144");
    SG_CUDA(cudaSetDevice(a->device));
    snapgpu_spacing *e = new snapgpu_spacing();
    e->device = a->device;
    e->filterFlags = filterFlags;
    e->forceSpacing = a->pparams.forceSpacing;
    e->window = window;
    e->minSpacing = a->pparams.minSpacing;
    e->maxSpacing = a->pparams.maxSpacing;
    cudaError_t err = cudaMalloc((void **)&e->d_window, (size_t)window * 8);
    if (err == cudaSuccess) err = cudaMalloc((void **)&e->d_sorted, (size_t)window * 8);
    if (err == cudaSuccess) err = cudaMallocHost((void **)&e->h_sorted, (size_t)window * 8);
    if (err == cudaSuccess) err = cudaMalloc((void **)&e->d_io, 24);
    if (err == cudaSuccess) err = cudaMallocHost((void **)&e->h_io, 24);
    if (err == cudaSuccess) err = cudaMalloc((void **)&e->d_ctrSave, sizeof(snapgpu_counters));
    if (err == cudaSuccess) err = cudaMalloc((void **)&e->d_ctr, sizeof(snapgpu_counters));
    if (err == cudaSuccess) err = cudaMallocHost((void **)&e->h_ctr, sizeof(snapgpu_counters));
    if (err == cudaSuccess) err = cub::DeviceRadixSort::SortKeys(nullptr, e->sortTempBytes, e->d_window, e->d_sorted, (int)window);
    if (err == cudaSuccess) err = cudaMalloc(&e->d_sortTemp, e->sortTempBytes);
    if (err != cudaSuccess) {
        spacing_free(e); delete e;
        return sg_fail(std::string("snapgpu_spacing_create: ") + cudaGetErrorString(err));
    }
    *out = e;
    return 0;
}

void snapgpu_spacing_destroy(snapgpu_spacing *e)
{
    if (!e) return;
    cudaSetDevice(e->device);
    spacing_free(e);
    delete e;
}

int snapgpu_spacing_get(const snapgpu_spacing *e, int32_t *minSpacing, uint32_t *maxSpacing, int64_t *samples, int64_t *updates)
{
    if (!e) return sg_fail("null argument");
    if (minSpacing) *minSpacing = e->minSpacing;
    if (maxSpacing) *maxSpacing = e->maxSpacing;
    if (samples) *samples = e->samples;
    if (updates) *updates = e->updates;
    return 0;
}

int snapgpu_spacing_timing(const snapgpu_spacing *e, int64_t *subLaunches, double *statSeconds)
{
    if (!e) return sg_fail("null argument");
    if (subLaunches) *subLaunches = e->subLaunches;
    if (statSeconds) *statSeconds = e->statSeconds;
    return 0;
}

static int spacing_reserve(snapgpu_spacing *e, int64_t nPairs)
{
    if (nPairs <= e->pairCap) return 0;
    cudaFree(e->d_dist); cudaFree(e->d_flag); cudaFree(e->d_pos); cudaFree(e->d_scanTemp);
    e->d_dist = nullptr; e->d_flag = e->d_pos = nullptr; e->d_scanTemp = nullptr; e->pairCap = 0;
    SG_CUDA(cudaMalloc((void **)&e->d_dist, (size_t)nPairs * 8));
    SG_CUDA(cudaMalloc((void **)&e->d_flag, (size_t)nPairs * 4));
    SG_CUDA(cudaMalloc((void **)&e->d_pos, (size_t)nPairs * 4));
    SG_CUDA(cub::DeviceScan::InclusiveSum(nullptr, e->scanTempBytes, e->d_flag, e->d_pos, (int)nPairs));
    SG_CUDA(cudaMalloc(&e->d_scanTemp, e->scanTempBytes));
    e->pairCap = nPairs;
    return 0;
}

// The window is full: sort it on the device, and compute the range on the host from the sorted copy.  The two sums must run in
// sorted order to give stock's bits, so on the device they would be one thread's chain of 2 x 262144 dependent double adds; the
// host was chosen on that reasoning, not on a timing of both (see DESIGN §3).  statSeconds times this whole function.
static int spacing_update(snapgpu_spacing *e, cudaStream_t st)
{
    const double t0 = sg_now_seconds();
    SG_CUDA(cub::DeviceRadixSort::SortKeys(e->d_sortTemp, e->sortTempBytes, e->d_window, e->d_sorted, (int)e->window, 0, 64, st));
    SG_CUDA(cudaMemcpyAsync(e->h_sorted, e->d_sorted, (size_t)e->window * 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    int32_t mn = 0, mx = 0;
    sg_spacing_range(e->h_sorted, e->window, &mn, &mx);
    e->minSpacing = mn;
    e->maxSpacing = (uint32_t)mx;            // IntersectingPairedEndAligner::setMaxSpacing(int) into an unsigned
    e->count = 0; e->windowPairs = 0; e->windowSamples = 0;
    e->updates++;
    e->statSeconds += sg_now_seconds() - t0;
    return 0;
}

static int align_paired_ins_impl(snapgpu_aligner *a, snapgpu_spacing *e, int64_t n, const char *d_bases, const char *d_quals,
                                 const uint64_t *d_offsets, const uint32_t *d_lens, snapgpu_paired_result *d_results,
                                 snapgpu_counters *d_counters, cudaStream_t st)
{
    if (spacing_reserve(e, n)) return 1;
    int64_t p = 0;
    int k = 0;                       // sub-launches since the last update in this call
    while (p < n) {
        const int64_t rem = n - p, d = e->window - e->count;
        int64_t c;
        if (k < 2 || rem <= d) c = std::min(rem, d);
        else if (k == 2 && e->windowSamples > 0) c = std::min(rem, std::max(d, (2 * d * e->windowPairs + e->windowSamples - 1) / e->windowSamples));
        else c = rem;
        const bool speculative = c > d;
        if (speculative && d_counters) SG_CUDA(cudaMemcpyAsync(e->d_ctrSave, d_counters, sizeof(snapgpu_counters), cudaMemcpyDeviceToDevice, st));
        a->pparams.minSpacing = a->pparamsBig.minSpacing = e->minSpacing;
        a->pparams.maxSpacing = a->pparamsBig.maxSpacing = e->maxSpacing;
        if (launch_align(a, c, d_bases, d_quals, d_offsets + 2 * p, d_lens + 2 * p, d_results + p, d_counters, st)) return 1;
        e->subLaunches++; k++;
        const int blocks = (int)((c + 255) / 256);
        sg_spacing_sample_kernel<<<blocks, 256, 0, st>>>(c, d_results + p, (const uint8_t *)d_bases, (const unsigned long long *)(d_offsets + 2 * p),
                                                         d_lens + 2 * p, a->params.minReadLength, (int)a->params.maxK, a->params.maxReadLen, e->filterFlags,
                                                         e->forceSpacing, e->d_dist, e->d_flag);
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cub::DeviceScan::InclusiveSum(e->d_scanTemp, e->scanTempBytes, e->d_flag, e->d_pos, (int)c, st));
        SG_CUDA(cudaMemsetAsync(e->d_io + 1, 0xff, 8, st));
        sg_spacing_append_kernel<<<blocks, 256, 0, st>>>(c, e->d_dist, e->d_pos, e->count, e->window, e->d_window, e->d_io);
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cudaMemcpyAsync(e->h_io, e->d_io, 16, cudaMemcpyDeviceToHost, st));
        e->h_io[2] = 0;
        SG_CUDA(cudaMemcpyAsync(&e->h_io[2], a->d_error, sizeof(int), cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        // a kernel error (an over-long read, an overflowed pool) leaves the estimator as it was before this sub-launch
        if (e->h_io[2] != 0) return snapgpu_aligner_check(a, st) ? 1 : sg_fail("aligner kernel reported an error");
        const int64_t cut = e->h_io[1];
        if (cut >= 0 && cut < c - 1) {
            // the window filled inside a speculative sub-launch: only [p, cut] belongs to the old range
            c = cut + 1;
            if (d_counters) {
                SG_CUDA(cudaMemcpyAsync(d_counters, e->d_ctrSave, sizeof(snapgpu_counters), cudaMemcpyDeviceToDevice, st));
                if (launch_align(a, c, d_bases, d_quals, d_offsets + 2 * p, d_lens + 2 * p, d_results + p, d_counters, st)) return 1;
                e->subLaunches++;
            }
        }
        const int64_t taken = std::min(e->h_io[0], d);
        e->count += taken; e->samples += taken;
        e->windowPairs += c; e->windowSamples += taken;
        p += c;
        if (e->count == e->window) {
            if (spacing_update(e, st)) return 1;
            k = 0;
        }
    }
    return 0;
}

// The handle is shared (the drop-in has one per device and one estimator per worker thread): its own range is put back after
// every call.
static int align_paired_ins(snapgpu_aligner *a, snapgpu_spacing *e, int64_t n, const char *d_bases, const char *d_quals,
                            const uint64_t *d_offsets, const uint32_t *d_lens, snapgpu_paired_result *d_results,
                            snapgpu_counters *d_counters, cudaStream_t st)
{
    const int32_t min0 = a->pparams.minSpacing, minBig0 = a->pparamsBig.minSpacing;
    const uint32_t max0 = a->pparams.maxSpacing, maxBig0 = a->pparamsBig.maxSpacing;
    const int rc = align_paired_ins_impl(a, e, n, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters, st);
    a->pparams.minSpacing = min0; a->pparamsBig.minSpacing = minBig0;
    a->pparams.maxSpacing = max0; a->pparamsBig.maxSpacing = maxBig0;
    return rc;
}

static int spacing_check(snapgpu_aligner *a, snapgpu_spacing *e, int64_t nPairs)
{
    if (!a->paired) return sg_fail("snapgpu_align_paired_ins called on a single-end aligner handle");
    if (e->device != a->device) return sg_fail("snapgpu_align_paired_ins: the estimator was created for another device");
    if (nPairs < 0 || 2 * nPairs > a->maxBatchReads) return sg_fail("pair count exceeds maxBatchPairs");
    return 0;
}

int snapgpu_align_paired_ins_device(snapgpu_aligner *a, snapgpu_spacing *e, int64_t nPairs, const char *d_bases, const char *d_quals,
                                    const uint64_t *d_offsets, const uint32_t *d_lens, snapgpu_paired_result *d_results,
                                    snapgpu_counters *d_counters, void *cudaStream)
{
    if (!a || !e || !d_bases || !d_quals || !d_offsets || !d_lens || !d_results) return sg_fail("null argument");
    if (spacing_check(a, e, nPairs)) return 1;
    if (nPairs == 0) return 0;
    SG_CUDA(cudaSetDevice(a->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : a->stream;
    return align_paired_ins(a, e, nPairs, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters, st);
}

// A host-buffer call that cannot hold a cut before its last pair (nPairs <= W - count; the drop-in's batches, mostly): the pipelined
// host path of snapgpu_align_paired under the estimator's range, then the samples from the host copies of the results and reads.
static int align_paired_ins_one_launch(snapgpu_aligner *a, snapgpu_spacing *e, int64_t nPairs, const char *bases, const char *quals,
                                       const uint64_t *offsets, const uint32_t *lens, snapgpu_paired_result *results, snapgpu_counters *counters)
{
    const int32_t min0 = a->pparams.minSpacing, minBig0 = a->pparamsBig.minSpacing;
    const uint32_t max0 = a->pparams.maxSpacing, maxBig0 = a->pparamsBig.maxSpacing;
    a->pparams.minSpacing = a->pparamsBig.minSpacing = e->minSpacing;
    a->pparams.maxSpacing = a->pparamsBig.maxSpacing = e->maxSpacing;
    const int rc = align_host(a, nPairs, 2, sizeof(snapgpu_paired_result), bases, quals, offsets, lens, (uint8_t *)results, counters);
    a->pparams.minSpacing = min0; a->pparamsBig.minSpacing = minBig0;
    a->pparams.maxSpacing = max0; a->pparamsBig.maxSpacing = maxBig0;
    if (rc) return 1;
    e->subLaunches++;
    int64_t taken = 0;
    for (int64_t i = 0; i < nPairs; i++) {
        bool useful[2], tooLong = false;
        for (int w = 0; w < 2; w++) {       // as sg_spacing_sample_kernel decides it
            const char *b = bases + offsets[2 * i + w];
            const uint32_t len = lens[2 * i + w];
            uint32_t countOfNs = 0;
            for (uint32_t k = 0; k < len; k++) countOfNs += b[k] == 'N';
            useful[w] = len >= a->params.minReadLength && countOfNs <= a->params.maxK;
            tooLong = tooLong || len > a->params.maxReadLen;
        }
        if (tooLong) useful[0] = useful[1] = false;
        const int64_t smp = sg_spacing_sample(results[i], useful, e->filterFlags, e->forceSpacing != 0, SNAPGPU_INVALID_LOCATION_32);
        if (smp >= 0) e->h_sorted[taken++] = smp;        // staging only: h_sorted is rewritten by the next update
    }
    if (taken) SG_CUDA(cudaMemcpy(e->d_window + e->count, e->h_sorted, (size_t)taken * 8, cudaMemcpyHostToDevice));
    e->count += taken; e->samples += taken;
    e->windowPairs += nPairs; e->windowSamples += taken;
    if (e->count == e->window && spacing_update(e, a->stream)) return 1;
    return 0;
}

int snapgpu_align_paired_ins(snapgpu_aligner *a, snapgpu_spacing *e, int64_t nPairs, const char *bases, const char *quals,
                             const uint64_t *offsets, const uint32_t *lens, snapgpu_paired_result *results, snapgpu_counters *counters)
{
    if (!a || !e || !bases || !quals || !offsets || !lens || !results) return sg_fail("null argument");
    if (spacing_check(a, e, nPairs)) return 1;
    if (nPairs == 0) return 0;
    SG_CUDA(cudaSetDevice(a->device));
    if (nPairs <= e->window - e->count) return align_paired_ins_one_launch(a, e, nPairs, bases, quals, offsets, lens, results, counters);
    // pack the reads back to back, as the device entry takes them
    std::vector<uint64_t> off((size_t)(2 * nPairs));
    size_t total = 0;
    for (int64_t i = 0; i < 2 * nPairs; i++) {
        if (lens[i] > SNAPGPU_MAX_READ_LENGTH) return sg_fail("read longer than MAX_READ_LENGTH");
        off[i] = total; total += lens[i];
    }
    if (nPairs > e->stagePairs) {
        cudaFree(e->d_offsets); cudaFree(e->d_lens); cudaFree(e->d_results);
        e->d_offsets = nullptr; e->d_lens = nullptr; e->d_results = nullptr; e->stagePairs = 0;
        SG_CUDA(cudaMalloc((void **)&e->d_offsets, (size_t)nPairs * 16));
        SG_CUDA(cudaMalloc((void **)&e->d_lens, (size_t)nPairs * 8));
        SG_CUDA(cudaMalloc((void **)&e->d_results, (size_t)nPairs * sizeof(snapgpu_paired_result)));
        e->stagePairs = nPairs;
    }
    if (total + 1 > e->stageBases) {
        cudaFree(e->d_bases); cudaFree(e->d_quals);
        e->d_bases = e->d_quals = nullptr; e->stageBases = 0;
        SG_CUDA(cudaMalloc((void **)&e->d_bases, total + 1));
        SG_CUDA(cudaMalloc((void **)&e->d_quals, total + 1));
        e->stageBases = total + 1;
    }
    cudaStream_t st = a->stream;
    bool contiguous = true;
    for (int64_t i = 0; i < 2 * nPairs && contiguous; i++) contiguous = offsets[i] == offsets[0] + off[i];
    if (contiguous) {
        SG_CUDA(cudaMemcpyAsync(e->d_bases, bases + offsets[0], total, cudaMemcpyHostToDevice, st));
        SG_CUDA(cudaMemcpyAsync(e->d_quals, quals + offsets[0], total, cudaMemcpyHostToDevice, st));
    } else {
        std::vector<char> b(total), q(total);
        for (int64_t i = 0; i < 2 * nPairs; i++) {
            memcpy(&b[off[i]], bases + offsets[i], lens[i]);
            memcpy(&q[off[i]], quals + offsets[i], lens[i]);
        }
        SG_CUDA(cudaMemcpyAsync(e->d_bases, b.data(), total, cudaMemcpyHostToDevice, st));
        SG_CUDA(cudaMemcpyAsync(e->d_quals, q.data(), total, cudaMemcpyHostToDevice, st));
        SG_CUDA(cudaStreamSynchronize(st));
    }
    SG_CUDA(cudaMemcpyAsync(e->d_offsets, off.data(), (size_t)nPairs * 16, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(e->d_lens, lens, (size_t)nPairs * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemsetAsync(e->d_ctr, 0, sizeof(snapgpu_counters), st));
    if (align_paired_ins(a, e, nPairs, e->d_bases, e->d_quals, e->d_offsets, e->d_lens, e->d_results, e->d_ctr, st)) {
        const std::string keep = g_lastError;
        cudaStreamSynchronize(st); cudaGetLastError();
        g_lastError = keep;
        return 1;
    }
    SG_CUDA(cudaMemcpyAsync(results, e->d_results, (size_t)nPairs * sizeof(snapgpu_paired_result), cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(snapgpu_counters), cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    if (snapgpu_aligner_check(a, nullptr)) return 1;
    if (counters) {
        int64_t *dst = (int64_t *)counters; const int64_t *src = (const int64_t *)e->h_ctr;
        for (size_t k = 0; k < sizeof(snapgpu_counters) / 8; k++) dst[k] += src[k];
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// FASTQ ingest
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// Output stage (SURVEY 8f N1): SAM records on the device.
// ONE OCTET OF THREADS PER READ (pair): the eight threads of an aligned octet of a warp are the eight SSE lanes of the reference's
// AffineGapVectorizedWithCigar vectors (sg_ag_cigar.h: SgV8) -- the DP that regenerates the CIGAR of every read with a mismatch is the
// bulk of the writer's work -- and run everything else of SAMFormat::writeRead / writePairs (sg_lv_cigar.h, sg_cigar.h, sg_sam.h)
// identically, storing the same values.  Four reads per warp.  Each record goes into a slot; a scan of the record lengths and a
// warp-per-record copy then pack the slots into contiguous text on the device, so only the text crosses the bus.
// ------------------------------------------------------------------------------------------------
struct SgSamScratchLayout { size_t lvInts, agVec, agRows, agRes, perOctet; uint32_t maxReadLen; };

static SgSamScratchLayout sam_layout(uint32_t maxReadLen)
{
    SgSamScratchLayout l;
    l.maxReadLen = maxReadLen;
    l.lvInts = sg_lv_cigar_scratch_ints(SG_MAX_K - 1);
    // vectors per row: unbanded ceil(P/8); banded numSeg * numVec < P/8 + numVec with numVec <= ceil(P/24) (banded only when P >= 3(2k+1))
    l.agVec = (size_t)maxReadLen / 8 + (size_t)maxReadLen / 24 + 4;
    l.agRows = (size_t)maxReadLen + SG_MAX_K + 8;
    l.agRes = 2 * l.agRows;
    size_t b = 0;
    b += sg_align_up(l.lvInts * 4, 256) * 2 + sg_align_up(l.lvInts, 256);                 // L, totalIndels, A
    b += sg_align_up((SG_MAX_K + 2) * 4, 256) * 2 + sg_align_up(SG_MAX_K + 2, 256);      // btMatched, btD, btAction
    b += sg_align_up(l.agVec * 8 * 2, 256) * 3 + sg_align_up(5 * l.agVec * 8 * 2, 256);  // H, Hm1, E, prof
    b += sg_align_up(l.agRows * l.agVec * 8, 256);                                        // bt
    b += sg_align_up(l.agRes, 256) + sg_align_up(l.agRes * 4, 256);                       // resAction, resCount
    b += sg_align_up((size_t)maxReadLen + 16, 256) * 4;                                   // data, quality x2
    l.perOctet = b;
    return l;
}

__device__ static void sam_carve(const SgSamScratchLayout &l, uint8_t *q, SgSamContext *C)
{
    C->lv.kmax = SG_MAX_K - 1;
    C->lv.L = (int *)q; q += sg_align_up(l.lvInts * 4, 256);
    C->lv.totalIndels = (int *)q; q += sg_align_up(l.lvInts * 4, 256);
    C->lv.A = q; q += sg_align_up(l.lvInts, 256);
    C->lv.btMatched = (int *)q; q += sg_align_up((SG_MAX_K + 2) * 4, 256);
    C->lv.btD = (int *)q; q += sg_align_up((SG_MAX_K + 2) * 4, 256);
    C->lv.btAction = q; q += sg_align_up(SG_MAX_K + 2, 256);
    C->agS.numVecMax = (int)l.agVec; C->agS.rowsMax = (int)l.agRows; C->agS.resMax = (int)l.agRes;
    C->agS.H = (int16_t *)q; q += sg_align_up(l.agVec * 8 * 2, 256);
    C->agS.Hm1 = (int16_t *)q; q += sg_align_up(l.agVec * 8 * 2, 256);
    C->agS.E = (int16_t *)q; q += sg_align_up(l.agVec * 8 * 2, 256);
    C->agS.prof = (int16_t *)q; q += sg_align_up(5 * l.agVec * 8 * 2, 256);
    C->agS.bt = q; q += sg_align_up(l.agRows * l.agVec * 8, 256);
    C->agS.resAction = q; q += sg_align_up(l.agRes, 256);
    C->agS.resCount = (int *)q; q += sg_align_up(l.agRes * 4, 256);
    C->data = q; q += sg_align_up((size_t)l.maxReadLen + 16, 256);
    C->quality = q; q += sg_align_up((size_t)l.maxReadLen + 16, 256);
    C->data2 = q; q += sg_align_up((size_t)l.maxReadLen + 16, 256);
    C->quality2 = q;
}

// MB = resident CTAs (of 256 threads = 32 octets) per SM the instantiation is compiled for: the kernel is bound by the latency of each
// read's serial chain, so more resident octets win as long as the register cap does not cost more in spills (see DESIGN.md).
extern "C++" {
template <int MB>
__global__ void __launch_bounds__(256, MB)
sg_sam_kernel(const __grid_constant__ SgIndexView ix, SgSamScratchLayout lay, uint8_t *scratch, const char *const *contigNames, const char *readGroupAux,
              SgAgParams ag, int useM, int useAffineGap, long long nUnits, int paired, const uint8_t *bases, const uint8_t *quals,
              const unsigned long long *offsets, const uint32_t *lens, const uint8_t *ids, const unsigned long long *idOffsets, const uint32_t *idLens,
              const snapgpu_single_result *single, const snapgpu_paired_result *pairs, const uint32_t *frontClipped, const uint32_t *clippedLens,
              char *slots, uint32_t slotBytes, uint32_t *recordBytes, int bam, const uint8_t *rgAuxBam, int rgAuxBamLen,
              long long *sortLocations, uint32_t *sortBytes)
{
    SgBamContext Bc; Bc.readGroupAux = rgAuxBam; Bc.readGroupAuxLen = rgAuxBamLen;
    const long long octet = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const long long nOctets = ((long long)gridDim.x * blockDim.x) >> 3;
    SgSamContext C;
    C.ix = &ix; C.contigName = contigNames; C.ag = ag; C.readGroupAux = readGroupAux; C.useM = useM != 0; C.useAffineGap = useAffineGap != 0;
    sam_carve(lay, scratch + (size_t)octet * lay.perOctet, &C);
    SgSortInfo si;
    C.sort = &si;
    for (long long u = octet; u < nUnits; u += nOctets) {
        char *out = slots + (size_t)u * slotBytes;
        uint32_t n;
        si.nRecords = 0;
        if (!paired) {
            SgSamRead R;
            R.unclippedData = bases + offsets[u]; R.unclippedQuality = quals + offsets[u]; R.unclippedLength = lens[u];
            R.frontClipped = frontClipped ? frontClipped[u] : 0u; R.dataLength = clippedLens ? clippedLens[u] : lens[u];      // quality clipping (Read::clip), if any
            R.id = ids + idOffsets[u]; R.idLength = idLens[u];
            R.additionalFrontClipping = 0; R.additionalBackClipping = 0;
            const snapgpu_single_result &r = single[u];
            SgSamResult sr;
            sr.status = r.status; sr.location = r.status == SNAPGPU_NOT_FOUND ? -1 : r.location; sr.direction = r.direction; sr.mapq = r.mapq; sr.score = r.score;
            sr.scorePriorToClipping = r.scorePriorToClipping; sr.usedAffineGapScoring = r.usedAffineGapScoring; sr.basesClippedBefore = r.basesClippedBefore;
            sr.basesClippedAfter = r.basesClippedAfter; sr.clippingForReadAdjustment = r.clippingForReadAdjustment;
            n = bam ? (uint32_t)sg_bam_write_single(C, Bc, R, sr, (uint8_t *)out) : (uint32_t)sg_sam_write_single(C, R, sr, out);
        } else {
            SgSamRead R[2];
            for (int w = 0; w < 2; w++) {
                const long long k = 2 * u + w;
                R[w].unclippedData = bases + offsets[k]; R[w].unclippedQuality = quals + offsets[k]; R[w].unclippedLength = lens[k];
                R[w].frontClipped = frontClipped ? frontClipped[k] : 0u; R[w].dataLength = clippedLens ? clippedLens[k] : lens[k];
                R[w].id = ids + idOffsets[k]; R[w].idLength = idLens[k];
                R[w].additionalFrontClipping = 0; R[w].additionalBackClipping = 0;
            }
            const snapgpu_paired_result &r = pairs[u];
            SgSamPairResult pr;
            for (int w = 0; w < 2; w++) {
                pr.status[w] = r.status[w]; pr.location[w] = r.location[w]; pr.direction[w] = r.direction[w]; pr.mapq[w] = r.mapq[w]; pr.score[w] = r.score[w];
                pr.usedAffineGapScoring[w] = r.usedAffineGapScoring[w]; pr.basesClippedBefore[w] = r.basesClippedBefore[w]; pr.basesClippedAfter[w] = r.basesClippedAfter[w];
                pr.clippingForReadAdjustment[w] = r.clippingForReadAdjustment[w];
            }
            pr.alignedAsPair = r.alignedAsPair;
            n = bam ? (uint32_t)sg_bam_write_pair(C, Bc, R[0], R[1], pr, out) : (uint32_t)sg_sam_write_pair(C, R[0], R[1], pr, out);
        }
        recordBytes[u] = n > slotBytes ? 0u : n;
        if ((threadIdx.x & 7) == 0) {          // what a sorting writer files each record under (row N4)
            const long long r0 = paired ? 2 * u : u;
            for (int k = 0; k < (paired ? 2 : 1); k++) {
                sortLocations[r0 + k] = k < si.nRecords ? (long long)si.location[k] : SG_SORT_UNALIGNED;
                sortBytes[r0 + k] = k < si.nRecords ? si.bytes[k] : 0u;
            }
        }
        __syncwarp(0xffu << (threadIdx.x & 24u));        // the octet leaves its scratch together
    }
}

}   // extern "C++"

// packs the slots: warp per record (pair of records)
__global__ void sg_sam_pack_kernel(const char *slots, uint32_t slotBytes, const uint32_t *recordBytes, const unsigned long long *recordOffsets, long long nUnits, char *text,
                                   unsigned long long textCapacity, int *overflow)
{
    const int lane = threadIdx.x & 31;
    const long long nW = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long u = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < nUnits; u += nW) {
        const uint32_t n = recordBytes[u];
        const unsigned long long off = recordOffsets[u];
        if (n == 0) { if (lane == 0) atomicMax(overflow, 1); continue; }                 // a record that could not be formatted
        if (off + n > textCapacity) { if (lane == 0) atomicMax(overflow, 2); continue; }
        const char *src = slots + (size_t)u * slotBytes;
        for (uint32_t k = lane; k < n; k += 32) text[off + k] = src[k];
    }
}

struct snapgpu_sam {
    const snapgpu_index *index = nullptr;
    int device = 0;
    SgSamScratchLayout lay;
    SgAgParams ag;
    int useM = 1, useAffineGap = 1;
    int64_t maxBatchReads = 0;
    int64_t nOctets = 0;
    int format = SNAPGPU_FORMAT_SAM;
    uint8_t *d_rgAuxBam = nullptr; int rgAuxBamLen = 0;
    int ctasPerSM = 4;
    uint32_t slotBytes = 0;
    size_t stageBases = 0;
    uint8_t *d_scratch = nullptr; size_t scratchBytes = 0;
    char *d_names = nullptr; const char **d_namePtrs = nullptr; char *d_rgAux = nullptr;
    uint32_t maxNameLen = 0;
    // staging of the host-buffer call
    uint8_t *d_bases = nullptr, *d_quals = nullptr, *d_ids = nullptr, *d_results = nullptr;
    unsigned long long *d_offsets = nullptr, *d_idOffsets = nullptr, *d_recordOffsets = nullptr;
    uint32_t *d_lens = nullptr, *d_idLens = nullptr, *d_recordBytes = nullptr, *d_front = nullptr, *d_clippedLens = nullptr;
    char *d_slots = nullptr; size_t slotsBytes = 0;
    char *d_text = nullptr; size_t textBytes = 0;
    void *d_cub = nullptr; size_t cubBytes = 0;
    int *d_overflow = nullptr;
    // row N4: what the last format call filed each RECORD under (2 per pair, in the order written), for snapgpu_sam_sort_device
    long long *d_sortLocations = nullptr; uint32_t *d_sortBytes = nullptr;
    int32_t *d_contigOriginal = nullptr;
    unsigned long long *d_sortKeys = nullptr, *d_sortKeysOut = nullptr, *d_recOffsets = nullptr, *d_sortedOffsets = nullptr;
    uint32_t *d_perm = nullptr, *d_permOut = nullptr, *d_sortedBytes = nullptr;
    int64_t lastRecords = 0, lastUnits = 0; int lastPaired = 0;
    unsigned long long *h_meta = nullptr;        // pinned: [0] last offset, [1] last length (low word), [2] overflow
    cudaStream_t stream = nullptr;
    // row N4 after the sort (snapgpu_bam_markdup_device / snapgpu_bam_index_device): work arrays, grown on demand
    void *d_post = nullptr; size_t postBytes = 0;
    int64_t *d_contigStartByOriginal = nullptr;
    std::vector<int64_t> h_contigStartByOriginal, h_contigSpan;
};

void snapgpu_sam_destroy(snapgpu_sam *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    cudaDeviceSynchronize();
    cudaFree(s->d_scratch); cudaFree(s->d_names); cudaFree((void *)s->d_namePtrs); cudaFree(s->d_rgAux); cudaFree(s->d_bases); cudaFree(s->d_quals); cudaFree(s->d_ids);
    cudaFree(s->d_results); cudaFree(s->d_offsets); cudaFree(s->d_idOffsets); cudaFree(s->d_lens); cudaFree(s->d_idLens); cudaFree(s->d_recordBytes); cudaFree(s->d_front); cudaFree(s->d_clippedLens); cudaFree(s->d_slots);
    cudaFree(s->d_recordOffsets); cudaFree(s->d_text); cudaFree(s->d_cub); cudaFree(s->d_overflow); cudaFreeHost(s->h_meta); cudaFree(s->d_rgAuxBam);
    cudaFree(s->d_sortLocations); cudaFree(s->d_sortBytes); cudaFree(s->d_contigOriginal); cudaFree(s->d_sortKeys); cudaFree(s->d_sortKeysOut); cudaFree(s->d_recOffsets);
    cudaFree(s->d_sortedOffsets); cudaFree(s->d_perm); cudaFree(s->d_permOut); cudaFree(s->d_sortedBytes); cudaFree(s->d_post); cudaFree(s->d_contigStartByOriginal);
    if (s->stream) cudaStreamDestroy(s->stream);
    delete s;
}

#define SG_SAM_MAX_ID 256

int snapgpu_sam_create(const snapgpu_index *idx, const snapgpu_params *params, int32_t useM, int64_t maxBatchReads, snapgpu_sam **out)
{
    if (!idx || !params || !out) return sg_fail("null argument");
    *out = nullptr;
    if (require_device(idx->device)) return 1;
    if (maxBatchReads <= 0) return sg_fail("maxBatchReads must be positive");
    snapgpu_sam *s = new (std::nothrow) snapgpu_sam;
    if (!s) return sg_fail("out of memory");
    s->index = idx; s->device = idx->device; s->maxBatchReads = maxBatchReads;
    s->ag = sg_ag_params(params->matchReward, params->subPenalty, params->gapOpenPenalty, params->gapExtendPenalty, 0, 0);
    s->useM = useM != 0; s->useAffineGap = params->useAffineGap != 0;
    cudaDeviceProp prop;
    SG_CUDA(cudaGetDeviceProperties(&prop, s->device));
    s->ctasPerSM = 4;                    // the fastest of 2, 4, 6 and 8 in a sweep
    if (const char *e = getenv("SNAPGPU_SAM_CTAS_PER_SM")) { const int v = atoi(e); if (v == 2 || v == 3 || v == 4 || v == 6 || v == 8) s->ctasPerSM = v; }
    s->nOctets = (int64_t)prop.multiProcessorCount * s->ctasPerSM * 256 / 8;
    // contig names and the default read group line (ReaderContext::defaultReadGroupAux for the default read group "FASTQ")
    std::string blob; std::vector<size_t> off;
    for (size_t c = 0; c < idx->h_contigName.size(); c++) {
        off.push_back(blob.size()); blob += idx->h_contigName[c]; blob.push_back('\0');
        if (idx->h_contigName[c].size() > s->maxNameLen) s->maxNameLen = (uint32_t)idx->h_contigName[c].size();
    }
    const char rg[] = "\tRG:Z:FASTQ\tPL:Z:Illumina\tPU:Z:pu\tLB:Z:lb\tSM:Z:sm";
    size_t c1 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, c1, (uint32_t *)nullptr, (unsigned long long *)nullptr, (int)maxBatchReads);
    size_t c2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, c2, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (int)maxBatchReads);
    s->cubBytes = (c1 > c2 ? c1 : c2) + 256;
    bool ok = cudaMalloc((void **)&s->d_names, blob.size() + 16) == cudaSuccess && cudaMalloc((void **)&s->d_namePtrs, (off.size() + 1) * sizeof(char *)) == cudaSuccess &&
              cudaMalloc((void **)&s->d_rgAux, sizeof(rg)) == cudaSuccess;
    ok = ok && cudaMalloc((void **)&s->d_ids, (size_t)maxBatchReads * SG_SAM_MAX_ID + 16) == cudaSuccess &&
         cudaMalloc((void **)&s->d_results, (size_t)maxBatchReads * sizeof(snapgpu_paired_result)) == cudaSuccess &&
         cudaMalloc((void **)&s->d_offsets, (size_t)maxBatchReads * 8) == cudaSuccess && cudaMalloc((void **)&s->d_idOffsets, (size_t)maxBatchReads * 8) == cudaSuccess &&
         cudaMalloc((void **)&s->d_lens, (size_t)maxBatchReads * 4) == cudaSuccess && cudaMalloc((void **)&s->d_idLens, (size_t)maxBatchReads * 4) == cudaSuccess &&
         cudaMalloc((void **)&s->d_recordBytes, (size_t)maxBatchReads * 4) == cudaSuccess && cudaMalloc((void **)&s->d_recordOffsets, (size_t)maxBatchReads * 8) == cudaSuccess &&
         cudaMalloc((void **)&s->d_front, (size_t)maxBatchReads * 4) == cudaSuccess && cudaMalloc((void **)&s->d_clippedLens, (size_t)maxBatchReads * 4) == cudaSuccess &&
         cudaMalloc((void **)&s->d_cub, s->cubBytes) == cudaSuccess && cudaMalloc((void **)&s->d_overflow, sizeof(int)) == cudaSuccess &&
         cudaMalloc((void **)&s->d_sortLocations, (size_t)maxBatchReads * 8) == cudaSuccess && cudaMalloc((void **)&s->d_sortBytes, (size_t)maxBatchReads * 4) == cudaSuccess &&
         cudaMalloc((void **)&s->d_sortKeys, (size_t)maxBatchReads * 8) == cudaSuccess && cudaMalloc((void **)&s->d_sortKeysOut, (size_t)maxBatchReads * 8) == cudaSuccess &&
         cudaMalloc((void **)&s->d_recOffsets, (size_t)maxBatchReads * 8) == cudaSuccess && cudaMalloc((void **)&s->d_sortedOffsets, (size_t)maxBatchReads * 8 + 8) == cudaSuccess &&
         cudaMalloc((void **)&s->d_perm, (size_t)maxBatchReads * 4) == cudaSuccess && cudaMalloc((void **)&s->d_permOut, (size_t)maxBatchReads * 4) == cudaSuccess &&
         cudaMalloc((void **)&s->d_sortedBytes, (size_t)maxBatchReads * 4) == cudaSuccess &&
         cudaMalloc((void **)&s->d_contigOriginal, idx->h_contigOriginal.size() * 4 + 16) == cudaSuccess &&
         cudaMallocHost((void **)&s->h_meta, 4 * sizeof(unsigned long long)) == cudaSuccess &&
         cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) == cudaSuccess;
    if (!ok) {
        std::string msg = std::string("snapgpu_sam_create: ") + cudaGetErrorString(cudaGetLastError());
        snapgpu_sam_destroy(s);
        return sg_fail(msg);
    }
    std::vector<const char *> ptrs;
    for (size_t c = 0; c < off.size(); c++) ptrs.push_back(s->d_names + off[c]);
    SG_CUDA(cudaMemcpy(s->d_names, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    if (!ptrs.empty()) SG_CUDA(cudaMemcpy((void *)s->d_namePtrs, ptrs.data(), ptrs.size() * sizeof(char *), cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(s->d_rgAux, rg, sizeof(rg), cudaMemcpyHostToDevice));
    if (idx->h_contigOriginal.size() != idx->h_contigStart.size()) { snapgpu_sam_destroy(s); return sg_fail("snapgpu_sam_create: index without original contig numbers"); }
    SG_CUDA(cudaMemcpy(s->d_contigOriginal, idx->h_contigOriginal.data(), idx->h_contigOriginal.size() * 4, cudaMemcpyHostToDevice));
    {
        // beginningLocation by ORIGINAL contig number (what a BAM record's refID is), and an upper bound of each contig's length
        const size_t nc = idx->h_contigStart.size();
        s->h_contigStartByOriginal.assign(nc, 0); s->h_contigSpan.assign(nc, 0);
        for (size_t c = 0; c < nc; c++) {
            const int32_t o = idx->h_contigOriginal[c];
            if (o < 0 || (size_t)o >= nc) { snapgpu_sam_destroy(s); return sg_fail("snapgpu_sam_create: original contig numbers are not a permutation"); }
            s->h_contigStartByOriginal[o] = idx->h_contigStart[c];
            s->h_contigSpan[o] = (c + 1 < nc ? idx->h_contigStart[c + 1] : (int64_t)idx->view.nBases) - idx->h_contigStart[c];
        }
        SG_CUDA(cudaMalloc((void **)&s->d_contigStartByOriginal, nc * 8 + 8));
        SG_CUDA(cudaMemcpy(s->d_contigStartByOriginal, s->h_contigStartByOriginal.data(), nc * 8, cudaMemcpyHostToDevice));
    }
    // the same read group line as BAM tags (ReaderContext::defaultReadGroupAux for a BAM writer): the literal's terminating NUL ends the last tag
    static const char rgBam[] = "RGZFASTQ\0PLZIllumina\0PUZpu\0LBZlb\0SMZsm";
    s->rgAuxBamLen = (int)sizeof(rgBam);
    SG_CUDA(cudaMalloc((void **)&s->d_rgAuxBam, sizeof(rgBam)));
    SG_CUDA(cudaMemcpy(s->d_rgAuxBam, rgBam, sizeof(rgBam), cudaMemcpyHostToDevice));
    *out = s;
    return 0;
}

// The file header in front of the records (host code: sg_samheader.h): SAM text, or the BAM header block when the handle is in SNAPGPU_FORMAT_BAM.
int snapgpu_sam_header(const snapgpu_sam *s, int sorted, const char *commandLine, const char *version, const char *rgLine, char *out, int64_t outCapacity, int64_t *outBytes)
{
    if (!s || !out || !outBytes) return sg_fail("null argument");
    *outBytes = 0;
    const snapgpu_index *ix = s->index;
    try {
        std::vector<SgHeaderContig> contigs;
        if (!sg_header_contigs(ix->h_contigName, ix->h_contigStart, ix->h_contigIsAlt, ix->h_contigOriginal, ix->view.nBases, ix->view.chromosomePadding, &contigs))
            return sg_fail("snapgpu_sam_header: the index has no usable contig table");
        std::vector<uint8_t> o;
        if (s->format == SNAPGPU_FORMAT_BAM) o = sg_bam_header(contigs, sorted != 0, commandLine, version, rgLine);
        else { const std::string t = sg_sam_header_text(contigs, sorted != 0, commandLine, version, rgLine); o.assign(t.begin(), t.end()); }
        if ((int64_t)o.size() > outCapacity) return sg_fail("snapgpu_sam_header: output buffer too small");
        memcpy(out, o.data(), o.size());
        *outBytes = (int64_t)o.size();
    } catch (const std::bad_alloc &) {
        return sg_fail("snapgpu_sam_header: out of host memory");
    }
    return 0;
}

int snapgpu_sam_set_format(snapgpu_sam *s, int format)
{
    if (!s) return sg_fail("null argument");
    if (format != SNAPGPU_FORMAT_SAM && format != SNAPGPU_FORMAT_BAM) return sg_fail("snapgpu_sam_set_format: unknown format");
    if (format == SNAPGPU_FORMAT_BAM) {
        // A BAM record's refID / next_refID index the header's reference table, which is in ORIGINAL contig order (BAMFormat::writeHeader, Bam.cpp:1012-1023);
        // the record writer here files the internal contig number.  The two differ only for a FASTA whose ALT contigs are not already last (the reference's
        // indexer then moves them behind the primary ones): found by the host-side sweep over an ALT-bearing index after the round's GPU budget was
        // spent, so the mapping is not in the kernel yet -- SAM records (names, not numbers) and the header are right on such an index, BAM is refused.
        const std::vector<int32_t> &o = s->index->h_contigOriginal;
        for (size_t c = 0; c < o.size(); c++)
            if (o[c] != (int32_t)c) return sg_fail("snapgpu_sam_set_format: BAM records on an index whose contigs were reordered (ALT contigs not last in the FASTA) "
                                                   "are not supported yet (refID is the original contig number); SAM is");
    }
    s->format = format;
    return 0;
}

// ---- BGZF (the container of a BAM file; reference SNAPLib/GzipDataWriter.cpp + Bam.cpp): the payload cut into members of at most 0xff00 bytes,
//      each a gzip member with the 'BC' extra field carrying its size.  The deflate stream of a member is ONE STORED block (BTYPE = 00): valid
//      BGZF that any BAM reader inflates to exactly the payload, without a compressor on the device. ----
#define SG_BGZF_PAYLOAD 0xff00u
// CRC-32 arithmetic on the reflected polynomial (zlib's crc32_combine): a * b mod P, and x^(8 n) mod P by squaring
__device__ __forceinline__ uint32_t sg_crc_multmodp(uint32_t a, uint32_t b)
{
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1u)) == 0) break; }
        m >>= 1;
        b = (b & 1u) ? (b >> 1) ^ 0xedb88320u : b >> 1;
    }
    return p;
}
__device__ __forceinline__ uint32_t sg_crc_x8n(const uint32_t *x2n, uint32_t nBytes)       // x2n[k] = x^(2^k) mod P
{
    uint32_t p = 1u << 31, k = 3;
    while (nBytes) { if (nBytes & 1u) p = sg_crc_multmodp(x2n[k & 31u], p); nBytes >>= 1; k++; }
    return p;
}
// One CTA per member.  The threads copy the payload; each also runs the table CRC over its own 1/256th of it, and thread 0 joins the 256 partial CRCs
// (crc(A || B) = crc(A) * x^(8 |B|) + crc(B) over GF(2)[x] / P): ~255 dependent table steps per thread and 255 modular products instead of 65 280
// steps on one thread.
__global__ void __launch_bounds__(256)
sg_bgzf_kernel(const uint8_t *in, unsigned long long nBytes, uint8_t *out, unsigned long long nBlocks)
{
    __shared__ uint32_t table[256];
    __shared__ uint32_t part[256];
    __shared__ uint32_t x2n[32];
    {
        uint32_t c = threadIdx.x;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (0xedb88320u ^ (c >> 1)) : (c >> 1);
        table[threadIdx.x] = c;
    }
    if (threadIdx.x == 0) { uint32_t v = 1u << 30; x2n[0] = v; for (int k = 1; k < 32; k++) { v = sg_crc_multmodp(v, v); x2n[k] = v; } }
    __syncthreads();
    for (unsigned long long b = blockIdx.x; b < nBlocks; b += gridDim.x) {
        const unsigned long long off = b * SG_BGZF_PAYLOAD;
        const uint32_t len = (uint32_t)((nBytes - off) < SG_BGZF_PAYLOAD ? (nBytes - off) : SG_BGZF_PAYLOAD);
        uint8_t *o = out + b * (unsigned long long)(SG_BGZF_PAYLOAD + 31u);      // members are laid at a fixed pitch; the host (or a scan) closes the gaps
        const uint8_t *src = in + off;
        for (uint32_t k = threadIdx.x; k < len; k += blockDim.x) o[23 + k] = src[k];
        const uint32_t slice = (len + 255u) / 256u;
        {
            const uint32_t lo = threadIdx.x * slice < len ? threadIdx.x * slice : len, hi = lo + slice < len ? lo + slice : len;
            uint32_t crc = 0xffffffffu;
            for (uint32_t k = lo; k < hi; k++) crc = table[(crc ^ src[k]) & 0xffu] ^ (crc >> 8);
            part[threadIdx.x] = crc ^ 0xffffffffu;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t xs = sg_crc_x8n(x2n, slice);
            uint32_t crc = part[0];
            for (uint32_t t = 1; t < 256u; t++) {
                const uint32_t lo = t * slice < len ? t * slice : len, hi = lo + slice < len ? lo + slice : len;
                if (hi == lo) break;
                crc = sg_crc_multmodp(hi - lo == slice ? xs : sg_crc_x8n(x2n, hi - lo), crc) ^ part[t];
            }
            const uint32_t total = len + 31u;
            const uint8_t hdr[18] = {31, 139, 8, 4, 0, 0, 0, 0, 0, 255, 6, 0, 'B', 'C', 2, 0, (uint8_t)((total - 1u) & 0xffu), (uint8_t)((total - 1u) >> 8)};
            for (int k = 0; k < 18; k++) o[k] = hdr[k];
            o[18] = 1; o[19] = (uint8_t)(len & 0xffu); o[20] = (uint8_t)(len >> 8); o[21] = (uint8_t)(~len & 0xffu); o[22] = (uint8_t)((~len >> 8) & 0xffu);
            uint8_t *t = o + 23 + len;
            t[0] = (uint8_t)crc; t[1] = (uint8_t)(crc >> 8); t[2] = (uint8_t)(crc >> 16); t[3] = (uint8_t)(crc >> 24);
            t[4] = (uint8_t)len; t[5] = (uint8_t)(len >> 8); t[6] = 0; t[7] = 0;
        }
        __syncthreads();
    }
}

// All but the last member are full (pitch = their size), so the output is already contiguous: nBlocks - 1 full members + the last one.
int snapgpu_bgzf_device(const char *d_in, int64_t nBytes, char *d_out, int64_t outCapacity, int64_t *outBytes, void *cudaStream)
{
    if (!d_in || !d_out || !outBytes || nBytes < 0) return sg_fail("bad argument");
    *outBytes = 0;
    if (nBytes == 0) return 0;
    const unsigned long long nBlocks = ((unsigned long long)nBytes + SG_BGZF_PAYLOAD - 1) / SG_BGZF_PAYLOAD;
    const unsigned long long total = (unsigned long long)nBytes + nBlocks * 31ull;
    if ((unsigned long long)outCapacity < total) return sg_fail("snapgpu_bgzf: output buffer too small (payload + 31 bytes per 65280-byte member)");
    const unsigned grid = (unsigned)(nBlocks < 8ull * sg_sms() ? nBlocks : 8ull * sg_sms());
    sg_bgzf_kernel<<<grid, 256, 0, (cudaStream_t)cudaStream>>>((const uint8_t *)d_in, (unsigned long long)nBytes, (uint8_t *)d_out, nBlocks);
    SG_CUDA(cudaGetLastError());
    *outBytes = (int64_t)total;
    return 0;
}

// ---- BGZF members with a compressor (sg_deflate.h): one block of 1024 threads per member, persistent over the members; each member is laid at a fixed
//      pitch, a scan of the member sizes and one copy per member then close the gaps. ----
extern "C++" {
__global__ void __launch_bounds__(1024, 1)
sg_bgzf_deflate_kernel(const uint8_t *in, unsigned long long nBytes, uint8_t *members, uint32_t *memberSizes, unsigned long long nMembers, uint16_t *arenas)
{
    extern __shared__ __align__(16) uint8_t sgDeflateSmem[];
    SgDeflateShared &S = *(SgDeflateShared *)sgDeflateSmem;
    SgDeflateArena G;
    uint16_t *a = arenas + (size_t)blockIdx.x * (SG_DEFLATE_ARENA_BYTES / 2);
    G.mlen = a; G.mdist = a + (SG_DEFLATE_MAX_PAYLOAD + 8); G.jumpA = a + 2 * (SG_DEFLATE_MAX_PAYLOAD + 8); G.jumpB = a + 3 * (SG_DEFLATE_MAX_PAYLOAD + 8);
    for (unsigned long long m = blockIdx.x; m < nMembers; m += gridDim.x) {
        const unsigned long long off = m * SG_DEFLATE_MAX_PAYLOAD;
        const uint32_t len = (uint32_t)((nBytes - off) < SG_DEFLATE_MAX_PAYLOAD ? (nBytes - off) : SG_DEFLATE_MAX_PAYLOAD);
        const uint32_t sz = sg_deflate_member(S, G, in + off, len, members + m * (unsigned long long)SG_DEFLATE_MEMBER_PITCH);
        if (threadIdx.x == 0) memberSizes[m] = sz;
        __syncthreads();
    }
}

__global__ void sg_bgzf_compact_kernel(const uint8_t *members, const uint32_t *memberSizes, const unsigned long long *memberOffsets, unsigned long long nMembers, uint8_t *out)
{
    for (unsigned long long m = blockIdx.x; m < nMembers; m += gridDim.x) {
        const uint8_t *src = members + m * (unsigned long long)SG_DEFLATE_MEMBER_PITCH;
        uint8_t *dst = out + memberOffsets[m];
        const uint32_t n = memberSizes[m];
        for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
    }
}
}

static int sam_post_reserve(snapgpu_sam *s, size_t bytes);

int snapgpu_bgzf_deflate_device(snapgpu_sam *s, const char *d_in, int64_t nBytes, char *d_out, int64_t outCapacity, int64_t *outBytes, uint64_t *memberOffsets,
                                void *cudaStream)
{
    if (!s || !d_in || !d_out || !outBytes || nBytes < 0) return sg_fail("bad argument");
    *outBytes = 0;
    if (memberOffsets) memberOffsets[0] = 0;
    if (nBytes == 0) return 0;
    SG_CUDA(cudaSetDevice(s->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : s->stream;
    const unsigned long long nMembers = ((unsigned long long)nBytes + SG_DEFLATE_MAX_PAYLOAD - 1) / SG_DEFLATE_MAX_PAYLOAD;
    if (nMembers >= 0x7fffffffULL) return sg_fail("snapgpu_bgzf_deflate_device: too many members for one call");
    int sms = 0;
    SG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device));
    const unsigned grid = (unsigned)(nMembers < (unsigned long long)sms ? nMembers : (unsigned long long)sms);
    size_t cubBytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, cubBytes, (uint32_t *)nullptr, (unsigned long long *)nullptr, (int)nMembers);
    const size_t need = (size_t)nMembers * SG_DEFLATE_MEMBER_PITCH + 256 + (size_t)nMembers * 4 + 256 + ((size_t)nMembers + 1) * 8 + 256 + cubBytes + 256 +
                        (size_t)grid * SG_DEFLATE_ARENA_BYTES + 256;
    if (sam_post_reserve(s, need)) return 1;
    uint8_t *base = (uint8_t *)s->d_post;
    size_t at = 0;
    auto take = [&](size_t bytes) { uint8_t *p = base + at; at += (bytes + 255) & ~(size_t)255; return p; };
    uint8_t *members = take((size_t)nMembers * SG_DEFLATE_MEMBER_PITCH);
    uint32_t *sizes = (uint32_t *)take((size_t)nMembers * 4);
    unsigned long long *offs = (unsigned long long *)take(((size_t)nMembers + 1) * 8);
    void *d_cub = take(cubBytes);
    uint16_t *arenas = (uint16_t *)take((size_t)grid * SG_DEFLATE_ARENA_BYTES);
    SG_CUDA(cudaFuncSetAttribute(sg_bgzf_deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SgDeflateShared)));      // (per device)
    sg_bgzf_deflate_kernel<<<grid, 1024, sizeof(SgDeflateShared), st>>>((const uint8_t *)d_in, (unsigned long long)nBytes, members, sizes, nMembers, arenas);
    SG_CUDA(cudaGetLastError());
    size_t cb = cubBytes;
    SG_CUDA(cub::DeviceScan::ExclusiveSum(d_cub, cb, sizes, offs, (int)nMembers, st));
    unsigned long long lastOff = 0; uint32_t lastSize = 0;
    SG_CUDA(cudaMemcpyAsync(&lastOff, offs + (nMembers - 1), 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(&lastSize, sizes + (nMembers - 1), 4, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    const unsigned long long total = lastOff + lastSize;
    if ((unsigned long long)outCapacity < total) return sg_fail("snapgpu_bgzf_deflate_device: output buffer too small");
    sg_bgzf_compact_kernel<<<(unsigned)(nMembers < 8ull * sg_sms() ? nMembers : 8ull * sg_sms()), 256, 0, st>>>(members, sizes, offs, nMembers, (uint8_t *)d_out);
    SG_CUDA(cudaGetLastError());
    if (memberOffsets) {
        SG_CUDA(cudaMemcpyAsync(memberOffsets, offs, (size_t)nMembers * 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        memberOffsets[nMembers] = total;
    }
    *outBytes = (int64_t)total;
    return 0;
}

// (Re)sizes the octets' scratch and the record slots for reads of up to maxLen bases.
static int sam_reserve(snapgpu_sam *s, uint32_t maxLen, int64_t nUnits, int paired)
{
    if (maxLen < 32) maxLen = 32;
    maxLen = (maxLen + 31u) / 32u * 32u;
    if (s->d_scratch == nullptr || maxLen > s->lay.maxReadLen) {
        const SgSamScratchLayout lay = sam_layout(maxLen);
        const size_t need = lay.perOctet * (size_t)s->nOctets;
        SG_CUDA(cudaStreamSynchronize(s->stream));
        cudaFree(s->d_scratch); s->d_scratch = nullptr;
        SG_CUDA(cudaMalloc((void **)&s->d_scratch, need));
        SG_CUDA(cudaMemsetAsync(s->d_scratch, 0, need, s->stream));
        s->lay = lay; s->scratchBytes = need;
    }
    // one record: QNAME, the fixed fields and RNAME / RNEXT, a CIGAR of up to SG_SAM_MAX_OPS operations (<= 6 characters each from 10000
    // bases on), SEQ and QUAL, the tags
    const uint32_t opChars = maxLen >= 10000 ? 6u : (maxLen >= 1000 ? 5u : 4u);
    const uint32_t one = 2 * maxLen + SG_SAM_MAX_ID + 2 * s->maxNameLen + 256 + (opChars + 1) * SG_SAM_MAX_OPS;
    const uint32_t slot = (paired ? 2 * one : one + 0u);
    const size_t need = (size_t)slot * (size_t)nUnits;
    if (slot > s->slotBytes || need > s->slotsBytes) {
        SG_CUDA(cudaStreamSynchronize(s->stream));
        cudaFree(s->d_slots); s->d_slots = nullptr;
        const size_t cap = (size_t)(slot > s->slotBytes ? slot : s->slotBytes) * (size_t)(paired ? (s->maxBatchReads + 1) / 2 : s->maxBatchReads);
        SG_CUDA(cudaMalloc((void **)&s->d_slots, cap));
        s->slotBytes = slot > s->slotBytes ? slot : s->slotBytes; s->slotsBytes = cap;
    }
    return 0;
}

// The device-resident core: every array already in HBM; the packed text is left in d_text (capacity textCapacity), *textBytes says how much.
static int sam_format_device(snapgpu_sam *s, int paired, int64_t nReads, uint32_t maxLen, const uint8_t *d_bases, const uint8_t *d_quals, const unsigned long long *d_offsets,
                             const uint32_t *d_lens, const uint8_t *d_ids, const unsigned long long *d_idOffsets, const uint32_t *d_idLens, const uint32_t *d_front,
                             const uint32_t *d_clippedLens, const void *d_results, char *d_text, int64_t textCapacity, int64_t *textBytes, cudaStream_t st)
{
    const int64_t nUnits = paired ? nReads / 2 : nReads;
    if (sam_reserve(s, maxLen, nUnits, paired)) return 1;
    int64_t octets = s->nOctets < nUnits ? s->nOctets : nUnits;
    int blocks = (int)((octets * 8 + 255) / 256);
    SG_CUDA(cudaMemsetAsync(s->d_overflow, 0, sizeof(int), st));
#define SG_SAM_LAUNCH(MB) sg_sam_kernel<MB><<<blocks, 256, 0, st>>>(s->index->view, s->lay, s->d_scratch, s->d_namePtrs, s->d_rgAux, s->ag, s->useM, s->useAffineGap, nUnits, paired, \
                                          d_bases, d_quals, d_offsets, d_lens, d_ids, d_idOffsets, d_idLens, \
                                          paired ? nullptr : (const snapgpu_single_result *)d_results, paired ? (const snapgpu_paired_result *)d_results : nullptr, \
                                          d_front, d_clippedLens, s->d_slots, s->slotBytes, s->d_recordBytes, s->format == SNAPGPU_FORMAT_BAM, s->d_rgAuxBam, s->rgAuxBamLen, \
                                          s->d_sortLocations, s->d_sortBytes)
    if (s->ctasPerSM == 8) SG_SAM_LAUNCH(8); else if (s->ctasPerSM == 6) SG_SAM_LAUNCH(6); else if (s->ctasPerSM == 4) SG_SAM_LAUNCH(4);
    else if (s->ctasPerSM == 3) SG_SAM_LAUNCH(3); else SG_SAM_LAUNCH(2);
#undef SG_SAM_LAUNCH
    SG_CUDA(cudaGetLastError());
    s->lastRecords = nReads; s->lastUnits = nUnits; s->lastPaired = paired;
    size_t cb = s->cubBytes;
    SG_CUDA(cub::DeviceScan::ExclusiveSum(s->d_cub, cb, s->d_recordBytes, s->d_recordOffsets, (int)nUnits, st));
    long long warps = nUnits < (long long)sg_sms() * 64 ? nUnits : (long long)sg_sms() * 64;
    sg_sam_pack_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(s->d_slots, s->slotBytes, s->d_recordBytes, s->d_recordOffsets, nUnits, d_text,
                                                                            (unsigned long long)textCapacity, s->d_overflow);
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[0], s->d_recordOffsets + (nUnits - 1), 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[1], s->d_recordBytes + (nUnits - 1), 4, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[2], s->d_overflow, 4, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    const int ov = (int)(s->h_meta[2] & 0xffffffffu);
    if (ov == 1) return sg_fail("snapgpu_sam_format: a record could not be formatted");
    if (ov == 2) return sg_fail("snapgpu_sam_format: text buffer too small");
    *textBytes = (int64_t)(s->h_meta[0] + (s->h_meta[1] & 0xffffffffu));
    return 0;
}

static int sam_format(snapgpu_sam *s, int paired, int64_t nReads, const char *bases, const char *quals, const uint64_t *offsets, const uint32_t *lens, const char *ids,
                      const uint64_t *idOffsets, const uint32_t *idLens, const uint32_t *frontClipped, const uint32_t *clippedLens, const void *results, char *text,
                      int64_t textCapacity, int64_t *textBytes)
{
    if (!s || !bases || !quals || !offsets || !lens || !ids || !idOffsets || !idLens || !results || !text || !textBytes) return sg_fail("null argument");
    if (nReads < 0 || nReads > s->maxBatchReads || (paired && (nReads & 1))) return sg_fail("snapgpu_sam_format: bad read count");
    if ((frontClipped == nullptr) != (clippedLens == nullptr)) return sg_fail("snapgpu_sam_format: frontClipped and clippedLens go together (both or neither)");
    *textBytes = 0;
    if (nReads == 0) return 0;
    SG_CUDA(cudaSetDevice(s->device));
    size_t totalBases = 0, totalIds = 0;
    uint32_t maxLen = 0;
    for (int64_t i = 0; i < nReads; i++) {
        if (lens[i] > SNAPGPU_MAX_READ_LENGTH) return sg_fail("a read is longer than MAX_READ_LENGTH");
        if (idLens[i] >= SG_SAM_MAX_ID) return sg_fail("a read id is longer than 255 characters");
        if (frontClipped && (uint64_t)frontClipped[i] + clippedLens[i] > lens[i]) return sg_fail("snapgpu_sam_format: clipped view outside the read");
        if (offsets[i] + lens[i] > totalBases) totalBases = (size_t)(offsets[i] + lens[i]);
        if (idOffsets[i] + idLens[i] > totalIds) totalIds = (size_t)(idOffsets[i] + idLens[i]);
        if (lens[i] > maxLen) maxLen = lens[i];
    }
    if (totalIds > (size_t)s->maxBatchReads * SG_SAM_MAX_ID) return sg_fail("snapgpu_sam_format: id buffer larger than the handle was sized for");
    cudaStream_t st = s->stream;
    // the staging of the reads and of the text grows with the batches seen
    if (s->d_text == nullptr || (size_t)textCapacity > s->textBytes) {
        SG_CUDA(cudaStreamSynchronize(st));
        cudaFree(s->d_text); s->d_text = nullptr;
        SG_CUDA(cudaMalloc((void **)&s->d_text, (size_t)textCapacity + 16));
        s->textBytes = (size_t)textCapacity;
    }
    if (s->d_bases == nullptr || totalBases + 16 > s->stageBases) {
        SG_CUDA(cudaStreamSynchronize(st));
        cudaFree(s->d_bases); cudaFree(s->d_quals); s->d_bases = s->d_quals = nullptr;
        SG_CUDA(cudaMalloc((void **)&s->d_bases, totalBases + 16));
        SG_CUDA(cudaMalloc((void **)&s->d_quals, totalBases + 16));
        s->stageBases = totalBases + 16;
    }
    SG_CUDA(cudaMemcpyAsync(s->d_bases, bases, totalBases, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(s->d_quals, quals, totalBases, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(s->d_ids, ids, totalIds, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(s->d_offsets, offsets, (size_t)nReads * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(s->d_idOffsets, idOffsets, (size_t)nReads * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(s->d_lens, lens, (size_t)nReads * 4, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(s->d_idLens, idLens, (size_t)nReads * 4, cudaMemcpyHostToDevice, st));
    if (frontClipped) {
        SG_CUDA(cudaMemcpyAsync(s->d_front, frontClipped, (size_t)nReads * 4, cudaMemcpyHostToDevice, st));
        SG_CUDA(cudaMemcpyAsync(s->d_clippedLens, clippedLens, (size_t)nReads * 4, cudaMemcpyHostToDevice, st));
    }
    const int64_t nUnits = paired ? nReads / 2 : nReads;
    SG_CUDA(cudaMemcpyAsync(s->d_results, results, (size_t)nUnits * (paired ? sizeof(snapgpu_paired_result) : sizeof(snapgpu_single_result)), cudaMemcpyHostToDevice, st));
    int64_t used = 0;
    if (sam_format_device(s, paired, nReads, maxLen, s->d_bases, s->d_quals, s->d_offsets, s->d_lens, s->d_ids, s->d_idOffsets, s->d_idLens,
                          frontClipped ? s->d_front : nullptr, frontClipped ? s->d_clippedLens : nullptr, s->d_results, s->d_text, textCapacity, &used, st)) return 1;
    SG_CUDA(cudaMemcpyAsync(text, s->d_text, (size_t)used, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    *textBytes = used;
    return 0;
}

int snapgpu_sam_format_single(snapgpu_sam *s, int64_t nReads, const char *bases, const char *quals, const uint64_t *offsets, const uint32_t *lens, const char *ids,
                              const uint64_t *idOffsets, const uint32_t *idLens, const uint32_t *frontClipped, const uint32_t *clippedLens,
                              const snapgpu_single_result *results, char *text, int64_t textCapacity, int64_t *textBytes)
{
    return sam_format(s, 0, nReads, bases, quals, offsets, lens, ids, idOffsets, idLens, frontClipped, clippedLens, results, text, textCapacity, textBytes);
}

int snapgpu_sam_format_paired(snapgpu_sam *s, int64_t nReads, const char *bases, const char *quals, const uint64_t *offsets, const uint32_t *lens, const char *ids,
                              const uint64_t *idOffsets, const uint32_t *idLens, const uint32_t *frontClipped, const uint32_t *clippedLens,
                              const snapgpu_paired_result *results, char *text, int64_t textCapacity, int64_t *textBytes)
{
    return sam_format(s, 1, nReads, bases, quals, offsets, lens, ids, idOffsets, idLens, frontClipped, clippedLens, results, text, textCapacity, textBytes);
}

// Device-resident forms: every array (and the text buffer) is a DEVICE pointer, so the records of a batch aligned with snapgpu_align_*_device
// are formatted without their results ever visiting the host; maxReadLen = the longest read of the batch.  Synchronises `cudaStream` once.
int snapgpu_sam_format_single_device(snapgpu_sam *s, int64_t nReads, uint32_t maxReadLen, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                                     const uint32_t *d_lens, const char *d_ids, const uint64_t *d_idOffsets, const uint32_t *d_idLens, const uint32_t *d_frontClipped,
                                     const uint32_t *d_clippedLens, const snapgpu_single_result *d_results, char *d_text, int64_t textCapacity, int64_t *textBytes,
                                     void *cudaStream)
{
    if (!s || !d_bases || !d_quals || !d_offsets || !d_lens || !d_ids || !d_idOffsets || !d_idLens || !d_results || !d_text || !textBytes) return sg_fail("null argument");
    if (nReads < 0 || nReads > s->maxBatchReads) return sg_fail("snapgpu_sam_format: bad read count");
    if ((d_frontClipped == nullptr) != (d_clippedLens == nullptr)) return sg_fail("snapgpu_sam_format: frontClipped and clippedLens go together (both or neither)");
    if (maxReadLen == 0 || maxReadLen > SNAPGPU_MAX_READ_LENGTH) return sg_fail("snapgpu_sam_format: maxReadLen out of range");
    *textBytes = 0;
    if (nReads == 0) return 0;
    SG_CUDA(cudaSetDevice(s->device));
    return sam_format_device(s, 0, nReads, maxReadLen, (const uint8_t *)d_bases, (const uint8_t *)d_quals, (const unsigned long long *)d_offsets, d_lens, (const uint8_t *)d_ids,
                             (const unsigned long long *)d_idOffsets, d_idLens, d_frontClipped, d_clippedLens, d_results, d_text, textCapacity, textBytes,
                             cudaStream ? (cudaStream_t)cudaStream : s->stream);
}

int snapgpu_sam_format_paired_device(snapgpu_sam *s, int64_t nReads, uint32_t maxReadLen, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                                     const uint32_t *d_lens, const char *d_ids, const uint64_t *d_idOffsets, const uint32_t *d_idLens, const uint32_t *d_frontClipped,
                                     const uint32_t *d_clippedLens, const snapgpu_paired_result *d_results, char *d_text, int64_t textCapacity, int64_t *textBytes,
                                     void *cudaStream)
{
    if (!s || !d_bases || !d_quals || !d_offsets || !d_lens || !d_ids || !d_idOffsets || !d_idLens || !d_results || !d_text || !textBytes) return sg_fail("null argument");
    if (nReads < 0 || nReads > s->maxBatchReads || (nReads & 1)) return sg_fail("snapgpu_sam_format: bad read count");
    if ((d_frontClipped == nullptr) != (d_clippedLens == nullptr)) return sg_fail("snapgpu_sam_format: frontClipped and clippedLens go together (both or neither)");
    if (maxReadLen == 0 || maxReadLen > SNAPGPU_MAX_READ_LENGTH) return sg_fail("snapgpu_sam_format: maxReadLen out of range");
    *textBytes = 0;
    if (nReads == 0) return 0;
    SG_CUDA(cudaSetDevice(s->device));
    return sam_format_device(s, 1, nReads, maxReadLen, (const uint8_t *)d_bases, (const uint8_t *)d_quals, (const unsigned long long *)d_offsets, d_lens, (const uint8_t *)d_ids,
                             (const unsigned long long *)d_idOffsets, d_idLens, d_frontClipped, d_clippedLens, d_results, d_text, textCapacity, textBytes,
                             cudaStream ? (cudaStream_t)cudaStream : s->stream);
}

// ------------------------------------------------------------------------------------------------
// Row N4 (SURVEY 8f), first piece: SortedDataFilter on the device.  The reference's sorting writer keeps, for every record, the key of the
// location SimpleReadWriter filed it under -- (original contig number, 1-based position in the contig), (0, 0) for location 0, (-1, 0) for
// an unaligned record, -1 comparing as unsigned, i.e. last (SortedDataFilter::onAdvance, SortedDataWriter.cpp:905-939) -- stable-sorts each write batch by it and copies the
// records out in that order (onNextBatch, :942-1010) as one sorted run of its later merge.  Here: keys from the locations the formatter
// kernel left, one stable radix sort of (key, record index), a scan of the permuted lengths, one warp per record to move the bytes.  A batch
// is whatever was formatted last; with HBM to hold the whole output that is the whole run and no merge is left to do.
// ------------------------------------------------------------------------------------------------
__global__ void sg_sort_keys_kernel(SgIndexView ix, const int32_t *contigOriginal, long long nRecords, int paired, const long long *sortLocations, const uint32_t *sortBytes,
                                    const unsigned long long *unitOffsets, unsigned long long *keys, uint32_t *perm, unsigned long long *recOffsets)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nRecords) return;
    const long long loc = sortLocations[r];
    unsigned long long key;
    if (loc == SG_SORT_UNALIGNED) key = 0xffffffffULL << 32;                               // contig -1 (compared UNSIGNED, Genome.h:156-182: after every contig), pos 0
    else if (loc == 0) key = 0;                                                             // contig 0, pos 0 (onAdvance's special case)
    else {
        const int c = sg_contig_at(ix, loc);
        key = ((unsigned long long)(uint32_t)contigOriginal[c] << 32) | (uint32_t)(loc - ix.contigStart[c] + 1);
    }
    keys[r] = key;
    perm[r] = (uint32_t)r;
    recOffsets[r] = paired ? unitOffsets[r >> 1] + ((r & 1) ? sortBytes[r - 1] : 0u) : unitOffsets[r];
}

__global__ void sg_sort_gather_bytes_kernel(long long nRecords, const uint32_t *perm, const uint32_t *sortBytes, uint32_t *sortedBytes)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < nRecords) sortedBytes[r] = sortBytes[perm[r]];
}

__global__ void sg_sort_move_kernel(long long nRecords, const uint32_t *perm, const uint32_t *sortedBytes, const unsigned long long *sortedOffsets,
                                    const unsigned long long *recOffsets, const char *text, char *sorted, unsigned long long capacity, int *overflow)
{
    const int lane = threadIdx.x & 31;
    const long long nW = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nRecords; r += nW) {
        const uint32_t n = sortedBytes[r];
        const unsigned long long to = sortedOffsets[r], from = recOffsets[perm[r]];
        if (to + n > capacity) { if (lane == 0) atomicMax(overflow, 2); continue; }
        for (uint32_t k = lane; k < n; k += 32) sorted[to + k] = text[from + k];
    }
}

int snapgpu_sam_sort_device(snapgpu_sam *s, const char *d_text, char *d_sorted, int64_t sortedCapacity, int64_t *sortedBytes, uint64_t *d_keysOut,
                            uint64_t *d_offsetsOut, void *cudaStream)
{
    if (!s || !d_sorted || !sortedBytes) return sg_fail("null argument");
    if (!d_text) d_text = s->d_text;             // the handle's own buffer: where a host-buffer format call left the records on the device
    if (!d_text) return sg_fail("snapgpu_sam_sort_device: nothing formatted yet");
    *sortedBytes = 0;
    const long long n = s->lastRecords;
    if (n == 0) return 0;
    SG_CUDA(cudaSetDevice(s->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : s->stream;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    SG_CUDA(cudaMemsetAsync(s->d_overflow, 0, sizeof(int), st));
    sg_sort_keys_kernel<<<blocks, 256, 0, st>>>(s->index->view, s->d_contigOriginal, n, s->lastPaired, s->d_sortLocations, s->d_sortBytes, s->d_recordOffsets,
                                                s->d_sortKeys, s->d_perm, s->d_recOffsets);
    SG_CUDA(cudaGetLastError());
    size_t cb = s->cubBytes;
    SG_CUDA(cub::DeviceRadixSort::SortPairs(s->d_cub, cb, s->d_sortKeys, s->d_sortKeysOut, s->d_perm, s->d_permOut, (int)n, 0, 64, st));      // (LSD radix sort: stable)
    sg_sort_gather_bytes_kernel<<<blocks, 256, 0, st>>>(n, s->d_permOut, s->d_sortBytes, s->d_sortedBytes);
    SG_CUDA(cudaGetLastError());
    cb = s->cubBytes;
    SG_CUDA(cub::DeviceScan::ExclusiveSum(s->d_cub, cb, s->d_sortedBytes, s->d_sortedOffsets, (int)n, st));
    const long long warps = n < (long long)sg_sms() * 64 ? n : (long long)sg_sms() * 64;
    sg_sort_move_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(n, s->d_permOut, s->d_sortedBytes, s->d_sortedOffsets, s->d_recOffsets, d_text, d_sorted,
                                                                             (unsigned long long)sortedCapacity, s->d_overflow);
    SG_CUDA(cudaGetLastError());
    if (d_keysOut) SG_CUDA(cudaMemcpyAsync(d_keysOut, s->d_sortKeysOut, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
    if (d_offsetsOut) SG_CUDA(cudaMemcpyAsync(d_offsetsOut, s->d_sortedOffsets, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[0], s->d_sortedOffsets + (n - 1), 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[1], s->d_sortedBytes + (n - 1), 4, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[2], s->d_overflow, 4, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    if ((int)(s->h_meta[2] & 0xffffffffu) != 0) return sg_fail("snapgpu_sam_sort_device: sorted buffer too small");
    *sortedBytes = (int64_t)(s->h_meta[0] + (s->h_meta[1] & 0xffffffffu));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Row N4 after the sort: duplicate marking and the BAM index of a coordinate-sorted stream of BAM records in HBM (sg_bampost.h has the semantics;
// here: the data-parallel plumbing around them).
// ------------------------------------------------------------------------------------------------
extern "C++" {
struct SgPostCarve {               // bump allocator over the handle's work buffer
    uint8_t *base; size_t used, cap;
    template <typename T> T *take(size_t n) { used = (used + 255) & ~(size_t)255; T *p = (T *)(base + used); used += n * sizeof(T); return p; }
};
}
static int sam_post_reserve(snapgpu_sam *s, size_t bytes)
{
    if (bytes <= s->postBytes) return 0;
    cudaFree(s->d_post); s->d_post = nullptr; s->postBytes = 0;
    SG_CUDA(cudaMalloc(&s->d_post, bytes));
    s->postBytes = bytes;
    return 0;
}

__global__ void sg_dup_fields_kernel(const uint8_t *records, const unsigned long long *offsets, long long n, const int64_t *contigStartByOriginal, int32_t nRef,
                                     SgDupFields *f, int32_t *flagRun, uint8_t *fragFlag, uint32_t *iota)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SgBamRec r; r.p = records + offsets[i];
    sg_dup_fields(r, contigStartByOriginal, nRef, &f[i]);
    flagRun[i] = -1; fragFlag[i] = 0; iota[i] = (uint32_t)i;
}

// where a run starting at record s would end, and where the run after it would start (jump[s]; n = there is none).  jump has n + 1 entries, jump[n] = n.
__global__ void sg_dup_runs_kernel(const SgDupFields *f, long long n, uint32_t *runEndOf, uint32_t *jump, uint8_t *mark)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > n) return;
    if (s == n) { jump[n] = (uint32_t)n; return; }
    mark[s] = s == 0 ? 1 : 0;
    if (f[s].logical == SG_DUP_INVALID_LOCATION) { runEndOf[s] = (uint32_t)(s + 1); jump[s] = (uint32_t)(s + 1); return; }
    const long long e = sg_dup_first_beyond(f, n, s, 2 * SG_DUP_RUN_REACH);
    runEndOf[s] = (uint32_t)e;
    jump[s] = (uint32_t)(e == n ? n : sg_dup_first_beyond(f, n, s, SG_DUP_RUN_REACH));
}

// one round of pointer jumping: everything marked marks what it jumps to; the jump doubles
__global__ void sg_dup_orbit_kernel(long long n, const uint32_t *jump, uint32_t *jumpNext, uint8_t *mark)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s > n) return;
    const uint32_t j = jump[s];
    if (s < n && mark[s] && j < n) mark[j] = 1;
    jumpNext[s] = jump[j];
}

__global__ void sg_dup_run_flags_kernel(const SgDupFields *f, long long n, const uint8_t *mark, uint8_t *isRun)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) isRun[s] = (mark[s] && f[s].logical != SG_DUP_INVALID_LOCATION) ? 1 : 0;
}

__global__ void sg_dup_run_table_kernel(const uint32_t *runStarts, const long long *nRuns, const uint32_t *runEndOf, long long *runStart, long long *runEnd)
{
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < *nRuns) { runStart[k] = runStarts[k]; runEnd[k] = runEndOf[runStarts[k]]; }
}

// sort keys of the current order `idx`: WHICH 0: the larger of (info, mateInfo), 1: the smaller, 2: the library, 3: info -- records without FLAG 0x1 sort last in the pair passes
__global__ void sg_dup_keys_kernel(const SgDupFields *f, long long n, const uint32_t *idx, int which, unsigned long long *keys)
{
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const SgDupFields &F = f[idx[j]];
    unsigned long long k;
    if (which == 3) k = F.info;
    else if (which == 4) k = F.lib;
    else if (!(F.flag & SG_BAM_FLAG_PAIRED)) k = ~0ULL;
    else if (which == 0) k = F.info > F.mateInfo ? F.info : F.mateInfo;
    else if (which == 1) k = F.info < F.mateInfo ? F.info : F.mateInfo;
    else k = F.lib;
    keys[j] = k;
}

__global__ void sg_dup_walk_kernel(const uint8_t *records, const unsigned long long *offsets, long long n, const SgDupFields *f, const long long *nRuns,
                                   const long long *runStart, const long long *runEnd, const uint32_t *order, int pairs, int32_t *flagRun, uint8_t *fragFlag)
{
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const SgDupFields &F = f[order[j]];
    if (pairs) {
        if (!(F.flag & SG_BAM_FLAG_PAIRED)) return;
        const uint64_t lo = F.info < F.mateInfo ? F.info : F.mateInfo, hi = F.info < F.mateInfo ? F.mateInfo : F.info;
        if (j > 0) {
            const SgDupFields &P = f[order[j - 1]];
            if ((P.flag & SG_BAM_FLAG_PAIRED) && P.lib == F.lib && (P.info < P.mateInfo ? P.info : P.mateInfo) == lo && (P.info < P.mateInfo ? P.mateInfo : P.info) == hi) return;   // not the head
        }
        long long e = j + 1;
        while (e < n) {
            const SgDupFields &Q = f[order[e]];
            if (!((Q.flag & SG_BAM_FLAG_PAIRED) && Q.lib == F.lib && (Q.info < Q.mateInfo ? Q.info : Q.mateInfo) == lo && (Q.info < Q.mateInfo ? Q.mateInfo : Q.info) == hi)) break;
            e++;
        }
        if (e - j < 2) return;
        SgDupView V; V.n = n; V.records = records; V.offsets = offsets; V.f = f; V.nRuns = *nRuns; V.runStart = runStart; V.runEnd = runEnd;
        sg_dup_walk_pair_key(V, order + j, e - j, lo, hi, flagRun);
    } else {
        if (j > 0) { const SgDupFields &P = f[order[j - 1]]; if (P.lib == F.lib && P.info == F.info) return; }
        long long e = j + 1;
        while (e < n && f[order[e]].lib == F.lib && f[order[e]].info == F.info) e++;
        if (e - j < 2) return;
        SgDupView V; V.n = n; V.records = records; V.offsets = offsets; V.f = f; V.nRuns = *nRuns; V.runStart = runStart; V.runEnd = runEnd;
        sg_dup_walk_fragment_key(V, order + j, e - j, flagRun, fragFlag);
    }
}

__global__ void sg_dup_apply_kernel(uint8_t *records, const unsigned long long *offsets, long long n, const SgDupFields *f, const int32_t *flagRun, const uint8_t *fragFlag,
                                    unsigned long long *marked)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if ((flagRun[i] >= 0 || fragFlag[i]) && !(f[i].flag & SG_BAM_FLAG_DUPLICATE)) {
        const uint32_t fl = f[i].flag | SG_BAM_FLAG_DUPLICATE;
        uint8_t *p = records + offsets[i];
        p[18] = (uint8_t)fl; p[19] = (uint8_t)(fl >> 8);
        atomicAdd(marked, 1ULL);
    }
}

int snapgpu_bam_markdup_device(snapgpu_sam *s, char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t *nMarked, void *cudaStream)
{
    if (!s || !d_records || !d_offsets || !nMarked) return sg_fail("null argument");
    *nMarked = 0;
    if (nRecords < 0 || nRecords >= 0x7fffffffLL) return sg_fail("snapgpu_bam_markdup_device: record count out of range");
    if (nRecords < 2) return 0;
    SG_CUDA(cudaSetDevice(s->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : s->stream;
    const long long n = nRecords;
    size_t cubSort = 0, cubSel = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, cubSort, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (uint32_t *)nullptr, (uint32_t *)nullptr, (int)n);
    cub::DeviceSelect::Flagged(nullptr, cubSel, (uint32_t *)nullptr, (uint8_t *)nullptr, (uint32_t *)nullptr, (long long *)nullptr, (int)n);
    const size_t cubBytes = (cubSort > cubSel ? cubSort : cubSel) + 256;
    const size_t need = (size_t)n * (sizeof(SgDupFields) + 4 * 4 + 2 * 8 + 3 * 4 + 2 * 8 + 4 + 3) + cubBytes + 64 * 256;
    if (sam_post_reserve(s, need)) return 1;
    SgPostCarve C{(uint8_t *)s->d_post, 0, s->postBytes};
    SgDupFields *f = C.take<SgDupFields>(n);
    uint32_t *runEndOf = C.take<uint32_t>(n + 1), *jumpA = C.take<uint32_t>(n + 1), *jumpB = C.take<uint32_t>(n + 1), *iota = C.take<uint32_t>(n);
    long long *runStart = C.take<long long>(n), *runEnd = C.take<long long>(n);
    uint32_t *runStarts = C.take<uint32_t>(n), *idxA = C.take<uint32_t>(n), *idxB = C.take<uint32_t>(n);
    unsigned long long *keysA = C.take<unsigned long long>(n), *keysB = C.take<unsigned long long>(n);
    int32_t *flagRun = C.take<int32_t>(n);
    uint8_t *mark = C.take<uint8_t>(n + 1), *isRun = C.take<uint8_t>(n), *fragFlag = C.take<uint8_t>(n);
    long long *d_nRuns = C.take<long long>(1);
    unsigned long long *d_marked = C.take<unsigned long long>(1);
    void *d_cub = C.take<uint8_t>(cubBytes);
    if (C.used > C.cap) return sg_fail("snapgpu_bam_markdup_device: work buffer accounting");
    const unsigned blocks = (unsigned)((n + 1 + 255) / 256);
    const uint8_t *rec = (const uint8_t *)d_records; const unsigned long long *off = (const unsigned long long *)d_offsets;
    SG_CUDA(cudaMemsetAsync(d_marked, 0, 8, st));
    sg_dup_fields_kernel<<<blocks, 256, 0, st>>>(rec, off, n, s->d_contigStartByOriginal, (int32_t)s->h_contigStartByOriginal.size(), f, flagRun, fragFlag, iota);
    sg_dup_runs_kernel<<<blocks, 256, 0, st>>>(f, n, runEndOf, jumpA, mark);
    SG_CUDA(cudaGetLastError());
    { uint32_t *a = jumpA, *b = jumpB; for (long long span = 1; span <= n; span <<= 1) { sg_dup_orbit_kernel<<<blocks, 256, 0, st>>>(n, a, b, mark); uint32_t *t = a; a = b; b = t; } }
    sg_dup_run_flags_kernel<<<blocks, 256, 0, st>>>(f, n, mark, isRun);
    SG_CUDA(cudaGetLastError());
    size_t cb = cubBytes;
    SG_CUDA(cub::DeviceSelect::Flagged(d_cub, cb, iota, isRun, runStarts, d_nRuns, (int)n, st));
    sg_dup_run_table_kernel<<<blocks, 256, 0, st>>>(runStarts, d_nRuns, runEndOf, runStart, runEnd);
    SG_CUDA(cudaGetLastError());
    // pair keys: stable LSD passes over (larger end, smaller end, library), then one thread per key
    const uint32_t *order = iota;
    uint32_t *out = idxA, *other = idxB;
    const int pairPasses[3] = {0, 1, 2}, fragPasses[2] = {3, 4};
    for (int p = 0; p < 3; p++) {
        sg_dup_keys_kernel<<<blocks, 256, 0, st>>>(f, n, order, pairPasses[p], keysA);
        cb = cubBytes;
        SG_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, cb, keysA, keysB, order, out, (int)n, 0, 64, st));
        order = out; uint32_t *t = out; out = other; other = t;
    }
    sg_dup_walk_kernel<<<blocks, 256, 0, st>>>(rec, off, n, f, d_nRuns, runStart, runEnd, order, 1, flagRun, fragFlag);
    SG_CUDA(cudaGetLastError());
    order = iota; out = idxA; other = idxB;
    for (int p = 0; p < 2; p++) {
        sg_dup_keys_kernel<<<blocks, 256, 0, st>>>(f, n, order, fragPasses[p], keysA);
        cb = cubBytes;
        SG_CUDA(cub::DeviceRadixSort::SortPairs(d_cub, cb, keysA, keysB, order, out, (int)n, 0, 64, st));
        order = out; uint32_t *t = out; out = other; other = t;
    }
    sg_dup_walk_kernel<<<blocks, 256, 0, st>>>(rec, off, n, f, d_nRuns, runStart, runEnd, order, 0, flagRun, fragFlag);
    sg_dup_apply_kernel<<<blocks, 256, 0, st>>>((uint8_t *)d_records, off, n, f, flagRun, fragFlag, d_marked);
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(&s->h_meta[0], d_marked, 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    *nMarked = (int64_t)s->h_meta[0];
    return 0;
}

// ---- the index ----
struct SgBaiRecord { int32_t ref; uint32_t bin; unsigned long long at; };
__global__ void sg_bai_records_kernel(const uint8_t *records, const unsigned long long *offsets, long long n, unsigned long long headerBytes, int32_t nRef,
                                      uint8_t *isHead, unsigned long long *composite, unsigned long long *refFirst, unsigned long long *refLast,
                                      unsigned long long *refMapped, unsigned long long *refUnmapped, uint32_t *iota)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    SgBamRec r; r.p = records + offsets[i];
    const int32_t ref = r.refID();
    const unsigned long long at = headerBytes + offsets[i];
    bool head = i == 0;
    if (!head) { SgBamRec q; q.p = records + offsets[i - 1]; head = q.refID() != ref || q.bin() != r.bin(); }
    isHead[i] = head ? 1 : 0;
    iota[i] = (uint32_t)i;
    unsigned long long c = 0;
    if (ref >= 0 && ref < nRef) {
        atomicMin(&refFirst[ref], at);
        atomicMax(&refLast[ref], at + (unsigned long long)r.size());
        if (r.flag() & SG_BAM_FLAG_UNMAPPED) atomicAdd(&refUnmapped[ref], 1ULL);
        else { atomicAdd(&refMapped[ref], 1ULL); c = ((unsigned long long)(ref + 1) << 32) | (unsigned long long)(sg_bai_linear_slot(r) + 1); }
    }
    composite[i] = c;
}

struct SgMaxU64 { __device__ __forceinline__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return a > b ? a : b; } };

__global__ void sg_bai_chunks_kernel(const uint8_t *records, const unsigned long long *offsets, long long n, unsigned long long headerBytes, unsigned long long totalBytes,
                                     const uint32_t *heads, const long long *nHeads, SgBaiRecord *chunkHead, unsigned long long *chunkEnd)
{
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= *nHeads) return;
    SgBamRec r; r.p = records + offsets[heads[k]];
    chunkHead[k].ref = r.refID(); chunkHead[k].bin = r.bin(); chunkHead[k].at = headerBytes + offsets[heads[k]];
    chunkEnd[k] = (k + 1 < *nHeads) ? headerBytes + offsets[heads[k + 1]] : totalBytes;
}

// a record sets the linear-index entry of its window iff no earlier record of its reference reached that far (addInterval only ever appends, Bam.cpp:3425-3440)
__global__ void sg_bai_linear_kernel(const unsigned long long *offsets, long long n, unsigned long long headerBytes, const unsigned long long *composite,
                                     const unsigned long long *prefixMax, const unsigned long long *refSlotBase, unsigned long long *intervals, unsigned long long *refSlots)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long c = composite[i];
    if (c == 0 || c <= prefixMax[i]) return;
    const uint32_t ref = (uint32_t)(c >> 32) - 1u, slot = (uint32_t)c - 1u;
    intervals[refSlotBase[ref] + slot] = headerBytes + offsets[i];
    atomicMax(&refSlots[ref], (unsigned long long)slot + 1ULL);
}

static int bam_index_impl(snapgpu_sam *s, const char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t recordBytes, int64_t headerBytes,
                          const uint64_t *memberOffsets, char *bai, int64_t baiCapacity, int64_t *baiBytes, void *cudaStream)
{
    if (!s || !bai || !baiBytes || (nRecords > 0 && (!d_records || !d_offsets))) return sg_fail("null argument");
    *baiBytes = 0;
    if (nRecords < 0 || nRecords >= 0x7fffffffLL || recordBytes < 0 || headerBytes < 0) return sg_fail("snapgpu_bam_index_device: argument out of range");
    SG_CUDA(cudaSetDevice(s->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : s->stream;
    const long long n = nRecords;
    const int32_t nRef = (int32_t)s->h_contigStartByOriginal.size();
    const unsigned long long total = (unsigned long long)headerBytes + (unsigned long long)recordBytes;
    std::vector<SgBaiChunk> chunks;
    std::vector<SgBaiRef> refs((size_t)nRef);
    if (n > 0) {
        std::vector<unsigned long long> slotBase((size_t)nRef + 1, 0);
        for (int32_t r = 0; r < nRef; r++) slotBase[r + 1] = slotBase[r] + (unsigned long long)(s->h_contigSpan[r] / 16384 + 3);
        const size_t nSlots = (size_t)slotBase[nRef];
        size_t cubSel = 0, cubScan = 0;
        cub::DeviceSelect::Flagged(nullptr, cubSel, (uint32_t *)nullptr, (uint8_t *)nullptr, (uint32_t *)nullptr, (long long *)nullptr, (int)n);
        cub::DeviceScan::ExclusiveScan(nullptr, cubScan, (unsigned long long *)nullptr, (unsigned long long *)nullptr, SgMaxU64(), 0ULL, (int)n);
        const size_t cubBytes = (cubSel > cubScan ? cubSel : cubScan) + 256;
        const size_t need = (size_t)n * (1 + 8 + 8 + 4 + 4 + sizeof(SgBaiRecord) + 8) + (size_t)nRef * 8 * 6 + nSlots * 8 + cubBytes + 64 * 256;
        if (sam_post_reserve(s, need)) return 1;
        SgPostCarve C{(uint8_t *)s->d_post, 0, s->postBytes};
        uint8_t *isHead = C.take<uint8_t>(n);
        unsigned long long *composite = C.take<unsigned long long>(n), *prefixMax = C.take<unsigned long long>(n);
        uint32_t *iota = C.take<uint32_t>(n), *heads = C.take<uint32_t>(n);
        SgBaiRecord *chunkHead = C.take<SgBaiRecord>(n);
        unsigned long long *chunkEnd = C.take<unsigned long long>(n);
        unsigned long long *refFirst = C.take<unsigned long long>(nRef), *refLast = C.take<unsigned long long>(nRef), *refMapped = C.take<unsigned long long>(nRef),
                           *refUnmapped = C.take<unsigned long long>(nRef), *refSlots = C.take<unsigned long long>(nRef), *d_slotBase = C.take<unsigned long long>(nRef + 1);
        unsigned long long *intervals = C.take<unsigned long long>(nSlots);
        long long *d_nHeads = C.take<long long>(1);
        void *d_cub = C.take<uint8_t>(cubBytes);
        if (C.used > C.cap) return sg_fail("snapgpu_bam_index_device: work buffer accounting");
        const unsigned blocks = (unsigned)((n + 255) / 256);
        const uint8_t *rec = (const uint8_t *)d_records; const unsigned long long *off = (const unsigned long long *)d_offsets;
        SG_CUDA(cudaMemsetAsync(refFirst, 0xff, (size_t)nRef * 8, st));
        SG_CUDA(cudaMemsetAsync(refLast, 0, (size_t)nRef * 8, st));
        SG_CUDA(cudaMemsetAsync(refMapped, 0, (size_t)nRef * 8, st));
        SG_CUDA(cudaMemsetAsync(refUnmapped, 0, (size_t)nRef * 8, st));
        SG_CUDA(cudaMemsetAsync(refSlots, 0, (size_t)nRef * 8, st));
        SG_CUDA(cudaMemsetAsync(intervals, 0xff, nSlots * 8, st));
        SG_CUDA(cudaMemcpyAsync(d_slotBase, slotBase.data(), (size_t)(nRef + 1) * 8, cudaMemcpyHostToDevice, st));
        sg_bai_records_kernel<<<blocks, 256, 0, st>>>(rec, off, n, (unsigned long long)headerBytes, nRef, isHead, composite, refFirst, refLast, refMapped, refUnmapped, iota);
        SG_CUDA(cudaGetLastError());
        size_t cb = cubBytes;
        SG_CUDA(cub::DeviceSelect::Flagged(d_cub, cb, iota, isHead, heads, d_nHeads, (int)n, st));
        sg_bai_chunks_kernel<<<blocks, 256, 0, st>>>(rec, off, n, (unsigned long long)headerBytes, total, heads, d_nHeads, chunkHead, chunkEnd);
        cb = cubBytes;
        SG_CUDA(cub::DeviceScan::ExclusiveScan(d_cub, cb, composite, prefixMax, SgMaxU64(), 0ULL, (int)n, st));
        sg_bai_linear_kernel<<<blocks, 256, 0, st>>>(off, n, (unsigned long long)headerBytes, composite, prefixMax, d_slotBase, intervals, refSlots);
        SG_CUDA(cudaGetLastError());
        long long nHeads = 0;
        SG_CUDA(cudaMemcpyAsync(&nHeads, d_nHeads, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        std::vector<SgBaiRecord> hHead((size_t)nHeads); std::vector<unsigned long long> hEnd((size_t)nHeads), hIntervals(nSlots);
        std::vector<unsigned long long> hFirst(nRef), hLast(nRef), hMapped(nRef), hUnmapped(nRef), hSlots(nRef);
        SG_CUDA(cudaMemcpy(hHead.data(), chunkHead, (size_t)nHeads * sizeof(SgBaiRecord), cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hEnd.data(), chunkEnd, (size_t)nHeads * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hIntervals.data(), intervals, nSlots * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hFirst.data(), refFirst, (size_t)nRef * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hLast.data(), refLast, (size_t)nRef * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hMapped.data(), refMapped, (size_t)nRef * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hUnmapped.data(), refUnmapped, (size_t)nRef * 8, cudaMemcpyDeviceToHost));
        SG_CUDA(cudaMemcpy(hSlots.data(), refSlots, (size_t)nRef * 8, cudaMemcpyDeviceToHost));
        chunks.resize((size_t)nHeads);
        for (long long k = 0; k < nHeads; k++) { chunks[k].ref = hHead[k].ref; chunks[k].bin = hHead[k].bin; chunks[k].start = hHead[k].at; chunks[k].end = hEnd[k]; }
        for (int32_t r = 0; r < nRef; r++) {
            SgBaiRef &R = refs[r];
            R.any = hMapped[r] + hUnmapped[r] > 0;
            R.firstStart = hFirst[r]; R.lastEnd = hLast[r]; R.mapped = hMapped[r]; R.unmapped = hUnmapped[r];
            R.intervals.assign(hIntervals.begin() + slotBase[r], hIntervals.begin() + slotBase[r] + hSlots[r]);
        }
    }
    std::vector<uint8_t> o = sg_bai_compose(nRef, chunks, refs, total, memberOffsets);
    if ((int64_t)o.size() > baiCapacity) return sg_fail("snapgpu_bam_index_device: bai buffer too small");
    memcpy(bai, o.data(), o.size());
    *baiBytes = (int64_t)o.size();
    return 0;
}

int snapgpu_bam_index_device(snapgpu_sam *s, const char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t recordBytes, int64_t headerBytes,
                             char *bai, int64_t baiCapacity, int64_t *baiBytes, void *cudaStream)
{
    return bam_index_impl(s, d_records, d_offsets, nRecords, recordBytes, headerBytes, nullptr, bai, baiCapacity, baiBytes, cudaStream);
}

int snapgpu_bam_index_members_device(snapgpu_sam *s, const char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t recordBytes, int64_t headerBytes,
                                     const uint64_t *memberOffsets, int64_t nMembers, char *bai, int64_t baiCapacity, int64_t *baiBytes, void *cudaStream)
{
    if (!memberOffsets) return sg_fail("null argument");
    if (recordBytes < 0 || headerBytes < 0 || nMembers != (int64_t)(((uint64_t)recordBytes + (uint64_t)headerBytes + 0xff00ULL - 1) / 0xff00ULL))
        return sg_fail("snapgpu_bam_index_members_device: nMembers is not the member count of headerBytes + recordBytes");
    return bam_index_impl(s, d_records, d_offsets, nRecords, recordBytes, headerBytes, memberOffsets, bai, baiCapacity, baiBytes, cudaStream);
}

int64_t snapgpu_sam_last_record_count(const snapgpu_sam *s) { return s ? s->lastRecords : 0; }

struct snapgpu_fastq {
    int device = 0;
    int64_t maxBytes = 0, maxReads = 0, nTilesMax = 0;
    uint8_t *d_text = nullptr, *d_bases = nullptr, *d_quals = nullptr;     // staging of the host-buffer path
    uint32_t *d_tileCounts = nullptr, *d_tileBase = nullptr, *d_nlPos = nullptr, *d_lens = nullptr, *d_idLens = nullptr, *d_front = nullptr;
    unsigned long long *d_offsets = nullptr, *d_idOffsets = nullptr;
    SgFastqRecord *d_rec = nullptr;
    long long *d_meta = nullptr, *h_meta = nullptr;
    int *d_status = nullptr, *h_status = nullptr;
    void *d_cub = nullptr; size_t cubBytes = 0;
    cudaStream_t stream = nullptr;
};

void snapgpu_fastq_destroy(snapgpu_fastq *f)
{
    if (!f) return;
    cudaSetDevice(f->device);
    cudaDeviceSynchronize();
    cudaFree(f->d_text); cudaFree(f->d_bases); cudaFree(f->d_quals); cudaFree(f->d_tileCounts); cudaFree(f->d_tileBase); cudaFree(f->d_nlPos);
    cudaFree(f->d_lens); cudaFree(f->d_idLens); cudaFree(f->d_front); cudaFree(f->d_offsets); cudaFree(f->d_idOffsets); cudaFree(f->d_rec);
    cudaFree(f->d_meta); cudaFreeHost(f->h_meta); cudaFree(f->d_status); cudaFreeHost(f->h_status); cudaFree(f->d_cub);
    if (f->stream) cudaStreamDestroy(f->stream);
    delete f;
}

int snapgpu_fastq_create(int device, int64_t maxBytes, int64_t maxReads, snapgpu_fastq **out)
{
    if (!out) return sg_fail("null argument");
    *out = nullptr;
    if (require_device(device)) return 1;
    if (maxBytes <= 0 || maxBytes >= (int64_t)0xfffffff0LL) return sg_fail("snapgpu_fastq_create: maxBytes must be in (0, 4 GiB)");
    if (maxReads <= 0) return sg_fail("snapgpu_fastq_create: maxReads must be positive");
    snapgpu_fastq *f = new (std::nothrow) snapgpu_fastq;
    if (!f) return sg_fail("out of memory");
    f->device = device; f->maxBytes = maxBytes; f->maxReads = maxReads;
    f->nTilesMax = (maxBytes + SG_FQ_TILE - 1) / SG_FQ_TILE;
    size_t c1 = 0, c2 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, c1, (uint32_t *)nullptr, (uint32_t *)nullptr, (int)(f->nTilesMax + 1));
    cub::DeviceScan::ExclusiveSum(nullptr, c2, (uint32_t *)nullptr, (unsigned long long *)nullptr, (int)maxReads);
    f->cubBytes = (c1 > c2 ? c1 : c2) + 256;
    const size_t maxLines = (size_t)maxReads * 4 + 4;
    cudaError_t e = cudaSuccess;
    #define SG_FQ_ALLOC(p, n) if (e == cudaSuccess) e = cudaMalloc((void **)&(p), (n))
    SG_FQ_ALLOC(f->d_text, (size_t)maxBytes + 16); SG_FQ_ALLOC(f->d_bases, (size_t)maxBytes / 2 + 16); SG_FQ_ALLOC(f->d_quals, (size_t)maxBytes / 2 + 16);
    SG_FQ_ALLOC(f->d_tileCounts, (size_t)(f->nTilesMax + 1) * 4); SG_FQ_ALLOC(f->d_tileBase, (size_t)(f->nTilesMax + 1) * 4);
    SG_FQ_ALLOC(f->d_nlPos, maxLines * 4); SG_FQ_ALLOC(f->d_lens, (size_t)maxReads * 4); SG_FQ_ALLOC(f->d_idLens, (size_t)maxReads * 4);
    SG_FQ_ALLOC(f->d_front, (size_t)maxReads * 4); SG_FQ_ALLOC(f->d_offsets, (size_t)maxReads * 8); SG_FQ_ALLOC(f->d_idOffsets, (size_t)maxReads * 8);
    SG_FQ_ALLOC(f->d_rec, (size_t)maxReads * sizeof(SgFastqRecord)); SG_FQ_ALLOC(f->d_meta, 4 * sizeof(long long)); SG_FQ_ALLOC(f->d_status, sizeof(int));
    SG_FQ_ALLOC(f->d_cub, f->cubBytes);
    #undef SG_FQ_ALLOC
    if (e == cudaSuccess) e = cudaMallocHost((void **)&f->h_meta, 4 * sizeof(long long));
    if (e == cudaSuccess) e = cudaMallocHost((void **)&f->h_status, sizeof(int));
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&f->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { std::string msg = std::string("snapgpu_fastq_create: ") + cudaGetErrorString(e); snapgpu_fastq_destroy(f); return sg_fail(msg); }
    *out = f;
    return 0;
}

int snapgpu_fastq_parse_device(snapgpu_fastq *f, const char *d_text, int64_t nBytes, int clippingType, char *d_bases, char *d_quals, uint64_t *d_offsets,
                               uint32_t *d_lens, uint64_t *d_idOffsets, uint32_t *d_idLens, uint32_t *d_frontClipped, int64_t *nReads,
                               int64_t *bytesConsumed, void *cudaStream)
{
    if (!f || !d_text || !d_bases || !d_quals || !d_offsets || !d_lens || !nReads || !bytesConsumed) return sg_fail("null argument");
    if (nBytes < 0 || nBytes > f->maxBytes) return sg_fail("snapgpu_fastq_parse: nBytes exceeds the handle's maxBytes");
    if (clippingType < 0 || clippingType > 3) return sg_fail("snapgpu_fastq_parse: clippingType must be 0..3");
    *nReads = 0; *bytesConsumed = 0;
    if (nBytes == 0) return 0;
    SG_CUDA(cudaSetDevice(f->device));
    cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : f->stream;
    const uint8_t *text = (const uint8_t *)d_text;
    const long long nTiles = (nBytes + SG_FQ_TILE - 1) / SG_FQ_TILE;
    int grid = (int)(nTiles < (long long)sg_sms() * 16 ? nTiles : (long long)sg_sms() * 16);
    SG_CUDA(cudaMemsetAsync(f->d_status, 0, sizeof(int), st));
    SG_CUDA(cudaMemsetAsync(f->d_tileCounts + nTiles, 0, 4, st));
    sg_fastq_count_kernel<<<grid, SG_FQ_THREADS, 0, st>>>(text, nBytes, f->d_tileCounts, nTiles);
    size_t cb = f->cubBytes;
    SG_CUDA(cub::DeviceScan::ExclusiveSum(f->d_cub, cb, f->d_tileCounts, f->d_tileBase, (int)(nTiles + 1), st));
    const long long maxLines = f->maxReads * 4 + 4;
    sg_fastq_positions_kernel<<<grid, SG_FQ_THREADS, 0, st>>>(text, nBytes, f->d_tileBase, f->d_nlPos, maxLines, nTiles);
    sg_fastq_meta_kernel<<<1, 1, 0, st>>>(text, nBytes, f->d_tileBase, nTiles, f->d_nlPos, f->maxReads, f->d_meta);
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(f->h_meta, f->d_meta, 3 * sizeof(long long), cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    const long long R = f->h_meta[1];
    *nReads = R; *bytesConsumed = f->h_meta[2];
    if (R == 0) return 0;
    sg_fastq_records_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(text, nBytes, f->d_nlPos, R, clippingType, (uint8_t)'#', (uint8_t)'#',
                                                                      (uint32_t)SNAPGPU_MAX_READ_LENGTH, f->d_rec, d_lens, (unsigned long long *)d_idOffsets,
                                                                      d_idLens, d_frontClipped, f->d_status);
    cb = f->cubBytes;
    SG_CUDA(cub::DeviceScan::ExclusiveSum(f->d_cub, cb, d_lens, (unsigned long long *)d_offsets, (int)R, st));
    long long warps = R < (long long)sg_sms() * 64 ? R : (long long)sg_sms() * 64;
    sg_fastq_copy_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(text, nBytes, f->d_rec, (const unsigned long long *)d_offsets, R,
                                                                              (uint8_t *)d_bases, (uint8_t *)d_quals);
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(f->h_status, f->d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    if (*f->h_status == SG_FQ_ERR_BLANK_LINE) return sg_fail("Syntax error in FASTQ file: blank line.");
    if (*f->h_status == SG_FQ_ERR_BAD_START) return sg_fail("FASTQ file has an invalid starting character on a line");
    if (*f->h_status == SG_FQ_ERR_TOO_LONG) return sg_fail("Saw a read longer than MAX_READ_LENGTH");
    return 0;
}

int snapgpu_fastq_parse(snapgpu_fastq *f, const char *text, int64_t nBytes, int clippingType, char *bases, char *quals, uint64_t *offsets, uint32_t *lens,
                        uint64_t *idOffsets, uint32_t *idLens, uint32_t *frontClipped, int64_t *nReads, int64_t *bytesConsumed)
{
    if (!f || !text || !bases || !quals || !offsets || !lens || !nReads || !bytesConsumed) return sg_fail("null argument");
    if (nBytes < 0 || nBytes > f->maxBytes) return sg_fail("snapgpu_fastq_parse: nBytes exceeds the handle's maxBytes");
    SG_CUDA(cudaSetDevice(f->device));
    SG_CUDA(cudaMemcpyAsync(f->d_text, text, (size_t)nBytes, cudaMemcpyHostToDevice, f->stream));
    if (snapgpu_fastq_parse_device(f, (const char *)f->d_text, nBytes, clippingType, (char *)f->d_bases, (char *)f->d_quals, (uint64_t *)f->d_offsets, f->d_lens,
                                   (uint64_t *)f->d_idOffsets, f->d_idLens, f->d_front, nReads, bytesConsumed, nullptr)) return 1;
    const int64_t R = *nReads;
    if (R == 0) return 0;
    SG_CUDA(cudaMemcpyAsync(offsets, f->d_offsets, (size_t)R * 8, cudaMemcpyDeviceToHost, f->stream));
    SG_CUDA(cudaMemcpyAsync(lens, f->d_lens, (size_t)R * 4, cudaMemcpyDeviceToHost, f->stream));
    if (idOffsets) SG_CUDA(cudaMemcpyAsync(idOffsets, f->d_idOffsets, (size_t)R * 8, cudaMemcpyDeviceToHost, f->stream));
    if (idLens) SG_CUDA(cudaMemcpyAsync(idLens, f->d_idLens, (size_t)R * 4, cudaMemcpyDeviceToHost, f->stream));
    if (frontClipped) SG_CUDA(cudaMemcpyAsync(frontClipped, f->d_front, (size_t)R * 4, cudaMemcpyDeviceToHost, f->stream));
    SG_CUDA(cudaStreamSynchronize(f->stream));
    const uint64_t total = offsets[R - 1] + lens[R - 1];
    if (total) {
        SG_CUDA(cudaMemcpyAsync(bases, f->d_bases, (size_t)total, cudaMemcpyDeviceToHost, f->stream));
        SG_CUDA(cudaMemcpyAsync(quals, f->d_quals, (size_t)total, cudaMemcpyDeviceToHost, f->stream));
        SG_CUDA(cudaStreamSynchronize(f->stream));
    }
    return 0;
}

int64_t snapgpu_aligner_launch_count(const snapgpu_aligner *a) { return a ? a->launches : 0; }

int64_t snapgpu_aligner_deferred_count(snapgpu_aligner *a)
{
    if (!a || a->paired || !a->twoPass || !a->d_retryCount) return -1;
    unsigned long long v = 0;
    if (cudaSetDevice(a->device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(&v, a->d_retryCount, 8, cudaMemcpyDeviceToHost) != cudaSuccess) { sg_fail(cudaGetErrorString(cudaGetLastError())); return -1; }
    return (int64_t)v;
}

static int leaf_scratch(int device, SgParams *p, int *threads, uint8_t **d_scratch, size_t *bytes, SgTables **d_tb)
{
    if (require_device(device)) return 1;
    memset(p, 0, sizeof(*p));
    p->poolSize = 1; p->tableSlots = 2; p->numWeightLists = 2; p->maxReadLen = 1000;
    *bytes = sg_align_up(sg_scratch_bytes(*p), 256);
    *threads = 64 * 32;
    if (const char *e = getenv("SNAPGPU_TEST_WORKERS")) { int v = atoi(e); if (v >= 32 && v <= 8192) *threads = v / 32 * 32; }   // leaf micro-benchmarks
    SG_CUDA(cudaMalloc((void **)d_scratch, *bytes * (size_t)*threads));
    SG_CUDA(cudaMemset(*d_scratch, 0, *bytes * (size_t)*threads));
    SgTables T;
    sg_init_tables(T, 20);
    SG_CUDA(cudaMalloc((void **)d_tb, sizeof(SgTables)));
    SG_CUDA(cudaMemcpy(*d_tb, &T, sizeof(SgTables), cudaMemcpyHostToDevice));
    return 0;
}

static int test_lv_impl(int device, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf, uint64_t patBytes,
                        const snapgpu_lv_job *jobs, int64_t nJobs, snapgpu_lv_out *out, int nWarps)
{
    SgParams p; int threads; uint8_t *d_scratch = nullptr; size_t bytes; SgTables *d_tb = nullptr;
    if (leaf_scratch(device, &p, &threads, &d_scratch, &bytes, &d_tb)) return 1;
    uint8_t *d_text, *d_pat, *d_qual; snapgpu_lv_job *d_jobs; snapgpu_lv_out *d_out;
    SG_CUDA(cudaMalloc((void **)&d_text, textBytes + 16)); SG_CUDA(cudaMalloc((void **)&d_pat, patBytes + 16)); SG_CUDA(cudaMalloc((void **)&d_qual, patBytes + 16));
    SG_CUDA(cudaMalloc((void **)&d_jobs, (size_t)nJobs * sizeof(*jobs) + 16)); SG_CUDA(cudaMalloc((void **)&d_out, (size_t)nJobs * sizeof(*out) + 16));
    SG_CUDA(cudaMemcpy(d_text, textBuf, textBytes, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d_pat, patBuf, patBytes, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d_qual, qualBuf, patBytes, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d_jobs, jobs, (size_t)nJobs * sizeof(*jobs), cudaMemcpyHostToDevice));
    if (nWarps > 0) {
        if (nWarps > threads) nWarps = threads;
        sg_test_lv_warp_kernel<<<nWarps, 32>>>(d_tb, p, d_scratch, bytes, d_text, d_pat, d_qual, d_jobs, nJobs, d_out);
    } else {
        sg_test_lv_kernel<<<threads / 32, 32>>>(d_tb, p, d_scratch, bytes, d_text, d_pat, d_qual, d_jobs, nJobs, d_out);
    }
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaDeviceSynchronize());
    SG_CUDA(cudaMemcpy(out, d_out, (size_t)nJobs * sizeof(*out), cudaMemcpyDeviceToHost));
    cudaFree(d_text); cudaFree(d_pat); cudaFree(d_qual); cudaFree(d_jobs); cudaFree(d_out); cudaFree(d_scratch); cudaFree(d_tb);
    return 0;
}

int snapgpu_test_lv(int device, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf, uint64_t patBytes,
                    const snapgpu_lv_job *jobs, int64_t nJobs, snapgpu_lv_out *out)
{
    return test_lv_impl(device, textBuf, textBytes, patBuf, qualBuf, patBytes, jobs, nJobs, out, 0);
}

int snapgpu_test_lv_warp(int device, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf, uint64_t patBytes,
                         const snapgpu_lv_job *jobs, int64_t nJobs, snapgpu_lv_out *out, int nWarps)
{
    return test_lv_impl(device, textBuf, textBytes, patBuf, qualBuf, patBytes, jobs, nJobs, out, nWarps < 1 ? 1 : nWarps);
}

static int test_ag_impl(int device, const snapgpu_ag_params *ap, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf,
                        uint64_t patBytes, const snapgpu_ag_job *jobs, int64_t nJobs, snapgpu_ag_out *out, int nWarps)
{
    SgParams p; int threads; uint8_t *d_scratch = nullptr; size_t bytes; SgTables *d_tb = nullptr;
    if (leaf_scratch(device, &p, &threads, &d_scratch, &bytes, &d_tb)) return 1;
    SgAgParams P = sg_ag_params(ap->matchReward, ap->subPenalty, ap->gapOpenPenalty, ap->gapExtendPenalty, ap->fivePrimeEndBonus, ap->threePrimeEndBonus);
    P.usePacked = 1;                 // leaf tests: the packed form unless SNAPGPU_TEST_AG_PACKED=0 (the tests run both)
    if (const char *e = getenv("SNAPGPU_TEST_AG_PACKED")) P.usePacked = atoi(e);        // 0 int form, 1 packed loop-compact, 2 packed unrolled
    uint8_t *d_text, *d_pat, *d_qual; snapgpu_ag_job *d_jobs; snapgpu_ag_out *d_out;
    SG_CUDA(cudaMalloc((void **)&d_text, textBytes + 16)); SG_CUDA(cudaMalloc((void **)&d_pat, patBytes + 16)); SG_CUDA(cudaMalloc((void **)&d_qual, patBytes + 16));
    SG_CUDA(cudaMalloc((void **)&d_jobs, (size_t)nJobs * sizeof(*jobs) + 16)); SG_CUDA(cudaMalloc((void **)&d_out, (size_t)nJobs * sizeof(*out) + 16));
    SG_CUDA(cudaMemcpy(d_text, textBuf, textBytes, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d_pat, patBuf, patBytes, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d_qual, qualBuf, patBytes, cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d_jobs, jobs, (size_t)nJobs * sizeof(*jobs), cudaMemcpyHostToDevice));
    if (nWarps > 0) {
        if (nWarps > threads) nWarps = threads;
        sg_test_ag_warp_kernel<<<nWarps, 32>>>(d_tb, p, P, d_scratch, bytes, d_text, d_pat, d_qual, d_jobs, nJobs, d_out);
        if (const char *e = getenv("SNAPGPU_TEST_REPEAT")) {           // leaf micro-benchmark: time R more launches of the same batch
            int reps = atoi(e);
            cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
            cudaEventRecord(e0);
            for (int r = 0; r < reps; r++) sg_test_ag_warp_kernel<<<nWarps, 32>>>(d_tb, p, P, d_scratch, bytes, d_text, d_pat, d_qual, d_jobs, nJobs, d_out);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
            fprintf(stderr, "snapgpu_test_ag_warp: %d jobs x %d launches on %d warps: %.3f ms per launch, %.1f ns per job\n", (int)nJobs, reps, nWarps,
                    ms / reps, 1e6 * ms / reps / (double)nJobs);
            cudaEventDestroy(e0); cudaEventDestroy(e1);
        }
    } else {
        sg_test_ag_kernel<<<threads / 32, 32>>>(d_tb, p, P, d_scratch, bytes, d_text, d_pat, d_qual, d_jobs, nJobs, d_out);
    }
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaDeviceSynchronize());
    SG_CUDA(cudaMemcpy(out, d_out, (size_t)nJobs * sizeof(*out), cudaMemcpyDeviceToHost));
    cudaFree(d_text); cudaFree(d_pat); cudaFree(d_qual); cudaFree(d_jobs); cudaFree(d_out); cudaFree(d_scratch); cudaFree(d_tb);
    return 0;
}

int snapgpu_test_ag(int device, const snapgpu_ag_params *ap, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf,
                    uint64_t patBytes, const snapgpu_ag_job *jobs, int64_t nJobs, snapgpu_ag_out *out)
{
    return test_ag_impl(device, ap, textBuf, textBytes, patBuf, qualBuf, patBytes, jobs, nJobs, out, 0);
}

int snapgpu_test_ag_warp(int device, const snapgpu_ag_params *ap, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf,
                         uint64_t patBytes, const snapgpu_ag_job *jobs, int64_t nJobs, snapgpu_ag_out *out, int nWarps)
{
    return test_ag_impl(device, ap, textBuf, textBytes, patBuf, qualBuf, patBytes, jobs, nJobs, out, nWarps < 1 ? 1 : nWarps);
}

} // extern "C"
