/*
 * snapgpu.h -- C ABI of the H100-native seed-and-extend engine that drops in behind SNAP's
 * per-thread aligner hook.
 *
 * Every entry point is plain C: pointers, sizes, POD structs.  No C++/torch types cross this line.
 * A SNAP maintainer binds these from `AlignerExtension::runIterationThread`
 * (reference SNAPLib/AlignerContext.h:145-180, call sites SingleAligner.cpp:102 and
 * PairedAligner.cpp:503); INTEGRATION.md shows the stub.
 *
 * Return convention: 0 = success, non-zero = failure and snapgpu_last_error() describes it
 * (the reference's own convention is WriteErrorMessage()+soft_exit(1), exit.cpp:30-42; a library
 * must not exit(), so errors are returned and the extension turns them into soft_exit).
 * There is NO CPU fallback: if no CUDA device / kernel image is usable every call fails loudly.
 */
#ifndef SNAPGPU_H
#define SNAPGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SNAPGPU_ABI_VERSION 9   /* 2: snapgpu_sam_format_* take frontClipped / clippedLens before `results`; 3: groups, replicate, host_alloc, random-sector rate;
                                 * 4: snapgpu_sam_sort_device; 5: snapgpu_bam_markdup_device, snapgpu_bam_index_device;
                                 * 6: snapgpu_align_single_secondary(_device) (-om), snapgpu_bgzf_deflate_device, snapgpu_bam_index_members_device, snapgpu_sam_header;
                                 * 7: snapgpu_contig, snapgpu_index_build_genome(_device), snapgpu_save_options, snapgpu_index_save_ex;
                                 * 8: snapgpu_aligner_deferred_count;
                                 * 9: snapgpu_spacing_* and snapgpu_align_paired_ins(_device) (`snap paired -ins`) */

/* AlignmentResult enum, reference SNAPLib/AlignmentResult.h:34 */
enum { SNAPGPU_NOT_FOUND = 0, SNAPGPU_SINGLE_HIT = 1, SNAPGPU_MULTIPLE_HITS = 2 };
/* Direction, reference SNAPLib/directions.h */
enum { SNAPGPU_FORWARD = 0, SNAPGPU_RC = 1 };

#define SNAPGPU_INVALID_LOCATION_32 0xffffffffLL /* InvalidGenomeLocation for 4-byte locations, GenomeIndex.cpp:511-517 */
#define SNAPGPU_UNUSED_SCORE 0xffff               /* BaseAligner::UnusedScoreValue, BaseAligner.h:141 */
#define SNAPGPU_MAX_K 127                         /* LandauVishkin.h:11 */
#define SNAPGPU_MAX_READ_LENGTH 1000              /* Read.h:49 */

/*
 * POD mirror of SingleAlignmentResult (reference SNAPLib/AlignmentResult.h:49-77), field for field,
 * minus alignmentTimeInNanoseconds (only meaningful with -at and measured by the caller).
 */
typedef struct snapgpu_single_result {
    int32_t  status;                    /* SNAPGPU_NOT_FOUND / SINGLE_HIT / MULTIPLE_HITS */
    int32_t  direction;                 /* SNAPGPU_FORWARD / SNAPGPU_RC */
    int64_t  location;                  /* GenomeLocation; SNAPGPU_INVALID_LOCATION_32 when not found */
    int64_t  origLocation;              /* location before indel adjustment */
    int32_t  score;                     /* edit distance */
    int32_t  scorePriorToClipping;
    int32_t  mapq;
    int32_t  clippingForReadAdjustment;
    int32_t  usedAffineGapScoring;
    int32_t  basesClippedBefore;
    int32_t  basesClippedAfter;
    int32_t  agScore;
    int32_t  supplementary;
    int32_t  seedOffset;
    double   matchProbability;
    double   probabilityAllCandidates;
    uint32_t popularSeedsSkipped;
    uint32_t reserved;
} snapgpu_single_result;               /* 88 bytes */

/*
 * The AlignerContext / AlignerOptions fields the hot path reads
 * (reference SNAPLib/AlignerContext.h:102-131, AlignerOptions.h:93-186, defaults AlignerOptions.cpp:39-121).
 * snapgpu_params_default() fills the 2.0.5 single-end defaults.
 */
typedef struct snapgpu_params {
    uint32_t struct_size;               /* sizeof(snapgpu_params), for ABI checking */
    uint32_t maxHits;                   /* -h   (300)  */
    uint32_t maxDist;                   /* -d   (14)   maxK */
    uint32_t numSeedsFromCommandLine;   /* -n   (25)   */
    double   seedCoverage;              /* -sc  (0.0); used when numSeedsFromCommandLine == 0 */
    uint32_t minWeightToCheck;          /* -ms  (1)    */
    uint32_t extraSearchDepth;          /* -D   (1)    */
    uint32_t minReadLength;             /* -mrl (50)   */
    int32_t  useAffineGap;              /* -G / -G-  (1) */
    int32_t  matchReward;               /* -gm  (1)  */
    int32_t  subPenalty;                /* -gs  (4)  */
    int32_t  gapOpenPenalty;            /* -go  (6)  */
    int32_t  gapExtendPenalty;          /* -ge  (1)  */
    int32_t  fivePrimeEndBonus;         /* -g5  (10) */
    int32_t  threePrimeEndBonus;        /* -g3  (7)  */
    /* DisabledOptimizations, AlignerOptions.h:78-88 */
    int32_t  noUkkonen;
    int32_t  noOrderedEvaluation;
    int32_t  noTruncation;
    int32_t  noEditDistance;            /* -ne */
    int32_t  noBandedAffineGap;
    int32_t  altAwareness;              /* -A- turns off (1) */
    int32_t  maxScoreGapToPreferNonAltAlignment; /* (64) */
    int32_t  explorePopularSeeds;       /* -x (0) */
    int32_t  stopOnFirstHit;            /* -f (0) */
    int32_t  maxSecondaryAlignmentAdditionalEditDistance; /* -om (-1 = off); >= 0: single-end handles only, through snapgpu_align_single_secondary */
    int32_t  ignoreAlignmentAdjustmentsForOm; /* (1) -- AlignmentAdjuster is off by default; only 1 supported */
} snapgpu_params;

typedef struct snapgpu_index_info {
    int64_t  countOfBases;              /* Genome::getCountOfBases() incl. inter-contig padding */
    uint32_t seedLen;
    uint32_t hashTableKeySize;          /* bytes of the seed kept as the in-table key */
    uint32_t nHashTables;
    uint32_t locationSize;              /* only 4 supported (lookupSeed32 path) */
    uint32_t largeHashTable;            /* 1 = `-large` two-value entries */
    uint32_t chromosomePadding;
    uint32_t nContigs;
    uint32_t reserved;
    uint64_t overflowTableSize;         /* in 32-bit words */
    uint64_t hashTableSlots;            /* total slots over all tables */
    uint64_t hbmBytes;                  /* bytes resident on the device for this index */
} snapgpu_index_info;

/*
 * POD mirror of PairedAlignmentResult (reference SNAPLib/AlignmentResult.h:86-129), field for field, minus the two
 * timing fields.  Index [r] = read r of the pair.
 */
typedef struct snapgpu_paired_result {
    int32_t  status[2];
    int32_t  direction[2];
    int64_t  location[2];
    int64_t  origLocation[2];
    int32_t  score[2];
    int32_t  scorePriorToClipping[2];
    int32_t  mapq[2];
    int32_t  clippingForReadAdjustment[2];
    int32_t  usedAffineGapScoring[2];
    int32_t  basesClippedBefore[2];
    int32_t  basesClippedAfter[2];
    int32_t  agScore[2];
    int32_t  supplementary[2];
    int32_t  seedOffset[2];
    int32_t  lvIndels[2];
    int32_t  usedGaplessClipping[2];
    int32_t  refSpan[2];
    int32_t  liftover[2];
    uint32_t popularSeedsSkipped[2];
    int32_t  alignedAsPair;
    int32_t  agForcedSingleAlignerCall;
    double   matchProbability[2];
    double   probabilityAllPairs;
} snapgpu_paired_result;                /* 200 bytes */

/*
 * The extra options `snap paired` reads (reference SNAPLib/PairedAligner.cpp:228-243, 288-364, AlignerOptions.cpp:101-111).
 * The shared ones come from snapgpu_params (for pairs: maxDist -d, numSeedsFromCommandLine -n (8), maxHits -h).
 */
typedef struct snapgpu_paired_params {
    uint32_t struct_size;
    int32_t  minSpacing;                /* -s min (0)    */
    uint32_t maxSpacing;                /* -s max (1000) */
    uint32_t intersectingAlignerMaxHits;/* -H   (4000)   */
    uint32_t maxCandidatePoolSize;      /* -mcp (1000000)*/
    uint32_t maxSeedsSingleEnd;         /* -N   (25) seeds for the chimeric single-end fallback */
    uint32_t maxDistForIndels;          /* -i   (40)     */
    int32_t  forceSpacing;              /* -fs  (0)      */
    int32_t  minScoreRealignment;       /* (3)  */
    int32_t  minScoreGapRealignmentALT; /* (3)  */
    int32_t  minAGScoreImprovement;     /* (24; 15 without soft clipping, PairedAligner.cpp:388) */
    int32_t  enableHammingScoringBaseAligner; /* -eh / -eh- (1) */
    int32_t  useSoftClipping;           /* -hc- / -hc (1) */
    int32_t  flattenMAPQAtOrBelow;      /* -fmb (3) */
} snapgpu_paired_params;

/* Per-call work counters (reference BaseAligner.h:106-111 + AlignerStats.h:41-97 subset). */
typedef struct snapgpu_counters {
    int64_t totalReads;
    int64_t uselessReads;               /* filtered up front: too short / too many Ns (SingleAligner.cpp:213) */
    int64_t singleHits;
    int64_t multiHits;
    int64_t notFound;
    int64_t nHashTableLookups;          /* lookupSeed32 calls */
    int64_t nHashEntriesProbed;         /* hash-table entries examined over both strand probes */
    int64_t nOverflowWordsRead;         /* overflow-table words touched (count word + hits used) */
    int64_t lvCalls;                    /* locations scored with Landau-Vishkin */
    int64_t affineGapCalls;             /* locations scored with affine gap */
    int64_t nHitsIgnoredBecauseOfTooHighPopularity;
    int64_t mapqHistogram[71];
} snapgpu_counters;

typedef struct snapgpu_index   snapgpu_index;   /* opaque: hash tables + overflow + bases resident in HBM */
typedef struct snapgpu_aligner snapgpu_aligner; /* opaque: per-host-thread stream, scratch arenas, staging */

const char *snapgpu_last_error(void);            /* thread-local, never NULL */
/* Page-locked host memory for callers that do not link CUDA themselves (the align calls DMA straight out of / into such buffers);
 * NULL on failure. */
void *snapgpu_host_alloc(size_t bytes);
void  snapgpu_host_free(void *p);
int  snapgpu_abi_version(void);
int  snapgpu_device_count(void);                 /* 0 if no usable CUDA device */
void snapgpu_params_default(snapgpu_params *p);  /* `snap single` 2.0.5 defaults, AlignerOptions.cpp:39-121 */

/*
 * Index.  Replaces GenomeIndex::loadFromDirectory (reference SNAPLib/GenomeIndex.cpp:1838-2093):
 * reads the four files `Genome`, `GenomeIndex`, `GenomeIndexHash`, `OverflowTable` written by
 * `snap-aligner index` (format v7.1, SURVEY 8a-F) and places them in HBM on `device`.
 */
int  snapgpu_index_open(const char *directory, int device, snapgpu_index **out);
/*
 * Builds the same lookup structure on the device from raw reference bases (one byte per base,
 * already including SNAP's lowercase-'n' contig padding), for when no pre-built directory exists.
 * Equivalent in *results* to GenomeIndex::BuildIndexToDirectory (GenomeIndex.cpp:527-1110): every
 * seed maps to the same hit set in the same (descending) order; slot layout is not part of the contract.
 * contigStarts[nContigs] are the beginningLocation values (first real base of each contig).
 * Memory: beside the finished index (bases, buckets or tables, overflow table), one sweep sorts every position at once in
 * 24 bytes each (~72 GB at 3 Gbp).  When that, or the 12 bytes per position it keeps while the index is allocated, does not fit
 * the free device memory, the build sorts the positions in key-range passes that each fit (SNAPGPU_BUILD_PASSES=n asks for at
 * least n); a 3 Gbp bucket index then builds on an 80 GB device.  The index is the same either way.
 */
int  snapgpu_index_build(const char *bases, int64_t nBases, const int64_t *contigStarts, uint32_t nContigs,
                         uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out);
/* Same, with the nBases bases already in HBM (DEVICE pointer); they are copied into the index image. */
int  snapgpu_index_build_device(const char *d_bases, int64_t nBases, const int64_t *contigStarts, uint32_t nContigs,
                                uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out);
/*
 * One contig of a genome, as the reference's Genome keeps it (Genome.h Contig) and writes it to the Genome file
 * (Genome::saveToFile): what `snap-aligner index` reads from a FASTA (names, ALT marking, ALT-last order) and an -altLiftoverFile.
 */
typedef struct snapgpu_contig {
    const char *name;                   /* NUL-terminated; written with spaces as '_' */
    int64_t  beginningLocation;         /* first base of the contig in the padded genome; ascending */
    int32_t  isAlt;                     /* ALT contig; ALT contigs come after every non-ALT one */
    int32_t  originalContigNumber;      /* the contig's place in the FASTA */
    int64_t  projBeginningLocation;     /* liftover: where the ALT contig projects (the Genome file's field, as is) */
    int32_t  projIsRC;                  /* liftover: the projection is reverse-complemented */
    int32_t  reserved;
    const char *projCigar;              /* liftover: the projection CIGAR; NULL without a liftover line */
} snapgpu_contig;
/*
 * snapgpu_index_build(_device) with the genome's contig descriptors: the index gets their names, ALT flags, original numbers and
 * liftover data, as snapgpu_index_open gives an index from a Genome file with ALT contigs, so it aligns ALT-aware (`snap paired`
 * liftover) like the same genome opened from a directory `snap-aligner index` wrote.  The lookup structure is built exactly as by
 * snapgpu_index_build.  Fails on a malformed projection CIGAR, a non-ALT contig after an ALT one, or locations that do not ascend.
 */
int  snapgpu_index_build_genome(const char *bases, int64_t nBases, const snapgpu_contig *contigs, uint32_t nContigs,
                                uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out);
int  snapgpu_index_build_genome_device(const char *d_bases, int64_t nBases, const snapgpu_contig *contigs, uint32_t nContigs,
                                       uint32_t seedLen, uint32_t chromosomePadding, int device, snapgpu_index **out);
/* The table geometry of a saved index: `snap-aligner index -keysize / -large / -h`. */
typedef struct snapgpu_save_options {
    uint32_t struct_size;               /* sizeof(snapgpu_save_options) */
    uint32_t keyBytes;                  /* 2..8 with 2*seedLen >= 8*keyBytes and 2*seedLen - 8*keyBytes <= 16 (2..6 for seeds 16..24) */
    uint32_t large;                     /* 1: -large tables (two values per entry, keyed by the canonical seed) */
    uint32_t reserved;
    double   slack;                     /* > 0: each table holds (1 + slack) x its distinct keys (at least 100 slots) */
} snapgpu_save_options;
/*
 * Writes the HBM-resident index out as a reference-format directory (the four files `snap-aligner index` produces,
 * SURVEY 8a-F) so stock SNAP can load an index built on the device.  The Genome file carries the contigs' names, ALT flags,
 * original numbers and liftover data as given.  A device-built bucket index has its buckets re-laid into the reference's tables of
 * the requested geometry, each table sized from its exact entry count, one range of tables at a time in buffers of at most the free
 * device memory (a staging slot of 8 bytes -- default tables with keys of up to 4 bytes -- or 16, plus the packed entry when its
 * size differs; SNAPGPU_BUILD_PASSES=n: at least n ranges).  A geometry with a single table needs it to fit whole.  An index in the
 * reference's layout (SNAPGPU_INDEX_LAYOUT=snap) saves only with the default options.
 */
int  snapgpu_index_save_ex(const snapgpu_index *idx, const char *directory, const snapgpu_save_options *opts);
/* snapgpu_index_save_ex with 4-byte keys, default tables and slack 0.3. */
int  snapgpu_index_save(const snapgpu_index *idx, const char *directory);
int  snapgpu_index_info_get(const snapgpu_index *idx, snapgpu_index_info *info);
/*
 * Second, third ... copy of an HBM-resident index on another device of the same process (SURVEY 8e: "replicate the full index image in
 * every GPU's HBM ... index upload can be done once"): device-to-device copies over NVLink / NVSwitch peer access instead of
 * N uploads from the host.  The copy is an independent index (close each one).
 */
int  snapgpu_index_replicate(const snapgpu_index *src, int device, snapgpu_index **out);
void snapgpu_index_close(snapgpu_index *idx);

/*
 * A group of CUDA devices driven by ONE process -- the SNAP extension runs one feeder thread per device -- with an NCCL communicator
 * per device (ncclCommInitAll; NCCL is loaded with dlopen at this call, not linked).  The path has exactly two collectives
 * (SURVEY 8e): the index broadcast at start-up (one upload from the index directory, then ncclBroadcast over NVLink / NVSwitch instead
 * of N uploads) and the all-reduce of the statistics at the end (AlignerStats.h:41-84; AlignerContext::finishThread adds the
 * per-thread stats on the host in the reference, AlignerContext.cpp:241-245).  Reads shard across the devices without any exchange.
 */
typedef struct snapgpu_group snapgpu_group;
int  snapgpu_group_create(const int *devices, int nDevices, snapgpu_group **out);
void snapgpu_group_destroy(snapgpu_group *g);
int  snapgpu_group_size(const snapgpu_group *g);
/* src lives on the group's first device; out[nDevices]: out[0] = src itself, out[k] = an independent copy on device k (close each). */
int  snapgpu_index_broadcast(snapgpu_group *g, snapgpu_index *src, snapgpu_index **out);
/* counters[nDevices] (HOST): each entry is replaced by the sum over the group (ncclAllReduce(SUM) on the devices). */
int  snapgpu_counters_allreduce(snapgpu_group *g, snapgpu_counters *counters);

/*
 * Batched GenomeIndex::lookupSeed32 (reference SNAPLib/GenomeIndex.cpp:2095-2157).
 * seeds: nSeeds * seedLen ASCII bases (host memory).  For seed i: nHits[2*i] forward, nHits[2*i+1] RC;
 * hits[(2*i+dir)*maxHitsPerSeed ...] receives the first min(nHits, maxHitsPerSeed) locations, descending
 * as in the overflow table.  Seeds with non-ACGT bases report 0/0 (Seed::DoesTextRepresentASeed, Seed.cpp:28).
 * probes[i] (optional) = hash entries examined for seed i.
 */
int  snapgpu_lookup_seeds(const snapgpu_index *idx, const char *seeds, int64_t nSeeds, uint32_t maxHitsPerSeed,
                          int64_t *nHits, uint32_t *hits, uint32_t *probes);

/*
 * Measurement utility (the denominator of bench.py's seed_phase; on no product path): the device's random-access ceiling.  nAccesses
 * aligned 32-byte sector reads at pseudo-random places of a scratch table of tableBytes, one independent read in flight per thread
 * (best of three launches, CUDA events).  A hash probe is exactly this access, so sector reads per second is the roofline of the
 * seed-lookup phase: lookups/s <= rate / sectors per lookup.
 */
int  snapgpu_measure_random_sector_rate(int device, uint64_t tableBytes, uint64_t nAccesses, double *sectorsPerSecond);

/* Same with DEVICE pointers (d_hits / d_probes may be NULL), enqueued on `cudaStream` without synchronising:
 * the seed-lookup phase in isolation, for its roofline measurement. */
int  snapgpu_lookup_seeds_device(const snapgpu_index *idx, const char *d_seeds, int64_t nSeeds, uint32_t maxHitsPerSeed,
                                 int64_t *d_nHits, uint32_t *d_hits, uint32_t *d_probes, void *cudaStream);

/*
 * Aligner handle.  One per host thread, like BaseAligner (reference SNAPLib/BaseAligner.h:19-20:
 * "NOT thread safe"); owns a CUDA stream, pinned staging and the device scratch arenas.
 * maxBatchReads bounds n in the align calls.
 */
int  snapgpu_aligner_create(const snapgpu_index *idx, const snapgpu_params *params, int64_t maxBatchReads,
                            snapgpu_aligner **out);
void snapgpu_aligner_destroy(snapgpu_aligner *a);

/*
 * Replaces the per-thread loop body `aligner->AlignRead(read, results, ...)` + pre-filter + updateStats
 * (reference SNAPLib/SingleAligner.cpp:197-338, BaseAligner.cpp:272-763) for a batch of n reads.
 * bases/quals: concatenated clipped views (Read::getData()/getQuality(), upper-cased), read i at
 * [offsets[i], offsets[i]+lens[i]).  HOST pointers; copies are done inside.  results[n] caller-owned.
 * counters may be NULL; when given it is *accumulated into*.
 * Page-locked buffers (cudaHostAlloc / cudaHostRegister) are detected and used for DMA directly -- reads that sit back to
 * back in pinned bases/quals skip the staging copy, pinned results are written in place; pageable memory works the same,
 * through the handle's own pinned staging.
 */
int  snapgpu_align_single(snapgpu_aligner *a, int64_t n, const char *bases, const char *quals,
                          const uint64_t *offsets, const uint32_t *lens,
                          snapgpu_single_result *results, snapgpu_counters *counters);

/*
 * Same, but all five arrays are DEVICE pointers and the kernels are enqueued on `cudaStream`
 * (a cudaStream_t / CUstream passed as void*; NULL = the aligner's own stream).  Does not synchronise.
 * d_counters may be NULL; otherwise a device snapgpu_counters that is accumulated into.
 */
int  snapgpu_align_single_device(snapgpu_aligner *a, int64_t n, const char *d_bases, const char *d_quals,
                                 const uint64_t *d_offsets, const uint32_t *d_lens,
                                 snapgpu_single_result *d_results, snapgpu_counters *d_counters,
                                 void *cudaStream);

/*
 * Secondary alignments, `snap single -om <d> [-omax <n>] [-mpc <n>]`: what AlignRead does when its caller passes a secondaryResults
 * buffer (reference SNAPLib/SingleAligner.cpp:250-318; recording in ScoreSet::updateBestScore, BaseAligner.cpp:2143-2299; pruning in
 * BaseAligner::finalizeSecondaryResults, :2422-2553).  The handle must have been created with
 * params.maxSecondaryAlignmentAdditionalEditDistance = <d> >= 0 (and <= extraSearchDepth, AlignerContext.cpp:784); such a handle only
 * takes these two calls.  maxSecondaryAlignments = -omax (0x7fffffff = no limit), maxSecondaryAlignmentsPerContig = -mpc (<= 0 = no limit).
 * results[n]: the primary results (they can differ from a run without -om: the "MAPQ cannot recover" early stop is off, :1512).
 * secondary[n * secondaryCapacityPerRead]: read i's secondary results at [i * secondaryCapacityPerRead, +nSecondary[i]), in the order the
 * reference leaves them in its buffer.  nSecondary[i] < 0: read i has -nSecondary[i] of them and they did not fit -- none were written;
 * call again with at least that capacity (the reference's caller doubles its buffer and calls AlignRead again, SingleAligner.cpp:250-263).
 */
int  snapgpu_align_single_secondary(snapgpu_aligner *a, int64_t n, const char *bases, const char *quals,
                                    const uint64_t *offsets, const uint32_t *lens, snapgpu_single_result *results,
                                    int32_t maxSecondaryAlignments, int32_t maxSecondaryAlignmentsPerContig,
                                    int64_t secondaryCapacityPerRead, snapgpu_single_result *secondary, int32_t *nSecondary,
                                    snapgpu_counters *counters);
/* Device-pointer form (see snapgpu_align_single_device).  A worker whose raw record buffer fills up latches an error that
 * snapgpu_aligner_check() reports (the host form grows the buffers and aligns the batch again by itself). */
int  snapgpu_align_single_secondary_device(snapgpu_aligner *a, int64_t n, const char *d_bases, const char *d_quals,
                                           const uint64_t *d_offsets, const uint32_t *d_lens, snapgpu_single_result *d_results,
                                           int32_t maxSecondaryAlignments, int32_t maxSecondaryAlignmentsPerContig,
                                           int64_t secondaryCapacityPerRead, snapgpu_single_result *d_secondary, int32_t *d_nSecondary,
                                           snapgpu_counters *d_counters, void *cudaStream);

/*
 * Paired-end aligner handle: the ChimericPairedEndAligner(IntersectingPairedEndAligner) stack that
 * PairedAlignerContext::runIterationThread builds per thread (reference SNAPLib/PairedAligner.cpp:547-638).
 * Scope: no secondary results (-om unset); on an index with ALT contigs the pairing is ALT-aware (two score sets, liftover of ALT pairs onto their primary contig) unless params->altAwareness = 0 (-A-).  Soft clipping (the default) runs the Hamming / gapless
 * passes of both aligners (IntersectingPairedEndAligner::alignHamming, BaseAligner::AlignRead(useHamming) +
 * alignAffineGap); useSoftClipping = 0 is `snap paired -hc`.
 */
void snapgpu_paired_params_default(snapgpu_paired_params *pp);   /* `snap paired` 2.0.5 defaults */
int  snapgpu_paired_aligner_create(const snapgpu_index *idx, const snapgpu_params *params, const snapgpu_paired_params *pparams,
                                   int64_t maxBatchPairs, snapgpu_aligner **out);

/*
 * Replaces the loop body `aligner->align(reads[0], reads[1], results, ...)` + the useful-read pre-filter
 * (reference SNAPLib/PairedAligner.cpp:640-800, ChimericPairedEndAligner.cpp:126-448,
 * IntersectingPairedEndAligner.cpp:169-252) for a batch of nPairs pairs.  Reads are laid out as in
 * snapgpu_align_single with pair i = reads 2i (first in pair) and 2i+1; offsets/lens hold 2*nPairs entries.
 * counters may be NULL; lvCalls / affineGapCalls count both the intersecting and the single-end fallback aligner.
 * Fields the reference itself leaves undefined (mapq / scorePriorToClipping of an end reported NotFound by the
 * single-end fallback: uninitialised stack there) are returned as 0.
 */
int  snapgpu_align_paired(snapgpu_aligner *a, int64_t nPairs, const char *bases, const char *quals,
                          const uint64_t *offsets, const uint32_t *lens,
                          snapgpu_paired_result *results, snapgpu_counters *counters);

/* Device-pointer form (see snapgpu_align_single_device).  Errors raised inside the kernel (a candidate pool that the
 * reference would soft_exit() on, an over-long read) are latched in the aligner: snapgpu_aligner_check() reports them. */
int  snapgpu_align_paired_device(snapgpu_aligner *a, int64_t nPairs, const char *d_bases, const char *d_quals,
                                 const uint64_t *d_offsets, const uint32_t *d_lens,
                                 snapgpu_paired_result *d_results, snapgpu_counters *d_counters,
                                 void *cudaStream);

/*
 * Insert-size inference (`snap paired -ins`, reference PairedAligner.cpp:889-925).  An estimator holds what stock keeps per worker
 * thread: a window of samples and the current (minSpacing, maxSpacing).  A pair that is not useless adds a sample when its
 * primary record passes the filters (`filterFlags`, after the -fs fix-up) and its ends are FORWARD/RC or RC/FORWARD: the distance
 * between the two locations.  When the window holds `window` samples it is sorted and the new range computed
 * (PairedAligner.cpp:424-458); the pair after the one that filled it is the first aligned with that range.
 *
 * snapgpu_spacing_create: the initial range is the aligner's -s range.  filterFlags takes the bits of AlignerOptions::filterFlags
 * (FilterUnaligned 0x1, FilterSingleHit 0x2, FilterMultipleHits 0x4, FilterBothMatesMatch 0x8, FilterTooShort 0x10; -F a is 0x16).  window 0 means 262144, stock's; any other value (4..262144) is a test
 * seam only and does not reproduce stock.  The estimator lives on the aligner's device and may be used with any paired aligner
 * handle on that device.
 */
typedef struct snapgpu_spacing snapgpu_spacing;
int  snapgpu_spacing_create(const snapgpu_aligner *a, int32_t filterFlags, int64_t window, snapgpu_spacing **out);
void snapgpu_spacing_destroy(snapgpu_spacing *est);
/* The current range, the samples taken so far and the number of range updates. */
int  snapgpu_spacing_get(const snapgpu_spacing *est, int32_t *minSpacing, uint32_t *maxSpacing, int64_t *samples, int64_t *updates);
/* Alignment sub-launches issued for this estimator, and the host seconds spent sorting full windows and computing their ranges. */
int  snapgpu_spacing_timing(const snapgpu_spacing *est, int64_t *subLaunches, double *statSeconds);

/* snapgpu_align_paired under insert-size inference: every pair is aligned with the range stock would use for it, and the
 * estimator's state carries over between calls, so results do not depend on how the pairs are split into calls.  The pairs run in
 * sub-launches; a call makes at most 5 per range update it performs, plus 5.  Counters count each pair once.  A kernel error
 * (see snapgpu_aligner_check) fails the call and leaves the estimator as it was before the sub-launch that raised it. */
int  snapgpu_align_paired_ins(snapgpu_aligner *a, snapgpu_spacing *est, int64_t nPairs, const char *bases, const char *quals,
                              const uint64_t *offsets, const uint32_t *lens,
                              snapgpu_paired_result *results, snapgpu_counters *counters);
/* Device-pointer form.  Not asynchronous: it synchronises `cudaStream` (NULL = the aligner's own) after every sub-launch to read the
 * sample count back.  d_counters (may be NULL) are added to, as snapgpu_align_paired_device does. */
int  snapgpu_align_paired_ins_device(snapgpu_aligner *a, snapgpu_spacing *est, int64_t nPairs, const char *d_bases, const char *d_quals,
                                     const uint64_t *d_offsets, const uint32_t *d_lens,
                                     snapgpu_paired_result *d_results, snapgpu_counters *d_counters, void *cudaStream);

/* Synchronises `cudaStream` (NULL = the aligner's own) and returns non-zero (message in snapgpu_last_error) if a
 * kernel of this aligner latched an error since the last check. */
int  snapgpu_aligner_check(snapgpu_aligner *a, void *cudaStream);

/*
 * FASTQ ingest (SURVEY 8f row N2).  Replaces, for a whole buffer of FASTQ text at once, FASTQReader::getReadFromBuffer
 * (reference SNAPLib/FASTQ.cpp:229-300), the upper-casing / '.' -> 'N' of Read::init (Read.h:465-492) and Read::clip
 * (Read.h:567-619), and leaves the reads in HBM in exactly the layout snapgpu_align_single_device /
 * snapgpu_align_paired_device take (for pairs from two files: parse each, interleave offsets/lens on the host, or hand an
 * interleaved FASTQ).  Only complete 4-line records are consumed; *bytesConsumed says where the next call must start.
 * clippingType: 0 none, 1 front, 2 back (SNAP's default, `-C-+`), 3 both (Read.h:88); quality '#' is what gets clipped.
 * Per read r: bases/quals at [offsets[r], offsets[r]+lens[r]) of the output buffers (already clipped and upper-cased),
 * idOffsets[r]/idLens[r] = the read name inside `text` (without '@', up to the first space), frontClipped[r] = bases
 * removed at the front.  Any of idOffsets / idLens / frontClipped may be NULL.
 * A syntax error the reference would exit on (blank line, bad first character of a line, read longer than
 * MAX_READ_LENGTH) makes the call fail with the reason in snapgpu_last_error().
 */
typedef struct snapgpu_fastq snapgpu_fastq;     /* opaque: workspace for buffers of up to maxBytes / maxReads */
int  snapgpu_fastq_create(int device, int64_t maxBytes, int64_t maxReads, snapgpu_fastq **out);
void snapgpu_fastq_destroy(snapgpu_fastq *f);
/* DEVICE pointers for text and all outputs; output buffers must hold nBytes/2 bytes and maxReads entries.  Synchronises
 * `cudaStream` (NULL = the handle's own) once, to learn the record count. */
int  snapgpu_fastq_parse_device(snapgpu_fastq *f, const char *d_text, int64_t nBytes, int clippingType,
                                char *d_bases, char *d_quals, uint64_t *d_offsets, uint32_t *d_lens,
                                uint64_t *d_idOffsets, uint32_t *d_idLens, uint32_t *d_frontClipped,
                                int64_t *nReads, int64_t *bytesConsumed, void *cudaStream);
/* HOST pointers; copies inside. */
int  snapgpu_fastq_parse(snapgpu_fastq *f, const char *text, int64_t nBytes, int clippingType,
                         char *bases, char *quals, uint64_t *offsets, uint32_t *lens,
                         uint64_t *idOffsets, uint32_t *idLens, uint32_t *frontClipped,
                         int64_t *nReads, int64_t *bytesConsumed);

/*
 * Output stage (SURVEY 8f row N1): SAM records from result records, formatted on the device.
 * snapgpu_sam_format_single replaces, for one batch, SimpleReadWriter::writeReads (reference SNAPLib/ReadWriter.cpp:170-330) ->
 * SAMFormat::writeRead (SAM.cpp:1897-2352) -> createSAMLine (:1423-1573) and computeCigarString (:2595-2766) with
 * LandauVishkinWithCigar (LandauVishkin.cpp:141-650) / AffineGapVectorizedWithCigar (AffineGapVectorized.cpp:159-1128);
 * snapgpu_sam_format_paired replaces SimpleReadWriter::writePairs (ReadWriter.cpp:362-560) -> SAMFormat::writePairs
 * (SAM.cpp:1574-1896) and fillMateInfo (:1308-1422): two records per pair, in genome order, with mate fields and QS.
 * Primary alignments, default tags (PG, NM, the default read group line); the header lines are the caller's.
 * reads / ids / results are HOST arrays in the layout of snapgpu_align_single / _paired (ids: concatenated, idOffsets / idLens per
 * read, at most 255 characters each); `text` receives the records back to back, *textBytes their total length.
 * `useM`: M instead of = / X operations (SNAP's default, -M).  Scoring parameters and useAffineGap are taken from `params`.
 * Quality clipping (Read::clip, reference SNAPLib/Read.h:567-619): hand over the UNCLIPPED reads plus, per read, frontClipped[i] (bases clipped
 * at the front) and clippedLens[i] (length of the view that was aligned) -- e.g. snapgpu_fastq_parse's frontClipped and lens outputs next to
 * the text's own sequence lines -- or NULL for both when nothing was clipped.  The records then carry the whole read with S operations,
 * like stock SNAP's.  One octet of threads per read: the eight threads are the eight lanes of the reference's SSE vectors in the CIGAR DP.
 */
typedef struct snapgpu_sam snapgpu_sam;
int  snapgpu_sam_create(const snapgpu_index *idx, const snapgpu_params *params, int32_t useM, int64_t maxBatchReads, snapgpu_sam **out);
void snapgpu_sam_destroy(snapgpu_sam *s);
int  snapgpu_sam_format_single(snapgpu_sam *s, int64_t nReads, const char *bases, const char *quals, const uint64_t *offsets, const uint32_t *lens,
                               const char *ids, const uint64_t *idOffsets, const uint32_t *idLens,
                               const uint32_t *frontClipped, const uint32_t *clippedLens,
                               const snapgpu_single_result *results, char *text, int64_t textCapacity, int64_t *textBytes);
int  snapgpu_sam_format_paired(snapgpu_sam *s, int64_t nReads, const char *bases, const char *quals, const uint64_t *offsets, const uint32_t *lens,
                               const char *ids, const uint64_t *idOffsets, const uint32_t *idLens,
                               const uint32_t *frontClipped, const uint32_t *clippedLens,
                               const snapgpu_paired_result *results, char *text, int64_t textCapacity, int64_t *textBytes);

/* SNAPGPU_FORMAT_BAM: the format calls write uncompressed BAM alignment records (block_size, the fixed fields, bin, CIGAR words, 4-bit
 * sequence, qualities, the default tags: BAMFormat::writeRead / writePairs, reference SNAPLib/Bam.cpp:1033-1310, 1312-1509, 1812-2031) back
 * to back instead of SAM text; snapgpu_bgzf_device wraps such a stream (or a header) into BGZF members, which is what a .bam file is made of. */
enum { SNAPGPU_FORMAT_SAM = 0, SNAPGPU_FORMAT_BAM = 1 };
int  snapgpu_sam_set_format(snapgpu_sam *s, int format);
/* The header that goes in front of the records (HOST buffers; no kernel): SAMFormat::writeHeader (reference SNAPLib/SAM.cpp:1203-1305) for FASTQ input --
 * @HD VN:1.6 GO:query | SO:coordinate (sorted), the read-group line (rgLine; NULL = the reference's fallback "@RG\tID:FASTQ\tSM:sample"; stock snap-aligner
 * passes "@RG\tID:FASTQ\tPL:Illumina\tPU:pu\tLB:lb\tSM:sm"), @PG ID:SNAP PN:SNAP CL:<commandLine> VN:<version>, one @SQ per contig in original order
 * (LN without the chromosome padding, AH:* for ALT contigs) -- or, in SNAPGPU_FORMAT_BAM, BAMFormat::writeHeader's block (Bam.cpp:969-1030): "BAM\1",
 * l_text, that text, n_ref, the reference table.  header || records, wrapped by snapgpu_bgzf_[deflate_]device and closed with the 28-byte BGZF
 * end-of-file member, is a complete .bam. */
int  snapgpu_sam_header(const snapgpu_sam *s, int sorted, const char *commandLine, const char *version, const char *rgLine,
                        char *out, int64_t outCapacity, int64_t *outBytes);
/* BGZF members (reference SNAPLib/GzipDataWriter.cpp; SAM spec 4.1) over nBytes of DEVICE data, written to d_out: members of up to 65280
 * payload bytes, each ONE STORED deflate block with its CRC-32 -- valid BGZF that inflates to exactly the payload (no compressor runs on
 * the device; the reference compresses, so files differ in size, not in content).  outCapacity >= nBytes + 31 per member.  Asynchronous on `cudaStream`. */
int  snapgpu_bgzf_device(const char *d_in, int64_t nBytes, char *d_out, int64_t outCapacity, int64_t *outBytes, void *cudaStream);
/* The same with a compressor on the device (reference: GzipCompressWorker hands every chunk to zlib's deflate(), SNAPLib/GzipDataWriter.cpp:153-276): every
 * member is ONE dynamic-Huffman deflate block over an LZ77 parse of its 65280 payload bytes, built by a thread block (snap_b200/csrc/sg_deflate.h: strided
 * hash match finding, the greedy parse by pointer jumping, minimum-redundancy codes, a prefix sum of token bit lengths); a member that would not shrink is
 * stored.  Any inflater gives back exactly the payload (CRC-32 / ISIZE checked); the compressed bytes differ from zlib's, as zlib's do between levels.
 * Members are contiguous in d_out; outCapacity >= nBytes + 31 per member is always enough.  memberOffsets (HOST, optional, one entry per member plus one):
 * where each member starts in d_out, the last entry = *outBytes -- what a .bai of the compressed file needs (snapgpu_bam_index_members_device).
 * `s` lends its work buffer and stream.  Synchronises `cudaStream` (NULL = the handle's own). */
int  snapgpu_bgzf_deflate_device(snapgpu_sam *s, const char *d_in, int64_t nBytes, char *d_out, int64_t outCapacity, int64_t *outBytes,
                                 uint64_t *memberOffsets, void *cudaStream);

/* SURVEY 8(f) row N4, the sort: the reference's sorting writer (`-so`; SortedDataFilter, reference SNAPLib/SortedDataWriter.cpp:905-1010) files
 * every record under the key of the genome location SimpleReadWriter passed to DataWriter::advance for it (ReadWriter.cpp:331, :601-615: the
 * record's own final location, its mate's when it is unaligned itself) -- (original contig number, 1-based position in the contig), (0, 0)
 * for location 0, (-1, 0) for an unaligned record with -1 compared as unsigned, so those come last -- stable-sorts each write batch by that key and copies the records
 * out in that order as one sorted run of its final merge.  snapgpu_sam_sort_device does that for the batch the LAST snapgpu_sam_format_*
 * call of `s` formatted (SAM or BAM records; d_text = where that call left them on the device, NULL = the handle's own staging buffer
 * after a host-buffer format call): one stable radix sort of the keys on the device, the
 * records moved by one warp each into d_sorted.  d_keysOut (optional, one uint64 per record, ascending: contig << 32 | position, contig 0xffffffff = unaligned) and
 * d_offsetsOut (optional, start of each sorted record) are what a merge of several runs, a BAM index or duplicate marking go on from; with
 * 180 GB of HBM a whole run's records can be ONE batch and no merge is left.  Synchronises `cudaStream` once.
 * Duplicate marking and the .bai index of the sorted stream: snapgpu_bam_markdup_device / snapgpu_bam_index_device below.  Not on the device: the k-way
 * merge of several runs (SortedDataFilterSupplier::mergeSort) -- a whole run is one batch here. */
int  snapgpu_sam_sort_device(snapgpu_sam *s, const char *d_text, char *d_sorted, int64_t sortedCapacity, int64_t *sortedBytes,
                             uint64_t *d_keysOut, uint64_t *d_offsetsOut, void *cudaStream);
int64_t snapgpu_sam_last_record_count(const snapgpu_sam *s);       /* records (2 per pair) of the last format call */

/* SURVEY 8(f) row N4, after the sort: what the reference's sorting BAM writer runs over the merged, coordinate-sorted record stream.
 * d_records: BAM alignment records back to back in DEVICE memory (snapgpu_sam_sort_device's output in SNAPGPU_FORMAT_BAM, or any sorted stream),
 * d_offsets[i]: where record i starts.
 *
 * snapgpu_bam_markdup_device = BAMDupMarkFilter (reference SNAPLib/Bam.cpp:2619-3121): sets FLAG 0x400 in place on every record the reference would set it
 * on -- fragments and pairs with the same library, unclipped 5' end(s) and strand(s); the copy with the largest sum of base qualities >= 15 (plus the
 * mate's QS tag for pairs) stays unmarked, ties go to the smaller tile / x / y of an Illumina read name, then to file order; a mapped pair beats a
 * fragment -- including the reference's windowing of the stream into overlapping runs of 2 x (MAX_READ_LENGTH + MAX_K) bases.  Bit-identical to the
 * reference for a stream it handles as one write batch.  On the device: the runs by pointer jumping, the records radix-sorted by key, one thread per key
 * (snap_b200/csrc/sg_bampost.h).  *nMarked = records newly flagged.  Synchronises `cudaStream` once.
 *
 * snapgpu_bam_index_device = BAMIndexSupplier (Bam.cpp:3229-3440): the .bai of the FILE whose uncompressed content is `headerBytes` bytes of BAM header
 * and reference table followed by these records, wrapped by snapgpu_bgzf_device as ONE stream (members of 0xff00 payload bytes) and closed with the
 * standard 28-byte end-of-file member.  Same bins, chunks (one per maximal stretch of equal (refID, bin)), per-reference metadata (pseudo-bin 37450:
 * file range, mapped / unmapped counts) and 16 Kbp linear index as the reference writes -- including its filing of a record under the window of its
 * END and 0 for windows no record opened -- with this file's virtual offsets; bins in ascending order.  `bai` is HOST memory; recordBytes = total size
 * of the records.  Synchronises `cudaStream`. */
int  snapgpu_bam_markdup_device(snapgpu_sam *s, char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t *nMarked, void *cudaStream);
int  snapgpu_bam_index_device(snapgpu_sam *s, const char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t recordBytes, int64_t headerBytes,
                              char *bai, int64_t baiCapacity, int64_t *baiBytes, void *cudaStream);
/* The .bai of the same content wrapped by snapgpu_bgzf_deflate_device (compressed members): memberOffsets / nMembers as that call reported them for the
 * stream header || records (nMembers = ceil((headerBytes + recordBytes) / 65280), memberOffsets[nMembers] = end of the last data member). */
int  snapgpu_bam_index_members_device(snapgpu_sam *s, const char *d_records, const uint64_t *d_offsets, int64_t nRecords, int64_t recordBytes, int64_t headerBytes,
                                      const uint64_t *memberOffsets, int64_t nMembers, char *bai, int64_t baiCapacity, int64_t *baiBytes, void *cudaStream);

/* Device-resident forms: every array, and the text buffer, is a DEVICE pointer -- the reads as parsed by snapgpu_fastq_parse_device, the
 * records as left by snapgpu_align_*_device -- so a batch goes from FASTQ text to SAM text without its reads or results visiting the
 * host.  maxReadLen = the longest read of the batch; ids: concatenated, idOffsets / idLens per read.  The packed text is left in d_text;
 * the call synchronises `cudaStream` (NULL = the handle's own) once, to learn *textBytes. */
int  snapgpu_sam_format_single_device(snapgpu_sam *s, int64_t nReads, uint32_t maxReadLen, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                                      const uint32_t *d_lens, const char *d_ids, const uint64_t *d_idOffsets, const uint32_t *d_idLens,
                                      const uint32_t *d_frontClipped, const uint32_t *d_clippedLens, const snapgpu_single_result *d_results,
                                      char *d_text, int64_t textCapacity, int64_t *textBytes, void *cudaStream);
int  snapgpu_sam_format_paired_device(snapgpu_sam *s, int64_t nReads, uint32_t maxReadLen, const char *d_bases, const char *d_quals, const uint64_t *d_offsets,
                                      const uint32_t *d_lens, const char *d_ids, const uint64_t *d_idOffsets, const uint32_t *d_idLens,
                                      const uint32_t *d_frontClipped, const uint32_t *d_clippedLens, const snapgpu_paired_result *d_results,
                                      char *d_text, int64_t textCapacity, int64_t *textBytes, void *cudaStream);

/* Number of kernel launches issued through this aligner since creation (bench.py's gpu_launches). */
int64_t snapgpu_aligner_launch_count(const snapgpu_aligner *a);
/* Reads the last two-pass launch of a single-end aligner handed from its first pass to its second (affine-gap) pass; -1 for an aligner
 * that has no two-pass launch (paired, or -ne).  Waits for the aligner's device to finish its work first. */
int64_t snapgpu_aligner_deferred_count(snapgpu_aligner *a);

/*
 * Leaf kernels exposed for parity tests (never used by the product path's callers).
 * Batched LandauVishkin<dir>::computeEditDistance (reference SNAPLib/LandauVishkin.h:100-351).
 * Job j: text = textBuf + textOff[j] (for dir=-1 the pointer is one past the first text char, as the
 * reference's callers pass it), pattern/quality at patOff[j].  Outputs per job.
 */
typedef struct snapgpu_lv_job {
    uint64_t textOff; uint64_t patOff; int32_t textLen; int32_t patternLen; int32_t k; int32_t dir;
} snapgpu_lv_job;
typedef struct snapgpu_lv_out {
    int32_t score; int32_t netIndel; int32_t totalIndels; int32_t textSpan; double matchProbability;
} snapgpu_lv_out;
int  snapgpu_test_lv(int device, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf,
                     uint64_t patBytes, const snapgpu_lv_job *jobs, int64_t nJobs, snapgpu_lv_out *out);

/*
 * Batched AffineGapVectorized<dir>::computeScore / computeScoreBanded
 * (reference SNAPLib/AffineGapVectorized.h:821-1339 / 256-819).
 */
typedef struct snapgpu_ag_job {
    uint64_t textOff; uint64_t patOff; int32_t textLen; int32_t patternLen; int32_t w; int32_t scoreInit;
    int32_t dir; int32_t isRC; int32_t banded; int32_t useClippingOptimizations;
} snapgpu_ag_job;
typedef struct snapgpu_ag_out {
    int32_t agScore; int32_t textOffset; int32_t patternOffset; int32_t nEdits; double matchProbability;
} snapgpu_ag_out;
typedef struct snapgpu_ag_params {
    int32_t matchReward, subPenalty, gapOpenPenalty, gapExtendPenalty, fivePrimeEndBonus, threePrimeEndBonus;
} snapgpu_ag_params;
int  snapgpu_test_ag(int device, const snapgpu_ag_params *p, const char *textBuf, uint64_t textBytes,
                     const char *patBuf, const char *qualBuf, uint64_t patBytes,
                     const snapgpu_ag_job *jobs, int64_t nJobs, snapgpu_ag_out *out);

/*
 * The same leaves in their warp-cooperative form (the form the alignment kernel uses): one job per warp over nWarps
 * warps.  With nWarps == 1 the jobs run in order on one scratch arena, i.e. with the call history of a sequential run.
 */
int  snapgpu_test_lv_warp(int device, const char *textBuf, uint64_t textBytes, const char *patBuf, const char *qualBuf,
                          uint64_t patBytes, const snapgpu_lv_job *jobs, int64_t nJobs, snapgpu_lv_out *out, int nWarps);
int  snapgpu_test_ag_warp(int device, const snapgpu_ag_params *p, const char *textBuf, uint64_t textBytes,
                          const char *patBuf, const char *qualBuf, uint64_t patBytes,
                          const snapgpu_ag_job *jobs, int64_t nJobs, snapgpu_ag_out *out, int nWarps);

#ifdef __cplusplus
}
#endif
#endif /* SNAPGPU_H */
