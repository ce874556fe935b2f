"""Python host-side mirror of the C ABI in include/snapgpu.h (ctypes over snap_b200/csrc/libsnapgpu.so).

This is plumbing for tests and bench.py; the product is the CUDA library.  There is no CPU path here: if the
library is missing, or no CUDA device is usable, every call raises.
Names mirror the reference's: Index ~ GenomeIndex (loadFromDirectory / lookupSeed32), SingleAligner ~ the
per-thread BaseAligner loop of SingleAligner.cpp:197-338.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SNAPGPU_LIB") or os.path.join(HERE, "csrc", "libsnapgpu.so")      # SNAPGPU_LIB: A/B builds of the same library


class SnapGpuError(RuntimeError):
    pass


class Params(C.Structure):
    """snapgpu_params (AlignerOptions / AlignerContext fields the hot path reads)."""
    _fields_ = [
        ("struct_size", C.c_uint32), ("maxHits", C.c_uint32), ("maxDist", C.c_uint32),
        ("numSeedsFromCommandLine", C.c_uint32), ("seedCoverage", C.c_double),
        ("minWeightToCheck", C.c_uint32), ("extraSearchDepth", C.c_uint32), ("minReadLength", C.c_uint32),
        ("useAffineGap", C.c_int32), ("matchReward", C.c_int32), ("subPenalty", C.c_int32),
        ("gapOpenPenalty", C.c_int32), ("gapExtendPenalty", C.c_int32), ("fivePrimeEndBonus", C.c_int32),
        ("threePrimeEndBonus", C.c_int32), ("noUkkonen", C.c_int32), ("noOrderedEvaluation", C.c_int32),
        ("noTruncation", C.c_int32), ("noEditDistance", C.c_int32), ("noBandedAffineGap", C.c_int32),
        ("altAwareness", C.c_int32), ("maxScoreGapToPreferNonAltAlignment", C.c_int32),
        ("explorePopularSeeds", C.c_int32), ("stopOnFirstHit", C.c_int32),
        ("maxSecondaryAlignmentAdditionalEditDistance", C.c_int32), ("ignoreAlignmentAdjustmentsForOm", C.c_int32),
    ]


class PairedParams(C.Structure):
    """snapgpu_paired_params (the extra options `snap paired` reads, PairedAligner.cpp:228-243)."""
    _fields_ = [
        ("struct_size", C.c_uint32), ("minSpacing", C.c_int32), ("maxSpacing", C.c_uint32), ("intersectingAlignerMaxHits", C.c_uint32),
        ("maxCandidatePoolSize", C.c_uint32), ("maxSeedsSingleEnd", C.c_uint32), ("maxDistForIndels", C.c_uint32), ("forceSpacing", C.c_int32),
        ("minScoreRealignment", C.c_int32), ("minScoreGapRealignmentALT", C.c_int32), ("minAGScoreImprovement", C.c_int32),
        ("enableHammingScoringBaseAligner", C.c_int32), ("useSoftClipping", C.c_int32), ("flattenMAPQAtOrBelow", C.c_int32),
    ]


class Contig(C.Structure):
    """snapgpu_contig: one contig as the reference's Genome file holds it (name, location, ALT flag, original number, liftover)."""
    _fields_ = [
        ("name", C.c_char_p), ("beginningLocation", C.c_int64), ("isAlt", C.c_int32), ("originalContigNumber", C.c_int32),
        ("projBeginningLocation", C.c_int64), ("projIsRC", C.c_int32), ("reserved", C.c_int32), ("projCigar", C.c_char_p),
    ]


class SaveOptions(C.Structure):
    """snapgpu_save_options: the table geometry of a saved index (`snap-aligner index -keysize / -large / -h`)."""
    _fields_ = [("struct_size", C.c_uint32), ("keyBytes", C.c_uint32), ("large", C.c_uint32), ("reserved", C.c_uint32), ("slack", C.c_double)]


class IndexInfo(C.Structure):
    _fields_ = [
        ("countOfBases", C.c_int64), ("seedLen", C.c_uint32), ("hashTableKeySize", C.c_uint32),
        ("nHashTables", C.c_uint32), ("locationSize", C.c_uint32), ("largeHashTable", C.c_uint32),
        ("chromosomePadding", C.c_uint32), ("nContigs", C.c_uint32), ("reserved", C.c_uint32),
        ("overflowTableSize", C.c_uint64), ("hashTableSlots", C.c_uint64), ("hbmBytes", C.c_uint64),
    ]


RESULT_DTYPE = np.dtype([
    ("status", "<i4"), ("direction", "<i4"), ("location", "<i8"), ("origLocation", "<i8"),
    ("score", "<i4"), ("scorePriorToClipping", "<i4"), ("mapq", "<i4"), ("clippingForReadAdjustment", "<i4"),
    ("usedAffineGapScoring", "<i4"), ("basesClippedBefore", "<i4"), ("basesClippedAfter", "<i4"),
    ("agScore", "<i4"), ("supplementary", "<i4"), ("seedOffset", "<i4"),
    ("matchProbability", "<f8"), ("probabilityAllCandidates", "<f8"),
    ("popularSeedsSkipped", "<u4"), ("reserved", "<u4"),
])
PAIRED_RESULT_DTYPE = np.dtype([
    ("status", "<i4", 2), ("direction", "<i4", 2), ("location", "<i8", 2), ("origLocation", "<i8", 2), ("score", "<i4", 2),
    ("scorePriorToClipping", "<i4", 2), ("mapq", "<i4", 2), ("clippingForReadAdjustment", "<i4", 2), ("usedAffineGapScoring", "<i4", 2),
    ("basesClippedBefore", "<i4", 2), ("basesClippedAfter", "<i4", 2), ("agScore", "<i4", 2), ("supplementary", "<i4", 2),
    ("seedOffset", "<i4", 2), ("lvIndels", "<i4", 2), ("usedGaplessClipping", "<i4", 2), ("refSpan", "<i4", 2), ("liftover", "<i4", 2),
    ("popularSeedsSkipped", "<u4", 2), ("alignedAsPair", "<i4"), ("agForcedSingleAlignerCall", "<i4"),
    ("matchProbability", "<f8", 2), ("probabilityAllPairs", "<f8"),
])
assert PAIRED_RESULT_DTYPE.itemsize == 200
COUNTER_FIELDS = ["totalReads", "uselessReads", "singleHits", "multiHits", "notFound", "nHashTableLookups",
                  "nHashEntriesProbed", "nOverflowWordsRead", "lvCalls", "affineGapCalls",
                  "nHitsIgnoredBecauseOfTooHighPopularity"]
N_COUNTERS = len(COUNTER_FIELDS) + 71

# every symbol include/snapgpu.h declares
EXPORTS = [
    "snapgpu_last_error", "snapgpu_abi_version", "snapgpu_device_count", "snapgpu_params_default",
    "snapgpu_index_open", "snapgpu_index_build", "snapgpu_index_build_device", "snapgpu_index_build_genome", "snapgpu_index_build_genome_device", "snapgpu_index_save", "snapgpu_index_save_ex", "snapgpu_index_info_get", "snapgpu_index_close", "snapgpu_index_replicate", "snapgpu_host_alloc", "snapgpu_host_free",
    "snapgpu_group_create", "snapgpu_group_destroy", "snapgpu_group_size", "snapgpu_index_broadcast", "snapgpu_counters_allreduce",
    "snapgpu_lookup_seeds", "snapgpu_lookup_seeds_device", "snapgpu_measure_random_sector_rate", "snapgpu_aligner_create", "snapgpu_aligner_destroy", "snapgpu_align_single",
    "snapgpu_align_single_device", "snapgpu_align_single_secondary", "snapgpu_align_single_secondary_device", "snapgpu_paired_params_default", "snapgpu_paired_aligner_create", "snapgpu_align_paired",
    "snapgpu_align_paired_device", "snapgpu_aligner_check", "snapgpu_fastq_create", "snapgpu_fastq_destroy", "snapgpu_fastq_parse_device",
    "snapgpu_fastq_parse", "snapgpu_sam_create", "snapgpu_sam_destroy", "snapgpu_sam_format_single", "snapgpu_sam_format_paired", "snapgpu_sam_format_single_device", "snapgpu_sam_format_paired_device", "snapgpu_sam_set_format", "snapgpu_sam_header", "snapgpu_bgzf_device", "snapgpu_bgzf_deflate_device", "snapgpu_bam_index_members_device", "snapgpu_sam_sort_device", "snapgpu_sam_last_record_count", "snapgpu_bam_markdup_device", "snapgpu_bam_index_device", "snapgpu_aligner_launch_count", "snapgpu_aligner_deferred_count",
    "snapgpu_spacing_create", "snapgpu_spacing_destroy", "snapgpu_spacing_get", "snapgpu_spacing_timing", "snapgpu_align_paired_ins", "snapgpu_align_paired_ins_device", "snapgpu_test_lv", "snapgpu_test_ag", "snapgpu_test_lv_warp", "snapgpu_test_ag_warp",
]

ABI_VERSION = 9          # include/snapgpu.h SNAPGPU_ABI_VERSION this mirror was written against
_lib = None


def lib():
    """Loads the CUDA library.  Raises (never falls back) if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SnapGpuError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        L.snapgpu_last_error.restype = C.c_char_p
        if L.snapgpu_abi_version() != ABI_VERSION:
            raise SnapGpuError("%s has ABI version %d, this mirror expects %d: rebuild (python -c 'import __graft_entry__ as g; g.build()')"
                               % (LIB_PATH, L.snapgpu_abi_version(), ABI_VERSION))
        L.snapgpu_params_default.argtypes = [C.POINTER(Params)]
        L.snapgpu_index_open.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
        L.snapgpu_index_build.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                          C.POINTER(C.c_void_p)]
        L.snapgpu_index_build_device.argtypes = L.snapgpu_index_build.argtypes
        L.snapgpu_index_build_genome.argtypes = [C.c_void_p, C.c_int64, C.POINTER(Contig), C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                                                 C.POINTER(C.c_void_p)]
        L.snapgpu_index_build_genome_device.argtypes = L.snapgpu_index_build_genome.argtypes
        L.snapgpu_index_save_ex.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(SaveOptions)]
        L.snapgpu_lookup_seeds_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.snapgpu_index_save.argtypes = [C.c_void_p, C.c_char_p]
        L.snapgpu_index_info_get.argtypes = [C.c_void_p, C.POINTER(IndexInfo)]
        L.snapgpu_index_close.argtypes = [C.c_void_p]
        L.snapgpu_index_replicate.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.snapgpu_group_create.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        L.snapgpu_group_destroy.argtypes = [C.c_void_p]
        L.snapgpu_group_size.argtypes = [C.c_void_p]
        L.snapgpu_index_broadcast.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.snapgpu_counters_allreduce.argtypes = [C.c_void_p, C.c_void_p]
        L.snapgpu_host_alloc.restype = C.c_void_p
        L.snapgpu_host_alloc.argtypes = [C.c_size_t]
        L.snapgpu_host_free.argtypes = [C.c_void_p]
        L.snapgpu_lookup_seeds.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.snapgpu_measure_random_sector_rate.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.POINTER(C.c_double)]
        L.snapgpu_aligner_create.argtypes = [C.c_void_p, C.POINTER(Params), C.c_int64, C.POINTER(C.c_void_p)]
        L.snapgpu_aligner_destroy.argtypes = [C.c_void_p]
        L.snapgpu_align_single.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 6
        L.snapgpu_align_single_device.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 7
        L.snapgpu_align_single_secondary.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5 + [C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.snapgpu_align_single_secondary_device.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 5 + [C.c_int32, C.c_int32, C.c_int64] + [C.c_void_p] * 4
        L.snapgpu_paired_params_default.argtypes = [C.POINTER(PairedParams)]
        L.snapgpu_paired_aligner_create.argtypes = [C.c_void_p, C.POINTER(Params), C.POINTER(PairedParams), C.c_int64, C.POINTER(C.c_void_p)]
        L.snapgpu_align_paired.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 6
        L.snapgpu_align_paired_device.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 7
        L.snapgpu_spacing_create.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_void_p)]
        L.snapgpu_spacing_destroy.argtypes = [C.c_void_p]
        L.snapgpu_spacing_get.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.snapgpu_spacing_timing.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        L.snapgpu_align_paired_ins.argtypes = [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 6
        L.snapgpu_align_paired_ins_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 7
        L.snapgpu_aligner_check.argtypes = [C.c_void_p, C.c_void_p]
        L.snapgpu_fastq_create.argtypes = [C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_void_p)]
        L.snapgpu_fastq_destroy.argtypes = [C.c_void_p]
        L.snapgpu_sam_create.argtypes = [C.c_void_p, C.POINTER(Params), C.c_int32, C.c_int64, C.POINTER(C.c_void_p)]
        L.snapgpu_sam_destroy.argtypes = [C.c_void_p]
        L.snapgpu_sam_format_single.argtypes = [C.c_void_p, C.c_int64] + [C.c_void_p] * 11 + [C.c_int64, C.POINTER(C.c_int64)]
        L.snapgpu_sam_format_paired.argtypes = L.snapgpu_sam_format_single.argtypes
        L.snapgpu_sam_format_single_device.argtypes = [C.c_void_p, C.c_int64, C.c_uint32] + [C.c_void_p] * 11 + [C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.snapgpu_sam_format_paired_device.argtypes = L.snapgpu_sam_format_single_device.argtypes
        L.snapgpu_sam_set_format.argtypes = [C.c_void_p, C.c_int]
        L.snapgpu_bgzf_device.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.snapgpu_sam_sort_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_void_p]
        L.snapgpu_bam_markdup_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.snapgpu_sam_header.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        L.snapgpu_bgzf_deflate_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p, C.c_void_p]
        L.snapgpu_bam_index_members_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                                       C.POINTER(C.c_int64), C.c_void_p]
        L.snapgpu_bam_index_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.snapgpu_sam_last_record_count.restype = C.c_int64
        L.snapgpu_sam_last_record_count.argtypes = [C.c_void_p]
        L.snapgpu_fastq_parse.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int] + [C.c_void_p] * 7 + [C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.snapgpu_fastq_parse_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int] + [C.c_void_p] * 7 + [C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_void_p]
        L.snapgpu_aligner_launch_count.restype = C.c_int64
        L.snapgpu_aligner_launch_count.argtypes = [C.c_void_p]
        L.snapgpu_aligner_deferred_count.restype = C.c_int64
        L.snapgpu_aligner_deferred_count.argtypes = [C.c_void_p]
        L.snapgpu_test_lv.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64, C.c_void_p]
        L.snapgpu_test_ag.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                      C.c_int64, C.c_void_p]
        L.snapgpu_test_lv_warp.argtypes = L.snapgpu_test_lv.argtypes + [C.c_int]
        L.snapgpu_test_ag_warp.argtypes = L.snapgpu_test_ag.argtypes + [C.c_int]
        _lib = L
    return _lib


def _check(rc: int) -> None:
    if rc != 0:
        raise SnapGpuError(lib().snapgpu_last_error().decode(errors="replace"))


def _p(a):
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)


def default_params(**kw) -> Params:
    p = Params()
    lib().snapgpu_params_default(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def default_paired_params(**kw) -> PairedParams:
    p = PairedParams()
    lib().snapgpu_paired_params_default(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def counters_dict(arr: np.ndarray) -> dict:
    d = {k: int(arr[i]) for i, k in enumerate(COUNTER_FIELDS)}
    d["mapqHistogram"] = [int(x) for x in arr[len(COUNTER_FIELDS):]]
    return d


class Index:
    """The genome index resident in HBM (GenomeIndex::loadFromDirectory, reference GenomeIndex.cpp:1838)."""

    def __init__(self, handle, device):
        self.handle = handle
        self.device = device

    @staticmethod
    def open(directory: str, device: int = 0) -> "Index":
        h = C.c_void_p()
        _check(lib().snapgpu_index_open(directory.encode(), device, C.byref(h)))
        return Index(h, device)

    @staticmethod
    def build(bases_with_padding: np.ndarray, contig_starts, seed_len: int = 20, chromosome_padding: int = 2000,
              device: int = 0) -> "Index":
        """Builds the lookup structure on the device from padded bases (see snapgpu_index_build)."""
        h = C.c_void_p()
        b = np.ascontiguousarray(bases_with_padding, dtype=np.uint8)
        cs = np.ascontiguousarray(contig_starts, dtype=np.int64)
        _check(lib().snapgpu_index_build(_p(b), b.size, _p(cs), cs.size, seed_len, chromosome_padding, device, C.byref(h)))
        return Index(h, device)

    @staticmethod
    def build_device(d_bases_ptr: int, n_bases: int, contig_starts, seed_len: int = 20, chromosome_padding: int = 2000,
                     device: int = 0) -> "Index":
        """Like build(), from bases already resident in HBM (device pointer as int)."""
        h = C.c_void_p()
        cs = np.ascontiguousarray(contig_starts, dtype=np.int64)
        _check(lib().snapgpu_index_build_device(C.c_void_p(d_bases_ptr), n_bases, _p(cs), cs.size, seed_len, chromosome_padding, device,
                                                C.byref(h)))
        return Index(h, device)

    @staticmethod
    def build_genome(bases, contigs, seed_len: int = 20, chromosome_padding: int = 2000, device: int = 0, d_bases_ptr: int = 0) -> "Index":
        """snapgpu_index_build_genome: padded bases (host array, or bases_ptr/n of device memory when d_bases_ptr is given) and one dict
        per contig with the snapgpu_contig fields (name as bytes; projCigar bytes or None)."""
        arr = (Contig * len(contigs))()
        for i, c in enumerate(contigs):
            for k, v in c.items():
                setattr(arr[i], k, v)
        h = C.c_void_p()
        if d_bases_ptr:
            _check(lib().snapgpu_index_build_genome_device(C.c_void_p(d_bases_ptr), int(bases), arr, len(contigs), seed_len, chromosome_padding,
                                                           device, C.byref(h)))
        else:
            b = np.ascontiguousarray(bases, dtype=np.uint8)
            _check(lib().snapgpu_index_build_genome(_p(b), b.size, arr, len(contigs), seed_len, chromosome_padding, device, C.byref(h)))
        return Index(h, device)

    def lookup_seeds_device(self, d_seeds: int, n: int, d_nhits: int, d_hits: int = 0, d_probes: int = 0, max_hits: int = 0, stream: int = 0):
        _check(lib().snapgpu_lookup_seeds_device(self.handle, C.c_void_p(d_seeds), n, max_hits, C.c_void_p(d_nhits), C.c_void_p(d_hits),
                                                 C.c_void_p(d_probes), C.c_void_p(stream)))

    def replicate(self, device: int) -> "Index":
        """A copy of this index on another device of the same process (device-to-device copies)."""
        h = C.c_void_p()
        _check(lib().snapgpu_index_replicate(self.handle, device, C.byref(h)))
        return Index(h, device)

    def save(self, directory: str) -> None:
        """Writes a reference-format index directory (loadable by stock `snap-aligner`)."""
        _check(lib().snapgpu_index_save(self.handle, directory.encode()))

    def save_ex(self, directory: str, key_bytes: int = 4, large: bool = False, slack: float = 0.3) -> None:
        """Writes a reference-format index directory in the given table geometry (snapgpu_index_save_ex)."""
        o = SaveOptions(C.sizeof(SaveOptions), key_bytes, 1 if large else 0, 0, slack)
        _check(lib().snapgpu_index_save_ex(self.handle, directory.encode(), C.byref(o)))

    def info(self) -> IndexInfo:
        info = IndexInfo()
        _check(lib().snapgpu_index_info_get(self.handle, C.byref(info)))
        return info

    def lookup_seeds(self, seeds: np.ndarray, n: int, max_hits: int = 512, want_hits: bool = True):
        """Batched lookupSeed32 (reference GenomeIndex.cpp:2095)."""
        nh = np.zeros(2 * n, dtype=np.int64)
        hits = np.zeros(2 * n * max_hits, dtype=np.uint32) if want_hits else None
        probes = np.zeros(n, dtype=np.uint32)
        _check(lib().snapgpu_lookup_seeds(self.handle, _p(np.ascontiguousarray(seeds, dtype=np.uint8)), n, max_hits, _p(nh), _p(hits), _p(probes)))
        return nh.reshape(n, 2), (hits.reshape(n, 2, max_hits) if want_hits else None), probes

    def close(self):
        if self.handle:
            lib().snapgpu_index_close(self.handle)
            self.handle = None


class Group:
    """The devices one process drives, with NCCL communicators over them (snapgpu_group_create): index broadcast + counters all-reduce."""

    def __init__(self, devices):
        self.devices = list(devices)
        arr = (C.c_int * len(self.devices))(*self.devices)
        h = C.c_void_p()
        _check(lib().snapgpu_group_create(arr, len(self.devices), C.byref(h)))
        self.handle = h

    def broadcast_index(self, index: Index):
        out = (C.c_void_p * len(self.devices))()
        _check(lib().snapgpu_index_broadcast(self.handle, index.handle, out))
        return [index] + [Index(C.c_void_p(out[k]), self.devices[k]) for k in range(1, len(self.devices))]

    def allreduce_counters(self, counters: np.ndarray) -> np.ndarray:
        """counters: int64 [nDevices, N_COUNTERS] (host); returns the array with every row replaced by the column sums."""
        c = np.ascontiguousarray(counters, dtype=np.int64).copy()
        assert c.shape == (len(self.devices), N_COUNTERS)
        _check(lib().snapgpu_counters_allreduce(self.handle, _p(c)))
        return c

    def close(self):
        if self.handle:
            lib().snapgpu_group_destroy(self.handle)
            self.handle = None


class SingleAligner:
    """One per host thread, like BaseAligner (reference BaseAligner.h:19-20)."""

    def __init__(self, index: Index, params: Params | None = None, max_batch_reads: int = 1 << 20):
        self.index = index
        self.params = params if params is not None else default_params()
        h = C.c_void_p()
        _check(lib().snapgpu_aligner_create(index.handle, C.byref(self.params), max_batch_reads, C.byref(h)))
        self.handle = h
        self.max_batch_reads = max_batch_reads

    def align(self, batch, out=None):
        """Host buffers in, host results out (copies inside): snapgpu_align_single.  `out`: optional preallocated result
        array (e.g. a view of page-locked memory, which the library then DMAs into directly)."""
        res = np.zeros(batch.n, dtype=RESULT_DTYPE) if out is None else out[:batch.n]
        ctr = np.zeros(N_COUNTERS, dtype=np.int64)
        done = 0
        while done < batch.n:
            m = min(self.max_batch_reads, batch.n - done)
            sub_off = batch.offsets[done:done + m]
            sub_len = batch.lens[done:done + m]
            _check(lib().snapgpu_align_single(self.handle, m, _p(batch.bases), _p(batch.quals), _p(sub_off), _p(sub_len),
                                               C.c_void_p(res.ctypes.data + done * RESULT_DTYPE.itemsize), _p(ctr)))
            done += m
        return res, counters_dict(ctr)

    def align_secondary(self, batch, capacity: int = 64, max_secondary: int = 0x7fffffff, max_per_contig: int = -1):
        """`snap single -om` (the handle's params carry maxSecondaryAlignmentAdditionalEditDistance >= 0): snapgpu_align_single_secondary.
        Returns (primary results [n], secondary results [n, capacity], counts [n] (negative: -count did not fit), counters)."""
        res = np.zeros(batch.n, dtype=RESULT_DTYPE)
        sec = np.zeros((batch.n, capacity), dtype=RESULT_DTYPE)
        nsec = np.zeros(batch.n, dtype=np.int32)
        ctr = np.zeros(N_COUNTERS, dtype=np.int64)
        done = 0
        while done < batch.n:
            m = min(self.max_batch_reads, batch.n - done)
            sub_off = batch.offsets[done:done + m]
            sub_len = batch.lens[done:done + m]
            _check(lib().snapgpu_align_single_secondary(self.handle, m, _p(batch.bases), _p(batch.quals), _p(sub_off), _p(sub_len),
                                                         C.c_void_p(res.ctypes.data + done * RESULT_DTYPE.itemsize), max_secondary, max_per_contig, capacity,
                                                         C.c_void_p(sec.ctypes.data + done * capacity * RESULT_DTYPE.itemsize),
                                                         C.c_void_p(nsec.ctypes.data + done * 4), _p(ctr)))
            done += m
        return res, sec, nsec, counters_dict(ctr)

    def align_secondary_device(self, n, d_bases, d_quals, d_offsets, d_lens, d_results, capacity, d_secondary, d_nsecondary, max_secondary=0x7fffffff,
                               max_per_contig=-1, d_counters=0, stream=0):
        """Device pointers (ints) in; enqueues on `stream`; no synchronisation: snapgpu_align_single_secondary_device."""
        _check(lib().snapgpu_align_single_secondary_device(self.handle, n, C.c_void_p(d_bases), C.c_void_p(d_quals), C.c_void_p(d_offsets), C.c_void_p(d_lens),
                                                            C.c_void_p(d_results), max_secondary, max_per_contig, capacity, C.c_void_p(d_secondary),
                                                            C.c_void_p(d_nsecondary), C.c_void_p(d_counters), C.c_void_p(stream)))

    def check(self, stream=0):
        _check(lib().snapgpu_aligner_check(self.handle, C.c_void_p(stream)))

    def align_device(self, n, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters=0, stream=0):
        """Device pointers (ints) in; enqueues on `stream`; no synchronisation: snapgpu_align_single_device."""
        _check(lib().snapgpu_align_single_device(self.handle, n, C.c_void_p(d_bases), C.c_void_p(d_quals), C.c_void_p(d_offsets),
                                                  C.c_void_p(d_lens), C.c_void_p(d_results), C.c_void_p(d_counters), C.c_void_p(stream)))

    def launch_count(self) -> int:
        return int(lib().snapgpu_aligner_launch_count(self.handle))

    def deferred_count(self) -> int:
        """Reads the last two-pass launch sent on to its affine-gap pass (-1 without a two-pass launch); waits for the device."""
        return int(lib().snapgpu_aligner_deferred_count(self.handle))

    def close(self):
        if self.handle:
            lib().snapgpu_aligner_destroy(self.handle)
            self.handle = None

    def __del__(self):       # a handle dropped without close() must not keep its arenas (tens of GB of HBM) until the process ends
        try:
            self.close()
        except Exception:
            pass


class PairedAligner:
    """ChimericPairedEndAligner(IntersectingPairedEndAligner) for batches of pairs (reference PairedAligner.cpp:547-800).
    Pair i = reads 2i, 2i+1 of the batch."""

    def __init__(self, index: Index, params: Params, pparams: PairedParams, max_batch_pairs: int = 1 << 19):
        self.index = index
        self.params = params
        self.pparams = pparams
        h = C.c_void_p()
        _check(lib().snapgpu_paired_aligner_create(index.handle, C.byref(params), C.byref(pparams), max_batch_pairs, C.byref(h)))
        self.handle = h
        self.max_batch_pairs = max_batch_pairs

    def align(self, batch, out=None):
        """Host buffers in, host results out (copies inside): snapgpu_align_paired.  `out` as in SingleAligner.align."""
        n_pairs = batch.n // 2
        res = np.zeros(n_pairs, dtype=PAIRED_RESULT_DTYPE) if out is None else out[:n_pairs]
        ctr = np.zeros(N_COUNTERS, dtype=np.int64)
        done = 0
        while done < n_pairs:
            m = min(self.max_batch_pairs, n_pairs - done)
            sub_off = batch.offsets[2 * done:2 * (done + m)]
            sub_len = batch.lens[2 * done:2 * (done + m)]
            _check(lib().snapgpu_align_paired(self.handle, m, _p(batch.bases), _p(batch.quals), _p(sub_off), _p(sub_len),
                                               C.c_void_p(res.ctypes.data + done * PAIRED_RESULT_DTYPE.itemsize), _p(ctr)))
            done += m
        return res, counters_dict(ctr)

    def align_device(self, n_pairs, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters=0, stream=0):
        """Device pointers (ints) in; enqueues on `stream`; no synchronisation: snapgpu_align_paired_device."""
        _check(lib().snapgpu_align_paired_device(self.handle, n_pairs, C.c_void_p(d_bases), C.c_void_p(d_quals), C.c_void_p(d_offsets),
                                                  C.c_void_p(d_lens), C.c_void_p(d_results), C.c_void_p(d_counters), C.c_void_p(stream)))

    def check(self, stream=0):
        _check(lib().snapgpu_aligner_check(self.handle, C.c_void_p(stream)))

    def launch_count(self) -> int:
        return int(lib().snapgpu_aligner_launch_count(self.handle))

    def close(self):
        if self.handle:
            lib().snapgpu_aligner_destroy(self.handle)
            self.handle = None

    def __del__(self):       # a handle dropped without close() must not keep its arenas (tens of GB of HBM) until the process ends
        try:
            self.close()
        except Exception:
            pass


class SpacingEstimator:
    """Insert-size inference of `snap paired -ins` for one worker's stream of pairs (reference PairedAligner.cpp:889-925):
    snapgpu_spacing_*.  `filter_flags` are AlignerOptions::filterFlags bits; `window` 0 is stock's 262144, other values are a
    test seam."""

    def __init__(self, aligner: "PairedAligner", filter_flags: int = 0, window: int = 0):
        h = C.c_void_p()
        _check(lib().snapgpu_spacing_create(aligner.handle, filter_flags, window, C.byref(h)))
        self.handle = h
        self.aligner = aligner

    def get(self) -> dict:
        mn, mx, s, u = C.c_int32(), C.c_uint32(), C.c_int64(), C.c_int64()
        _check(lib().snapgpu_spacing_get(self.handle, C.byref(mn), C.byref(mx), C.byref(s), C.byref(u)))
        return {"minSpacing": mn.value, "maxSpacing": mx.value, "samples": s.value, "updates": u.value}

    def timing(self) -> dict:
        n, t = C.c_int64(), C.c_double()
        _check(lib().snapgpu_spacing_timing(self.handle, C.byref(n), C.byref(t)))
        return {"subLaunches": n.value, "statSeconds": t.value}

    def align(self, batch, out=None):
        """Host buffers in, host results out: snapgpu_align_paired_ins, in calls of at most the aligner's max_batch_pairs."""
        n_pairs = batch.n // 2
        res = np.zeros(n_pairs, dtype=PAIRED_RESULT_DTYPE) if out is None else out[:n_pairs]
        ctr = np.zeros(N_COUNTERS, dtype=np.int64)
        done = 0
        while done < n_pairs:
            m = min(self.aligner.max_batch_pairs, n_pairs - done)
            sub_off = batch.offsets[2 * done:2 * (done + m)]
            sub_len = batch.lens[2 * done:2 * (done + m)]
            _check(lib().snapgpu_align_paired_ins(self.aligner.handle, self.handle, m, _p(batch.bases), _p(batch.quals), _p(sub_off),
                                                  _p(sub_len), C.c_void_p(res.ctypes.data + done * PAIRED_RESULT_DTYPE.itemsize), _p(ctr)))
            done += m
        return res, counters_dict(ctr)

    def align_device(self, n_pairs, d_bases, d_quals, d_offsets, d_lens, d_results, d_counters=0, stream=0):
        """Device pointers (ints) in: snapgpu_align_paired_ins_device (synchronises `stream` between its sub-launches)."""
        _check(lib().snapgpu_align_paired_ins_device(self.aligner.handle, self.handle, n_pairs, C.c_void_p(d_bases), C.c_void_p(d_quals),
                                                      C.c_void_p(d_offsets), C.c_void_p(d_lens), C.c_void_p(d_results), C.c_void_p(d_counters),
                                                      C.c_void_p(stream)))

    def close(self):
        if self.handle:
            lib().snapgpu_spacing_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SamFormatter:
    """SAM records of a batch from its result records (SimpleReadWriter::writeReads / writePairs + SAMFormat for a whole batch)."""

    def __init__(self, index, params, max_batch_reads: int, use_m: bool = True):
        h = C.c_void_p()
        _check(lib().snapgpu_sam_create(index.handle, C.byref(params), 1 if use_m else 0, max_batch_reads, C.byref(h)))
        self.handle = h
        self.max_batch_reads = max_batch_reads

    def set_format(self, bam: bool) -> None:
        """False: SAM text (default); True: uncompressed BAM alignment records (snapgpu_sam_set_format)."""
        _check(lib().snapgpu_sam_set_format(self.handle, 1 if bam else 0))

    @staticmethod
    def pack_ids(ids):
        """ids (one bytes object per read) -> (concatenated uint8 array, offsets, lengths) as the C ABI takes them."""
        id_buf = np.frombuffer(b"".join(ids) + b"\0", dtype=np.uint8).copy()
        id_lens = np.array([len(x) for x in ids], dtype=np.uint32)
        id_offs = np.concatenate([[0], np.cumsum(id_lens[:-1], dtype=np.uint64)]).astype(np.uint64)
        return id_buf, id_offs, id_lens

    def format_arrays(self, batch, id_buf, id_offs, id_lens, results, paired: bool = False, text=None, front_clipped=None, clipped_lens=None):
        """The C ABI call itself (snapgpu_sam_format_single / _paired); returns (text buffer, bytes used)."""
        if text is None:
            text = np.zeros(int(batch.n) * (2 * int(batch.lens.max()) + 1024) + 4096, dtype=np.uint8)
        used = C.c_int64(0)
        fn = lib().snapgpu_sam_format_paired if paired else lib().snapgpu_sam_format_single
        fc = None if front_clipped is None else _p(np.ascontiguousarray(front_clipped, dtype=np.uint32))
        cl = None if clipped_lens is None else _p(np.ascontiguousarray(clipped_lens, dtype=np.uint32))
        _check(fn(self.handle, batch.n, _p(batch.bases), _p(batch.quals), _p(batch.offsets), _p(batch.lens), _p(id_buf), _p(id_offs), _p(id_lens), fc, cl,
                  _p(results), _p(text), text.size, C.byref(used)))
        return text, used.value

    def format_device(self, n_reads, max_read_len, d_bases, d_quals, d_offsets, d_lens, d_ids, d_id_offsets, d_id_lens, d_results, d_text, text_capacity,
                      paired: bool = False, d_front=0, d_clipped_lens=0, stream=0) -> int:
        """Device pointers (ints) in, packed SAM text left in d_text; returns the bytes used (snapgpu_sam_format_*_device)."""
        used = C.c_int64(0)
        fn = lib().snapgpu_sam_format_paired_device if paired else lib().snapgpu_sam_format_single_device
        _check(fn(self.handle, n_reads, max_read_len, C.c_void_p(d_bases), C.c_void_p(d_quals), C.c_void_p(d_offsets), C.c_void_p(d_lens), C.c_void_p(d_ids),
                  C.c_void_p(d_id_offsets), C.c_void_p(d_id_lens), C.c_void_p(d_front), C.c_void_p(d_clipped_lens), C.c_void_p(d_results), C.c_void_p(d_text),
                  text_capacity, C.byref(used), C.c_void_p(stream)))
        return used.value

    def sort_device(self, d_text, d_sorted, sorted_capacity, d_keys_out=0, d_offsets_out=0, stream=0) -> int:
        """Coordinate-sorts the records the last format_device call left in d_text into d_sorted (device pointers as ints); returns the bytes
        written (snapgpu_sam_sort_device: SortedDataFilter's per-batch stable sort, on the device)."""
        used = C.c_int64(0)
        _check(lib().snapgpu_sam_sort_device(self.handle, C.c_void_p(d_text), C.c_void_p(d_sorted), sorted_capacity, C.byref(used), C.c_void_p(d_keys_out),
                                             C.c_void_p(d_offsets_out), C.c_void_p(stream)))
        return used.value

    def last_record_count(self) -> int:
        return int(lib().snapgpu_sam_last_record_count(self.handle))

    def markdup_device(self, d_records, d_offsets, n_records, stream=0) -> int:
        """BAMDupMarkFilter over a coordinate-sorted stream of BAM records in device memory (pointers as ints): FLAG 0x400 set in place; returns
        the number of records newly flagged (snapgpu_bam_markdup_device)."""
        marked = C.c_int64(0)
        _check(lib().snapgpu_bam_markdup_device(self.handle, C.c_void_p(d_records), C.c_void_p(d_offsets), n_records, C.byref(marked), C.c_void_p(stream)))
        return marked.value

    def header(self, command_line: bytes, version: bytes, rg_line: bytes | None = b"@RG\tID:FASTQ\tPL:Illumina\tPU:pu\tLB:lb\tSM:sm", sorted_: bool = False) -> bytes:
        """The file header in front of the records: SAM text, or the BAM header block after set_format(bam=True) (snapgpu_sam_header)."""
        buf = np.zeros(1 << 20, dtype=np.uint8)
        used = C.c_int64(0)
        _check(lib().snapgpu_sam_header(self.handle, 1 if sorted_ else 0, command_line, version, rg_line, _p(buf), buf.size, C.byref(used)))
        return buf[:used.value].tobytes()

    def bgzf_deflate_device(self, d_in, n_bytes, d_out, out_capacity, stream=0):
        """Compressed BGZF members over device data (snapgpu_bgzf_deflate_device); returns (bytes written to d_out, member offsets [nMembers + 1])."""
        n_members = (int(n_bytes) + 0xff00 - 1) // 0xff00
        offs = np.zeros(n_members + 1, dtype=np.uint64)
        used = C.c_int64(0)
        _check(lib().snapgpu_bgzf_deflate_device(self.handle, C.c_void_p(d_in), n_bytes, C.c_void_p(d_out), out_capacity, C.byref(used), _p(offs), C.c_void_p(stream)))
        return int(used.value), offs

    def index_device(self, d_records, d_offsets, n_records, record_bytes, header_bytes, stream=0, member_offsets=None) -> bytes:
        """The .bai of header ‖ records as snapgpu_bgzf_device lays the file out (snapgpu_bam_index_device) or, given the member offsets
        snapgpu_bgzf_deflate_device reported, as that call laid it out (snapgpu_bam_index_members_device)."""
        cap = 1 << 20
        mo = None if member_offsets is None else np.ascontiguousarray(member_offsets, dtype=np.uint64)
        while True:
            out = np.empty(cap, dtype=np.uint8); used = C.c_int64(0)
            if mo is not None:
                rc = lib().snapgpu_bam_index_members_device(self.handle, C.c_void_p(d_records), C.c_void_p(d_offsets), n_records, record_bytes, header_bytes,
                                                            _p(mo), mo.size - 1, out.ctypes.data_as(C.c_void_p), cap, C.byref(used), C.c_void_p(stream))
            else:
                rc = lib().snapgpu_bam_index_device(self.handle, C.c_void_p(d_records), C.c_void_p(d_offsets), n_records, record_bytes, header_bytes,
                                                    out.ctypes.data_as(C.c_void_p), cap, C.byref(used), C.c_void_p(stream))
            if rc != 0 and b"too small" in lib().snapgpu_last_error() and cap < (1 << 32):
                cap *= 8
                continue
            _check(rc)
            return out[:used.value].tobytes()

    def format(self, batch, ids, results, paired: bool = False, front_clipped=None, clipped_lens=None) -> bytes:
        """batch: synth.ReadBatch (host arrays); ids: one bytes object per read; results: the aligner's records (one per read, or one
        per pair with paired=True)."""
        id_buf, id_offs, id_lens = self.pack_ids(ids)
        b = type(batch)(np.ascontiguousarray(batch.bases), np.ascontiguousarray(batch.quals), np.ascontiguousarray(batch.offsets), np.ascontiguousarray(batch.lens))
        text, used = self.format_arrays(b, id_buf, id_offs, id_lens, np.ascontiguousarray(results), paired, front_clipped=front_clipped, clipped_lens=clipped_lens)
        return text[:used].tobytes()

    def close(self):
        if self.handle:
            lib().snapgpu_sam_destroy(self.handle)
            self.handle = None

    def __del__(self):       # a handle dropped without close() must not keep its arenas (tens of GB of HBM) until the process ends
        try:
            self.close()
        except Exception:
            pass


class FastqParser:
    """FASTQ text -> clipped, upper-cased reads in the aligners' layout (FASTQReader::getReadFromBuffer + Read::clip for a whole buffer)."""

    CLIP_NONE, CLIP_FRONT, CLIP_BACK, CLIP_FRONT_AND_BACK = 0, 1, 2, 3

    def __init__(self, max_bytes: int, max_reads: int, device: int = 0):
        h = C.c_void_p()
        _check(lib().snapgpu_fastq_create(device, max_bytes, max_reads, C.byref(h)))
        self.handle = h
        self.max_bytes, self.max_reads = max_bytes, max_reads

    def parse(self, text: np.ndarray, clipping: int = 2):
        """Host buffer in (uint8 array), host arrays out: (bases, quals, offsets, lens, id_offsets, id_lens, front_clipped, bytes_consumed)."""
        text = np.ascontiguousarray(text, dtype=np.uint8)
        n = C.c_int64(0)
        used = C.c_int64(0)
        bases = np.zeros(text.size // 2 + 16, dtype=np.uint8)
        quals = np.zeros(text.size // 2 + 16, dtype=np.uint8)
        offs = np.zeros(self.max_reads, dtype=np.uint64)
        lens = np.zeros(self.max_reads, dtype=np.uint32)
        ido = np.zeros(self.max_reads, dtype=np.uint64)
        idl = np.zeros(self.max_reads, dtype=np.uint32)
        fc = np.zeros(self.max_reads, dtype=np.uint32)
        _check(lib().snapgpu_fastq_parse(self.handle, _p(text), text.size, clipping, _p(bases), _p(quals), _p(offs), _p(lens), _p(ido), _p(idl), _p(fc),
                                          C.byref(n), C.byref(used)))
        r = n.value
        total = int(offs[r - 1] + lens[r - 1]) if r else 0
        return bases[:total], quals[:total], offs[:r], lens[:r], ido[:r], idl[:r], fc[:r], used.value

    def parse_device(self, d_text, n_bytes, clipping, d_bases, d_quals, d_offsets, d_lens, d_id_offsets=0, d_id_lens=0, d_front=0, stream=0):
        n = C.c_int64(0)
        used = C.c_int64(0)
        _check(lib().snapgpu_fastq_parse_device(self.handle, C.c_void_p(d_text), n_bytes, clipping, C.c_void_p(d_bases), C.c_void_p(d_quals),
                                                 C.c_void_p(d_offsets), C.c_void_p(d_lens), C.c_void_p(d_id_offsets), C.c_void_p(d_id_lens), C.c_void_p(d_front),
                                                 C.byref(n), C.byref(used), C.c_void_p(stream)))
        return n.value, used.value

    def close(self):
        if self.handle:
            lib().snapgpu_fastq_destroy(self.handle)
            self.handle = None

    def __del__(self):       # a handle dropped without close() must not keep its arenas (tens of GB of HBM) until the process ends
        try:
            self.close()
        except Exception:
            pass


def bgzf_device(d_in: int, n_bytes: int, d_out: int, out_capacity: int, stream: int = 0) -> int:
    """BGZF members (stored deflate blocks + CRC-32) over device data; returns the bytes written to d_out (snapgpu_bgzf_device)."""
    used = C.c_int64(0)
    _check(lib().snapgpu_bgzf_device(C.c_void_p(d_in), n_bytes, C.c_void_p(d_out), out_capacity, C.byref(used), C.c_void_p(stream)))
    return used.value


def measure_random_sector_rate(table_bytes: int, n_accesses: int = 1 << 26, device: int = 0) -> float:
    """Random 32-byte sector reads per second over a table of table_bytes (the roofline of hash probing)."""
    r = C.c_double(0.0)
    _check(lib().snapgpu_measure_random_sector_rate(device, table_bytes, n_accesses, C.byref(r)))
    return r.value


def test_lv(text, pat, qual, jobs, out_dtype, device=0, warps=0):
    """warps == 0: scalar leaf, one job per thread; warps >= 1: warp-cooperative leaf, one job per warp."""
    out = np.zeros(jobs.size, dtype=out_dtype)
    if warps:
        _check(lib().snapgpu_test_lv_warp(device, _p(text), text.size, _p(pat), _p(qual), pat.size, _p(jobs), jobs.size, _p(out), warps))
    else:
        _check(lib().snapgpu_test_lv(device, _p(text), text.size, _p(pat), _p(qual), pat.size, _p(jobs), jobs.size, _p(out)))
    return out


def test_ag(text, pat, qual, jobs, out_dtype, params, device=0, warps=0):
    out = np.zeros(jobs.size, dtype=out_dtype)
    params = np.ascontiguousarray(params, dtype=np.int32)
    if warps:
        _check(lib().snapgpu_test_ag_warp(device, _p(params), _p(text), text.size, _p(pat), _p(qual), pat.size, _p(jobs), jobs.size, _p(out), warps))
    else:
        _check(lib().snapgpu_test_ag(device, _p(params), _p(text), text.size, _p(pat), _p(qual), pat.size, _p(jobs), jobs.size, _p(out)))
    return out
