"""Host-build checks of what the device index build and save rest on when they run in passes (snap_b200/csrc/sg_bucket.h,
sg_host.h): recovering a bucket slot's seed from the slot and its bucket, re-laying buckets into the reference's tables, and
planning key-range / table-range passes."""
import numpy as np
import pytest

import buildsim_lib as hs


def _revcomp(x: int, n: int) -> int:
    r = 0
    for _ in range(n):
        r = (r << 2) | (3 - (x & 3))
        x >>= 2
    return r


@pytest.mark.parametrize("bits", [32, 34, 40, 46, 48])
def test_bucket_unmix_inverts_mix(bits):
    rng = np.random.default_rng(bits)
    for c in [0, (1 << bits) - 1] + [int(v) for v in rng.integers(0, 1 << bits, size=2000, dtype=np.uint64)]:
        h = hs.bucket_mix(c, bits)
        assert h < (1 << bits)
        assert hs.bucket_unmix(h, bits) == c


@pytest.mark.parametrize("seed_len", [16, 20, 24])
@pytest.mark.parametrize("load", [0.3, 0.5, 0.9])
def test_slot_decode_round_trip(seed_len, load):
    """Bucket images at the smallest bucket count the tags allow, filled through sg_bucket_insert_seq around the wrap from the last
    bucket to bucket 0 (keys chosen by their h, so their homes straddle it) to the given load, plus seeds that are their own reverse
    complement.  Every used slot must decode to the seed and orientation it was inserted with."""
    bits = 2 * seed_len
    n_buckets = hs.bucket_min_count(bits)
    assert n_buckets == (1 << (bits - 30)) * 256
    window = min(n_buckets, 8192)
    rng = np.random.default_rng(seed_len * 10 + int(load * 10))
    span = (window // 2) * (1 << bits) // n_buckets                  # h values whose home is within window / 2 buckets of the wrap
    want_entries = int(load * 4 * window)
    keys = []                                                        # (canonical, orientation, seed)
    seen = set()
    last = (1 << bits) - (1 << bits) // n_buckets                    # the first dozen keys all have the last bucket as home
    while len(keys) < want_entries:
        if len(keys) < 12:
            h = last + int(rng.integers(0, (1 << bits) - last))
        else:
            h = (int(rng.integers(0, 2 * span)) - span) % (1 << bits)
        c = hs.bucket_unmix(h, bits)
        rc = _revcomp(c, seed_len)
        if c > rc or c in seen:
            continue
        seen.add(c)
        r = rng.random()
        for o in ((0,) if r < 0.4 else (1,) if r < 0.7 else (0, 1)):
            keys.append((c, o, c if o == 0 else rc))
    for _ in range(40):                                              # own reverse complements: only orientation 0 exists
        half = int(rng.integers(0, 1 << seed_len))
        c = (half << seed_len) | _revcomp(half, seed_len // 2)
        assert _revcomp(c, seed_len) == c
        if c not in seen:
            seen.add(c)
            keys.append((c, 0, c))
    img = hs.bucket_image(n_buckets)
    inserted = [hs.bucket_insert_seq(img, n_buckets, bits, c, o, i) for i, (c, o, _) in enumerate(keys)]
    assert sum(inserted) >= 0.97 * len(keys)
    used = np.nonzero((img & np.uint64(0xffffffff)) != np.uint64(0xffffffff))[0]
    assert used.size == sum(inserted)
    seeds, orients = hs.bucket_decode(img, n_buckets, seed_len, used)
    values = (img[used] & np.uint64(0xffffffff)).astype(np.int64)
    wrapped = 0
    for s, v, sd, o in zip(used, values, seeds, orients):
        c, want_o, want_seed = keys[v]
        assert (int(sd), int(o)) == (want_seed, want_o), (int(s), v)
        home = (hs.bucket_mix(c, bits) * n_buckets) >> bits
        wrapped += int(s) // 4 < home
    assert wrapped > 0                                               # some keys went past the last bucket to the first ones


def test_buckets_to_tables_reproduces_the_reference_tables(small_cfg):
    """The reference-built directory, re-laid into buckets and back into its own table geometry: for the seed at every genome
    position (whose lookup gives both strands) the hit sets and their order equal the original tables', and so do the per-table
    used counts."""
    orig = hs.BsIndex(small_cfg.idx)
    back = hs.BsIndex(small_cfg.idx).relayout().buckets_to_tables()
    assert np.array_equal(orig.table_used(), back.table_used())
    assert int(orig.table_used().sum()) > 0
    seeds = np.concatenate([np.lib.stride_tricks.sliding_window_view(c, 20) for c in small_cfg.contigs])
    seeds = np.ascontiguousarray(seeds)
    step = 20000
    n_hits = 0
    for a in range(0, len(seeds), step):
        chunk = np.ascontiguousarray(seeds[a:a + step])
        n1, h1 = orig.lookup(chunk, len(chunk))
        n2, h2 = back.lookup(chunk, len(chunk))
        assert np.array_equal(n1, n2), a
        k = np.minimum(n1, 512)
        mask = np.arange(512)[None, None, :] < k[:, :, None]
        assert np.array_equal(np.where(mask, h1, 0), np.where(mask, h2, 0)), a
        n_hits += int(n1.sum())
    assert n_hits >= len(seeds)                                      # every valid position finds at least itself


def _check_plan(bounds, bin_bytes, budget):
    assert bounds[0] == 0 and bounds[-1] == len(bin_bytes)
    assert np.all(np.diff(bounds) > 0)
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        assert int(np.sum(bin_bytes[lo:hi], dtype=np.uint64)) <= budget


def test_plan_passes():
    rng = np.random.default_rng(5)
    bins = rng.integers(0, 1000, size=4096).astype(np.uint64) * 24
    bins[rng.random(4096) < 0.2] = 0
    total = int(bins.sum())
    nonempty = int((bins > 0).sum())
    # everything fits: one pass
    b, bad = hs.plan_passes(bins, total)
    assert bad is None and list(b) == [0, 4096]
    b, _ = hs.plan_passes(bins, total * 10)
    assert list(b) == [0, 4096]
    # tighter budgets: contiguous ranges covering every bin, each within the budget, no more than needed
    for div in (2, 3, 10, 100):
        budget = total // div
        b, bad = hs.plan_passes(bins, budget)
        assert bad is None
        _check_plan(b, bins, budget)
        assert len(b) - 1 >= div
        sums = [int(bins[lo:hi].sum()) for lo, hi in zip(b[:-1], b[1:])]
        assert all(sums[i] + sums[i + 1] > budget for i in range(len(sums) - 1))      # greedy: no two neighbours would fit together
    # a forced minimum is honoured, up to one pass per non-empty bin
    for m in (2, 3, 7, nonempty, nonempty + 50):
        b, bad = hs.plan_passes(bins, total, m)
        assert bad is None
        _check_plan(b, bins, total)
        assert len(b) - 1 >= min(m, nonempty)
    b, _ = hs.plan_passes(bins, total, nonempty)
    assert len(b) - 1 == nonempty
    assert all(int((bins[lo:hi] > 0).sum()) == 1 for lo, hi in zip(b[:-1], b[1:]))
    # a few heavy bins among light ones still give the forced count
    lop = np.array([1, 1, 1, 1000, 0, 1, 5000, 1], dtype=np.uint64)
    b, _ = hs.plan_passes(lop, 10 ** 6, 5)
    _check_plan(b, lop, 10 ** 6)
    assert len(b) - 1 >= 5
    # a bin larger than the budget is refused, and named
    big = bins.copy()
    big[1234] = total
    b, bad = hs.plan_passes(big, total - 1)
    assert b is None and bad == 1234
