"""The device index build in key-range passes and the save in table-range passes (SNAPGPU_BUILD_PASSES forces them on a small
genome): the index must be the one a single sweep builds, and the saved directory the reference's own format with the same hits."""
import os
import struct

import numpy as np
import pytest

from conftest import OPTION_SETS, PAIRED_OPTION_SETS, differing, differing_pairs

pytestmark = pytest.mark.gpu

INFO_FIELDS = ("countOfBases", "nHashTables", "overflowTableSize", "hashTableSlots", "hbmBytes")


@pytest.fixture(scope="module")
def engine():
    from snap_b200 import engine as e
    assert e.lib().snapgpu_device_count() >= 1, "no CUDA device: the CUDA path has no fallback"
    return e


@pytest.fixture(scope="module")
def genomes(small_cfg):
    """small_cfg's padded genome, and a copy with runs of 'N' planted inside its contigs."""
    bases, starts = small_cfg.padded_bases()
    with_n = bases.copy()
    rng = np.random.default_rng(77)
    for s in starts:
        for _ in range(12):
            o = int(s) + int(rng.integers(100, 119_000))
            with_n[o:o + int(rng.integers(1, 60))] = ord("N")
    return {"plain": (bases, starts), "with_n": (with_n, starts)}


@pytest.fixture(scope="module")
def ref_gidx(engine, small_cfg):
    ix = engine.Index.open(small_cfg.idx)
    yield ix
    ix.close()


def _build(engine, monkeypatch, bases, starts, seed_len=20, layout="bucket", entry="host", passes=None):
    if passes is None:
        monkeypatch.delenv("SNAPGPU_BUILD_PASSES", raising=False)
    else:
        monkeypatch.setenv("SNAPGPU_BUILD_PASSES", str(passes))
    if layout == "snap":
        monkeypatch.setenv("SNAPGPU_INDEX_LAYOUT", "snap")
    else:
        monkeypatch.delenv("SNAPGPU_INDEX_LAYOUT", raising=False)
    try:
        if entry == "host":
            return engine.Index.build(bases, starts, seed_len=seed_len, chromosome_padding=2000)
        import torch
        d = torch.from_numpy(np.ascontiguousarray(bases)).cuda()
        ix = engine.Index.build_device(d.data_ptr(), d.numel(), starts, seed_len=seed_len, chromosome_padding=2000)
        torch.cuda.synchronize()
        return ix
    finally:
        monkeypatch.delenv("SNAPGPU_BUILD_PASSES", raising=False)
        monkeypatch.delenv("SNAPGPU_INDEX_LAYOUT", raising=False)


def _position_seeds(bases, seed_len):
    """The seed at every genome position (the lookup of a seed also gives its reverse complement's hits)."""
    return np.ascontiguousarray(np.lib.stride_tricks.sliding_window_view(bases, seed_len))


def _same_hits(a, b, seeds, max_hits=100, step=60000):
    for lo in range(0, len(seeds), step):
        chunk = np.ascontiguousarray(seeds[lo:lo + step])
        n1, h1, _ = a.lookup_seeds(chunk, len(chunk), max_hits)
        n2, h2, _ = b.lookup_seeds(chunk, len(chunk), max_hits)
        assert np.array_equal(n1, n2), lo
        mask = np.arange(max_hits)[None, None, :] < np.minimum(n1, max_hits)[:, :, None]
        assert np.array_equal(np.where(mask, h1, 0), np.where(mask, h2, 0)), lo


def _same_info(a, b):
    ia, ib = a.info(), b.info()
    for f in INFO_FIELDS:
        assert getattr(ia, f) == getattr(ib, f), f


@pytest.mark.parametrize("layout", ["bucket", "snap"])
@pytest.mark.parametrize("entry", ["host", "device"])
def test_forced_passes_build_the_one_pass_index(engine, genomes, ref_gidx, monkeypatch, layout, entry):
    for name, (bases, starts) in genomes.items():
        one = _build(engine, monkeypatch, bases, starts, layout=layout, entry=entry)
        seeds = _position_seeds(bases, 20)
        if name == "plain":
            _same_hits(ref_gidx, one, seeds)
        for passes in (2, 3, 7):
            ix = _build(engine, monkeypatch, bases, starts, layout=layout, entry=entry, passes=passes)
            _same_info(one, ix)
            _same_hits(one, ix, seeds)
            if name == "plain":
                _same_hits(ref_gidx, ix, seeds)
            ix.close()
        one.close()


@pytest.mark.parametrize("seed_len", [16, 24])
@pytest.mark.parametrize("layout", ["bucket", "snap"])
def test_forced_passes_other_seed_lengths(engine, genomes, monkeypatch, seed_len, layout):
    bases, starts = genomes["with_n"]
    one = _build(engine, monkeypatch, bases, starts, seed_len=seed_len, layout=layout)
    seeds = _position_seeds(bases, seed_len)
    for passes in (3, 7):
        ix = _build(engine, monkeypatch, bases, starts, seed_len=seed_len, layout=layout, entry="device" if passes == 7 else "host", passes=passes)
        _same_info(one, ix)
        _same_hits(one, ix, seeds)
        ix.close()
    one.close()


def test_one_pass_per_key_range(engine, genomes, ref_gidx, monkeypatch):
    """SNAPGPU_BUILD_PASSES above the number of non-empty key ranges: one pass per non-empty range of the seed's top 16 bits."""
    bases, starts = genomes["plain"]
    one = _build(engine, monkeypatch, bases, starts)
    ix = _build(engine, monkeypatch, bases, starts, passes=65536)
    _same_info(one, ix)
    _same_hits(ref_gidx, ix, _position_seeds(bases, 20))
    ix.close()
    one.close()


def test_multi_pass_index_aligns_like_the_reference(engine, genomes, small_cfg, reflib, monkeypatch):
    bases, starts = genomes["plain"]
    ix = _build(engine, monkeypatch, bases, starts, passes=3)
    ridx = reflib.RefIndex(small_cfg.idx)
    for opt in ("default_d14", "ne_d20", "d8_h20"):
        kw = OPTION_SETS[opt]
        al = engine.SingleAligner(ix, engine.default_params(**kw), 4096)
        for name in ("std150", "noisy150"):
            want, _ = reflib.RefSingleAligner(ridx, reflib.default_params(**kw)).align(small_cfg.reads[name])
            got, _ = al.align(small_cfg.reads[name])
            assert differing(want, got) == [], (opt, name)
        al.close()
    for opt in ("default_d14", "hc_d14"):
        kw, pkw = PAIRED_OPTION_SETS[opt]
        al = engine.PairedAligner(ix, engine.default_params(**{"numSeedsFromCommandLine": 8, **kw}), engine.default_paired_params(**pkw), 2048)
        for name in ("std150", "noisy150"):
            pb = small_cfg.pairs[name]
            want, _ = reflib.RefPairedAligner(ridx, reflib.default_params_paired(**kw), reflib.default_paired_params(**pkw)).align(pb)
            got, _ = al.align(pb)
            assert differing_pairs(want, got) == [], (opt, name)
        al.close()
    ix.close()


def _table_headers(directory):
    """(size, used) of every table in a GenomeIndexHash file (HashTable.cpp:199-260 headers)."""
    out = []
    with open(os.path.join(directory, "GenomeIndexHash"), "rb") as f:
        data = f.read()
    off = 0
    while off < len(data):
        magic, size, used, ks, vs, vc, _ = struct.unpack_from("<IQQIIII", data, off)
        assert magic == 0xb111b010 and ks == 4 and vs == 4 and vc == 1
        out.append((size, used))
        off += 36 + size * 8
    assert off == len(data)
    return out


def test_save_in_table_range_passes(engine, genomes, small_cfg, reflib, ref_gidx, monkeypatch, tmp_path):
    bases, starts = genomes["plain"]
    one = _build(engine, monkeypatch, bases, starts)
    d1 = str(tmp_path / "one")
    one.save(d1)
    ix = _build(engine, monkeypatch, bases, starts, passes=3)
    d = str(tmp_path / "passes")
    monkeypatch.setenv("SNAPGPU_BUILD_PASSES", "5")
    ix.save(d)
    monkeypatch.delenv("SNAPGPU_BUILD_PASSES")
    assert _table_headers(d) == _table_headers(d1)
    assert len(_table_headers(d)) == 256
    # the unmodified reference loads it, with the hits of the reference-built directory
    ridx, r0 = reflib.RefIndex(d), reflib.RefIndex(small_cfg.idx)
    seeds = _position_seeds(bases, 20)
    for i in range(0, len(seeds), 3):
        s = seeds[i].tobytes()
        a, w = ridx.lookup(s, 512), r0.lookup(s, 512)
        assert a[0] == w[0] and a[1] == w[1] and np.array_equal(a[2], w[2]) and np.array_equal(a[3], w[3]), i
    p = reflib.default_params(maxDist=14)
    for name in ("std150", "noisy150"):
        want, _ = reflib.RefSingleAligner(r0, p).align(small_cfg.reads[name])
        got, _ = reflib.RefSingleAligner(ridx, p).align(small_cfg.reads[name])
        assert differing(want, got) == [], name
    # and the library re-opens it to the same records
    back = engine.Index.open(d)
    _same_hits(ref_gidx, back, seeds)
    q = engine.default_params(maxDist=14)
    r1, _ = engine.SingleAligner(ref_gidx, q, 4096).align(small_cfg.reads["noisy150"])
    r2, _ = engine.SingleAligner(back, q, 4096).align(small_cfg.reads["noisy150"])
    assert differing(r1, r2) == []
    back.close()
    ix.close()
    one.close()


def test_save_seed16_single_table(engine, genomes, reflib, monkeypatch, tmp_path):
    """Seed length 16 has one table: forced passes cannot split it, and the save still writes it whole."""
    bases, starts = genomes["with_n"]
    ix = _build(engine, monkeypatch, bases, starts, seed_len=16, passes=4)
    d = str(tmp_path / "s16")
    monkeypatch.setenv("SNAPGPU_BUILD_PASSES", "4")
    ix.save(d)
    monkeypatch.delenv("SNAPGPU_BUILD_PASSES")
    h = _table_headers(d)
    assert len(h) == 1 and h[0][1] > 0
    snap = _build(engine, monkeypatch, bases, starts, seed_len=16, layout="snap")
    back = engine.Index.open(d)
    _same_hits(snap, back, _position_seeds(bases, 16))
    back.close()
    snap.close()
    ix.close()
