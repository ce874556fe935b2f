"""SNAPGPU_SINGLE_AG_NARROW: the second pass of the two-pass single-end launch rescores bands of up to 32 columns with the two-unit
form (`duo`, sg_warp_ag_duo.cuh) or the one-unit form (`rows`, sg_warp_ag_rows_banded4).  Both settings must give the same records,
field for field, and the same counters, on `-d 14` reads and on a `-d 20 -G` set."""
import numpy as np
import pytest

from conftest import differing

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    from snap_b200 import engine as e
    assert e.lib().snapgpu_device_count() >= 1, "no CUDA device: the CUDA path has no fallback"
    return e


@pytest.fixture(scope="module")
def gidx(engine, small_cfg):
    ix = engine.Index.open(small_cfg.idx)
    yield ix
    ix.close()


def _run(engine, gidx, kw, rb, setting, monkeypatch):
    monkeypatch.setenv("SNAPGPU_SINGLE_AG_NARROW", setting)
    al = engine.SingleAligner(gidx, engine.default_params(**kw), 4096)
    try:
        got, ctr = al.align(rb)
        deferred = al.deferred_count()
    finally:
        al.close()
    return got, ctr, deferred


@pytest.mark.parametrize("kw", [dict(maxDist=14), dict(maxDist=20, useAffineGap=1)], ids=["d14", "d20_G"])
@pytest.mark.parametrize("reads", ["std150", "noisy150"])
def test_narrow_band_forms_give_the_same_records_and_counters(engine, gidx, small_cfg, reflib, monkeypatch, kw, reads):
    rb = small_cfg.reads[reads]
    rows, crows, drows = _run(engine, gidx, kw, rb, "rows", monkeypatch)
    duo, cduo, dduo = _run(engine, gidx, kw, rb, "duo", monkeypatch)
    assert drows == dduo and dduo > 0                       # reads did go through the second pass
    assert crows["affineGapCalls"] > 0
    assert differing(rows, duo) == []
    assert rows.tobytes() == duo.tobytes()
    for k in crows:
        assert np.array_equal(np.asarray(crows[k]), np.asarray(cduo[k])), k
    # and both are the reference's answer
    ridx = reflib.RefIndex(small_cfg.idx)
    want, wctr = reflib.RefSingleAligner(ridx, reflib.default_params(**kw)).align(rb)
    assert differing(want, duo) == []
    assert wctr["affineGapCalls"] == cduo["affineGapCalls"]


def test_narrow_band_switch_refuses_other_values(engine, gidx, monkeypatch):
    monkeypatch.setenv("SNAPGPU_SINGLE_AG_NARROW", "fast")
    with pytest.raises(Exception, match="SNAPGPU_SINGLE_AG_NARROW"):
        engine.SingleAligner(gidx, engine.default_params(maxDist=14), 4096)
