"""ALT-aware `snap paired` (the default; -A- turns it off) on an index with ALT contigs and a liftover file, host build of the engine's
headers against the compiled reference: every PairedAlignmentResult field, one-launch and staged forms (with the same LV / affine-gap call
counts), with the reference's pool sizes and with tiny ones (pairs that outgrow them are redone by a full-size aligner, as on the GPU)."""
import os

import pytest

import alt_pairing_data as AD
import hostsim_lib as hs
from conftest import differing_pairs

_HC = dict(fivePrimeEndBonus=5, threePrimeEndBonus=5)
_HCP = dict(useSoftClipping=0, minAGScoreImprovement=15)
ALT_PAIRED_SETS = {
    "stock": (dict(maxDist=27), dict()),
    "d14": (dict(maxDist=14), dict()),
    "gap2": (dict(maxDist=27, maxScoreGapToPreferNonAltAlignment=2), dict()),
    "hc": (dict(maxDist=27, **_HC), dict(**_HCP)),
    "noag_hc": (dict(maxDist=27, useAffineGap=0, **_HC), dict(**_HCP)),
    "esd3": (dict(maxDist=27, extraSearchDepth=3), dict()),
    "msgra0": (dict(maxDist=27), dict(minScoreGapRealignmentALT=0)),
    "msgra10": (dict(maxDist=27), dict(minScoreGapRealignmentALT=10)),
}


@pytest.fixture(scope="module")
def alt_pairs(tmp_path_factory, reflib):
    lift, nolift, cs = AD.build(str(tmp_path_factory.mktemp("altpair")), reflib.SNAP_ALIGNER)
    return lift, nolift, AD.pairs(cs, 2000, seed=4243)


def contig_starts(idx):
    lines = open(os.path.join(idx, "Genome"), "rb").read(4000).split(b"\n")
    n = int(lines[0].split()[1])
    return {l.split()[7]: int(l.split()[0]) for l in lines[1:n + 1]}


def test_index_keeps_the_projection(alt_pairs):
    """What `snap index -altLiftoverFile` writes per contig line: the projection start, the RC flag and the CIGAR."""
    lift, nolift, _ = alt_pairs
    lines = {l.split()[7]: l.split() for l in open(os.path.join(lift, "Genome"), "rb").read(4000).split(b"\n")[1:7]}
    starts = contig_starts(lift)
    assert int(lines[b"chr1_KI270762v1_alt"][3]) == starts[b"chr1"] + 20_000 and lines[b"chr1_KI270762v1_alt"][8] == b"12000M4I9000M3D8997M600S"
    assert int(lines[b"chr2_KI270763v1_alt"][4], 16) == 1 and lines[b"chr2_KI270763v1_alt"][8] == b"800S20000M"
    assert lines[b"HLA-A*01:01:01:01"][8] == b"*"
    assert all(l.split()[8] == b"*" for l in open(os.path.join(nolift, "Genome"), "rb").read(4000).split(b"\n")[1:7])


@pytest.mark.parametrize("opt", list(ALT_PAIRED_SETS))
def test_alt_aware_pairs_match_reference(reflib, alt_pairs, opt):
    lift, nolift, pairs = alt_pairs
    kw, pkw = ALT_PAIRED_SETS[opt]
    rp, pp = reflib.default_params_paired(**kw), reflib.default_paired_params(**pkw)
    for idx in (lift, nolift):
        want, _ = reflib.RefPairedAligner(reflib.RefIndex(idx), rp, pp).align(pairs)
        hidx = hs.HsIndex(idx)
        work = {}
        for staged in (False, True):
            for caps in ((0, 0), (16, 4)):
                al = hs.HsPairedAligner(hidx, rp, pp, pool_cap=caps[0], cand_cap=caps[1])
                al.set_staged(staged)
                got, nlv, nag = al.align(pairs, reflib.PAIRED_RESULT_DTYPE)
                bad = differing_pairs(want, got)
                assert bad == [], (opt, idx, staged, caps, bad[:5])
                work[(staged, caps)] = (nlv, nag)
                if caps[0]:
                    assert al.retried() > 0
        # the LV / affine-gap call counts do not depend on the launch form (with small pools the redone pairs count in the second aligner)
        assert work[(False, (0, 0))] == work[(True, (0, 0))] and work[(False, (16, 4))] == work[(True, (16, 4))], (opt, idx, work)


def test_alt_awareness_is_live_on_this_data(reflib, alt_pairs):
    """The checks above are not vacuous: on this data the reference lifts pairs over, undoes a liftover, lets an ALT pair keep the single-end
    aligner away (agForcedSingleAlignerCall differs from an -A- run) and returns other pairs than with ALT awareness off."""
    lift, _, pairs = alt_pairs
    ridx = reflib.RefIndex(lift)
    pp = reflib.default_paired_params()
    on, _ = reflib.RefPairedAligner(ridx, reflib.default_params_paired(maxDist=27), pp).align(pairs)
    off, _ = reflib.RefPairedAligner(ridx, reflib.default_params_paired(maxDist=27, altAwareness=0), pp).align(pairs)
    assert int((on["liftover"] == 1).all(axis=1).sum()) > 0
    # both ends on the reverse-complemented ALT contig and still there: its projection is valid everywhere, so the liftover was undone
    starts = contig_starts(lift)
    lo, hi = starts[b"chr2_KI270763v1_alt"], starts[b"HLA-A*01:01:01:01"]
    on_rc_alt = ((on["location"] >= lo) & (on["location"] < hi) & (on["status"] != 0)).all(axis=1)
    assert int((on_rc_alt & (on["liftover"] == 0).all(axis=1)).sum()) > 0
    assert (on["agForcedSingleAlignerCall"] != off["agForcedSingleAlignerCall"]).any()
    assert len(differing_pairs(on, off)) > 20
