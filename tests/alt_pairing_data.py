"""A GRCh38-style reference in miniature for ALT-aware pairing: two primary contigs and ALT contigs whose projection onto the
primary ones (the liftover SAM of `snap index -altLiftoverFile`, the format of bwa-kit's hs38DH.fa.alt) is known by construction.

- chr1_KI270762v1_alt: chr1[20000, 50000) with 0.5 % substitutions, a 4-base insertion and a 3-base deletion, then 600 bases of unrelated
  sequence: CIGAR 12000M4I9000M3D8997M600S.  Reads in the tail project into the soft clip (getProjLocation gives InvalidGenomeLocation).
- chr2_KI270763v1_alt: the reverse complement of chr2[60000, 80000) with 1 % substitutions, followed by 800 bases of unrelated sequence,
  flag 16: against chr2's forward strand it is 800S20000M, a leading soft clip.  Pairs in the unrelated tail lift over to a place they
  do not align to, so the liftover is undone.
- HLA-A*01:01:01:01: a 1 % copy of chr1[70000, 85000) without a liftover line.
- chrUn_KN707606v1_decoy_alt: unrelated sequence.

`build(dir, snap_aligner)` writes the FASTA and the liftover file and indexes the reference twice, with and without the liftover file."""
import os
import subprocess

import numpy as np

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
NAMES = [b"chr1", b"chr1_KI270762v1_alt", b"chr2", b"chr2_KI270763v1_alt", b"HLA-A*01:01:01:01", b"chrUn_KN707606v1_decoy_alt"]


def _mutate(rng, c, rate):
    c = c.copy()
    m = rng.random(c.size) < rate
    c[m] = ACGT[rng.integers(0, 4, int(m.sum()))]
    return c


def contigs():
    from snap_b200 import synth
    rng = np.random.default_rng(4242)
    chr1, chr2 = synth.make_contigs(2, 100_000, seed=4241, repeat_frac=0.1)
    a = _mutate(rng, chr1[20_000:50_000], 0.005)
    alt1 = np.concatenate([a[:12_000], ACGT[rng.integers(0, 4, 4)], a[12_000:21_000], a[21_003:], ACGT[rng.integers(0, 4, 600)]])
    alt2 = np.concatenate([synth.revcomp(_mutate(rng, chr2[60_000:80_000], 0.01)), ACGT[rng.integers(0, 4, 800)]])
    hla = _mutate(rng, chr1[70_000:85_000], 0.01)
    decoy = ACGT[rng.integers(0, 4, 12_000)]
    return [chr1, alt1, chr2, alt2, hla, decoy]


LIFTOVER = [
    (b"chr1_KI270762v1_alt", 0, b"chr1", 20_001, b"12000M4I9000M3D8997M600S"),
    (b"chr2_KI270763v1_alt", 16, b"chr2", 60_001, b"800S20000M"),
]


def build(d, snap_aligner):
    """-> (index with liftover, index without, contigs)"""
    cs = contigs()
    fa = os.path.join(d, "ref.fa")
    with open(fa, "wb") as f:
        for n, c in zip(NAMES, cs):
            f.write(b">" + n + b"\n")
            for i in range(0, c.size, 100):
                f.write(c[i:i + 100].tobytes() + b"\n")
    alt_sam = os.path.join(d, "alt.sam")
    with open(alt_sam, "wb") as f:
        f.write(b"@SQ\tSN:chr1\tLN:100000\n@SQ\tSN:chr2\tLN:100000\n")
        for name, flag, ref, pos, cigar in LIFTOVER:
            f.write(b"\t".join([name, b"%d" % flag, ref, b"%d" % pos, b"60", cigar, b"*", b"0", b"0", b"*", b"*"]) + b"\n")
    out = []
    for sub, extra in (("idx_lift", ["-altLiftoverFile", alt_sam]), ("idx_nolift", [])):
        idx = os.path.join(d, sub)
        os.makedirs(idx, exist_ok=True)
        res = subprocess.run([snap_aligner, "index", fa, idx, "-s", "20", "-t8"] + extra, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if res.returncode != 0 or not os.path.exists(os.path.join(idx, "GenomeIndexHash")):
            raise RuntimeError("snap-aligner index failed:\n" + res.stdout)
        out.append(idx)
    return out[0], out[1], cs


def pairs(cs, n, seed):
    """Pairs from every contig in proportion to its length (so from the ALT stretches and their primary twins), with noise, chimeric
    pairs, N runs and short ends."""
    from snap_b200 import synth
    return synth.make_pairs(cs, n, 150, seed=seed, sub_rate=0.01, ins_rate=0.002, del_rate=0.002, chimeric_frac=0.03, n_run_frac=0.03, short_frac=0.03)
