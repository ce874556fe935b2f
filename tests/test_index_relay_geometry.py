"""Host-build checks of saving a bucket index in any of the reference's table geometries (snap_b200/csrc/sg_bucket.h, sg_host.h: the
same mapping, staging form, probe sequence and packing snapgpu_index_save_ex runs on the device), and of the Genome file writer.

The buckets come from the reference's `snap-aligner index -keysize 4` directory for each seed length; each is written in a target
geometry and compared with the reference's own directory built in that geometry."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import alt_pairing_data as AD
import buildsim_lib as hs
import relaysim_lib as rs

# (seed length, the target's `snap-aligner index` options, key bytes, -large)
TARGETS = [
    (16, ["-locationSize", "4", "-keysize", "2"], 2, False),
    (16, ["-locationSize", "4", "-keysize", "3"], 3, False),
    (16, ["-locationSize", "4", "-keysize", "4"], 4, False),
    (20, [], 4, False),
    (20, ["-large"], 4, True),
    (22, ["-keysize", "4"], 4, False),
    (22, [], 5, False),
    (24, [], 5, False),
    (24, ["-keysize", "6"], 6, False),
    (24, ["-large"], 5, True),
]


def _ref_index(snap_aligner, fasta, out, opts):
    os.makedirs(out, exist_ok=True)
    res = subprocess.run([snap_aligner, "index", fasta, out, "-t8"] + opts, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0 or not os.path.exists(os.path.join(out, "GenomeIndexHash")):
        raise RuntimeError("snap-aligner index failed:\n" + res.stdout)
    return out


def table_used(directory):
    """Per-table used counts from a GenomeIndexHash file's table headers."""
    fields = open(os.path.join(directory, "GenomeIndex")).read().split()
    n_tables, key_bytes, small = int(fields[2]), int(fields[6]), int(fields[8])
    entry = (4 if small else 8) + key_bytes
    used = []
    with open(os.path.join(directory, "GenomeIndexHash"), "rb") as f:
        for _ in range(n_tables):
            magic, size, u, ks, vs, vc, _inv = struct.unpack("<IQQIIII", f.read(36))
            assert magic == 0xb111b010 and ks == key_bytes and vs == 4 and vc == (1 if small else 2)
            used.append(u)
            f.seek(size * entry, 1)
        assert f.read(1) == b""
    return np.array(used, dtype=np.uint64)


@pytest.fixture(scope="module")
def geometry_data(small_cfg, reflib, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("relaygeom"))
    src = {}
    for s in sorted({t[0] for t in TARGETS}):
        src[s] = _ref_index(reflib.SNAP_ALIGNER, small_cfg.fasta, os.path.join(d, "src%d" % s), ["-s", str(s), "-keysize", "4", "-locationSize", "4"])
    return d, src


def _seeds(contigs, seed_len):
    return np.ascontiguousarray(np.concatenate([np.lib.stride_tricks.sliding_window_view(c, seed_len) for c in contigs]))


@pytest.mark.parametrize("seed_len,opts,key_bytes,large", TARGETS, ids=["s%d_k%d%s" % (t[0], t[2], "_large" if t[3] else "") for t in TARGETS])
def test_buckets_saved_in_every_geometry_match_the_reference(small_cfg, reflib, geometry_data, seed_len, opts, key_bytes, large):
    d, src = geometry_data
    tag = "s%d_k%d%s" % (seed_len, key_bytes, "L" if large else "")
    want_dir = _ref_index(reflib.SNAP_ALIGNER, small_cfg.fasta, os.path.join(d, "ref_" + tag), ["-s", str(seed_len)] + opts)
    got_dir = os.path.join(d, "got_" + tag)
    rs.HostIndex(src[seed_len], relayout=True).relay_save(got_dir, key_bytes, large)
    # the header: geometry as the reference writes it (the hash file's size differs: the tables are sized from exact counts)
    want_hdr, got_hdr = open(os.path.join(want_dir, "GenomeIndex")).read().split(), open(os.path.join(got_dir, "GenomeIndex")).read().split()
    for i in (0, 1, 2, 4, 5, 6, 8, 9):
        assert want_hdr[i] == got_hdr[i], (i, want_hdr, got_hdr)
    assert int(got_hdr[6]) == key_bytes and got_hdr[8] == ("0" if large else "1")
    assert np.array_equal(table_used(want_dir), table_used(got_dir))
    assert open(os.path.join(want_dir, "Genome"), "rb").read() == open(os.path.join(got_dir, "Genome"), "rb").read()
    # every genome position's hits, through the host loader over all positions ...
    want, got = hs.BsIndex(want_dir), hs.BsIndex(got_dir)
    seeds = _seeds(small_cfg.contigs, seed_len)
    n_hits = 0
    for a in range(0, len(seeds), 20000):
        chunk = np.ascontiguousarray(seeds[a:a + 20000])
        n1, h1 = want.lookup(chunk, len(chunk))
        n2, h2 = got.lookup(chunk, len(chunk))
        assert np.array_equal(n1, n2), a
        k = np.minimum(n1, 512)
        mask = np.arange(512)[None, None, :] < k[:, :, None]
        assert np.array_equal(np.where(mask, h1, 0), np.where(mask, h2, 0)), a
        n_hits += int(n1.sum())
    assert n_hits >= len(seeds)
    # ... and through the unmodified reference's loader and lookupSeed32 on a sample of them
    rw, rg = reflib.RefIndex(want_dir), reflib.RefIndex(got_dir)
    for i in range(0, len(seeds), 97):
        s = seeds[i].tobytes()
        a, b = rw.lookup(s), rg.lookup(s)
        assert a[:2] == b[:2] and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), i


@pytest.fixture(scope="module")
def alt_dirs(reflib, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("relayalt"))
    lift, nolift, _ = AD.build(d, reflib.SNAP_ALIGNER)
    return lift, nolift


@pytest.mark.parametrize("which", ["small_cfg", "alt_lift", "alt_nolift"])
def test_genome_writer_reproduces_stock_genome_files(small_cfg, alt_dirs, tmp_path, which):
    """Contig lines parsed from a stock Genome file (names, ALT flags, original numbers, liftover fields) written back by
    sg_genome_file_header with the bases: byte for byte the file `snap-aligner index` wrote."""
    src = {"small_cfg": small_cfg.idx, "alt_lift": alt_dirs[0], "alt_nolift": alt_dirs[1]}[which]
    out = str(tmp_path / "Genome")
    rs.HostIndex(src).write_genome(out)
    want = open(os.path.join(src, "Genome"), "rb").read()
    assert open(out, "rb").read() == want
    if which == "alt_lift":
        assert b"12000M4I9000M3D8997M600S" in want[:4096]


def test_loader_refuses_a_malformed_liftover_cigar_and_alt_contigs_out_of_order(alt_dirs, tmp_path):
    src = alt_dirs[0]
    for name, edit in (("cigar", lambda t: t.replace(b"12000M4I9000M3D8997M600S", b"12000M4I9000M3D8997M60?S")),
                       ("order", None)):
        d = tmp_path / name
        shutil.copytree(src, d)
        g = open(d / "Genome", "rb").read()
        head_end = 0
        lines = g.split(b"\n")
        n_contigs = int(lines[0].split()[1])
        head_end = sum(len(x) + 1 for x in lines[:1 + n_contigs])
        head, bases = g[:head_end], g[head_end:]
        if edit:
            head = edit(head)
        else:                      # mark the first (primary) contig ALT: ALT contigs no longer form the tail
            hl = head.split(b"\n")
            f = hl[1].split(b" ")
            f[1] = b"1"
            hl[1] = b" ".join(f)
            head = b"\n".join(hl)
        open(d / "Genome", "wb").write(head + bases)
        with pytest.raises(RuntimeError) as e:
            rs.HostIndex(str(d))
        assert ("malformed projection CIGAR" if name == "cigar" else "ALT contigs must come last") in str(e.value)
