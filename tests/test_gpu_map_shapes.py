"""Shapes of the map stage that the other map tests never reach, against the reference binary:

* long reads past one thread slice of k_map_long: each of its 128 threads rolls max(64, ceil(nk / 128)) k-mers, so reads of more than
  8192 k-mers give slices longer than 64.  Reads sit on and around the slice boundaries (nk = 8191 ... 24577) and at 30-40 kbp.
* a contig past 2^24 bases: the contig table keeps a k-mer's position in 24 bits, as the reference's r_links bit-field does
  (newhash.h), so positions past 2^24 wrap and parse1read's read positions come out 2^24 short.  One random 17.5 Mbp genome, tiled
  with error-free pairs, makes a single unipath: the GPU pregraph walks it on one thread, then `map` runs on the reference's contig.

The contig case takes a few minutes of reference CPU time; set PGB200_SKIP_CONFIG_TESTS=1 to skip it."""
import filecmp
import gzip
import os
import subprocess
import time

import numpy as np
import pytest

from soapdenovo2_b200 import api, synth
from tests import util
from tests.test_gpu_map import MAP_OUT, _copy, _graph, _stderr_lines
from tests.test_gpu_map_long import _map_both

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")]

SLICE_NK = [8191, 8192, 8193, 8255, 8256, 8257, 16385, 24577]   # 128 x 64, 127 x 65, 128 x 65 - 63, 128 x 128 + 1, 128 x 192 + 1


def _long_cfg(d, K):
    g = synth.genome(150_000, 41, repeat=(500, 3))
    r1, r2 = synth.pe_reads(g, 15000, 150, 300, 0.002, 42)
    synth.write_fastq(os.path.join(d, "pe_1.fq"), r1, "p")
    synth.write_fastq(os.path.join(d, "pe_2.fq"), r2, "p")
    lengths = [nk + K - 1 for nk in SLICE_NK] + [30_000, 33_333, 36_001, 40_000]
    reads = synth.long_reads_of_lengths(g, lengths, seed=43) + synth.long_reads(g, 40, 200, 3000, seed=44)
    synth.write_long(os.path.join(d, "long.fa"), reads, fastq=False)
    cfg = os.path.join(d, "long.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=150\n[LIB]\navg_ins=300\nreverse_seq=0\nasm_flags=3\nrank=1\nq1={d}/pe_1.fq\nq2={d}/pe_2.fq\n"
                f"[LIB]\nasm_flags=4\nrd_len_cutoff=50000\nf={d}/long.fa\n")
    return cfg


@pytest.mark.parametrize("K", [31, 63, 91])
def test_long_reads_past_one_slice(tmp_path, monkeypatch, K):
    d = str(tmp_path)
    cfg = _long_cfg(d, K)
    f127 = K > 63
    g = _graph(d, cfg, K, flavour127=f127)
    _, _, err = _map_both(g, cfg, ["-p", "8"], flavour127=f127)
    assert "long read len 50000" in err   # the library's rd_len_cutoff
    _map_both(g, cfg, ["-p", "8", "-f"], flavour127=f127, tag="f")
    if K == 31:
        monkeypatch.setenv("PGB200_MAP_GROUPS", "1")
        _map_both(g, cfg, ["-p", "8"], tag="g1")


def _slice_end_reads(contigs, K, rng, with_b=True):
    """Long reads whose .longReadInGap record hangs on the k-mer at the end of one k_map_long slice.  Each read is junk (absent from
    the genome) with 1500 bases of contig A, placing it, and a short piece of contig B whose first k-mer is the last one of slice s.
    A read is written only when it hits two contig groups (parse1read's footprint: counter2 > 1, where below K = 32 a group needs two
    hits), so B is one k-mer (K > 32) or two (K < 32) and nothing else; without its slice-end k-mer no read is written."""
    ids = sorted(contigs, key=lambda c: -len(contigs[c]))
    a, b = contigs[ids[0]], contigs[ids[1]]
    m = K + 1 if K < 32 else K
    assert len(a) >= 1700 and len(b) >= m + 100
    out = []
    for nk in (8192, 8193, 8257, 16385, 24577):
        per = max(64, -(-nk // 128))
        L = nk + K - 1
        for s in (0, 1, 60):
            j = (s + 1) * per - 1
            r = bytearray(synth._ACGT[rng.integers(0, 4, size=L)].tobytes())
            if with_b:
                r[j:j + m] = b[100:100 + m].encode()
            at = 200 if j > L // 2 else L - 1700
            r[at:at + 1500] = a[100:1600].encode()
            out.append(bytes(r))
    return out


@pytest.mark.parametrize("K", [31, 63, 91])
def test_slice_end_kmer_decides_the_footprint(tmp_path, K):
    d = str(tmp_path)
    cfg = _long_cfg(d, K)
    f127 = K > 63
    g = _graph(d, cfg, K, flavour127=f127)
    contigs = _contigs(f"{g}.contig")
    synth.write_long(os.path.join(d, "long.fa"), _slice_end_reads(contigs, K, np.random.default_rng(45)), fastq=False)
    ref, _, _ = _map_both(g, cfg, ["-p", "8"], flavour127=f127)
    _map_both(g, cfg, ["-p", "8", "-f"], flavour127=f127, tag="f")
    # the same reads without contig B's piece: the reference writes none of them
    synth.write_long(os.path.join(d, "nob.fa"), _slice_end_reads(contigs, K, np.random.default_rng(45), with_b=False), fastq=False)
    nob_cfg = os.path.join(d, "nob.cfg")
    open(nob_cfg, "w").write(open(cfg).read().replace(f"{d}/long.fa", f"{d}/nob.fa"))
    nob = _copy(g, "nob")
    util.run([util.REF127 if f127 else util.REF63, "map", "-s", nob_cfg, "-g", nob, "-p", "8"])
    assert os.path.getsize(f"{ref}.longReadInGap") > 0 and os.path.getsize(f"{nob}.longReadInGap") == 0


# ---------------------------------------------------------------- a contig past 2^24
BIG = 17_500_000
WRAP = 1 << 24
STEP, RD, INS = 10, 150, 300


def _contigs(path):
    out, cid, seq = {}, None, []
    for line in open(path):
        if line.startswith(">"):
            if cid is not None:
                out[cid] = "".join(seq)
            cid, seq = int(line[1:].split()[0]), []
        else:
            seq.append(line.strip())
    if cid is not None:
        out[cid] = "".join(seq)
    return out


def wrapped_positions(genome, contig_path, roc_path, K):
    """Read positions in .readOnContig.gz on the long contig's own strand, against the truth from the tiling.  Returns
    (reads checked before 2^24, reads checked past 2^24, list of mismatches)."""
    ctgs = _contigs(contig_path)
    cid, seq = max(ctgs.items(), key=lambda kv: len(kv[1]))
    L = len(seq)
    gb = genome.tobytes()
    s_arr = np.frombuffer(seq.encode(), dtype=np.uint8)
    o = gb.find(s_arr[:200].tobytes())
    forward = o >= 0
    if not forward:
        o = gb.find(synth._COMP[s_arr[-200:][::-1]].tobytes())
    assert o >= 0
    seg = genome[o:o + L]
    assert np.array_equal(seg if forward else synth._COMP[seg[::-1]], s_arr), "the long contig is not a piece of the genome"
    before = past = 0
    bad = []
    with gzip.open(roc_path, "rt") as f:
        next(f)
        for line in f:
            rn, c, pos, orien = line.split()
            if int(c) != cid or orien != "+":
                continue
            p, mate = divmod(int(rn) - 1, 2)
            s = p * STEP
            # on the contig's own strand: mate 1 if the contig is the genome's forward strand, mate 2 if it is the reverse
            if forward != (mate == 0):
                bad.append((rn, c, pos, orien, "strand"))
                continue
            t = s - o if forward else (o + L) - (s + INS)
            if t + RD + K <= WRAP:
                before += 1
                want = t
            elif t >= WRAP:
                past += 1
                want = t - WRAP
            else:
                continue
            if int(pos) != want:
                bad.append((rn, c, pos, orien, want))
    return before, past, bad


def big_inputs(d):
    g = synth.genome(BIG, 17)
    r1, r2 = synth.tiled_pairs(g, STEP, RD, INS)
    synth.write_fasta_fast(os.path.join(d, "t_1.fa"), r1, "t")
    synth.write_fasta_fast(os.path.join(d, "t_2.fa"), r2, "t")
    cfg = os.path.join(d, "t.cfg")
    synth.write_config(cfg, RD, [{"avg_ins": INS, "files": [("f1", os.path.join(d, "t_1.fa")), ("f2", os.path.join(d, "t_2.fa"))]}])
    return g, cfg


def test_contig_past_2_24(tmp_path):
    if os.environ.get("PGB200_SKIP_CONFIG_TESTS"):
        pytest.skip("PGB200_SKIP_CONFIG_TESTS set")
    d = str(tmp_path)
    K = 63
    genome, cfg = big_inputs(d)
    ref, gpu = os.path.join(d, "ref"), os.path.join(d, "gpu")
    t0 = time.time()
    util.run([util.REF63, "pregraph", "-s", cfg, "-K", str(K), "-p", "8", "-R", "-o", ref], timeout=3000)
    t_ref = time.time() - t0
    t0 = time.time()
    r = subprocess.run([api.BIN63, "pregraph", "-s", cfg, "-K", str(K), "-p", "8", "-R", "-o", gpu], capture_output=True, text=True,
                       timeout=3000, env=dict(os.environ, PGB200_VERBOSE="1"))
    t_gpu = time.time() - t0
    assert r.returncode == 0, r.stderr[-4000:]
    print(f"\nreference pregraph {t_ref:.1f} s, GPU pregraph {t_gpu:.1f} s wall; GPU stage lines:")
    print("\n".join(l for l in r.stderr.splitlines() if l.startswith("[pgb200]")))
    util.compare(ref, gpu, util.SUFFIXES_R)

    util.run([util.REF63, "contig", "-g", ref, "-R"], timeout=3000)
    lens = sorted(len(s) for s in _contigs(f"{ref}.contig").values())
    print(f"contigs: {len(lens)}, longest {lens[-1]}")
    assert lens[-1] > WRAP + 1000
    rm, gm = _copy(ref, "mref"), _copy(ref, "mgpu")
    e_ref = util.run([util.REF63, "map", "-s", cfg, "-g", rm, "-p", "8"], timeout=3000)
    e_gpu = util.run([api.BIN63, "map", "-s", cfg, "-g", gm, "-p", "8"], timeout=3000)
    bad = [s for s in MAP_OUT if not filecmp.cmp(f"{rm}.{s}", f"{gm}.{s}", shallow=False)]
    assert not bad, f"map outputs differ: {bad}"
    assert _stderr_lines(e_gpu.replace(gm, rm)) == _stderr_lines(e_ref)
    before, past, wrong = wrapped_positions(genome, f"{ref}.contig", f"{gm}.readOnContig.gz", K)
    print(f"reads on the long contig's strand: {before} before 2^24, {past} past it (reported 2^24 short)")
    assert not wrong, wrong[:10]
    assert before > 1000 and past > 1000
