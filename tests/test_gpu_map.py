"""The GPU `map` stage against the reference binary: each case builds its graph with the reference's own `pregraph` and `contig`, runs
`map` twice on copies of that graph (the reference and the GPU CLI) and compares the files byte for byte and the stderr lines without
the time lines.  Needs oracle/_ref (the reference binaries built by oracle/Makefile)."""
import filecmp
import os
import re
import shutil
import subprocess

import pytest

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")]

GRAPH = ["contig", "ContigIndex", "preGraphBasic", "updated.edge", "Arc", "edge.gz", "preArc", "vertex", "kmerFreq", "markOnEdge", "path"]
MAP_OUT = ["readOnContig.gz", "readInGap.gz", "peGrads"]
FILL_OUT = ["shortreadInGap.gz", "PEreadOnContig.gz"]
_TIME = re.compile(r"^(Time spent|Overall time|\[pgb200\])")


def _stderr_lines(text):
    lines = text.splitlines()
    start = next(i for i, s in enumerate(lines) if s.startswith("****"))   # the reference's main() prints its version first
    return [s for s in lines[start:] if not _TIME.match(s)]


def _graph(d, cfg, K, flavour127=False):
    ref = util.REF127 if flavour127 else util.REF63
    g = os.path.join(d, "g")
    util.run([ref, "pregraph", "-s", cfg, "-K", str(K), "-p", "4", "-o", g, "-R"])
    util.run([ref, "contig", "-g", g, "-R"])
    return g


def _copy(g, name):
    out = os.path.join(os.path.dirname(g), name)
    for s in GRAPH:
        if os.path.exists(f"{g}.{s}"):
            shutil.copy(f"{g}.{s}", f"{out}.{s}")
    return out


def _map_both(g, cfg, args=(), flavour127=False, tag=""):
    ref_bin, gpu_bin = (util.REF127, api.BIN127) if flavour127 else (util.REF63, api.BIN63)
    ref, gpu = _copy(g, "ref" + tag), _copy(g, "gpu" + tag)
    e_ref = util.run([ref_bin, "map", "-s", cfg, "-g", ref, *args])
    e_gpu = util.run([gpu_bin, "map", "-s", cfg, "-g", gpu, *args])
    suffixes = MAP_OUT + (FILL_OUT if "-f" in args else [])
    bad = [s for s in suffixes if not filecmp.cmp(f"{ref}.{s}", f"{gpu}.{s}", shallow=False)]
    assert not bad, f"map outputs differ: {bad}"
    assert _stderr_lines(e_gpu.replace(gpu, ref)) == _stderr_lines(e_ref)
    return ref, gpu


def _with_max_rd_len(cfg, n, out):
    txt = re.sub(r"^max_rd_len=\d+", f"max_rd_len={n}", open(cfg).read(), flags=re.M)
    open(out, "w").write(txt)
    return out


def test_map_pe_fastq_k31(tmp_path):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 31)
    ref, gpu = _map_both(g, cfg, ["-p", "8"])
    # the scaffolder reads the map files: the same scaffolds from either
    util.run([util.REF63, "scaff", "-g", ref])
    util.run([util.REF63, "scaff", "-g", gpu])
    assert filecmp.cmp(f"{ref}.scafSeq", f"{gpu}.scafSeq", shallow=False)


@pytest.mark.parametrize("K", [31, 63])
def test_map_multilib(tmp_path, K):
    """asm_flags=2 library, skipped single-end files, rd_len_cutoff, reverse_seq, libraries sorted by avg_ins"""
    cfg = synth.scenario_multilib(str(tmp_path))
    g = _graph(str(tmp_path), cfg, K)
    _map_both(g, cfg, ["-p", "8"])


def test_map_threads_are_a_layout_parameter(tmp_path):
    """-p 1 and -p 8 give different reference .readInGap.gz files; the GPU matches each"""
    cfg = synth.scenario_multilib(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 31)
    for p in ("1", "8"):
        _map_both(g, cfg, ["-p", p], tag=p)


def test_map_multi_batch(tmp_path):
    """max_rd_len=30000 cuts the reads into batches of 3336; a library change falls inside a batch"""
    cfg = synth.scenario_multilib(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 31)
    big = _with_max_rd_len(cfg, 30000, os.path.join(str(tmp_path), "big.cfg"))
    _map_both(g, big, ["-p", "3"])


def test_map_small_k_and_fill(tmp_path):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 31)
    _map_both(g, cfg, ["-p", "8", "-k", "25"], tag="k")
    _map_both(g, cfg, ["-p", "8", "-f"], tag="f")


@pytest.mark.parametrize("K", [91, 127])
def test_map_127mer(tmp_path, K):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    g = _graph(str(tmp_path), cfg, K, flavour127=True)
    _map_both(g, cfg, ["-p", "8"], flavour127=True)


def test_map_adversarial(tmp_path):
    """N and '.' bases, lower case, reads shorter than K+1; mapped as pairs (p= and q1/q2) of an avg_ins=2000 library, which
    raises ALIGNLEN read by read"""
    d = str(tmp_path)
    cfg = synth.scenario_adversarial(d)
    g = _graph(d, cfg, 31)
    pcfg = os.path.join(d, "adv_pairs.cfg")
    shutil.copy(os.path.join(d, "adv.fq"), os.path.join(d, "adv2.fq"))   # the reference refuses q2 == q1
    with open(pcfg, "w") as f:
        f.write(f"max_rd_len=100\n[LIB]\navg_ins=2000\nreverse_seq=0\nasm_flags=3\nrank=2\npair_num_cutoff=3\n"
                f"p={d}/adv.fa\nq1={d}/adv.fq\nq2={d}/adv2.fq\n")
    _map_both(g, pcfg, ["-p", "8", "-f"])


def test_map_paired_asm2_reverse_map_len(tmp_path):
    """A paired asm_flags=2 library with reverse_seq=1 and map_len, a paired asm_flags=1 library that map must skip, and a library
    with map_len above the default: .peGrads shows which libraries contributed reads"""
    d = str(tmp_path)
    synth.scenario_multilib(d)
    g = _graph(d, os.path.join(d, "multi.cfg"), 31)
    cfg = os.path.join(d, "maplibs.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=150\n"
                f"[LIB]\navg_ins=500\nasm_flags=2\nreverse_seq=1\nmap_len=40\nrank=2\npair_num_cutoff=4\nf1={d}/m_a1.fa\nf2={d}/m_a2.fa\n"
                f"[LIB]\navg_ins=350\nasm_flags=1\nq1={d}/m_q1.fq\nq2={d}/m_q2.fq\n"
                f"[LIB]\navg_ins=200\nasm_flags=3\nrd_len_cutoff=140\nmap_len=60\nrank=1\nq1={d}/m_q1.fq\nq2={d}/m_q2.fq\n")
    ref, _ = _map_both(g, cfg, ["-p", "8", "-f"])
    grads = open(f"{ref}.peGrads").read().splitlines()
    assert grads[0].startswith("grads&num: 2\t7000\t")
    assert [int(x.split("\t")[0]) for x in grads[1:]] == [200, 500]


@pytest.mark.parametrize("case", ["fastq_no_plus", "fasta_two_line_sequence"])
def test_map_refuses_malformed_mate2(tmp_path, case):
    """A malformed record in the last chunk of the last file (here: the whole mate-2 file) is refused with the engine's message"""
    d = str(tmp_path)
    cfg = synth.scenario_pe_fastq(d)
    g = _graph(d, cfg, 31)
    if case == "fastq_no_plus":
        lines = open(f"{d}/pe_2.fq").read().splitlines(keepends=True)
        lines[4 * 100 + 2] = "x\n"
        open(f"{d}/bad_2.fq", "w").writelines(lines)
        body = f"q1={d}/pe_1.fq\nq2={d}/bad_2.fq\n"
    else:
        recs = open(f"{d}/pe_1.fq").read().splitlines()
        with open(f"{d}/ok_1.fa", "w") as f1, open(f"{d}/bad_2.fa", "w") as f2:
            for i in range(0, len(recs), 4):
                f1.write(f">{i}\n{recs[i + 1]}\n")
                f2.write(f">{i}\n{recs[i + 1][:70]}\n{recs[i + 1][70:]}\n" if i in (400, 800) else f">{i}\n{recs[i + 1]}\n")
        body = f"f1={d}/ok_1.fa\nf2={d}/bad_2.fa\n"
    bad_cfg = os.path.join(d, "bad.cfg")
    open(bad_cfg, "w").write(f"max_rd_len=150\n[LIB]\navg_ins=300\n{body}")
    gpu = _copy(g, "gpu")
    r = subprocess.run([api.BIN63, "map", "-s", bad_cfg, "-g", gpu], capture_output=True, text=True, timeout=300)
    assert r.returncode == 255
    assert "readseqInLib return error! please make sure input file is correct fastq/fasta file" in r.stderr
    assert "input is not single-line FASTA / 4-line FASTQ" in r.stderr


B63 = os.path.join(util.ROOT, "oracle", "_ref", "SOAPdenovo-63mer-b200")


@pytest.mark.skipif(not os.path.exists(B63), reason="drop-in binary not linked")
def test_dropin_map(tmp_path):
    """The reference's main() with the shim's call_align: `map` through the drop-in binary writes the reference's files"""
    cfg = synth.scenario_multilib(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 31)
    ref, gpu = _copy(g, "ref"), _copy(g, "dropin")
    e_ref = util.run([util.REF63, "map", "-s", cfg, "-g", ref, "-p", "8", "-f"])
    e_gpu = util.run([B63, "map", "-s", cfg, "-g", gpu, "-p", "8", "-f"])
    for s in MAP_OUT + FILL_OUT:
        assert filecmp.cmp(f"{ref}.{s}", f"{gpu}.{s}", shallow=False), s
    assert _stderr_lines(e_gpu.replace(gpu, ref)) == _stderr_lines(e_ref)
