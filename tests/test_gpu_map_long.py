"""The GPU `map` stage with long-read libraries (asm_flags=4) against the reference binary, as in test_gpu_map.py: each case builds its
graph with the reference's `pregraph` and `contig`, runs `map` with both binaries on copies of it and compares every output byte for
byte -- .longReadInGap (and .RlongReadInGap with -f) besides the short pass's files -- and the stderr lines without the time lines.
Also: the short-read scenarios with PGB200_MAP_LONG=all (the short pass through k_map_long as well), the overflow rounds of the
kernel's group table forced with PGB200_MAP_GROUPS, and the refusals of reads that would overflow the reference's buffers."""
import filecmp
import os
import subprocess

import pytest

from soapdenovo2_b200 import api, synth
from tests import util
from tests.test_gpu_map import GRAPH, MAP_OUT, FILL_OUT, _copy, _graph, _stderr_lines, _with_max_rd_len

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")]

LONG_OUT = ["longReadInGap"]
LONG_FILL = ["RlongReadInGap"]
B63 = os.path.join(util.ROOT, "oracle", "_ref", "SOAPdenovo-63mer-b200")


def _map_both(g, cfg, args=(), flavour127=False, tag="", gpu_bin=None, long=True):
    ref_bin = util.REF127 if flavour127 else util.REF63
    gpu_bin = gpu_bin or (api.BIN127 if flavour127 else api.BIN63)
    ref, gpu = _copy(g, "ref" + tag), _copy(g, "gpu" + tag)
    e_ref = util.run([ref_bin, "map", "-s", cfg, "-g", ref, *args])
    e_gpu = util.run([gpu_bin, "map", "-s", cfg, "-g", gpu, *args])
    fill = "-f" in args
    suffixes = MAP_OUT + (FILL_OUT if fill else []) + ((LONG_OUT + (LONG_FILL if fill else [])) if long else [])
    bad = [s for s in suffixes if not filecmp.cmp(f"{ref}.{s}", f"{gpu}.{s}", shallow=False)]
    assert not bad, f"map outputs differ: {bad}"
    assert _stderr_lines(e_gpu.replace(gpu, ref)) == _stderr_lines(e_ref)
    return ref, gpu, e_ref


@pytest.mark.parametrize("K", [31, 63])
def test_long_map(tmp_path, K):
    d = str(tmp_path)
    cfg = synth.scenario_long(d)
    g = _graph(d, cfg, K)
    ref, _, err = _map_both(g, cfg, ["-p", "8"])
    assert "long read len 5000" in err and "Map_len 40." in err and "reads in gaps." in err
    assert os.path.getsize(f"{ref}.longReadInGap") > 0
    assert open(f"{ref}.peGrads").readline().split("\t")[2].strip() == "5000"


def test_long_map_threads_fill_small_k(tmp_path):
    """-p 1 and -p 8 give different .longReadInGap files (the rcSeq[1] bytes); -f adds .RlongReadInGap; -k 25 maps with K < 32"""
    d = str(tmp_path)
    cfg = synth.scenario_long(d, fastq=True)
    g = _graph(d, cfg, 31)
    a, _, _ = _map_both(g, cfg, ["-p", "1"], tag="1")
    b, _, _ = _map_both(g, cfg, ["-p", "8"], tag="8")
    assert not filecmp.cmp(f"{a}.longReadInGap", f"{b}.longReadInGap", shallow=False)
    _map_both(g, cfg, ["-p", "8", "-f"], tag="f")
    _map_both(g, cfg, ["-p", "8", "-k", "25"], tag="k")


def test_long_map_127mer(tmp_path):
    d = str(tmp_path)
    cfg = synth.scenario_long(d)
    g = _graph(d, cfg, 91, flavour127=True)
    _map_both(g, cfg, ["-p", "8", "-f"], flavour127=True)


def test_long_map_two_libraries(tmp_path):
    """two long libraries with their own map_len and rd_len_cutoff (reads cut at 1500 in one), FASTA and FASTQ, beside the paired one"""
    d = str(tmp_path)
    synth.scenario_long(d)
    g0 = synth.genome(60000, 3, repeat=(400, 3))
    synth.write_long(os.path.join(d, "l2.fq"), synth.long_reads(g0, 200, 100, 2500, seed=33), fastq=True)
    cfg = os.path.join(d, "two.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=150\n[LIB]\navg_ins=300\nasm_flags=3\nrank=1\nq1={d}/pe_1.fq\nq2={d}/pe_2.fq\n"
                f"[LIB]\navg_ins=10\nasm_flags=4\nrd_len_cutoff=1500\nmap_len=60\nq={d}/l2.fq\n"
                f"[LIB]\navg_ins=20\nasm_flags=4\nrd_len_cutoff=4000\nmap_len=30\nf={d}/long.fa\n")
    g = _graph(d, cfg, 31)
    _map_both(g, cfg, ["-p", "8", "-f"])


@pytest.mark.parametrize("n_long", [250, 200])
def test_long_map_batches(tmp_path, n_long):
    """rd_len_cutoff 1000030 at K = 31 makes batches of 100 long reads: 250 reads end in a partial batch, 200 fill the last one
    exactly (no `Output ... reads in gaps.` line)"""
    d = str(tmp_path)
    cfg = synth.scenario_long(d, n_long=n_long, rd_len_cutoff=1000030)
    g = _graph(d, cfg, 31)
    _, _, err = _map_both(g, cfg, ["-p", "3"])
    assert ("reads in gaps." in err) == (n_long == 250)


def test_long_map_group_overflow(tmp_path, monkeypatch):
    """two group slots per CTA: every read that hits three or more contigs goes through the overflow rounds"""
    d = str(tmp_path)
    cfg = synth.scenario_long(d, min_len=1500, max_len=6000, rd_len_cutoff=8000)
    g = _graph(d, cfg, 31)
    monkeypatch.setenv("PGB200_MAP_GROUPS", "2")
    _map_both(g, cfg, ["-p", "8", "-f"])
    monkeypatch.setenv("PGB200_MAP_GROUPS", "1")
    _map_both(g, cfg, ["-p", "8"], tag="1")


@pytest.mark.parametrize("case", ["pe_fastq", "multilib63", "multi_batch", "adversarial", "k91"])
def test_short_scenarios_through_long_kernel(tmp_path, monkeypatch, case):
    d = str(tmp_path)
    K, fl127, args = 31, False, ["-p", "8"]
    if case == "pe_fastq":
        cfg = synth.scenario_pe_fastq(d)
        args = ["-p", "8", "-f"]
    elif case == "multilib63":
        cfg, K = synth.scenario_multilib(d), 63
    elif case == "multi_batch":
        cfg = synth.scenario_multilib(d)
    elif case == "adversarial":
        cfg = synth.scenario_adversarial(d)
    else:
        cfg, K, fl127 = synth.scenario_pe_fastq(d), 91, True
    g = _graph(d, cfg, K, flavour127=fl127)
    if case == "multi_batch":
        cfg = _with_max_rd_len(cfg, 30000, os.path.join(d, "big.cfg"))
        args = ["-p", "3"]
    monkeypatch.setenv("PGB200_MAP_LONG", "all")
    monkeypatch.setenv("PGB200_MAP_GROUPS", "2")
    _map_both(g, cfg, args, flavour127=fl127, long=False)


def test_scaff_fills_gaps_from_either_map(tmp_path):
    d = str(tmp_path)
    cfg = synth.scenario_long(d)
    g = _graph(d, cfg, 31)
    ref, gpu, _ = _map_both(g, cfg, ["-p", "8"])
    e_ref = util.run([util.REF63, "scaff", "-g", ref, "-F"])
    util.run([util.REF63, "scaff", "-g", gpu, "-F"])
    assert "Filled gap number" in e_ref
    assert filecmp.cmp(f"{ref}.scafSeq", f"{gpu}.scafSeq", shallow=False)


@pytest.mark.skipif(not os.path.exists(B63), reason="drop-in binary not linked")
def test_dropin_map_long(tmp_path):
    d = str(tmp_path)
    cfg = synth.scenario_long(d)
    g = _graph(d, cfg, 31)
    _map_both(g, cfg, ["-p", "8", "-f"], gpu_bin=B63)


@pytest.mark.parametrize("case", ["long_read_past_long_len", "short_read_past_max_rd_len"])
def test_overflowing_reads_are_refused(tmp_path, case):
    """The reference would write past seqBuffer: a long read longer than longReadLen (a cutoff-free long library beside a larger
    max_rd_len), or a short read longer than max_rd_len once the long pass has raised maxReadLen4all.  No output is written."""
    d = str(tmp_path)
    synth.scenario_long(d)
    g = _graph(d, synth.scenario_pe_fastq(d), 31)
    gpu = _copy(g, "gpu")
    g0 = synth.genome(60000, 3, repeat=(400, 3))
    if case == "long_read_past_long_len":
        synth.write_long(os.path.join(d, "l.fa"), synth.long_reads(g0, 50, 100, 140, seed=2), fastq=False)
        synth.write_long(os.path.join(d, "m.fa"), synth.long_reads(g0, 50, 1000, 1200, seed=3), fastq=False)
        body = f"[LIB]\navg_ins=5\nasm_flags=4\nrd_len_cutoff=1100\nf={d}/l.fa\n[LIB]\navg_ins=6\nasm_flags=4\nf={d}/m.fa\n"
        cfg_txt = f"max_rd_len=2000\n[LIB]\navg_ins=300\nq1={d}/pe_1.fq\nq2={d}/pe_2.fq\n" + body
    else:
        synth.write_long(os.path.join(d, "s.fa"), synth.long_reads(g0, 50, 151, 200, seed=4), fastq=False)
        cfg_txt = (f"max_rd_len=150\n[LIB]\navg_ins=300\nq1={d}/pe_1.fq\nq2={d}/pe_2.fq\np={d}/s.fa\n"
                   f"[LIB]\nasm_flags=4\nrd_len_cutoff=5000\nf={d}/long.fa\n")
    cfg = os.path.join(d, "over.cfg")
    open(cfg, "w").write(cfg_txt)
    before = set(os.listdir(d))
    r = subprocess.run([api.BIN63, "map", "-s", cfg, "-g", gpu], capture_output=True, text=True, timeout=300)
    assert r.returncode == 255
    assert "the reference would write past its read buffer" in r.stderr
    assert set(os.listdir(d)) == before
