"""The `map` stage's command line and input checks, which run before any GPU work, and the reference behaviour the stage's model of
.readInGap.gz rests on (only where oracle/_ref exists)."""
import filecmp
import os
import shutil
import subprocess

import pytest

from soapdenovo2_b200 import api, synth
from tests import util


def _map(args):
    return subprocess.run([api.BIN63, "map", *args], capture_output=True, text=True, timeout=120)


def test_map_usage_without_s_or_g(tmp_path):
    for args in (["-g", str(tmp_path / "x")], ["-s", str(tmp_path / "x.cfg")], []):
        r = _map(args)
        assert r.returncode == 1
        assert "\nmap -s configFile -g inputGraph [-f] [-p n_cpu -k kmer_R2C] [-h contig_total_length]\n" in r.stderr
        assert "kmer_R2C(min 13, max 63)" in r.stderr


def test_map_missing_contig(tmp_path):
    cfg = synth.scenario_pe_fastq(str(tmp_path), genome_len=5000, n_pairs=100)
    g = str(tmp_path / "none")
    r = _map(["-s", cfg, "-g", g])
    assert r.returncode == 255
    assert r.stderr.rstrip().endswith(f"Cannot open {g}.contig. Now exit to system...")


def _fake_graph(d):
    g = os.path.join(d, "g")
    with open(g + ".contig", "w") as f:
        f.write(">1 length 40 cvg_1.0_tip_0\n" + "ACGT" * 10 + "\n")
    return g


@pytest.mark.parametrize("line,msg", [("asm_flags=4", "long-read libraries (asm_flags=4) are not supported"),
                                      ("b=reads.bam", "BAM input (b=) is not supported")])
def test_map_refuses_long_reads_and_bam(tmp_path, line, msg):
    d = str(tmp_path)
    g = _fake_graph(d)
    cfg = os.path.join(d, "x.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=100\n[LIB]\navg_ins=300\n{line}\nq1={d}/a.fq\nq2={d}/b.fq\n")
    r = _map(["-s", cfg, "-g", g])
    assert r.returncode == 255
    assert msg in r.stderr
    assert not os.path.exists(g + ".readOnContig.gz")


@pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")
def test_reference_readingap_depends_on_threads(tmp_path):
    """The premise of the stage's rcSeq[1] model: the reference's .readOnContig.gz and .peGrads do not depend on -p, its
    .readInGap.gz does (stale bits of the buffer thread 0 shares).  If this fails, the model in map_stage.cpp has lost its premise."""
    d = str(tmp_path)
    cfg = synth.scenario_multilib(d)
    g = os.path.join(d, "g")
    util.run([util.REF63, "pregraph", "-s", cfg, "-K", "31", "-p", "4", "-o", g, "-R"])
    util.run([util.REF63, "contig", "-g", g, "-R"])
    outs = {}
    for p in ("3", "8"):
        o = os.path.join(d, "p" + p)
        for s in ("contig", "ContigIndex", "preGraphBasic"):
            shutil.copy(f"{g}.{s}", f"{o}.{s}")
        util.run([util.REF63, "map", "-s", cfg, "-g", o, "-p", p])
        outs[p] = o
    assert filecmp.cmp(f"{outs['3']}.readOnContig.gz", f"{outs['8']}.readOnContig.gz", shallow=False)
    assert filecmp.cmp(f"{outs['3']}.peGrads", f"{outs['8']}.peGrads", shallow=False)
    assert not filecmp.cmp(f"{outs['3']}.readInGap.gz", f"{outs['8']}.readInGap.gz", shallow=False), \
        "the reference's .readInGap.gz no longer depends on -p: the rcSeq[1] model of map_stage.cpp lost its premise"


def test_dropin_links_gpu_map():
    """The drop-in binaries take call_align from the shim and leave the reference's map objects out"""
    if not os.path.isdir(os.path.join(util.ROOT, "oracle", "_ref", "o63")):
        pytest.skip("oracle/_ref objects absent (built where the reference sources exist)")
    subprocess.run(["bash", os.path.join(util.ROOT, "scripts", "link_dropin.sh")], check=True, capture_output=True)
    for fl in ("63", "127"):
        exe = os.path.join(util.ROOT, "oracle", "_ref", f"SOAPdenovo-{fl}mer-b200")
        und = subprocess.run(["nm", "-D", "--undefined-only", exe], capture_output=True, text=True).stdout
        full = subprocess.run(["nm", exe], capture_output=True, text=True).stdout
        assert "pgb200_map_main" in und
        assert " T call_align" in full and " T call_scaffold" in full
        assert "prlRead2Ctg" not in full and "prlContig2nodes" not in full
