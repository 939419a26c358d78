"""GPU parity, pass 1, with the aggregation's record collapse forced on, forced off and adaptive (PGB200_SKM_COLLAPSE, which
applies to 256-bit keys: K <= 63 always collapses): the distinct-record buffer is filled through the dedup table (on), by copying every staged window
with count 1 (off), or per CTA by whichever the distinct share of its recent buckets calls for (auto).  All three are exact, so
every shape must give the C model's table dump and .kmerFreq, and the CLI the reference's pregraph files: the collapse-stress reads
of test_gpu_skm_collapse.py (records repeated up to hundreds of times, 1 bucket), and the stress shapes of test_gpu_pass1.py (1-4
buckets, a tiny table that grows, spills past the shared-memory table, mid-stream flushes).  65536 buckets give every CTA enough
buckets for auto to switch."""
import os
import subprocess

import pytest

from soapdenovo2_b200 import api, synth
from tests import util
from tests.test_gpu_skm_collapse import _scenario as _repeated_reads

pytestmark = pytest.mark.gpu

MODES = ["on", "off", "auto"]


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("buckets", ["0", "1"])
@pytest.mark.parametrize("K", [65, 99])   # (the reads are 100 bases long)
def test_repeated_records_modes(tmp_path, monkeypatch, K, buckets, mode):
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_SKM_COLLAPSE", mode)
    if buckets != "0":
        monkeypatch.setenv("PGB200_SKM_BUCKETS", buckets)
    cfg = _repeated_reads(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL127, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=1, max_rd_len=100)
    for mate, fn in enumerate(("c_1.fq", "c_2.fq")):
        eng.feed_text(open(tmp_path / fn, "rb").read(), fastq=True, ord_base=mate, ord_stride=2)
    eng.finish_pass1()
    hist, _, _ = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()
    eng.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("K,buckets,arena_mb,every", [(127, "1", "0", "0"), (127, "2", "0", "0"), (127, "4", "1", "3"), (99, "3", "1", "2"),
                                                     (127, "65536", "0", "0"), (65, "65536", "0", "0")])
def test_stress_paths_modes(tmp_path, monkeypatch, K, buckets, arena_mb, every, mode):
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_SKM_COLLAPSE", mode)
    monkeypatch.setenv("PGB200_SKM_BUCKETS", buckets)
    if arena_mb != "0":
        monkeypatch.setenv("PGB200_SKM_ARENA_MB", arena_mb)
    if every != "0":
        monkeypatch.setenv("PGB200_SKM_FLUSH_EVERY", every)
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL127, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=1, max_rd_len=150, table_slots=2048)
    for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
        lines = open(tmp_path / fn, "rb").read().split(b"\n")[:-1]
        recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines), 4)]
        for i in range(0, len(recs), 700):
            eng.feed_text(b"".join(recs[i:i + 700]), fastq=True, ord_base=2 * i + mate, ord_stride=2)
    st = eng.finish_pass1()
    assert st.table_slots > 2048
    hist, _, _ = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()
    eng.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("K,buckets", [(99, "0"), (99, "1"), (65, "0")])
def test_cli_vs_reference_modes(tmp_path, K, buckets, mode):
    """The CLI's pregraph files on the repeated reads against the reference (or the C model where it is not shipped)."""
    cfg = _repeated_reads(str(tmp_path))
    want = str(tmp_path / "want")
    if util.have_ref():
        util.run_ref(util.REF127, cfg, want, K, 4, ("-a", "1"))
    else:
        util.run_model(util.MODEL127, cfg, want, K, 4, ("-a", "1"))
    env = dict(os.environ, PGB200_SKM="1", PGB200_SKM_COLLAPSE=mode)
    if buckets != "0":
        env["PGB200_SKM_BUCKETS"] = buckets
    gpu = str(tmp_path / "gpu")
    r = subprocess.run([api.BIN127, "pregraph", "-s", cfg, "-K", str(K), "-p", "4", "-a", "1", "-o", gpu],
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    util.compare(want, gpu, util.SUFFIXES)


def test_bad_collapse_value(monkeypatch):
    """An unknown PGB200_SKM_COLLAPSE value is an error, not a silent default."""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_SKM_COLLAPSE", "sometimes")
    eng = api.PregraphEngine(K=31, P=1, initG=1, max_rd_len=100)
    try:
        eng.feed_text(b">r\n" + b"ACGTTGCAAGGCTTACCGATCGATCGGATCCAGTACGATCAGT\n", fastq=False, ord_base=0)
        with pytest.raises(Exception, match="PGB200_SKM_COLLAPSE"):
            eng.finish_pass1()
    finally:
        eng.close()
