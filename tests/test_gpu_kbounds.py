"""Every GPU kernel at the K where the k-mer algebra changes shape (make_kparams: top_word / top_shift, kprev, kprev_reg, krc_n).
At K = 33, 65 and 97 the first base opens a new 64-bit word and is alone in it (top_shift = 0); at K = 63, 95 and 127 the (K+1)-mer
fills its words exactly; K = 35, 61, 67, 93 and 125 sit one base off those edges; K <= 63 in the 127-mer build leaves whole words
empty.  Checked against the reference binary (all pregraph files; map files and stderr) and against the C model (the pass-1 table
dump in reference iteration order), under both insert paths of pass 1."""
import os
import subprocess

import pytest

from soapdenovo2_b200 import api, synth
from tests import util
from tests.test_gpu_map import _graph, _map_both
from tests.test_gpu_map_long import _map_both as _map_both_long

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")]

# (K, 127-mer build, -p, extra pregraph options)
CLI = [(33, False, 8, ("-R", "-a", "1")), (35, False, 4, ("-d", "1")), (61, False, 8, ("-R",)),
       (33, True, 4, ("-a", "1")), (63, True, 8, ("-R", "-d", "1")), (65, True, 8, ("-R", "-a", "1")), (67, True, 3, ()),
       (93, True, 8, ("-d", "1", "-a", "1")), (95, True, 8, ("-R",)), (97, True, 4, ("-R", "-a", "1")), (125, True, 8, ("-d", "1"))]


@pytest.mark.parametrize("K,f127,P,extra", CLI, ids=[f"K{K}-{127 if f else 63}mer" for K, f, _, _ in CLI])
def test_cli_parity_at_word_boundary_k(tmp_path, K, f127, P, extra):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    ref = str(tmp_path / "ref")
    util.run_ref(util.REF127 if f127 else util.REF63, cfg, ref, K, P, extra)
    suffixes = util.SUFFIXES_R if "-R" in extra else util.SUFFIXES
    for skm in ("0", "1"):   # per-instance inserts, aggregated super-k-mer records
        gpu = str(tmp_path / f"gpu{skm}")
        r = subprocess.run([api.BIN127 if f127 else api.BIN63, "pregraph", "-s", cfg, "-K", str(K), "-p", str(P), "-o", gpu, *extra],
                           capture_output=True, text=True, timeout=600, env=dict(os.environ, PGB200_SKM=skm))
        assert r.returncode == 0, r.stderr[-4000:]
        util.compare(ref, gpu, suffixes)


@pytest.fixture(scope="module")
def _oracle():
    util.build_oracle()


def _pass1_dump(tmp_path, K, f127, chunk=None):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL127 if f127 else util.MODEL63, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=int(f127), max_rd_len=150, table_slots=2048 if chunk else 0)
    for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
        data = open(tmp_path / fn, "rb").read()
        if not chunk:
            eng.feed_text(data, fastq=True, ord_base=mate, ord_stride=2)
            continue
        lines = data.split(b"\n")[:-1]
        recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines), 4)]
        for i in range(0, len(recs), chunk):
            eng.feed_text(b"".join(recs[i:i + chunk]), fastq=True, ord_base=2 * i + mate, ord_stride=2)
    st = eng.finish_pass1()
    assert st.instances == 12000 * (150 - K + 1)
    hist, _, _ = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()
    eng.close()


@pytest.mark.parametrize("mode", ["direct", "aggregated"])
@pytest.mark.parametrize("K,f127", [(33, False), (65, True), (95, True), (97, True)])
def test_pass1_table_dump_at_word_boundary_k(tmp_path, monkeypatch, _oracle, K, f127, mode):
    monkeypatch.setenv("PGB200_SKM", "0" if mode == "direct" else "1")
    _pass1_dump(tmp_path, K, f127)


@pytest.mark.parametrize("K", [65, 97])
def test_pass1_aggregation_stress_at_word_boundary_k(tmp_path, monkeypatch, _oracle, K):
    """three buckets (almost every k-mer spills past the shared-memory table), a 1 MB arena (mid-stream flushes), 700-read chunks"""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_SKM_BUCKETS", "3")
    monkeypatch.setenv("PGB200_SKM_ARENA_MB", "1")
    _pass1_dump(tmp_path, K, True, chunk=700)


# chunk_mb: map's default short-pass reader in chunks of that size, which each 1.9 MB read file crosses
MAP = [(33, False, None), (33, True, None), (65, True, None), (95, True, None), (97, True, None), (33, False, "1")]


@pytest.mark.parametrize("K,f127,chunk_mb", MAP, ids=[f"{K}-{f127}" + (f"-chunk{c}mb" if c else "") for K, f127, c in MAP])
def test_map_at_word_boundary_k(tmp_path, monkeypatch, K, f127, chunk_mb):
    if chunk_mb:
        monkeypatch.setenv("PGB200_CHUNK_MB", chunk_mb)
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    g = _graph(str(tmp_path), cfg, K, flavour127=f127)
    _map_both(g, cfg, ["-p", "8"], flavour127=f127)


def test_map_small_k_on_k63_graph(tmp_path):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 63)
    _map_both(g, cfg, ["-p", "8", "-k", "33"])


def test_map_two_word_keys_on_k97_graph(tmp_path):
    """-k 63 and -k 65 on a K = 97 graph in the 127-mer build: the map engine's keys go from four words to two"""
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    g = _graph(str(tmp_path), cfg, 97, flavour127=True)
    _map_both(g, cfg, ["-p", "8", "-k", "63"], flavour127=True, tag="63")
    _map_both(g, cfg, ["-p", "8", "-k", "65"], flavour127=True, tag="65")


def test_long_map_at_k65(tmp_path, monkeypatch):
    """a long-read library at K = 65, the short pass through k_map_long as well"""
    d = str(tmp_path)
    cfg = synth.scenario_long(d)
    g = _graph(d, cfg, 65, flavour127=True)
    monkeypatch.setenv("PGB200_MAP_LONG", "all")
    _map_both_long(g, cfg, ["-p", "8", "-f"], flavour127=True)
