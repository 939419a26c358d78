"""GPU tip clipping and edge emission on designed graph motifs (soapdenovo2_b200.synth.MOTIFS), node by node.

The engine restates the reference's order-dependent loops in parallel: THIN rounds, speculated minor-sweep windows that commit a
clean prefix (dirty frontiers, dead-end barriers, re-queued candidates), and claim/resolve rounds for the edges.  Each test checks
the result against the reference (or the C model) and, through the PGB200_VERBOSE counters, that the branch it is about ran:
  - per node: the table after remove_tips equals the model's -U dump byte for byte, over K, -p, -d 0 / 1 and -a 1 / growth replay;
  - forced windows: PGB200_TIP_WINDOW = 1, 2, 3, 64 split every conflict across windows and must not change a single node;
  - CLI: all seven files and the counter lines of every motif scenario of tests/test_graph_motifs_host.py."""
import gzip
import json
import os
import re

import pytest

from soapdenovo2_b200 import api, synth
from tests import util
from tests.test_gpu_full import _engine, _oracle
from tests.test_graph_motifs_host import EDGE_KINDS, GOLD_PATH, SCENARIOS, counter_lines, scenario, suffixes

pytestmark = pytest.mark.gpu

ALL = [k for k in synth.MOTIFS if k != "large"]
TIPS_RE = re.compile(r"remove_tips: (\d+) THIN round\(s\), (\d+) minor window\(s\), (\d+) dirty frontier\(s\), (\d+) barrier frontier\(s\), "
                     r"(\d+) re-queued, (\d+) new dead end\(s\) queued ahead, (\d+) behind")
EDGES_RE = re.compile(r"build_edges: (\d+) start\(s\), (\d+) claim/resolve round\(s\), (\d+) emitted start\(s\) without a reverse start")
TIP_KEYS = ("thin_rounds", "windows", "dirty", "barriers", "requeued", "ahead", "behind")


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def tip_counters(log):
    m = TIPS_RE.findall(log)
    assert len(m) == 1, log[-3000:]
    return dict(zip(TIP_KEYS, map(int, m[0])))


def tips_dump(cfg, K, P, D, initG, capfd):
    """finish_pass1 -> sweeps -> build_layout -> remove_tips -> dump_nodes through the C-ABI; returns (dump, tip counters)"""
    mrl, plan = api.plan_files(cfg)
    eng = api.PregraphEngine(K=K, P=P, initG=initG, D=D, flavour127=int(K > 63), max_rd_len=mrl, verbose=1)
    n = 0
    for mate, fq, rev, cut, path in plan:
        n += eng.feed_text(open(path, "rb").read(), fastq=bool(fq), ord_base=n, reverse_seq=rev, maxlen=cut)
    capfd.readouterr()
    eng.finish_pass1(); eng.sweeps(); eng.build_layout(); eng.remove_tips()
    dump = eng.dump_nodes()
    eng.close()
    return dump, tip_counters(capfd.readouterr().err)


def model_tips(cfg, d, K, P, extra):
    mod = os.path.join(d, "mod")
    util.run_model(util.MODEL127 if K > 63 else util.MODEL63, cfg, mod, K, P, ("-U", mod + ".tips", *extra))
    return open(mod + ".tips", "rb").read()


# (-p, -d, -a): the THIN pass and none, static tables and growth replay
OPTS = [(1, 0, 1), (3, 1, 1), (8, 0, 0), (3, 1, 0)]


@pytest.mark.parametrize("P,D,initG", OPTS, ids=[f"p{p}-d{d}-{'a1' if a else 'grow'}" for p, d, a in OPTS])
@pytest.mark.parametrize("K", [21, 31, 63, 65, 95, 127])
def test_nodes_after_tips(tmp_path, capfd, K, P, D, initG):
    d = str(tmp_path)
    cfg, _ = synth.write_motif_scenario(d, ALL, K, 12)
    want = model_tips(cfg, d, K, P, ("-d", str(D)) + (("-a", str(initG)) if initG else ()))
    got, c = tips_dump(cfg, K, P, D, initG, capfd)
    assert len(got) == len(want)
    if got != want:
        rec = (4 if K > 63 else 2) * 8 + 10
        i = next(i for i in range(0, len(got), rec) if got[i:i + rec] != want[i:i + rec]) // rec
        pytest.fail(f"node {i} (iteration order) differs after the tips: engine {got[i * rec:(i + 1) * rec].hex()} model {want[i * rec:(i + 1) * rec].hex()}")
    assert c["dirty"] > 0                       # the conflict motifs: a later tip read the junction an earlier clip writes
    assert c["requeued"] > 0
    if D == 0:
        assert c["thin_rounds"] >= 3            # three single tips on each side of one k-mer: one THIN commit per round


@pytest.mark.parametrize("K", [31, 95])
def test_forced_tip_windows(tmp_path, capfd, monkeypatch, K):
    d = str(tmp_path)
    cfg, _ = synth.write_motif_scenario(d, ["conflict", "cascade", "barrier", "thin_orphan"], K, 120)
    want = model_tips(cfg, d, K, 3, ("-a", "1"))
    total = dict.fromkeys(TIP_KEYS, 0)
    for w in (1, 2, 3, 64):
        monkeypatch.setenv("PGB200_TIP_WINDOW", str(w))
        got, c = tips_dump(cfg, K, 3, 0, 1, capfd)
        assert got == want, f"PGB200_TIP_WINDOW={w}: the table after the tips differs from the model"
        assert c["windows"] > 1
        for k in TIP_KEYS:
            total[k] += c[k]
    assert total["dirty"] > 0 and total["barriers"] > 0 and total["requeued"] > 0 and total["ahead"] > 0 and total["behind"] > 0, total


def edge_headers(prefix):
    """(length, from k-mer words, to k-mer words, bal_edge) of every .edge.gz record"""
    out = []
    for l in gzip.open(prefix + ".edge.gz", "rt"):
        if l.startswith(">"):
            f = l[1:].split(",")
            out.append((int(f[0].split()[1]), f[1], f[2], int(f[4])))
    return out


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_cli_on_motifs(tmp_path, name):
    d = str(tmp_path)
    cfg, _, K, P, extra = scenario(d, name)
    ref, gpu = os.path.join(d, "ref"), os.path.join(d, "gpu")
    lr = _oracle(int(K > 63), cfg, ref, K, P, extra)
    lg = _engine(int(K > 63), cfg, gpu, K, P, extra, env={"PGB200_VERBOSE": "1"})
    util.compare(ref, gpu, suffixes(extra))
    # the counter lines (tips per minor cycle among them) against the reference, or its stored lines where it was not built
    want = counter_lines(lr) if util.have_ref() else json.load(open(GOLD_PATH))[name]["counters"]
    assert [l for l in counter_lines(lg) if not l.startswith("[pgb200]")] == want
    c = tip_counters(lg)
    assert len(EDGES_RE.findall(lg)) == 1
    kinds = SCENARIOS[name][0]
    if kinds == ["conflict"]:
        assert c["dirty"] > 0
    if kinds == ["cascade"]:
        assert c["ahead"] > 0 and c["behind"] > 0 and c["requeued"] > 0
    if kinds == ["barrier"]:                    # X, made a dead end by A's clip, stops the window before c
        assert c["barriers"] > 0
    if kinds == EDGE_KINDS:
        h = edge_headers(gpu)
        lens = {x[0] for x in h}
        assert any(x[3] == 0 for x in h)        # the hairpin: a palindromic unipath, start == rev(start)
        assert any(x[1] == x[2] and x[3] == 1 for x in h)   # lollipop and figure-eight loops: leave and re-enter one junction
        assert {1, 100, 101, 200, 201} <= lens  # length-1 bubbles (the patch table) and the 100-column text wrapping
        assert int(re.search(r"edge\(s\) and (\d+) extra node", lg).group(1)) > 0
    if kinds[0] == "thin_orphan":
        assert c["thin_rounds"] >= 3
    if kinds == ["large"]:
        assert c["windows"] > 1                 # the default adaptive window crosses boundaries by itself
