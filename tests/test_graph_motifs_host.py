"""The tip and edge phases on designed graph motifs (soapdenovo2_b200.synth.MOTIFS), CPU only.

1. The motif builders make the graphs they claim (node, dead-end and junction counts, every tip walk's length and end node),
   checked by a plain Python de Bruijn graph of the reads, so that a mislabelled motif fails here and not as a GPU mismatch.
2. The C model (oracle/pregraph_model.c) writes the reference's seven files and counter lines on every motif scenario.  Where
   oracle/_ref was built the reference binary is run; otherwise the stored reference results (tests/golden/motif_ref.json) are used.
3. The reference's own log pins where the cut falls (chains of up to 2K-1 linear nodes are clipped, 2K are not), that a tie with
   the strongest link is kept, and that the cascades take at least three minor cycles.
PGB200_WRITE_MOTIF_REF=<file>: write the reference binary's digests and counter lines of every scenario to <file> (needs oracle/_ref)."""
import json
import os

import pytest

from soapdenovo2_b200 import synth
from tests import util

GOLD_PATH = os.path.join(util.ROOT, "tests", "golden", "motif_ref.json")

# name -> (motif kinds, K, -p, extra options, instances of each kind)
EDGE_KINDS = ["lollipop", "hairpin", "figure8", "bubble", "ring", "isolated"]
SCENARIOS = {
    "cut_k31": (["cut"], 31, 3, ("-R",), 200),
    "cut_k127": (["cut"], 127, 8, (), 100),
    "tie_k63": (["tie"], 63, 3, ("-d", "1"), 200),
    "conflict_k31": (["conflict"], 31, 3, (), 200),
    "conflict_k95": (["conflict"], 95, 1, ("-R",), 100),
    "cascade_k31": (["cascade"], 31, 8, ("-R",), 200),
    "cascade_k65": (["cascade"], 65, 3, (), 100),
    "thin_k31": (["thin_orphan", "thin_multi"], 31, 3, ("-R",), 200),
    "thin_k127": (["thin_orphan", "thin_multi"], 127, 3, (), 60),
    "edges_k21": (EDGE_KINDS, 21, 3, ("-R",), 40),
    "edges_k63": (EDGE_KINDS, 63, 8, ("-R",), 40),
    "edges_k127": (EDGE_KINDS, 127, 3, ("-R",), 24),
    "barrier_k31": (["barrier"], 31, 3, (), 200),
    "barrier_k95": (["barrier"], 95, 8, ("-R",), 100),
    "large_k21": (["large"], 21, 3, (), 510),
}
SEEDS = {"large_k21": 4}   # seeds 0..3 of the large instance collide on a k-mer across instances (write_motif_scenario refuses those)
COUNTERS = ("node(s) allocated", "tip(s) removed", "linear node(s) marked", "edge(s) and", "vertex(es) output", "kmer(s) removed")


def counter_lines(log):
    """the reference's counter lines that the model prints too"""
    return [l.strip() for l in log.splitlines() if any(k in l for k in COUNTERS)]


def cycles(lines):
    """tips removed per minor cycle, from the counter lines"""
    return [int(l.split()[0]) for l in lines if " removed in cycle " in l]


def scenario(d, name):
    kinds, K, P, extra, copies = SCENARIOS[name]
    cfg, sets = synth.write_motif_scenario(d, kinds, K, copies, SEEDS.get(name, 0))
    return cfg, sets, K, P, extra


def suffixes(extra):
    return util.SUFFIXES_R if "-R" in extra else util.SUFFIXES


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


@pytest.mark.parametrize("K", [21, 31, 63, 127])
@pytest.mark.parametrize("kind", synth.MOTIFS)
def test_motif_builds_the_graph_it_claims(kind, K):
    if kind == "large" and K > 31:
        pytest.skip("the large instance is built at small K only")
    synth.check_motifs([synth.motif_reads(kind, K, 30)], K)


_written = {}


def reference_result(name, cfg, d, K, P, extra):
    """(digests, counter lines) of the reference on this scenario: run here when the binary exists, else the stored result"""
    if util.have_ref():
        ref = os.path.join(d, "ref")
        log = util.run_ref(util.REF127 if K > 63 else util.REF63, cfg, ref, K, P, extra)
        res = (util.digests(ref, suffixes(extra)), counter_lines(log))
        if os.environ.get("PGB200_WRITE_MOTIF_REF"):
            _written[name] = {"digests": res[0], "counters": res[1]}
            json.dump(_written, open(os.environ["PGB200_WRITE_MOTIF_REF"], "w"), indent=1, sort_keys=True)
        return res
    gold = json.load(open(GOLD_PATH))[name]
    return gold["digests"], gold["counters"]


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_model_matches_reference_on_motifs(tmp_path, name):
    d = str(tmp_path)
    cfg, sets, K, P, extra = scenario(d, name)
    mod = os.path.join(d, "mod")
    log = util.run_model(util.MODEL127 if K > 63 else util.MODEL63, cfg, mod, K, P, ("-U", mod + ".tips", *extra))
    digests, lines = reference_result(name, cfg, d, K, P, extra)
    assert util.digests(mod, suffixes(extra)) == digests
    assert counter_lines(log) == lines
    # -U: one record per node, after the tips
    assert os.path.getsize(mod + ".tips") == int(lines[0].split()[0]) * ((4 if K > 63 else 2) * 8 + 10)

    # what the reference's log says about each motif
    kinds, copies = SCENARIOS[name][0], SCENARIOS[name][4]
    c = cycles(lines)
    if kinds == ["cut"]:          # m = 2K-2, 2K-1 clipped; 2K, 2K+1 not
        assert c[0] == copies // 2 and sum(c) == copies // 2
    if kinds == ["tie"]:          # equal to the strongest link: kept; one below: clipped
        assert c[0] == copies // 2 and sum(c) == copies // 2
    if kinds == ["cascade"]:      # each instance clips 4 times; some instances need a cycle per clip
        assert sum(c) == 4 * copies and len([x for x in c if x]) >= 3
    if kinds == ["conflict"]:     # every instance clips all but its strongest tip; the rest clip at J2 or stay
        n2 = (copies + 1) // 2
        assert sum(c) >= n2 * 1 + (copies - n2) * 2 and len([x for x in c if x]) >= 2
    if kinds[0] == "thin_orphan":  # every frequency-one tip goes in the THIN pass; the orphan-chain ends go in the minor pass
        assert lines[2] == f"Total {copies * 7} tip(s) removed." and c[0] == copies
    if kinds == ["barrier"]:      # A, X and c clip in every instance; c clips in the first cycle only when it comes after X
        assert sum(c) == 3 * copies and len([x for x in c if x]) >= 2
    if name == "large_k21":
        assert c[0] == 20400 and sum(c) == 20400
