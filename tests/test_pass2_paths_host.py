"""Pass 2 and the -R outputs on designed long reads (soapdenovo2_b200.synth.figure8_long), CPU only.

Every scenario of tests/test_gpu_pass2_paths.py is run through the C model (oracle/pregraph_model.c): all seven files must equal the
reference's, run here where oracle/_ref was built, else its stored digests (tests/golden/pass2_ref.json).  The .path file is then
parsed: every figure-eight read of 2+ turns must have a record of (revs + 1) & 255 entries (one of 1 turn, a 2-edge path, none), so
that the generator cannot drift into a graph in which the wrap of the reference's unsigned char count is never reached; and every read
of a branch-free ring must be counted as deleted (parse1read keeps no segment of a k-mer outside the edges).
PGB200_WRITE_PASS2_REF=<file>: write the reference binary's digests and counter lines of every scenario to <file> (needs oracle/_ref)."""
import json
import os
import re

import pytest

from soapdenovo2_b200 import synth
from tests import util

GOLD_PATH = os.path.join(util.ROOT, "tests", "golden", "pass2_ref.json")

# paths of 255, 256, 257, 258, 511, 512, 513 and 700 entries, and of 2 (no record), 3 and 4
WRAP = [1, 2, 3, 254, 255, 256, 257, 510, 511, 512, 699]
WRAP127 = [1, 2, 3, 254, 255, 256, 257]                  # reads of up to about 34,300 bases
STAGE = [1, 2, 3, 10, 16]

# name -> (K, -p, extra options, synth.write_pass2_scenario arguments, engine environment)
SCENARIOS = {
    "wrap_k13_p1": (13, 1, ("-R",), dict(revs=WRAP, rings=3), {}),
    "wrap_k13_p8_a1": (13, 8, ("-a", "1", "-R"), dict(revs=WRAP, seed=1), {}),
    "wrap_k31_p1_a1": (31, 1, ("-a", "1", "-R"), dict(revs=WRAP, seed=2), {}),
    "wrap_k31_p8": (31, 8, ("-R",), dict(revs=WRAP, seed=3, rings=2), {}),
    "wrap_k127_p8_a1": (127, 8, ("-a", "1", "-R"), dict(revs=WRAP127, seed=4, rings=1), {}),
    # about 6 MB of reads in 1 MB chunks: the .path offsets (reclen -> recoff scan) run across chunks
    "wrap_k31_chunks": (31, 8, ("-a", "1", "-R"), dict(revs=WRAP, inst=20, seed=5), {"PGB200_CHUNK_MB": "1"}),
    # the two copies of each read as mates of one f1/f2 library: read ordinals step by 2 within a file
    "wrap_k31_pe": (31, 3, ("-R",), dict(revs=WRAP, seed=6, paired=True), {}),
    # packed words per read W64 = ceil(max_rd_len / 32): pass 1 stages 256 x W64 x 8 B (48 KB at W64 = 24), pass 2 128 x W64 x 8 B
    # (48 KB at W64 = 48, the unstaged loop above); an odd W64 with a read count that is not a multiple of 128 ends in a partial tile
    "stage_w24": (31, 8, ("-a", "1", "-R"), dict(revs=STAGE, seed=7, max_rd_len=768, n_genome=600), {}),
    "stage_w47": (31, 3, ("-R",), dict(revs=STAGE, seed=8, max_rd_len=1504, n_genome=1001), {}),
    "stage_w48": (63, 8, ("-a", "1", "-R"), dict(revs=STAGE, seed=9, max_rd_len=1536, n_genome=700), {}),
    "stage_w49": (31, 8, ("-R", "-d", "1"), dict(revs=STAGE, seed=10, max_rd_len=1568, n_genome=700), {}),
}
COUNTERS = ("node(s) allocated", "tip(s) removed", "linear node(s) marked", "edge(s) and", "vertex(es) output", "pre-arc(s) added",
            "read(s) deleted", "kmer(s) removed")


def counter_lines(log):
    """the reference's counter lines that the engine prints too (the model prints its pass-2 totals on a line of its own)"""
    return [l.strip() for l in log.splitlines() if any(k in l for k in COUNTERS) and "(model)" not in l]


def scenario(d, name):
    K, P, extra, args, env = SCENARIOS[name]
    cfg, counts, rings = synth.write_pass2_scenario(d, K, **args)
    return cfg, counts, rings, K, P, extra, env


def deleted_reads(lines):
    return int(re.search(r"(\d+) read\(s\) deleted", "\n".join(lines)).group(1))


def check_paths(name, prefix, lines, counts, rings):
    """the .path record counts, and (where only designed reads were fed) the deleted-read count: the ring reads exactly"""
    mixed = "n_genome" in SCENARIOS[name][3]
    check_counts(path_counts(prefix), counts, mixed)
    if not mixed:
        assert deleted_reads(lines) == rings


def path_counts(prefix):
    """the count byte of every .path record, in order"""
    b = open(prefix + ".path", "rb").read()
    out, i = [], 0
    while i < len(b):
        out.append(b[i])
        i += 1 + 4 * b[i]
    assert i == len(b), "truncated .path record"
    return out


def check_counts(got, want, mixed):
    """want: the figure-eight reads' counts in read order.  Alone (mixed = False) they are the whole file; mixed with genome reads
    they must appear in order among the genome reads' records"""
    if not mixed:
        assert got == want
        return
    it = iter(got)
    assert all(any(c == w for c in it) for w in want), (got, want)


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


@pytest.mark.parametrize("K", [13, 31, 127])
def test_figure8_builds_the_graph_it_claims(K):
    M, expect = synth.figure8_long(K, [1, 2, 3, 5, 40])
    synth.check_motifs([M], K)
    assert expect == [None, 3, 4, 6, 41]
    assert max(len(s) for s, _ in synth.figure8_long(127, [257])[0].reads) <= 34500


_written = {}


def reference_result(name, cfg, d, K, P, extra):
    """(digests, counter lines) of the reference on this scenario: run here when the binary exists, else the stored result"""
    if util.have_ref():
        ref = os.path.join(d, "ref")
        log = util.run_ref(util.REF127 if K > 63 else util.REF63, cfg, ref, K, P, extra)
        res = (util.digests(ref, util.SUFFIXES_R), counter_lines(log))
        if os.environ.get("PGB200_WRITE_PASS2_REF"):
            _written[name] = {"digests": res[0], "counters": res[1]}
            json.dump(_written, open(os.environ["PGB200_WRITE_PASS2_REF"], "w"), indent=1, sort_keys=True)
        return res
    gold = json.load(open(GOLD_PATH))[name]
    return gold["digests"], gold["counters"]


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_model_matches_reference_on_long_paths(tmp_path, name):
    d = str(tmp_path)
    cfg, counts, rings, K, P, extra, _ = scenario(d, name)
    mod = os.path.join(d, "mod")
    util.run_model(util.MODEL127 if K > 63 else util.MODEL63, cfg, mod, K, P, extra)
    digests, lines = reference_result(name, cfg, d, K, P, extra)
    assert util.digests(mod, util.SUFFIXES_R) == digests
    if util.have_ref() and not os.environ.get("PGB200_WRITE_PASS2_REF"):
        assert digests == json.load(open(GOLD_PATH))[name]["digests"], "the stored digests are stale"
    check_paths(name, mod, lines, counts, rings)
