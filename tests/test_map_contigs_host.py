"""The `map` stage's `.contig` reader and contig table on designed inputs, on the CPU.

- The stage's reader (read_contigs, run by tests/host_read_contigs.cpp) against a Python transcription of the reference's two
  passes (tests/map_model.py) on `.contig` shapes that the reference's `contig` never writes: fgets piece boundaries, long headers,
  CRLF, '#' lines, names with leading whitespace or no digits, bases before the first header.
- Where oracle/_ref exists, the transcription and the placement model against the reference `map` itself: its stats line, node and
  k-mer counts, and, read by read, `.readOnContig.gz` and the heads of the `.readInGap.gz` records."""
import gzip
import os
import random
import subprocess

import pytest

from tests import map_designs as md
from tests import map_model, util

K = 31
_need_ref = pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")


@pytest.fixture(scope="module")
def reader(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("read_contigs") / "host_read_contigs")
    src = [os.path.join(util.ROOT, *p) for p in (("tests", "host_read_contigs.cpp"), ("soapdenovo2_b200", "csrc", "stage_io.cpp"),
                                                 ("soapdenovo2_b200", "csrc", "deflate.cu"))]
    subprocess.run([util.NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, *src, "-lz"],
                   check=True, capture_output=True)
    return exe


def _driver(exe, d, text, k):
    g = os.path.join(d, "c")
    open(g + ".contig", "wb").write(text)
    r = subprocess.run([exe, g, str(k)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stderr.strip(), r.stdout.splitlines()


def _expected(text, k):
    stats, kept, kmers = map_model.read_contigs(text, k)
    return stats, [f"kmers {kmers}"] + [f"{cid} {len(c)} {map_model.digest(c)}" for cid, c in kept]


_CASES = md.reader_cases(K)


@pytest.mark.parametrize("name,text", _CASES, ids=[c[0] for c in _CASES])
def test_reader_matches_transcription(reader, tmp_path, name, text):
    for k in (K, 21):
        assert _driver(reader, str(tmp_path), text, k) == _expected(text, k), (name, k)


# The four shapes whose reading the reference settles (K = 31, contig A of 20 000 bp as >1, B of 3 000 bp as >3): what the reference
# printed for each, and where a read from A at 19 700 lands
def _four(rng):
    A, B = md.seq(rng, 20000), md.seq(rng, 3000)
    w = lambda s: md.wrap(s, 100)   # noqa: E731
    return A, B, {
        "a_one_line": (f">1\n{A}\n>3\n{w(B)}\n", "2 contig(s), maximum sequence length 19996", 22936, 19700),
        "header_space": (f">1\n{w(A)}\n> 3 length 3000\n{w(B)}\n", "2 contig(s), maximum sequence length 20000", 22940, 19700),
        "bases_before": (f"{A[:77]}\n>1\n{w(A)}\n>3\n{w(B)}\n", "2 contig(s), maximum sequence length 20000", 22940, 19700),
        "long_header": (f">1 {'x' * 6000}\n{w(A)}\n>3\n{w(B)}\n", "2 contig(s), maximum sequence length 21054", 23944, 20704),
    }


def _four_pairs(A, B):
    return [(A[19700:19800], md.rc(A[19900:20000])), (B[100:200], md.rc(B[300:400])), (A[5000:5100], md.rc(B[2000:2100]))]


@pytest.mark.parametrize("case", ["a_one_line", "header_space", "bases_before", "long_header"])
def test_four_reference_shapes(reader, tmp_path, case):
    """Fixed numbers; each fails with a reader that counts whole lines, takes the name from s[1], keeps bases before the first
    '>' or skips a whole header line"""
    A, B, cases = _four(random.Random(4))
    text, stats, kmers, pos_a = cases[case]
    text = text.encode()
    got_stats, lines = _driver(reader, str(tmp_path), text, K)
    assert got_stats.startswith(stats) and lines[0] == f"kmers {kmers}"
    assert [ln.split()[0] for ln in lines[1:]] == ["1", "3"]   # B is contig 3 under "> 3 length 3000"
    pairs = _four_pairs(A, B)
    index = "Edge_num 4 2\nindex\tlength\treverseComplement\n1\t19969\t1\n3\t2969\t1\n"
    p = md.predict(text, index, pairs, K)
    assert p["on"][0] == f"1\t1\t{pos_a}\t+" and p["on"][2].split("\t")[1] == "3"
    if util.have_ref():
        g, cfg = md.write_graph(str(tmp_path), "four", text, index, K, pairs, 100)
        err = util.run([util.REF63, "map", "-s", cfg, "-g", g, "-p", "4"])
        assert md.ref_stats(err) == (p["stats"], p["table"].distinct(), kmers)
        assert _ref_on(g) == p["on"]


def _ref_on(g):
    return gzip.open(g + ".readOnContig.gz", "rt").read().splitlines()[1:]


@_need_ref
@pytest.mark.parametrize("name,text", _CASES, ids=[c[0] for c in _CASES])
def test_transcription_matches_reference(tmp_path, name, text):
    """The stats line, node and k-mer counts and the placements of reads drawn from the kept contigs"""
    p = md.predict(text, "Edge_num 0 0\n", [], K)
    n_records = text.count(b">") + 1
    index = md.contig_index(p["kept"], K, n_min=n_records)
    pairs = md.sample_pairs(random.Random(len(text)), p["kept"], 100) or [("A" * 100, "C" * 100)]
    p = md.predict(text, index, pairs, K)
    g, cfg = md.write_graph(str(tmp_path), "r", text, index, K, pairs, 100)
    err = util.run([util.REF63, "map", "-s", cfg, "-g", g, "-p", "4"], timeout=300)
    assert md.ref_stats(err) == (p["stats"], p["table"].distinct(), p["kmers"])
    assert _ref_on(g) == p["on"]


def _rules(p, K):
    """how often each designed rule fired in one run of the model"""
    t, pl = p["table"], p["placements"]
    return {
        "keys seen 3+ times": sum(1 for n in t.seen.values() if n >= 3),
        "deleted keys": sum(1 for e in t.t.values() if e is map_model.DELETED),
        "ties to the earlier group": sum(1 for x in pl if x.ctg and x.tie),
        "later group with one more hit": sum(1 for x in pl if x.ctg and len(x.groups) > 1 and x.groups[-1][1] == max(f for _, f in x.groups)
                                             and x.groups[-1][1] == x.groups[0][1] + 1),
        "reads with only deleted hits": sum(1 for x in pl if x.deleted and not x.groups),
        "one-hit groups beside a placement": sum(1 for x in pl if x.ctg and any(f == 1 for _, f in x.groups) and len(x.groups) > 1),
        "footprint reads": sum(x.footprint for x in pl),
        "minus-strand placements": sum(1 for x in pl if x.orien == "-"),
        "negative positions": sum(1 for x in pl if x.ctg and x.pos < 0),
        "kept contigs": len(p["kept"]),
    }


_TABLE_RUNS = [(31, ()), (31, ("-k", "21")), (31, ("-k", "25")), (63, ()), (65, ()), (127, ())]


@_need_ref
@pytest.mark.parametrize("Kg,args", _TABLE_RUNS, ids=[f"K{kg}{''.join(a)}" for kg, a in _TABLE_RUNS])
def test_table_model_matches_reference(tmp_path, Kg, args):
    """The designed contig set: the model's table and placements against the reference `map`, read by read; every rule the set is
    there for fires"""
    contig, index, pairs, L = md.table_set(Kg)
    k = int(args[1]) if args else Kg
    p = md.predict(contig, index, pairs, k)
    g, cfg = md.write_graph(str(tmp_path), "t", contig, index, Kg, pairs, L)
    ref = util.REF127 if Kg > 63 else util.REF63
    err = util.run([ref, "map", "-s", cfg, "-g", g, "-p", "4", *args], timeout=300)
    assert md.ref_stats(err) == (p["stats"], p["table"].distinct(), p["kmers"])
    on = _ref_on(g)
    for i, (a, b) in enumerate(zip(on, p["on"])):
        assert a == b, f"line {i}: reference {a!r}, model {b!r}; read {b.split()[0]}: {p['placements'][int(b.split()[0]) - 1]}"
    assert len(on) == len(p["on"])
    assert map_model.read_gap_heads(gzip.open(g + ".readInGap.gz").read()) == p["gap"]
    rules = _rules(p, k)
    print(f"K {Kg} {' '.join(args)}: {rules}")
    must = ["keys seen 3+ times", "deleted keys", "ties to the earlier group", "later group with one more hit", "reads with only deleted hits",
            "footprint reads", "minus-strand placements", "negative positions", "kept contigs"]
    if k < 32:
        must.append("one-hit groups beside a placement")
    assert all(rules[r] > 0 for r in must), rules
    # the cutoff: contigs of K + 1 bases are dropped, of K + 2 kept with 2 k-mers
    lens = [len(c) for _, c in p["kept"]]
    assert k + 1 not in lens and k + 2 in lens
