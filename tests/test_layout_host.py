"""The reference's table layout on designed set histories (tests/layout_designs.py), CPU only.

1. Every design reaches the branch it is about, by the Python model of put_kmerset / encap_kmerset: a set that ends exactly at its growth
   threshold grows once more or not as the design says, and flipping that one decision changes the key order (a design that the old
   "always grow at the end" rule, or its opposite, would pass proves nothing); the chain designs grow one set several times through long
   displacement chains; the -a 1 designs wrap their probe chains past slot 0.
2. The Python model's key order equals the key column of the C model's -T dump.
3. The C model writes the reference's files.  Where oracle/_ref was built the reference binary is run; otherwise the stored digests
   (tests/golden/layout_ref.json) are used.
PGB200_WRITE_LAYOUT_REF=<file>: write the reference binary's digests of every scenario to <file> (needs oracle/_ref)."""
import json
import os

import pytest

from tests import layout_designs as D
from tests import util

GOLD_PATH = os.path.join(util.ROOT, "tests", "golden", "layout_ref.json")


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def options(name):
    return D.SCENARIOS[name][4]


def initG(name):
    extra = options(name)
    return int(extra[extra.index("-a") + 1]) if "-a" in extra else 0


def suffixes(name):
    return util.SUFFIXES_R if "-R" in options(name) else util.SUFFIXES


def run_model(name, reads, rule="reference"):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    return D.model(reads, K, P, f127, initG(name), rule)


@pytest.mark.parametrize("name", list(D.SCENARIOS))
def test_design_reaches_its_branch(name):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    reads, paired, last = D.stream(name)
    sets, order = run_model(name, reads)
    s0 = sets[0]
    if fam == "threshold":
        target = args[0]
        assert s0.count == target and D.set_of(last, P, f127) == 0
        # the last key is set 0's last new key: no key of set 0 is first seen after it
        keys = [k for r in reads for k in D.chop(r, K) if D.set_of(k, P, f127) == 0]
        assert keys.index(last) == max(keys.index(k) for k in set(keys))
        if expect is None:   # contrast: one below or one above the threshold, so neither counterfactual rule applies
            assert s0.count != D.threshold(s0.size)
            assert run_model(name, reads, "always")[1] == order
            return
        grown = D.threshold(s0.size) > s0.count
        assert grown == expect
        # the growth would have happened at the first instance after the last key: the size before it has the count as threshold
        sizes = D.dynamic_sizes(6)
        assert (sizes[s0.growths - 1] if grown else sizes[s0.growths])[1] == target
        flipped = run_model(name, reads, "never" if expect else "always")[1]
        assert flipped != order, "the design does not tell the two growth rules apart"
        if args[1] == "rc":
            assert all(D.value(r[j:j + K]) != last for r in reads for j in range(len(r) - K + 1) if len(r) > K)
        if args[1] == "short":
            assert D.bases(last, K) in reads and len(reads[-1]) == K
        if args[1].startswith("pair"):
            # the last key ends mate 1 of the last pair (an even ordinal), as a forward or a reverse-complement instance
            assert paired and len(reads) % 2 == 0 and last in (D.value(reads[-2][-K:]), D.revcomp(D.value(reads[-2][-K:]), K))
    elif fam == "chains":
        assert s0.growths >= 3 and s0.max_chain >= 10 and s0.max_probe >= 1000
        assert run_model(name, reads, "always")[1] == order   # no set ends at its threshold
    else:
        size = D.static_size(initG(name), P, f127)
        assert s0.size == size and s0.growths == 0
        assert s0.wraps >= 1000 and s0.max_probe >= 2000
        assert any(k % size >= size - 4 and i < 1000 for i, k in s0.slot.items())   # keys homed at the end sit past slot 0
        if K > 63:
            assert any(k >> 128 for k in order)   # the upper words are in use


@pytest.mark.parametrize("name", list(D.SCENARIOS))
def test_python_model_equals_c_model(tmp_path, name):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    d = str(tmp_path)
    cfg, reads = D.write_scenario(d, name)
    dump = os.path.join(d, "mod.T")
    util.run_model(util.MODEL127 if f127 else util.MODEL63, cfg, os.path.join(d, "mod"), K, P, ("-1", "-T", dump, *extra))
    assert D.dump_keys(open(dump, "rb").read(), f127) == run_model(name, reads)[1]


_written = {}


def reference_digests(name, cfg, d):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    if util.have_ref():
        ref = os.path.join(d, "ref")
        util.run_ref(util.REF127 if f127 else util.REF63, cfg, ref, K, P, extra)
        got = util.digests(ref, suffixes(name))
        if os.environ.get("PGB200_WRITE_LAYOUT_REF"):
            _written[name] = got
            json.dump(_written, open(os.environ["PGB200_WRITE_LAYOUT_REF"], "w"), indent=1, sort_keys=True)
        return got
    return json.load(open(GOLD_PATH))[name]


@pytest.mark.parametrize("name", list(D.SCENARIOS))
def test_c_model_matches_reference(tmp_path, name):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    d = str(tmp_path)
    cfg, _ = D.write_scenario(d, name)
    mod = os.path.join(d, "mod")
    util.run_model(util.MODEL127 if f127 else util.MODEL63, cfg, mod, K, P, extra)
    assert util.digests(mod, suffixes(name)) == reference_digests(name, cfg, d)
