"""GPU table layout on the designed set histories of tests/layout_designs.py.

  - per node: finish_pass1 -> sweeps -> build_layout -> dump_nodes equals the C model's -T dump byte for byte, with both pass-1 insert
    paths (PGB200_SKM=0 / 1: the first-occurrence rank the layout reads comes from either), and once through the CLI-sized settings
    that make the GPU table grow and split the reads into chunks;
  - CLI: all files of every scenario against the reference (or its stored digests);
  - the verbose layout line shows that the threshold decision ran and what it decided."""
import json
import os
import re

import pytest

from soapdenovo2_b200 import api
from tests import layout_designs as D
from tests import util
from tests.test_gpu_full import _engine
from tests.test_layout_host import GOLD_PATH, initG, suffixes

pytestmark = pytest.mark.gpu

LATE_RE = re.compile(r"layout: (\d+) set\(s\) end at a growth threshold, (\d+) grow at a later instance, (\d+) read\(s\) scanned")


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def late_line(log):
    m = LATE_RE.findall(log)
    assert len(m) == 1, log[-3000:]
    return tuple(map(int, m[0]))


def engine_dump(name, cfg, capfd):
    """the table in iteration order through the C-ABI (files fed as the stage feeds them: mates interleave as 2*pair + mate)"""
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    mrl, plan = api.plan_files(cfg)
    D_ = int(extra[extra.index("-d") + 1]) if "-d" in extra else 0
    eng = api.PregraphEngine(K=K, P=P, initG=initG(name), D=D_, flavour127=int(f127), max_rd_len=mrl, verbose=1)
    n, i = 0, 0
    while i < len(plan):
        mate, fq, rev, cut, path = plan[i]
        if mate == 0:
            n1 = eng.feed_text(open(path, "rb").read(), fastq=bool(fq), ord_base=n, ord_stride=2, reverse_seq=rev, maxlen=cut)
            mate, fq, rev, cut, path = plan[i + 1]
            eng.feed_text(open(path, "rb").read(), fastq=bool(fq), ord_base=n + 1, ord_stride=2, reverse_seq=rev, maxlen=cut)
            n, i = n + 2 * n1, i + 2
        else:
            n, i = n + eng.feed_text(open(path, "rb").read(), fastq=bool(fq), ord_base=n, reverse_seq=rev, maxlen=cut), i + 1
    capfd.readouterr()
    eng.finish_pass1(); eng.sweeps(); eng.build_layout()
    dump = eng.dump_nodes()
    eng.close()
    return dump, capfd.readouterr().err


def model_dump(name, cfg, d):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    dump = os.path.join(d, "mod.T")
    util.run_model(util.MODEL127 if f127 else util.MODEL63, cfg, os.path.join(d, "mod"), K, P, ("-1", "-T", dump, *extra))
    return open(dump, "rb").read()


def check_late(name, log, reads):
    """the verbose layout line against the Python model: the sets that end at a growth threshold, and those a later instance grows"""
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    if initG(name):
        assert not LATE_RE.search(log)   # static sets never grow: no decision, no scan
        return
    sets, _ = D.model(reads, K, P, f127)
    thresholds = {t for _, t in D.dynamic_sizes(8)}
    flagged = [s for s in sets if s.count in thresholds]
    grow = [s for s in flagged if D.threshold(s.size) > s.count]
    n_late, n_grow, scanned = late_line(log)
    assert (n_late, n_grow) == (len(flagged), len(grow))
    assert (scanned > 0) == (n_late > 0)
    if fam == "threshold" and expect is not None:
        assert sets[0] in flagged and (sets[0] in grow) == expect


def first_difference(got, want, f127):
    rec = (4 if f127 else 2) * 8 + 10
    if len(got) != len(want):
        return f"{len(got) // rec} nodes, model {len(want) // rec}"
    i = next(i for i in range(0, len(got), rec) if got[i:i + rec] != want[i:i + rec]) // rec
    return f"node {i} (iteration order) differs: engine {got[i * rec:(i + 1) * rec].hex()} model {want[i * rec:(i + 1) * rec].hex()}"


@pytest.mark.parametrize("skm", ["0", "1"])
@pytest.mark.parametrize("name", list(D.SCENARIOS))
def test_nodes_in_reference_order(tmp_path, capfd, monkeypatch, name, skm):
    monkeypatch.setenv("PGB200_SKM", skm)
    d = str(tmp_path)
    cfg, reads = D.write_scenario(d, name)
    want = model_dump(name, cfg, d)
    got, log = engine_dump(name, cfg, capfd)
    assert got == want, first_difference(got, want, D.SCENARIOS[name][3])
    check_late(name, log, reads)


@pytest.mark.parametrize("name", ["last_t3_p1", "other_t3_p8", "pair_early_t1_p3", "pair_late_t1_p3", "chains_k63_p3", "wrap_k127_p3"])
def test_cli_small_table_and_chunks(tmp_path, name):
    """PGB200_TABLE_SLOTS=2048: the GPU table grows during pass 1; PGB200_CHUNK_MB=1 with 80000 reads shorter than K+1 in the middle of
    the stream: the design's reads lie in several chunks with ordinals far apart.  Checked against the C model (the short reads shift
    the read ids of the -R outputs, so the stored reference digests do not apply)."""
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    d = str(tmp_path)
    cfg, reads = D.write_scenario(d, name, pad=80000)
    assert os.path.getsize(cfg.replace("lib.cfg", "r1.fa" if "pair" in name else "r.fa")) > (1 << 20)
    gpu, mod = os.path.join(d, "gpu"), os.path.join(d, "mod")
    log = _engine(int(f127), cfg, gpu, K, P, extra, env={"PGB200_VERBOSE": "1", "PGB200_TABLE_SLOTS": "2048", "PGB200_CHUNK_MB": "1"})
    assert "growing k-mer table" in log
    util.run_model(util.MODEL127 if f127 else util.MODEL63, cfg, mod, K, P, extra)
    util.compare(mod, gpu, suffixes(name))
    check_late(name, log, reads)


@pytest.mark.parametrize("name", list(D.SCENARIOS))
def test_cli_on_layout_designs(tmp_path, name):
    fam, K, P, f127, extra, args, expect = D.SCENARIOS[name]
    d = str(tmp_path)
    cfg, reads = D.write_scenario(d, name)
    gpu = os.path.join(d, "gpu")
    log = _engine(int(f127), cfg, gpu, K, P, extra, env={"PGB200_VERBOSE": "1"})
    if util.have_ref():
        ref = os.path.join(d, "ref")
        util.run_ref(util.REF127 if f127 else util.REF63, cfg, ref, K, P, extra)
        util.compare(ref, gpu, suffixes(name))
    assert util.digests(gpu, suffixes(name)) == json.load(open(GOLD_PATH))[name]
    check_late(name, log, reads)
