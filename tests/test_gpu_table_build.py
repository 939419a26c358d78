"""GPU parity of the pass-1 table build, under both PGB200_TABLE_BUILD values: `region` (the pass's first aggregation launch stores its
aggregates into bins and k_table_build makes the table region by region, no table clear) and `merge` (every launch merges into a cleared
table with the CAS protocol).  Every case checks the C model's table dump and .kmerFreq, and in region mode that the branch it is about
ran, from the engine's PGB200_VERBOSE line ("region build: ... bin overflow B, carries C, remnant list N of CAP").  Tiny regions
(PGB200_TABLE_REGION) make carries and bin overflow common (the first launch of a test-sized pass defers most buckets, so its bins are sparse); a tiny remnant list (PGB200_TABLE_REMNANT_CAP) makes the launch run again in
merge mode."""
import os
import re

import pytest
import torch

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = pytest.mark.gpu

BUILDS = ["region", "merge"]
REGION_LINE = re.compile(r"region build: (\d+) regions of (\d+) slots, bin overflow (\d+), carries (\d+), remnant list (\d+) of (\d+)(.*)")


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def _region_stats(err):
    """(bin overflow, carries, ran again in merge mode) of every region build the engine reported"""
    return [(int(m.group(3)), int(m.group(4)), "merge mode" in m.group(7)) for m in REGION_LINE.finditer(err)]


def _model(tmp_path, K, D=0):
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    extra = ("-1", "-T", dump, "-a", "1") + (("-d", str(D)) if D else ())
    util.run_model(util.MODEL127 if K > 63 else util.MODEL63, cfg, mod, K, 4, extra)
    return mod, dump


def _pass(eng, tmp_path, chunk=0):
    for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
        data = open(tmp_path / fn, "rb").read()
        if not chunk:
            eng.feed_text(data, fastq=True, ord_base=mate, ord_stride=2)
            continue
        lines = data.split(b"\n")[:-1]
        recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines), 4)]
        for i in range(0, len(recs), chunk):
            eng.feed_text(b"".join(recs[i:i + chunk]), fastq=True, ord_base=2 * i + mate, ord_stride=2)
    return eng.finish_pass1()


def _check(eng, mod, dump):
    hist, lin, rem = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    assert (hist, lin, rem) == eng.sweeps()
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("K,D,region", [(31, 0, "0"), (63, 0, "0"), (127, 0, "0"), (63, 1, "0"), (31, 2, "8"), (63, 0, "8"), (127, 1, "8")])
def test_table_build(tmp_path, monkeypatch, capfd, build, K, D, region):
    """One launch per pass at K = 31, 63, 127, with and without -d; regions of 8 slots make carries (keys whose probe runs off
    their region's end, merged after the build and swept from the spill list)."""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_TABLE_BUILD", build)
    if region != "0":
        monkeypatch.setenv("PGB200_TABLE_REGION", region)
    mod, dump = _model(tmp_path, K, D)
    eng = api.PregraphEngine(K=K, P=4, initG=1, D=D, flavour127=int(K > 63), max_rd_len=150, table_slots=1 << 20, verbose=1)
    _pass(eng, tmp_path)
    _check(eng, mod, dump)
    eng.close()
    stats = _region_stats(capfd.readouterr().err)
    if build == "merge":
        assert stats == []
    else:
        assert len(stats) == 1 and not stats[0][2]
        if region != "0":
            assert stats[0][1] > 0


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("K,D", [(63, 0), (127, 1)])
def test_bin_overflow(tmp_path, monkeypatch, capfd, build, K, D):
    """Regions of 1 slot: every bin that receives a second entry overflows into the remnant list; the build then
    sweeps nothing (a key may have partials on the list) and k_sweep sweeps the whole table."""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_TABLE_BUILD", build)
    monkeypatch.setenv("PGB200_TABLE_REGION", "1")
    mod, dump = _model(tmp_path, K, D)
    eng = api.PregraphEngine(K=K, P=4, initG=1, D=D, flavour127=int(K > 63), max_rd_len=150, table_slots=1 << 23, verbose=1)
    _pass(eng, tmp_path)
    _check(eng, mod, dump)
    eng.close()
    stats = _region_stats(capfd.readouterr().err)
    if build == "region":
        assert len(stats) == 1 and stats[0][0] > 0 and not stats[0][2]   # (a 1-slot bin's entry always claims its slot: no carries)


@pytest.mark.parametrize("K", [31, 127])
def test_remnant_list_full(tmp_path, monkeypatch, capfd, K):
    """A remnant list too short for the bin overflow and carries: the launch runs again in merge mode, with the same result."""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_TABLE_REGION", "1")
    monkeypatch.setenv("PGB200_TABLE_REMNANT_CAP", "64")
    mod, dump = _model(tmp_path, K)
    eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=int(K > 63), max_rd_len=150, table_slots=1 << 23, verbose=1)
    _pass(eng, tmp_path)
    _check(eng, mod, dump)
    eng.close()
    stats = _region_stats(capfd.readouterr().err)
    assert len(stats) == 1 and stats[0][2]


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("K,D,buckets,slots", [(63, 0, "2", 1 << 17), (127, 1, "3", 1 << 17), (63, 0, "3", 2048), (127, 0, "4096", 2048)])
def test_spills_and_deferred_buckets(tmp_path, monkeypatch, capfd, build, K, D, buckets, slots):
    """2-3 buckets: almost every k-mer spills past the shared-memory table, so its partials reach the bins both from the spills and
    from the flush of the keys the shared-memory table did hold.  A table of 2048 slots: buckets are deferred, the built table grows,
    the deferred buckets merge into it."""
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_TABLE_BUILD", build)
    monkeypatch.setenv("PGB200_SKM_BUCKETS", buckets)
    mod, dump = _model(tmp_path, K, D)
    eng = api.PregraphEngine(K=K, P=4, initG=1, D=D, flavour127=int(K > 63), max_rd_len=150, table_slots=slots, verbose=1)
    st = _pass(eng, tmp_path)
    if slots == 2048:
        assert st.table_slots > 2048
    _check(eng, mod, dump)
    eng.close()
    err = capfd.readouterr().err
    assert len(_region_stats(err)) == (1 if build == "region" else 0)
    if slots == 2048:
        assert "growing k-mer table" in err


@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("skm", ["0", "1"])
def test_second_pass_on_dirty_table(tmp_path, monkeypatch, capfd, build, skm):
    """Two passes in one engine: reset_pass1 no longer clears the table.  The second pass finds the first one's table: the per-instance
    inserts (host text, PGB200_SKM=0) clear it before their first write, the region build overwrites every slot; a mid-stream
    launch after the build merges into the built table."""
    monkeypatch.setenv("PGB200_SKM", skm)
    monkeypatch.setenv("PGB200_TABLE_BUILD", build)
    mod, dump = _model(tmp_path, 63)
    eng = api.PregraphEngine(K=63, P=4, initG=1, max_rd_len=150, table_slots=1 << 17, verbose=1)
    other = tmp_path / "other"
    other.mkdir()
    synth.scenario_pe_fastq(str(other), seed=7)   # other reads: keys of the first pass must not survive into the second
    _pass(eng, other)
    eng.sweeps()
    eng.reset_pass1()
    if skm == "1":
        monkeypatch.setenv("PGB200_SKM_FLUSH_EVERY", "3")
    _pass(eng, tmp_path, chunk=1000 if skm == "1" else 0)
    _check(eng, mod, dump)
    eng.close()
    stats = _region_stats(capfd.readouterr().err)
    assert len(stats) == (2 if build == "region" and skm == "1" else 0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("build", BUILDS)
def test_two_gpus(tmp_path, monkeypatch, build):
    """Two engines, one process: each GPU builds the table of the buckets it owns."""
    monkeypatch.setenv("PGB200_TABLE_BUILD", build)
    mod, dump = _model(tmp_path, 63)
    engs = [api.PregraphEngine(K=63, P=4, initG=1, max_rd_len=150, device=r, world=2, rank=r) for r in range(2)]
    for e in engs:
        e.xchg_setup(1 << 20)
    for r, e in enumerate(engs):
        e.xchg_import_ptr(1 - r, 1 - r, engs[1 - r].xchg_base())
    for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
        engs[mate].feed_text(open(tmp_path / fn, "rb").read(), fastq=True, ord_base=mate, ord_stride=2)
    for e in engs:
        e.xchg_fence()
    for e in engs:
        e.flush()
        e.finish_pass1()
    engs[0].absorb(engs[1])
    _check(engs[0], mod, dump)
    for e in engs:
        e.close()
