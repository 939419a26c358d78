"""GPU parity of the pipelined region build (k_table_build) at the shapes its pipeline adds: a CTA takes every gridDim-th region and
double-buffers them, so the grid is run with one region per CTA, with some CTAs taking one more region than others (odd and even
counts side by side), with bins larger than a stage (copied in pieces), and with bins that are sparse or mostly empty (a bin with no
entries arrives on its stage's barrier without a copy).  At the default region size the grid is 4 CTAs per SM at K <= 63 and 2
above, 528 and 264 CTAs on a 132-SM H100.  Each case checks the C model's table dump and .kmerFreq, and from the engine's
PGB200_VERBOSE line the number of regions the build ran over."""
import pytest

from soapdenovo2_b200 import api, synth
from tests import util
from tests.test_gpu_table_build import _check, _pass, _region_stats, REGION_LINE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def _model(tmp_path, K, D):
    # a small read set (about 7e4 distinct 63-mers), so that tables of 2^17 slots hold it
    cfg = synth.scenario_pe_fastq(str(tmp_path), genome_len=20000, n_pairs=600)
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    extra = ("-1", "-T", dump, "-a", "1") + (("-d", str(D)) if D else ())
    util.run_model(util.MODEL127 if K > 63 else util.MODEL63, cfg, mod, K, 4, extra)
    return mod, dump


@pytest.mark.parametrize("K,D,slots,region,regions", [
    (63, 0, 1 << 17, "0", 256),       # fewer regions than CTAs: one region each; bins of about 250 entries, some in two pieces
    (63, 1, 1 << 19, "512", 1024),    # just above the grid: CTAs of 1 and of 2 regions
    (63, 0, 1 << 19, "256", 2048),    # odd and even counts side by side
    (127, 1, 1 << 18, "0", 512),      # 256-bit keys
    (127, 0, 1 << 16, "0", 128),      # bins of about 300 entries, more than a 256-entry stage: copied in two pieces
    (63, 0, 1 << 23, "0", 16384),     # sparse bins: about 4 entries each
    (63, 1, 1 << 23, "16", 524288),   # mostly empty bins, 512-byte regions
    (127, 0, 1 << 23, "8", 1048576),
])
def test_pipeline_shapes(tmp_path, monkeypatch, capfd, K, D, slots, region, regions):
    monkeypatch.setenv("PGB200_SKM", "1")
    monkeypatch.setenv("PGB200_TABLE_BUILD", "region")
    if region != "0":
        monkeypatch.setenv("PGB200_TABLE_REGION", region)
    mod, dump = _model(tmp_path, K, D)
    eng = api.PregraphEngine(K=K, P=4, initG=1, D=D, flavour127=int(K > 63), max_rd_len=150, table_slots=slots, verbose=1)
    _pass(eng, tmp_path)
    _check(eng, mod, dump)
    eng.close()
    err = capfd.readouterr().err
    stats = _region_stats(err)
    assert len(stats) == 1 and not stats[0][2]
    assert int(REGION_LINE.search(err).group(1)) == regions
