"""GPU parity of the window-staged aggregation kernel (k_skm_apply): table dump and .kmerFreq equal the oracle's when every bucket
spans many staging windows (1 or 3 buckets for the whole read set) and when a launch reads many segments, most of whose ranges
are empty for a given bucket (small chunks: over 100 segments per mate), at K = 31, 63 and 127."""
import os

import pytest

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


@pytest.mark.parametrize("K,flav,buckets,chunk", [(63, 0, "1", 700), (31, 0, "3", 700), (127, 1, "3", 700),
                                                   (31, 0, "0", 50), (63, 0, "0", 50), (127, 1, "0", 50)])
def test_staged_windows_and_many_segments(tmp_path, monkeypatch, K, flav, buckets, chunk):
    if os.environ.get("PGB200_SKM") == "0":
        pytest.skip("aggregated path only")
    monkeypatch.setenv("PGB200_SKM", "1")
    if buckets != "0":
        monkeypatch.setenv("PGB200_SKM_BUCKETS", buckets)
    cfg = synth.scenario_pe_fastq(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL127 if flav else util.MODEL63, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=flav, max_rd_len=150)
    n_chunks = 0
    for mate, fn in enumerate(("pe_1.fq", "pe_2.fq")):
        lines = open(tmp_path / fn, "rb").read().split(b"\n")[:-1]
        recs = [b"\n".join(lines[i:i + 4]) + b"\n" for i in range(0, len(lines), 4)]
        for i in range(0, len(recs), chunk):
            eng.feed_text(b"".join(recs[i:i + chunk]), fastq=True, ord_base=2 * i + mate, ord_stride=2)
            n_chunks += 1
    assert n_chunks > 100 or chunk > 100
    eng.finish_pass1()
    hist, _, _ = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()
    eng.close()
