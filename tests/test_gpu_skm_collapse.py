"""GPU parity, pass 1, on reads made of exact copies: every super-k-mer record of the aggregated pass 1 occurs tens to hundreds of
times in its bucket, so the aggregation collapses them into distinct records with counts (skm_apply.cu, k_skm_apply) and applies each k-mer
once per distinct record, weighted by its count.  Counts past 255 saturate the coverage and past 63 the links.  The .kmerFreq and
the full node table dump must equal the C model's, with the default bucket count and with ONE bucket (the distinct-record buffer
drains many times per window and every k-mer past the shared-memory table goes to the global table with its weight)."""
import os
import subprocess

import numpy as np
import pytest

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


def _scenario(d):
    """Error-free pairs at every position of a 4 kbp genome (tiled_pairs, step 1), plus 8 reads repeated 300 times each, on both
    strands: records repeat from a few times up to several hundred times."""
    g = synth.genome(4000, 17)
    r1, r2 = synth.tiled_pairs(g, 1, 100, 240)
    rng = np.random.default_rng(18)
    starts = rng.integers(0, len(g) - 100, 8)
    rep = np.repeat(np.stack([g[s:s + 100] for s in starts]), 300, axis=0)
    r1 = np.concatenate([r1, rep])
    r2 = np.concatenate([r2, synth._revcomp(rep)])
    synth.write_fastq(os.path.join(d, "c_1.fq"), r1, "c")
    synth.write_fastq(os.path.join(d, "c_2.fq"), r2, "c")
    cfg = os.path.join(d, "c.cfg")
    synth.write_config(cfg, 100, [{"avg_ins": 240, "files": [("q1", os.path.join(d, "c_1.fq")), ("q2", os.path.join(d, "c_2.fq"))]}])
    return cfg


@pytest.mark.parametrize("skm", ["1", "0"])
@pytest.mark.parametrize("buckets", ["0", "1"])
@pytest.mark.parametrize("K,flav", [(31, 0), (63, 0), (65, 1), (99, 1)])
def test_repeated_records_table_dump(tmp_path, monkeypatch, K, flav, buckets, skm):
    if skm == "0" and buckets != "0":
        pytest.skip("buckets only exist on the aggregated path")
    monkeypatch.setenv("PGB200_SKM", skm)
    if buckets != "0":
        monkeypatch.setenv("PGB200_SKM_BUCKETS", buckets)
    cfg = _scenario(str(tmp_path))
    mod, dump = str(tmp_path / "mod"), str(tmp_path / "mod.table")
    util.run_model(util.MODEL127 if flav else util.MODEL63, cfg, mod, K, 4, ("-1", "-T", dump, "-a", "1"))
    eng = api.PregraphEngine(K=K, P=4, initG=1, flavour127=flav, max_rd_len=100)
    for mate, fn in enumerate(("c_1.fq", "c_2.fq")):
        eng.feed_text(open(tmp_path / fn, "rb").read(), fastq=True, ord_base=mate, ord_stride=2)
    eng.finish_pass1()
    hist, _, _ = eng.sweeps()
    assert api.kmerfreq_text(hist) == open(mod + ".kmerFreq", "rb").read()
    assert hist[255] > 0   # coverage saturates
    eng.build_layout()
    assert eng.dump_nodes() == open(dump, "rb").read()
    eng.close()


@pytest.mark.parametrize("buckets", ["0", "1"])
def test_repeated_records_cli_vs_reference(tmp_path, buckets):
    """The CLI's pregraph files on the same reads, aggregated pass 1, against the reference (or the C model where it is not shipped)."""
    cfg = _scenario(str(tmp_path))
    want = str(tmp_path / "want")
    if util.have_ref():
        util.run_ref(util.REF63, cfg, want, 63, 4, ("-a", "1"))
    else:
        util.run_model(util.MODEL63, cfg, want, 63, 4, ("-a", "1"))
    env = dict(os.environ, PGB200_SKM="1")
    if buckets != "0":
        env["PGB200_SKM_BUCKETS"] = buckets
    gpu = str(tmp_path / "gpu")
    r = subprocess.run([api.BIN63, "pregraph", "-s", cfg, "-K", "63", "-p", "4", "-a", "1", "-o", gpu], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    util.compare(want, gpu, util.SUFFIXES)
