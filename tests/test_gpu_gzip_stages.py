"""GPU end to end: `pregraph` (with -R) and `map` (with -f, and a long-read library) write their .gz files with the GPU writer
(PGB200_GZ=gpu, the default) and with zlib (PGB200_GZ=host); both runs must equal the reference's files byte for byte, and the
reference's `contig` and `scaff` must run on the GPU-written files and produce the same results.  Needs oracle/_ref."""
import filecmp
import os
import shutil

import pytest

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")]

GRAPH = ["contig", "ContigIndex", "preGraphBasic", "updated.edge", "Arc", "edge.gz", "preArc", "vertex", "kmerFreq", "markOnEdge", "path"]


def _env(mode):
    return dict(os.environ, PGB200_GZ=mode)


def _run(cmd, mode):
    import subprocess
    r = subprocess.run(cmd, capture_output=True, text=True, env=_env(mode), timeout=900)
    assert r.returncode == 0, f"{' '.join(cmd)} (PGB200_GZ={mode})\n{r.stderr[-3000:]}"
    return r.stderr


def _same(a, b, suffixes):
    bad = [s for s in suffixes if not filecmp.cmp(f"{a}.{s}", f"{b}.{s}", shallow=False)]
    assert not bad, f"files differ: {bad} ({a} vs {b})"


@pytest.mark.parametrize("scenario,K", [("se_fasta", 31), ("pe_fastq", 63), ("multilib", 31)])
def test_pregraph_edge_gz_both_modes(tmp_path, scenario, K):
    d = str(tmp_path)
    cfg = getattr(synth, "scenario_" + scenario)(d)
    ref = os.path.join(d, "ref")
    util.run([util.REF63, "pregraph", "-s", cfg, "-K", str(K), "-p", "4", "-o", ref, "-R"])
    outs = {}
    for mode in ("gpu", "host"):
        out = os.path.join(d, mode)
        _run([api.BIN63, "pregraph", "-s", cfg, "-K", str(K), "-p", "4", "-o", out, "-R"], mode)
        _same(ref, out, util.SUFFIXES_R)
        outs[mode] = out
    # the reference's contig and scaff on the GPU-written .edge.gz
    for p in (ref, outs["gpu"]):
        util.run([util.REF63, "contig", "-g", p, "-R"])
    _same(ref, outs["gpu"], ["contig", "updated.edge", "Arc"])


def _graph_copy(g, name):
    out = os.path.join(os.path.dirname(g), name)
    for s in GRAPH:
        if os.path.exists(f"{g}.{s}"):
            shutil.copy(f"{g}.{s}", f"{out}.{s}")
    return out


@pytest.mark.parametrize("scenario,args", [("pe_fastq", ["-p", "8", "-f"]), ("multilib", ["-p", "3"]), ("long", ["-p", "8", "-f"])])
def test_map_gz_both_modes(tmp_path, scenario, args):
    d = str(tmp_path)
    cfg = getattr(synth, "scenario_" + scenario)(d)
    g = os.path.join(d, "g")
    util.run([util.REF63, "pregraph", "-s", cfg, "-K", "31", "-p", "4", "-o", g, "-R"])
    util.run([util.REF63, "contig", "-g", g, "-R"])
    ref = _graph_copy(g, "ref")
    util.run([util.REF63, "map", "-s", cfg, "-g", ref, *args])
    suffixes = ["readOnContig.gz", "readInGap.gz", "peGrads"] + (["shortreadInGap.gz", "PEreadOnContig.gz"] if "-f" in args else [])
    if os.path.exists(f"{ref}.longReadInGap"):
        suffixes.append("longReadInGap")
    for mode in ("gpu", "host"):
        out = _graph_copy(g, mode)
        _run([api.BIN63, "map", "-s", cfg, "-g", out, *args], mode)
        _same(ref, out, suffixes)
    # the reference's scaff reads the GPU-written map files: the same scaffolds
    util.run([util.REF63, "scaff", "-g", ref])
    util.run([util.REF63, "scaff", "-g", os.path.join(d, "gpu")])
    _same(ref, os.path.join(d, "gpu"), ["scafSeq"])
