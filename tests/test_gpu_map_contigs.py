"""The GPU `map` stage against the reference `map` on designed inputs (tests/map_designs.py): the `.contig` shapes the reference's
`contig` never writes, and the contig set whose k-mers repeat on purpose, with reads on its ties, deleted keys and one-hit groups.
Every output byte and the stderr lines (without the time lines) must match; the host side of each case is pinned on the CPU by
test_map_contigs_host.py.  When `.readOnContig.gz` differs, the message names the first differing reads with the model's account
of each (tests/map_model.py): its groups in first-hit order and its hits on deleted keys."""
import filecmp
import gzip
import os
import random
import shutil

import pytest

from soapdenovo2_b200 import api
from tests import map_designs as md
from tests import util
from tests.test_gpu_map import FILL_OUT, MAP_OUT, _stderr_lines

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not util.have_ref(), reason="oracle/_ref reference binaries not built")]


def _copy(g, name):
    out = os.path.join(os.path.dirname(g), name)
    for s in ("contig", "ContigIndex", "preGraphBasic"):
        shutil.copy(f"{g}.{s}", f"{out}.{s}")
    return out


def _explain(ref, gpu, model):
    a = gzip.open(ref + ".readOnContig.gz", "rt").read().splitlines()
    b = gzip.open(gpu + ".readOnContig.gz", "rt").read().splitlines()
    out = []
    for x, y in zip(a, b):
        if x != y and len(out) < 5:
            rd = int(x.split("\t")[0]) - 1
            out.append(f"reference {x!r}, GPU {y!r}; model for read {rd + 1}: {model['placements'][rd]}")
    if len(a) != len(b):
        out.append(f"{len(a)} lines from the reference, {len(b)} from the GPU")
    return "\n".join(out)


def _map_both(g, cfg, args, model=None, flavour127=False, tag="", long=False):
    ref_bin, gpu_bin = (util.REF127, api.BIN127) if flavour127 else (util.REF63, api.BIN63)
    ref, gpu = _copy(g, "ref" + tag), _copy(g, "gpu" + tag)
    e_ref = util.run([ref_bin, "map", "-s", cfg, "-g", ref, *args])
    e_gpu = util.run([gpu_bin, "map", "-s", cfg, "-g", gpu, *args])
    suffixes = MAP_OUT + (FILL_OUT if "-f" in args else []) + (["longReadInGap"] + (["RlongReadInGap"] if "-f" in args else []) if long else [])
    bad = [s for s in suffixes if not filecmp.cmp(f"{ref}.{s}", f"{gpu}.{s}", shallow=False)]
    assert not bad, f"map outputs differ: {bad}\n" + (_explain(ref, gpu, model) if model and "readOnContig.gz" in bad else "")
    assert _stderr_lines(e_gpu.replace(gpu, ref)) == _stderr_lines(e_ref)
    return ref, e_ref


_SHAPES = md.reader_cases(31)


@pytest.mark.parametrize("name,text", _SHAPES, ids=[c[0] for c in _SHAPES])
def test_map_contig_shapes(tmp_path, name, text):
    """Each .contig shape at K 31, with read pairs drawn from its kept contigs"""
    d = str(tmp_path)
    p = md.predict(text, "Edge_num 0 0\n", [], 31)
    index = md.contig_index(p["kept"], 31, n_min=text.count(b">") + 1)
    pairs = md.sample_pairs(random.Random(len(text)), p["kept"], 100) or [("A" * 100, "C" * 100)]
    g, cfg = md.write_graph(d, "s", text, index, 31, pairs, 100)
    _map_both(g, cfg, ["-p", "4", "-f"], model=md.predict(text, index, pairs, 31))


_RUNS = [(31, (), False), (31, ("-k", "21"), False), (31, ("-k", "25"), False), (63, (), False), (65, (), True), (127, (), True)]


@pytest.mark.parametrize("Kg,args,flavour127", _RUNS, ids=[f"K{kg}{''.join(a)}" for kg, a, _ in _RUNS])
def test_map_designed_table(tmp_path, Kg, args, flavour127):
    """The designed contig set on the 63-mer binary at K 31 and 63 and at -k 21 and 25, and on the 127-mer binary at K 65 and 127
    (map_lookup's widest key); with -f"""
    contig, index, pairs, L = md.table_set(Kg)
    g, cfg = md.write_graph(str(tmp_path), "t", contig, index, Kg, pairs, L)
    model = md.predict(contig, index, pairs, int(args[1]) if args else Kg)
    _map_both(g, cfg, ["-p", "8", "-f", *args], model=model, flavour127=flavour127)


_VARIANTS = {
    "map_long_all": ({"PGB200_MAP_LONG": "all"}, ["-p", "8"], False),
    "map_groups_1": ({"PGB200_MAP_GROUPS": "1", "PGB200_MAP_LONG": "all"}, ["-p", "8"], False),
    "reader_fgets": ({"PGB200_MAP_READER": "fgets"}, ["-p", "8"], False),
    "p1": ({}, ["-p", "1"], False),
    "p8_k21": ({}, ["-p", "8", "-k", "21"], False),
    "long_library": ({}, ["-p", "8", "-f"], True),
    "long_library_k21": ({}, ["-p", "3", "-k", "21"], True),
}


@pytest.mark.parametrize("variant", list(_VARIANTS))
def test_map_designed_table_variants(tmp_path, monkeypatch, variant):
    """The K 31 set through k_map_long for the short pass, with one group slot (every read takes the overflow rounds), through the
    fgets reader, at -p 1 and -p 8, and with an asm_flags=4 library whose reads (two mates joined, wrapped at 70) meet deleted keys
    and ties in .longReadInGap"""
    env, args, long = _VARIANTS[variant]
    for k, v in env.items():   # read by the GPU stage only
        monkeypatch.setenv(k, v)
    contig, index, pairs, L = md.table_set(31)
    g, cfg = md.write_graph(str(tmp_path), "t", contig, index, 31, pairs, L, long_reads=long)
    model = md.predict(contig, index, pairs, int(args[args.index("-k") + 1]) if "-k" in args else 31)
    _, err = _map_both(g, cfg, args, model=model, long=long)
    if long:
        assert "reads in gaps." in err
