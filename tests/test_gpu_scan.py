"""device_scan (scan.cuh) against closed forms on the GPU: tests/gpu_scan.cu scans inputs computed from the index alone (all ones,
i % 7, all zeros, a hashed sparse pattern) and checks every prefix, the value passed with it, the number of visits and the device total,
at sizes around one tile, around the largest single-level input (4096 x 262144 elements: beyond it the tile sums take a second scan
level, which the layout reaches with a large enough -a) and past 2^32 elements; through device_scan and through the split
device_scan_total + device_scan_finish.  The scratch buffer is exactly scan_scratch_elems(n) long and followed by a canary region."""
import os
import subprocess

import pytest

from tests import util

pytestmark = pytest.mark.gpu

ONE_LEVEL = 4096 * 262144
SIZES = [0, 1, 15, 16, 17, 4095, 4096, 4097, ONE_LEVEL - 1, ONE_LEVEL, ONE_LEVEL + 1, 2**32 - 1, 2**32 + 4097]


@pytest.fixture(scope="module")
def scans(tmp_path_factory):
    d = tmp_path_factory.mktemp("scan")
    exe = str(d / "gpu_scan")
    c = subprocess.run([util.NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                        os.path.join(util.ROOT, "tests", "gpu_scan.cu")], capture_output=True, text=True)
    assert c.returncode == 0, c.stdout[-2000:] + c.stderr[-4000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    rows = {}
    for line in r.stdout.splitlines():
        _, name, entry, n, tiles, bad, first, visits, total, want, canary = line.split()
        rows[(name, entry, int(n))] = dict(tiles=int(tiles), bad=int(bad), first=int(first), visits=int(visits), total=int(total),
                                           want=int(want), canary=canary == "1")
    return rows


def test_scan_covers_both_levels(scans):
    tiles = {n: scans[("ones", "whole", n)]["tiles"] for n in SIZES}
    print("\n".join(f"n = {n}: {t} tiles, {'two levels' if t > 262144 else 'one level'}" for n, t in tiles.items()))
    assert tiles[ONE_LEVEL] == 262144 and tiles[ONE_LEVEL + 1] == 262145
    assert len(scans) == 4 * 2 * len(SIZES)


@pytest.mark.parametrize("entry", ["whole", "split"])
@pytest.mark.parametrize("name", ["ones", "mod7", "zeros", "sparse"])
def test_scan_against_closed_form(scans, name, entry):
    for n in SIZES:
        s = scans[(name, entry, n)]
        where = f"{name} {entry} n={n} ({s['tiles']} tiles)"
        assert s["bad"] == 0, f"{where}: {s['bad']} wrong prefixes, first at index {s['first']}"
        assert s["visits"] == n, f"{where}: the output functor ran {s['visits']} times"
        assert s["total"] == s["want"], f"{where}: total {s['total']}, want {s['want']}"
        assert s["canary"], f"{where}: the scan wrote past scan_scratch_elems(n)"
    if name == "ones":
        assert scans[(name, entry, 2**32 + 4097)]["total"] == 2**32 + 4097   # prefixes past 32 bits
