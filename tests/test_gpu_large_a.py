"""The layout's scan past one level, through the CLI: with -a the reference sizes its P k-mer sets from the memory the user names, not
from the data (prlHashReads.c:369-390), and the GPU layout scans that whole geometry (layout.cu).  Past 4096 x 262144 slots the scan's
tile sums take a second level (scan.cuh).  A small input is run with -p 8 and -a values picked from the set-size rule on both sides of
that boundary, and all seven pregraph files are compared with the reference's.

The reference allocates about -a GiB of host memory (calloc'd, so mostly untouched); a case is skipped when MemAvailable is below twice
that.  The GPU CLI runs with its default settings, as a user runs it: its k-mer table is sized from -a too, and must leave HBM for the
layout (pass1.cu: create_table_if_needed).  The engine's own count of reference slots and scan tiles (PGB200_VERBOSE) is checked
against the set-size rule, so each case is known to take the scan level it is meant to.
Set PGB200_SKIP_CONFIG_TESTS=1 to skip them."""
import os
import subprocess

import numpy as np
import pytest

from soapdenovo2_b200 import api, synth
from tests import util

pytestmark = pytest.mark.gpu

SCAN_TILE = 4096
ONE_LEVEL_TILES = 4096 * 64   # k_scan_small takes at most this many tile sums
P = 8


@pytest.fixture(autouse=True)
def _need():
    if os.environ.get("PGB200_SKIP_CONFIG_TESTS"):
        pytest.skip("PGB200_SKIP_CONFIG_TESTS set")
    if not util.have_ref():
        pytest.skip("oracle/_ref not shipped")


# ---- the reference's set geometry (newhash.c:142-233, prlHashReads.c:369-390), restated as engine_impl.cuh does
def _is_prime(n):
    if n < 4:
        return True
    if n % 2 == 0:
        return False
    mx = int(np.sqrt(np.float32(n)))   # float sqrt, strict '<'
    return all(n % i for i in range(3, mx, 2))


def _next_prime(n):
    if n % 2 == 0:
        n += 1
    while not _is_prime(n):
        n += 2
    return n


def set_size(a, p, f127):
    want = int(a * 1024.0 ** 3 / p / (40 if f127 else 24))
    k = max(1, -(-want // 0xFFFFFF))
    return max(3, _next_prime(k * 0xFFFFFF))


def tiles(a, f127):
    return -(-P * set_size(a, P, f127) // SCAN_TILE)


def _pick(f127):
    """(largest -a whose layout scan has one level, smallest -a that needs two)"""
    one = max(a for a in range(1, 64) if tiles(a, f127) <= ONE_LEVEL_TILES)
    two = min(a for a in range(1, 64) if tiles(a, f127) > ONE_LEVEL_TILES)
    return one, two


# 63-mer build: -a 20 is the largest one-level value at -p 8, -a 21 the smallest two-level one (262 145 tiles); 127-mer build: -a 35
CASES = [(91, 35, True), (63, 20, False), (63, 21, False), (63, 32, False)]   # the largest allocation first


def test_set_size_restatement():
    """the restatement gives the known answer of the engine's own ref_static_set_size (tests/host_kat.cu), and CASES sit where
    the set-size rule puts the scan's level boundary"""
    assert set_size(1, 3, False) == 16777259
    assert _pick(False) == (20, 21) and _pick(True) == (34, 35)


def _mem_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


@pytest.mark.parametrize("K,a,f127", CASES, ids=[f"K{K}-a{a}" for K, a, _ in CASES])
def test_layout_scan_levels_match_reference(tmp_path, K, a, f127):
    size = set_size(a, P, f127)
    total = P * size
    t = -(-total // SCAN_TILE)
    print(f"\n-p {P} -a {a} ({'127' if f127 else '63'}-mer build): {P} sets of {size} slots = {total} slots, {t} tiles, "
          f"{'two scan levels' if t > ONE_LEVEL_TILES else 'one scan level'}")
    ref_bytes = total * (40 if f127 else 24) + P * ((size + 15) // 16 * 4)
    if _mem_available() < 2 * ref_bytes:
        pytest.skip(f"MemAvailable {_mem_available() >> 30} GiB < twice the {ref_bytes >> 30} GiB the reference allocates at -a {a}")
    cfg = synth.scenario_se_fasta(str(tmp_path))
    ref, gpu = str(tmp_path / "ref"), str(tmp_path / "gpu")
    args = ["-s", cfg, "-K", str(K), "-p", str(P), "-a", str(a), "-R"]
    util.run([util.REF127 if f127 else util.REF63, "pregraph", *args, "-o", ref], timeout=1800)
    env = {k: v for k, v in os.environ.items() if k != "PGB200_TABLE_SLOTS"}
    r = subprocess.run([api.BIN127 if f127 else api.BIN63, "pregraph", *args, "-o", gpu], capture_output=True, text=True, timeout=1800,
                       env=dict(env, PGB200_VERBOSE="1"))
    assert r.returncode == 0, r.stderr[-4000:]
    print("\n".join(l for l in r.stderr.splitlines() if l.startswith("[pgb200] k-mer table") or l.startswith("[pgb200] layout")))
    assert f"[pgb200] layout: {total} reference slots in {P} sets, {t} scan tiles" in r.stderr
    util.compare(ref, gpu, util.SUFFIXES_R)
