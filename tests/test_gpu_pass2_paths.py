"""GPU pass 2 and the -R outputs on designed long reads: every scenario of tests/test_pass2_paths_host.py through the CLI.

All seven files must equal the reference's (or the C model's where the reference was not built), and the counter lines (pre-arcs
added, reads deleted, ...) the reference's, run or stored.  The scenarios reach what the short-read parity cases never do:
  - .path records of 256+ edges, whose unsigned char count wraps in the reference (k_write_paths writes the last wrap's entries);
  - reads of up to about 34,000 bases: paths of 700 edges, arc ranks at large path indices, k_pass2's unstaged read loop;
  - the staged tiles at their size limits: 48 KB in pass 1 (W64 = 24) and in pass 2 (W64 = 48), W64 = 49 just past it, an odd W64
    with a partial last tile;
  - the .path offsets across 1 MB read chunks, and an f1/f2 library (read ordinals stepping by 2);
  - paths of exactly 2 edges (arcs, no record) and 3, and reads wholly in a branch-free ring (counted as deleted).
Not covered here: restarts inside a clipped tip, a stop at a deleted node after two kept segments, and a missing (K+1)-mer between
consecutive junctions; no designed read set yet shows those branches in the outputs."""
import json
import os

import pytest

from tests import util
from tests.test_gpu_full import _engine, _oracle
from tests.test_pass2_paths_host import GOLD_PATH, SCENARIOS, check_paths, counter_lines, scenario

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _build():
    util.build_oracle()


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_cli_on_long_paths(tmp_path, name):
    d = str(tmp_path)
    cfg, counts, rings, K, P, extra, env = scenario(d, name)
    ref, gpu = os.path.join(d, "ref"), os.path.join(d, "gpu")
    lr = _oracle(int(K > 63), cfg, ref, K, P, extra)
    lg = _engine(int(K > 63), cfg, gpu, K, P, extra, env=env)
    util.compare(ref, gpu, util.SUFFIXES_R)
    want = counter_lines(lr) if util.have_ref() else json.load(open(GOLD_PATH))[name]["counters"]
    got = [l for l in counter_lines(lg) if not l.startswith("[pgb200]")]
    assert got == want
    check_paths(name, gpu, got, counts, rings)
