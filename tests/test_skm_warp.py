"""The warp partition of the aggregated pass 1 (skm_warp_scan_read, soapdenovo2_b200/csrc/skm.cuh) must make exactly the runs of its
host definition skm_scan_read: every odd K from 13 to 127, 1 / 2 / 3 / 65536 buckets, short, boundary and long reads, random bases,
homopolymers and repeats.  See tests/host_skm_warp.cu.  The harness compiles for sm_90a anywhere; it runs on the GPU."""
import os
import subprocess

import pytest

from tests import util


def _compile(tmp_path):
    exe = str(tmp_path / "host_skm_warp")
    subprocess.run([util.NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                    os.path.join(util.ROOT, "tests", "host_skm_warp.cu")], check=True, capture_output=True)
    return exe


def test_warp_partition_harness_compiles(tmp_path):
    assert os.path.exists(_compile(tmp_path))


@pytest.mark.gpu
def test_warp_partition_equals_host_scan(tmp_path):
    r = subprocess.run([_compile(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "ALL OK"
    assert len(lines) == 1 + len(range(13, 128, 2)) and all("errors=0" in l for l in lines[:-1])
