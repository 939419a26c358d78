"""CPU: the aggregation kernel builds each k-mer instance from a record staged in shared memory plus the record's reversed bases
(skm_rec_reverse / skm_instance_staged, soapdenovo2_b200/csrc/skm.cuh).  For every odd K from 13 to 127, both key widths, every run
length, has_prev / last and random bases, the result must equal skm_instance_rec.  See tests/host_skm_stage.cu."""
import os
import subprocess

from tests import util


def test_staged_instances_equal_record_instances_on_host(tmp_path):
    exe = str(tmp_path / "host_skm_stage")
    subprocess.run([util.NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                    os.path.join(util.ROOT, "tests", "host_skm_stage.cu")], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    lines = r.stdout.strip().splitlines()
    assert lines[-1].startswith("ALL OK")
    assert len(lines) == 1 + len(range(13, 128, 2)) and all("errors=0" in l for l in lines[:-1])
