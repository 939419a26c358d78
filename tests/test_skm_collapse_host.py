"""CPU: the record collapse of the aggregated pass 1 -- the weighted update payload_apply_n against repeated payload_apply, and a
sequential restatement of the distinct-record buffer against applying every instance.  See tests/host_skm_collapse.cu."""
import os
import subprocess

from tests import util


def test_record_collapse_on_host(tmp_path):
    exe = str(tmp_path / "host_skm_collapse")
    subprocess.run([util.NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
                    os.path.join(util.ROOT, "tests", "host_skm_collapse.cu")], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    lines = r.stdout.strip().splitlines()
    assert lines[-1] == "ALL OK"
    assert len(lines) == 9 and all("errors=0" in l for l in lines[:-1])
    def field(line, name):
        return int(line.split(name + "=")[1].split()[0].rstrip(":"))
    # the tiled cases really collapse (counts past the saturation of the links at K = 31 and 65) and drain buckets more than once;
    # records of 32 k-mers occur at K = 63 and 127
    tiled = [l for l in lines if " tiled " in l]
    assert all(field(l, "max_count") > 1 and field(l, "drains") > field(l, "buckets") for l in tiled)
    assert all(field(l, "max_count") > 63 for l in tiled if l.startswith(("K=31 ", "K=65 ")))
    assert all(field(l, "n32") > 0 for l in lines if l.startswith(("K=63 ", "K=127 ")))
