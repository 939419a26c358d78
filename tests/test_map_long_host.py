"""The long-read pass of `map` on the CPU: k_map_long's group reduction against a literal parse1read (tests/host_map_group.cu, the
overflow rounds forced by small tables), and the refusals that come from the config before any GPU work or output file."""
import os
import subprocess

import pytest

from soapdenovo2_b200 import api
from tests import util


def test_group_reduction_equals_parse1read(tmp_path):
    exe = str(tmp_path / "host_map_group")
    subprocess.run(["g++", "-std=c++17", "-O2", "-x", "c++", os.path.join(util.ROOT, "tests", "host_map_group.cu"), "-o", exe],
                   check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "ALL OK"
    assert "errors=0" in r.stdout


def _fake_graph(d):
    g = os.path.join(d, "g")
    with open(g + ".contig", "w") as f:
        f.write(">1 length 40 cvg_1.0_tip_0\n" + "ACGT" * 10 + "\n")
    return g


@pytest.mark.parametrize("files", ["f1={d}/a.fa\nf2={d}/b.fa\n", "q1={d}/a.fq\nq2={d}/b.fq\n", "f={d}/s.fa\nq1={d}/a.fq\nq2={d}/b.fq\n"])
def test_long_library_with_two_file_pairs_is_refused(tmp_path, files):
    d = str(tmp_path)
    g = _fake_graph(d)
    cfg = os.path.join(d, "x.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=100\n[LIB]\navg_ins=300\nq1={d}/p.fq\nq2={d}/p2.fq\n"
                f"[LIB]\navg_ins=500\nasm_flags=4\nrd_len_cutoff=5000\n" + files.format(d=d))
    r = subprocess.run([api.BIN63, "map", "-s", cfg, "-g", g], capture_output=True, text=True, timeout=120)
    assert r.returncode == 255
    assert "long-read libraries (asm_flags=4) are not supported with two-file pairs (f1/f2, q1/q2)" in r.stderr
    assert sorted(os.listdir(d)) == ["g.contig", "x.cfg"]


def test_long_library_bam_is_refused(tmp_path):
    d = str(tmp_path)
    g = _fake_graph(d)
    cfg = os.path.join(d, "x.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=100\n[LIB]\nasm_flags=4\nrd_len_cutoff=5000\nf={d}/s.fa\nb={d}/r.bam\n")
    r = subprocess.run([api.BIN63, "map", "-s", cfg, "-g", g], capture_output=True, text=True, timeout=120)
    assert r.returncode == 255
    assert "BAM input (b=) is not supported" in r.stderr
    assert sorted(os.listdir(d)) == ["g.contig", "x.cfg"]
