"""How the stages read their input.  CPU: the one chunked reader both stages use (read_chunks, with pass 1's record rule), run by
tests/host_read_chunks.cpp with small chunks over FASTA and FASTQ files made here, and the check of PGB200_CHUNK_MB through both CLIs.
GPU: a read file that cannot be read (a directory) ends either stage before any output file is written."""
import os
import random
import subprocess

import pytest

from soapdenovo2_b200 import api, synth
from tests import util


@pytest.fixture(scope="module")
def reader(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("read_chunks") / "host_read_chunks")
    src = [os.path.join(util.ROOT, *p) for p in (("tests", "host_read_chunks.cpp"), ("soapdenovo2_b200", "csrc", "stage_io.cpp"),
                                                 ("soapdenovo2_b200", "csrc", "deflate.cu"))]
    subprocess.run([util.NVCC, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, *src, "-lz"],
                   check=True, capture_output=True)
    return exe


def _run(exe, path, fastq, cap, out):
    r = subprocess.run([exe, path, "fastq" if fastq else "fasta", str(cap), out], capture_output=True, text=True)
    calls = [tuple(int(x) for x in line.split()[1:]) for line in r.stdout.splitlines()]
    return r, calls


def _records(rng, n, fastq):
    """n records with ragged lengths; FASTQ quality lines often start with '@'"""
    out = []
    for i in range(n):
        seq = "".join(rng.choice("ACGTN") for _ in range(rng.randrange(1, 150)))
        if fastq:
            qual = "".join(rng.choice("@I#") for _ in seq)
            out.append(f"@r{i} x\n{seq}\n+\n{qual}\n".encode())
        else:
            out.append(f">r{i} x\n{seq}\n".encode())
    return out


def _cases():
    rng = random.Random(20261018)
    cases = []
    for fastq in (False, True):
        recs = _records(rng, 300, fastq)
        body = b"".join(recs)
        for tail in (b"", b"\n", b"\n\n\n"):
            cases.append((f"{'fq' if fastq else 'fa'}_tail{len(tail)}", fastq, recs, body + tail))
    return cases


@pytest.mark.parametrize("name,fastq,recs,data", _cases(), ids=[c[0] for c in _cases()])
def test_read_chunks_takes_whole_records(reader, tmp_path, name, fastq, recs, data):
    path, out = str(tmp_path / name), str(tmp_path / "taken")
    open(path, "wb").write(data)
    starts, o = set(), 0
    for r in recs:
        starts.add(o)
        o += len(r)
    body = data.rstrip(b"\n") + b"\n"   # the file without its trailing blank lines
    longest = max(len(r) for r in recs)
    # a FASTQ chunk is cut only once the next record's '+' line is in it: two records is the least that always goes forward
    for cap in (2 * longest + 3, 3 * longest, 4096, len(data), len(data) + 1):
        r, calls = _run(reader, path, fastq, cap, out)
        assert r.returncode == 0, r.stderr
        assert open(out, "rb").read() == body, cap
        assert [c[1] for c in calls] == [0] * (len(calls) - 1) + [1], cap   # at_eof on the last call and on no other
        at = 0
        for n, _, taken in calls:
            assert n <= cap and at in starts, cap   # every piece starts at a record start: none is split
            at += taken
        assert at == len(body)


def test_read_chunks_empty_and_blank_files(reader, tmp_path):
    out = str(tmp_path / "taken")
    for data, calls_expected in ((b"", []), (b"\n", [(1, 1, 0)]), (b"\n\n", [(2, 1, 0)])):
        path = str(tmp_path / "in")
        open(path, "wb").write(data)
        r, calls = _run(reader, path, False, 64, out)
        assert r.returncode == 0 and calls == calls_expected and open(out, "rb").read() == b"", data


@pytest.mark.parametrize("fastq", [False, True])
def test_read_chunks_refuses_a_record_longer_than_the_chunk(reader, tmp_path, fastq):
    seq = "A" * ((1 << 20) + 100)
    rec = f"@big\n{seq}\n+\n{'I' * len(seq)}\n" if fastq else f">big\n{seq}\n"
    path = str(tmp_path / "big")
    open(path, "w").write((">a\nACGT\n" if not fastq else "@a\nACGT\n+\nIIII\n") + rec + rec)
    r, _ = _run(reader, path, fastq, 1 << 20, str(tmp_path / "taken"))
    assert r.returncode == 1 and r.stderr == "pgb200: a single record exceeds the 1 MB chunk\n"


def test_read_chunks_open_and_read_errors(reader, tmp_path):
    missing = str(tmp_path / "absent.fa")
    r, calls = _run(reader, missing, False, 64, str(tmp_path / "taken"))
    assert r.returncode == 1 and calls == [] and r.stderr == f"Cannot open {missing}. Now exit to system...\n"
    # a directory opens on Linux; reading it fails
    d = str(tmp_path / "dir.fa")
    os.mkdir(d)
    r, calls = _run(reader, d, False, 64, str(tmp_path / "taken"))
    assert r.returncode == 1 and calls == [] and r.stderr == f"pgb200: read error on {d}\n"


def _outputs(d, prefix):
    return sorted(f for f in os.listdir(d) if f.startswith(prefix + "."))


@pytest.mark.parametrize("stage", ["pregraph", "map"])
@pytest.mark.parametrize("value", ["0", "abc", "-1", "4096"])
def test_cli_refuses_a_bad_chunk_size(tmp_path, stage, value):
    """Checked with the stage's other settings, before any engine exists: no GPU is needed to see it"""
    d = str(tmp_path)
    cfg = synth.scenario_se_fasta(d, genome_len=2000, n_reads=50)
    if stage == "pregraph":
        args = ["pregraph", "-s", cfg, "-K", "31", "-o", os.path.join(d, "out")]
    else:
        args = ["map", "-s", cfg, "-g", os.path.join(d, "out")]
    r = subprocess.run([api.BIN63, *args], capture_output=True, text=True, timeout=120, env=dict(os.environ, PGB200_CHUNK_MB=value))
    assert r.returncode == 255
    assert r.stderr.endswith(f'\npgb200: PGB200_CHUNK_MB must be a whole number of MB from 1 to 4095, not "{value}"\n'), r.stderr
    assert _outputs(d, "out") == []


@pytest.mark.gpu
@pytest.mark.parametrize("stage", ["pregraph", "map"])
def test_stage_refuses_an_unreadable_read_file(tmp_path, stage):
    d = str(tmp_path)
    reads = os.path.join(d, "reads.fa")
    os.mkdir(reads)
    cfg = os.path.join(d, "dir.cfg")
    open(cfg, "w").write(f"max_rd_len=100\n[LIB]\navg_ins=300\nf={reads}\np={reads}\n")
    g = os.path.join(d, "g")
    if stage == "pregraph":
        args = ["pregraph", "-s", cfg, "-K", "31", "-o", g]
    else:
        open(g + ".contig", "w").write(">1 length 40 cvg_1.0_tip_0\n" + "ACGT" * 10 + "\n")
        args = ["map", "-s", cfg, "-g", g]
    r = subprocess.run([api.BIN63, *args], capture_output=True, text=True, timeout=300)
    assert r.returncode == 255
    assert r.stderr.endswith(f"Import reads from file:\n {reads}\npgb200: read error on {reads}\n" if stage == "pregraph"
                             else f"\npgb200: read error on {reads}\n"), r.stderr[-2000:]
    assert _outputs(d, "g") == ([] if stage == "pregraph" else ["g.contig"])
