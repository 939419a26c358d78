"""GPU: the gzip writer of soapdenovo2_b200/csrc/deflate.cu writes exactly zlib.compressobj(6, DEFLATED, 31)'s bytes (the stream
gzopen(path, "w") + gzwrite write): on the shapes the CPU fuzz uses, on inputs of hundreds of MB that take several buffer rounds,
for any piece sizes, for host- and device-resident input, and past 4 GiB (ISIZE wraps)."""
import os
import random
import zlib

import numpy as np
import pytest

from soapdenovo2_b200 import api
from tests import test_deflate_host as shapes

pytestmark = pytest.mark.gpu


def zgz(data):
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    return co.compress(data) + co.flush()


def big(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "dna":
        return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()
    if kind == "random":
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    if kind == "read_on_contig":   # tab-separated integers, one record per line, like the map stage's .readOnContig
        m = n // 20 + 1
        ids = np.arange(1, m + 1)
        ctg = rng.integers(1, 2_000_000, m)
        pos = rng.integers(0, 30000, m)
        ori = np.where(rng.integers(0, 2, m) == 1, "+", "-")
        text = "".join(f"{a}\t{b}\t{c}\t{d}\n" for a, b, c, d in zip(ids.tolist(), ctg.tolist(), pos.tolist(), ori.tolist()))
        return text.encode()[:n]
    if kind == "edge":   # headers + 100-column DNA lines with repeats, like .edge
        unit = shapes.edge_text(random.Random(seed), 2000)
        reps = n // len(unit) + 1
        return (unit * reps)[:n]
    raise ValueError(kind)


def test_gate_accepts_this_zlib():
    assert api.gz_gpu_exact(0), "the GPU writer's bytes differ from this zlib's on the probe text"


def test_small_shapes_equal_zlib():
    bad = [k for k, v in shapes.cases().items() if api.gzip_bytes(v) != zgz(v)]
    assert not bad, f"differ from zlib: {bad}"


@pytest.mark.parametrize("kind,n", [("dna", 150 << 20), ("read_on_contig", 200 << 20), ("random", 80 << 20), ("edge", 120 << 20)])
def test_large_equal_zlib(kind, n):
    data = big(kind, n, 11)
    assert api.gzip_bytes(data) == zgz(data)


def test_pieces_equal_one_write(tmp_path, monkeypatch):
    """Small GPU rounds (5 MB buffers): pieces of 1 byte, pieces across block and window boundaries, pieces of several MB."""
    monkeypatch.setenv("PGB200_GZ_CHUNK_MB", "5")
    rng = random.Random(5)
    data = big("read_on_contig", 12 << 20, 3) + big("dna", 9 << 20, 4) + big("random", 3 << 20, 5) + b"N" * (2 << 20)
    want = zgz(data)
    path = tmp_path / "p.gz"
    with api.GpuGzWriter(path) as w:
        at = 0
        for _ in range(3000):   # 1-byte pieces first
            w.write(data[at:at + 1])
            at += 1
        while at < len(data):
            n = rng.choice([1, 2, 3, 255, 32768, 32506, 65536, rng.randrange(1, 70000), rng.randrange(1, 3 << 20)])
            w.write(data[at:at + n])
            at += n
    assert path.read_bytes() == want
    monkeypatch.setenv("PGB200_GZ_CHUNK_MB", "5")
    assert api.gzip_bytes(data) == want   # one write, the same small rounds


def test_device_input_equals_host_input(tmp_path):
    import torch
    data = big("dna", 40 << 20, 8) + big("read_on_contig", 30 << 20, 9)
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    torch.cuda.synchronize()
    path = tmp_path / "d.gz"
    with api.GpuGzWriter(path) as w:
        half = len(data) // 2 + 12345
        w.write(t.data_ptr(), half, on_device=True)
        w.write(t.data_ptr() + half, len(data) - half, on_device=True)
    assert path.read_bytes() == zgz(data) == api.gzip_bytes(data)


def test_host_mode_is_zlib(tmp_path, monkeypatch):
    monkeypatch.setenv("PGB200_GZ", "host")
    data = big("edge", 3 << 20, 2)
    assert api.gzip_bytes(data) == zgz(data)


def test_past_4gib_isize_wraps(tmp_path):
    """4.25 GiB in 1 GiB sub-writes from the device: ISIZE is the length mod 2^32, the CRC spans every round.  The text repeats with
    a 16 KB period, inside the window, so zlib (the reference here) runs at its fast long-match speed."""
    import torch
    unit = big("dna", 8 << 10, 21) + big("read_on_contig", 8 << 10, 22)
    n = (4 << 30) + (256 << 20) + 7
    dev = torch.frombuffer(bytearray(unit), dtype=torch.uint8).cuda().repeat(n // len(unit) + 1)[:n].contiguous()
    torch.cuda.synchronize()
    path = tmp_path / "huge.gz"
    with api.GpuGzWriter(path) as w:
        for at in range(0, n, 1 << 30):
            w.write(dev.data_ptr() + at, min(1 << 30, n - at), on_device=True)
    del dev
    co = zlib.compressobj(6, zlib.DEFLATED, 31)
    piece = unit * ((256 << 20) // len(unit))   # 256 MB, a whole number of periods
    with open(path, "rb") as f:
        got = f.read()
    at, pos, ok = 0, 0, True
    while at < n:
        z = co.compress(piece[:min(len(piece), n - at)])
        ok = ok and got[pos:pos + len(z)] == z
        pos += len(z)
        at += len(piece)
    z = co.flush()
    ok = ok and got[pos:] == z
    assert got[-4:] == (n % (1 << 32)).to_bytes(4, "little")
    assert ok, "differs from zlib"
