"""CPU: the zlib-exact deflate pieces (soapdenovo2_b200/csrc/deflate.cuh) run one after another by tests/host_deflate.cu must write
exactly zlib.compressobj(6, DEFLATED, 31)'s gzip bytes -- the stream gzopen(name, "w") + gzwrite writes -- on seeded inputs that
reach every rule: tiny inputs, the window sizes, long runs (258-byte matches, long chains), random bytes (stored blocks), DNA and the
map / pregraph text shapes (the reduced chain), far length-3 matches (TOO_FAR), and streams of exactly n x 16383 symbols with and
without an empty last block.  The driver also checks the CRC combine and the composed bit-offset maps against direct computation."""
import os
import random
import subprocess
import zlib

import pytest

from tests import util


def de_bruijn_prefix(n):
    """First n bytes of a byte string whose 3-byte substrings are all distinct (so deflate emits only literals)."""
    out = bytearray()
    seen = set()
    rng = random.Random(7)
    a, b = 0, 1
    out += bytes([a, b])
    while len(out) < n:
        for c in rng.sample(range(256), 256):
            if (a, b, c) not in seen:
                seen.add((a, b, c))
                out.append(c)
                a, b = b, c
                break
        else:
            raise AssertionError("stuck")
    return bytes(out[:n])


def read_on_contig(rng, n_lines):
    return b"read\tcontig\tpos\n" + b"".join(
        b"%d\t%d\t%d\t%c\n" % (i + 1, rng.randrange(1, 40000), rng.randrange(0, 5000), rng.choice(b"+-")) for i in range(n_lines))


def read_in_gap(rng, n_recs):
    out = bytearray()
    for _ in range(n_recs):   # binary records: len, contig, pos, packed read
        out += rng.randrange(50, 151).to_bytes(4, "little") + rng.randrange(1, 1 << 20).to_bytes(4, "little")
        out += rng.randrange(0, 1 << 16).to_bytes(4, "little") + bytes(rng.getrandbits(8) for _ in range(38))
    return bytes(out)


def edge_text(rng, n_edges):
    out = []
    for i in range(n_edges):
        L = rng.randrange(1, 400)
        out.append(b">length %d,%d,%d,%d,%d\n" % (L, rng.randrange(1 << 20), rng.randrange(1 << 20), rng.choice([-1, 0, 1]), rng.randrange(40)))
        seq = bytes(rng.choice(b"ACGT") for _ in range(L + 62))
        out += [seq[j:j + 100] + b"\n" for j in range(0, len(seq), 100)]
    return b"".join(out)


def too_far_text(rng, n):
    """Random bytes where many 3-byte strings recur only more than 4096 bytes back."""
    base = bytes(rng.getrandbits(8) for _ in range(5000))
    out = bytearray(base)
    while len(out) < n:
        k = rng.randrange(0, len(base) - 4)
        out += base[k:k + 3] + bytes(rng.getrandbits(8) for _ in range(rng.randrange(1, 6)))
    return bytes(out[:n])


def cases():
    rng = random.Random(20261016)
    dna = lambda n: bytes(rng.choice(b"ACGT") for _ in range(n))
    c = {"empty": b"", "one": b"x", "two": b"xy", "three": b"xyz", "three_same": b"aaa", "four_same": b"aaaa"}
    for n in (32505, 32506, 32507, 32767, 32768, 32769, 65273, 65274, 65275, 65535, 65536, 65537, 65536 + 32768 + 7):
        c[f"dna_{n}"] = dna(n)
    for n in (32506, 65274, 65536):
        c[f"rand_{n}"] = bytes(rng.getrandbits(8) for _ in range(n))
        c[f"run_{n}"] = b"G" * n
    c["runs_mixed"] = b"".join(bytes([rng.choice(b"ACGTN")]) * rng.randrange(1, 700) for _ in range(3000))
    c["rand_300k"] = bytes(rng.getrandbits(8) for _ in range(300000))
    c["one_letter_1m"] = b"A" * 1000000
    c["dna_400k"] = dna(400000)
    c["read_on_contig"] = read_on_contig(rng, 60000)
    c["read_in_gap"] = read_in_gap(rng, 8000)
    c["edge"] = edge_text(rng, 1500)
    c["too_far"] = too_far_text(rng, 200000)
    c["text_and_random"] = b"".join((read_on_contig(rng, 200) if rng.random() < 0.5 else bytes(rng.getrandbits(8) for _ in range(9000)))
                                    for _ in range(40))
    db = de_bruijn_prefix(3 * 16383 + 10)
    for k in (1, 2, 3):   # k x 16383 literals: the final pending literal fills the last block
        c[f"syms_{k}x16383_lit"] = db[:k * 16383]
    for k in (1, 2):      # k x 16383 - 1 literals + a final match: the in-loop flush takes the last symbol, an empty block follows
        c[f"syms_{k}x16383_match"] = db[:k * 16383 - 1] + db[k * 16383 - 1 - 20000 if k == 2 else 100:][:6]
    return c


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("deflate")
    exe = str(d / "host_deflate")
    subprocess.run([util.NVCC, "-std=c++17", "-O2", "-o", exe, os.path.join(util.ROOT, "tests", "host_deflate.cu")],
                   check=True, capture_output=True)
    return d, exe


def test_host_deflate_equals_zlib(driver):
    d, exe = driver
    cs = cases()
    args = []
    for k, v in cs.items():
        (d / f"{k}.in").write_bytes(v)
        args += [str(d / f"{k}.in"), str(d / f"{k}.gz")]
    r = subprocess.run([exe] + args, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    stats = {}
    for line in r.stdout.splitlines():
        name, *kv = line.split()
        stats[os.path.basename(name)[:-3]] = {a: int(b) for a, b in (x.split("=") for x in kv)}
    bad = []
    for k, v in cs.items():
        co = zlib.compressobj(6, zlib.DEFLATED, 31)
        if (d / f"{k}.gz").read_bytes() != co.compress(v) + co.flush():
            bad.append(k)
    assert not bad, f"streams differ from zlib: {bad}"
    # the rules the inputs are there for really ran
    assert stats["rand_300k"]["stored"] > 0 and stats["rand_32506"]["stored"] > 0
    assert stats["one_letter_1m"]["maxlen"] == 258 and stats["dna_400k"]["dyn"] > 1
    assert stats["empty"]["fixed"] == 1 and stats["empty"]["blocks"] == 1
    assert stats["too_far"]["toofar"] > 100
    assert stats["read_on_contig"]["reduced"] > 0 and stats["edge"]["reduced"] > 0
    for k in (1, 2, 3):
        s = stats[f"syms_{k}x16383_lit"]
        assert s["syms"] == k * 16383 and s["blocks"] == k
    for k in (1, 2):
        s = stats[f"syms_{k}x16383_match"]
        assert s["syms"] == k * 16383 and s["blocks"] == k + 1
