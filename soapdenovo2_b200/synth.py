"""Seeded synthetic read sets for the pregraph path (host-side numpy; test + bench plumbing, not the product path).

Recipe follows SURVEY.md section 8(d): uniform i.i.d. ACGT genome, uniform fragment starts, i.i.d. substitution
errors, constant quality 'I'.  Files avoid the reference reader's quirks (SURVEY.md A.9): single-line FASTA,
4-line FASTQ, trailing newline, sizes that are not a multiple of 32768 bytes.
"""
from __future__ import annotations

import os
import numpy as np

_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_COMP = np.zeros(256, dtype=np.uint8)
for _a, _b in zip(b"ACGTNacgtn", b"TGCANtgcan"):
    _COMP[_a] = _b


def genome(n: int, seed: int, repeat: tuple[int, int] | None = None) -> np.ndarray:
    rng = np.random.default_rng(seed)
    g = _ACGT[rng.integers(0, 4, size=n)]
    if repeat is not None:  # (length, copies): plant an exact repeat so the graph has real branches
        ln, copies = repeat
        unit = g[:ln].copy()
        for c in range(1, copies):
            p = (c * n) // copies
            g[p:p + ln] = unit
    return g


def _mutate(reads: np.ndarray, err: float, rng) -> np.ndarray:
    if err <= 0:
        return reads
    mask = rng.random(reads.shape) < err
    idx = np.searchsorted(_ACGT, reads[mask])  # 0..3 in "ACGT" order
    reads[mask] = _ACGT[(idx + rng.integers(1, 4, size=idx.shape)) % 4]
    return reads


def _sample(g: np.ndarray, n_reads: int, rd_len: int, rng, starts=None) -> np.ndarray:
    if starts is None:
        starts = rng.integers(0, len(g) - rd_len + 1, size=n_reads)
    return g[starts[:, None] + np.arange(rd_len)[None, :]].copy()


def _revcomp(reads: np.ndarray) -> np.ndarray:
    return _COMP[reads[:, ::-1]]


def _pad_if_32k(path: str) -> None:
    """The reference's AIO reader mis-handles files whose size is k*32768 (SURVEY.md A.9): dodge by renaming a read."""
    if os.path.getsize(path) % 32768 == 0:
        with open(path, "rb") as f:
            data = f.read()
        nl = data.index(b"\n")
        with open(path, "wb") as f:
            f.write(data[:nl] + b"x" + data[nl:])


def write_fasta(path: str, reads: np.ndarray, tag: str = "r") -> None:
    n, L = reads.shape
    with open(path, "wb") as f:
        for i in range(n):
            f.write(b">" + f"{tag}{i}".encode() + b"\n")
            f.write(reads[i].tobytes() + b"\n")
    _pad_if_32k(path)


def write_fastq(path: str, reads: np.ndarray, tag: str = "r") -> None:
    n, L = reads.shape
    q = b"I" * L
    with open(path, "wb") as f:
        for i in range(n):
            f.write(b"@" + f"{tag}{i}".encode() + b"\n" + reads[i].tobytes() + b"\n+\n" + q + b"\n")
    _pad_if_32k(path)


def se_reads(g, n_reads, rd_len, err, seed, both_strands=True):
    rng = np.random.default_rng(seed)
    r = _sample(g, n_reads, rd_len, rng)
    if both_strands:
        flip = rng.random(n_reads) < 0.5
        r[flip] = _revcomp(r[flip])
    return _mutate(r, err, rng)


def pe_reads(g, n_pairs, rd_len, insert, err, seed):
    rng = np.random.default_rng(seed)
    starts = rng.integers(0, len(g) - insert + 1, size=n_pairs)
    r1 = _sample(g, n_pairs, rd_len, rng, starts)
    r2 = _revcomp(_sample(g, n_pairs, rd_len, rng, starts + insert - rd_len))
    flip = rng.random(n_pairs) < 0.5  # fragment strand
    r1f, r2f = r1.copy(), r2.copy()
    r1f[flip], r2f[flip] = r2[flip], r1[flip]
    return _mutate(r1f, err, rng), _mutate(r2f, err, rng)


def write_config(path: str, max_rd_len: int, libs: list[dict]) -> None:
    """libs: [{'avg_ins':200, 'reverse_seq':0, 'asm_flags':3, 'rd_len_cutoff':None, 'files':[('q1',p),('q2',p),...]}]"""
    with open(path, "w") as f:
        f.write(f"max_rd_len={max_rd_len}\n")
        for lib in libs:
            f.write("[LIB]\n")
            f.write(f"avg_ins={lib.get('avg_ins', 200)}\n")
            f.write(f"reverse_seq={lib.get('reverse_seq', 0)}\n")
            f.write(f"asm_flags={lib.get('asm_flags', 3)}\n")
            if lib.get("rd_len_cutoff"):
                f.write(f"rd_len_cutoff={lib['rd_len_cutoff']}\n")
            f.write("rank=1\n")
            for k, p in lib["files"]:
                f.write(f"{k}={p}\n")


# ---------------------------------------------------------------- canned scenarios (SURVEY.md Appendix B list)
def scenario_se_fasta(d: str, genome_len=20000, n_reads=4000, rd_len=100, err=0.005, seed=1) -> str:
    g = genome(genome_len, seed)
    write_fasta(os.path.join(d, "se.fa"), se_reads(g, n_reads, rd_len, err, seed + 100))
    cfg = os.path.join(d, "se.cfg")
    write_config(cfg, rd_len, [{"avg_ins": 200, "files": [("f", os.path.join(d, "se.fa"))]}])
    return cfg


def scenario_pe_fastq(d: str, genome_len=60000, n_pairs=6000, rd_len=150, insert=300, err=0.004, seed=3,
                      repeat=(400, 3)) -> str:
    g = genome(genome_len, seed, repeat=repeat)
    r1, r2 = pe_reads(g, n_pairs, rd_len, insert, err, seed + 100)
    write_fastq(os.path.join(d, "pe_1.fq"), r1, "p")
    write_fastq(os.path.join(d, "pe_2.fq"), r2, "p")
    cfg = os.path.join(d, "pe.cfg")
    write_config(cfg, rd_len, [{"avg_ins": insert, "files": [("q1", os.path.join(d, "pe_1.fq")), ("q2", os.path.join(d, "pe_2.fq"))]}])
    return cfg


def scenario_multilib(d: str, genome_len=40000, seed=5) -> str:
    """4 libraries, mixed FASTA/FASTQ/SE/PE, rd_len_cutoff, reverse_seq, N's + lower case, an asm_flags=2 lib to ignore."""
    g = genome(genome_len, seed, repeat=(300, 2))
    rng = np.random.default_rng(seed + 7)
    a1, a2 = pe_reads(g, 1500, 100, 500, 0.004, seed + 1)
    write_fasta(os.path.join(d, "m_a1.fa"), a1, "a"); write_fasta(os.path.join(d, "m_a2.fa"), a2, "a")
    s = se_reads(g, 1500, 120, 0.004, seed + 2)
    nmask = rng.random(s.shape) < 0.002
    s[nmask] = ord("N")
    low = rng.random(s.shape[0]) < 0.3
    s[low] = np.char.lower(s[low].view("S1")).view(np.uint8) if low.any() else s[low]
    write_fasta(os.path.join(d, "m_s.fa"), s, "s")
    q1, q2 = pe_reads(g, 2000, 150, 200 + 100, 0.004, seed + 3)
    write_fastq(os.path.join(d, "m_q1.fq"), q1, "q"); write_fastq(os.path.join(d, "m_q2.fq"), q2, "q")
    rq = se_reads(g, 1200, 130, 0.004, seed + 4)
    write_fastq(os.path.join(d, "m_rq.fq"), rq, "z")
    ig = se_reads(g, 500, 100, 0.0, seed + 5)
    write_fasta(os.path.join(d, "m_ig.fa"), ig, "i")
    cfg = os.path.join(d, "multi.cfg")
    j = lambda n: os.path.join(d, n)
    write_config(cfg, 150, [
        {"avg_ins": 500, "files": [("f1", j("m_a1.fa")), ("f2", j("m_a2.fa"))]},
        {"avg_ins": 200, "rd_len_cutoff": 140, "files": [("f", j("m_s.fa")), ("q1", j("m_q1.fq")), ("q2", j("m_q2.fq"))]},
        {"avg_ins": 2000, "reverse_seq": 1, "files": [("q", j("m_rq.fq"))]},
        {"avg_ins": 300, "asm_flags": 2, "files": [("f", j("m_ig.fa"))]},
    ])
    return cfg


def scenario_adversarial(d: str, seed=9, crlf=False, K_hint=31) -> str:
    """Edge cases the reference's readers / counters / edge builder care about: ragged read lengths (incl. shorter than K+1
    and exactly K+1), N's, lower case, '.', a poly-A stretch (counter saturation: links 63, coverage 255), tandem repeats,
    a reverse-complement palindrome (bal_edge = 0 edges), optional CRLF line ends (the '\\r' is dropped, readseq1by1.c:182-200)."""
    rng = np.random.default_rng(seed)
    g = genome(12000, seed)
    unit = g[100:137].copy()
    g[3000:3000 + 37 * 6] = np.tile(unit, 6)                       # tandem repeat
    g[5000:5400] = ord("A")                                         # poly-A
    half = g[7000:7150].copy()
    g[7150:7300] = _COMP[half[::-1]]                                # palindrome: half + revcomp(half)
    nl = b"\r\n" if crlf else b"\n"
    reads = []
    for i in range(3500):
        L = int(rng.choice([K_hint - 3, K_hint, K_hint + 1, K_hint + 2, 60, 75, 100, 100, 100]))
        s = int(rng.integers(0, len(g) - L))
        r = g[s:s + L].copy()
        if rng.random() < 0.5:
            r = _COMP[r[::-1]]
        m = rng.random(L) < 0.004
        r[m] = _ACGT[rng.integers(0, 4, size=int(m.sum()))]
        if rng.random() < 0.05:
            r[int(rng.integers(0, L))] = ord("N")
        if rng.random() < 0.05:
            r[int(rng.integers(0, L))] = ord(".")
        if rng.random() < 0.2:
            r = np.frombuffer(r.tobytes().lower(), dtype=np.uint8).copy()
        reads.append(r.tobytes())
    for i in range(600):                                            # deep poly-A coverage -> saturated counters
        reads.append(b"A" * int(rng.choice([80, 100])))
    order = rng.permutation(len(reads))
    fa, fq = os.path.join(d, "adv.fa"), os.path.join(d, "adv.fq")
    with open(fa, "wb") as f:
        for j in order[: len(order) // 2]:
            f.write(b">r%d" % j + nl + reads[j] + nl)
    with open(fq, "wb") as f:
        for j in order[len(order) // 2:]:
            f.write(b"@r%d" % j + nl + reads[j] + nl + b"+" + nl + b"I" * len(reads[j]) + nl)
    for p in (fa, fq):
        _pad_if_32k(p)
    cfg = os.path.join(d, "adv.cfg")
    write_config(cfg, 100, [{"avg_ins": 200, "files": [("f", fa), ("q", fq)]}])
    return cfg


def long_reads(g: np.ndarray, n_reads: int, min_len: int, max_len: int, seed: int, err=0.01, n_rate=0.001, short_frac=0.05,
               K_hint=31) -> list[bytes]:
    """Seeded long reads for a gap-closing library (asm_flags=4): lengths uniform in [min_len, max_len], both strands, i.i.d.
    substitution errors, scattered N's, and a share `short_frac` of reads of 1..K_hint bases (shorter than K+1: they map nowhere)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_reads):
        L = int(rng.integers(1, K_hint + 1)) if rng.random() < short_frac else int(rng.integers(min_len, max_len + 1))
        L = min(L, len(g))
        s = int(rng.integers(0, len(g) - L + 1))
        r = g[s:s + L].copy()
        if rng.random() < 0.5:
            r = _COMP[r[::-1]]
        r = _mutate(r, err, rng)
        r[rng.random(L) < n_rate] = ord("N")
        out.append(r.tobytes())
    return out


def long_reads_of_lengths(g: np.ndarray, lengths: list[int], seed: int, err=0.01, n_rate=0.001) -> list[bytes]:
    """long_reads() with the read lengths given: one read per length, drawn as long_reads() draws them"""
    rng = np.random.default_rng(seed)
    out = []
    for L in lengths:
        s = int(rng.integers(0, len(g) - L + 1))
        r = g[s:s + L].copy()
        if rng.random() < 0.5:
            r = _COMP[r[::-1]]
        r = _mutate(r, err, rng)
        r[rng.random(L) < n_rate] = ord("N")
        out.append(r.tobytes())
    return out


def tiled_pairs(g: np.ndarray, step: int, rd_len: int, insert: int) -> tuple[np.ndarray, np.ndarray]:
    """Error-free pairs at every `step`-th genome position: pair i has mate 1 = g[s:s+rd_len] and mate 2 = the reverse complement of
    g[s+insert-rd_len:s+insert], s = i*step, for every s <= len(g) - insert (so every base is covered when step <= rd_len)."""
    starts = np.arange(0, len(g) - insert + 1, step, dtype=np.int64)
    win = np.lib.stride_tricks.sliding_window_view(g, rd_len)   # no per-base index array (millions of reads)
    return win[starts], _revcomp(win[starts + insert - rd_len])


def _wrapped(s: bytes, width) -> bytes:
    """s as lines of `width` bytes, or of the widths of a list taken in turn (one line for an empty s)"""
    if width is None or not s:
        return s + b"\n"
    widths = [width] if isinstance(width, int) else list(width)
    out, i, k = [], 0, 0
    while i < len(s):
        w = widths[k % len(widths)]
        out.append(s[i:i + w])
        i += w
        k += 1
    return b"\n".join(out) + b"\n"


def write_long(path: str, reads: list[bytes], fastq: bool, tag: str = "L", width=None) -> None:
    """Single-line FASTA or 4-line FASTQ, one record per read.  `width` wraps the sequence lines (and the FASTQ quality lines) at
    that many columns, or, given a list, at its widths in turn (ragged wrapping)."""
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            name = f"{tag}{i}".encode()
            f.write(b"@" + name + b"\n" + _wrapped(r, width) + b"+\n" + _wrapped(b"I" * len(r), width) if fastq
                    else b">" + name + b"\n" + _wrapped(r, width))
    _pad_if_32k(path)


def scenario_long(d: str, n_long=300, min_len=200, max_len=3000, rd_len_cutoff=5000, map_len=40, seed=21, fastq=False) -> str:
    """scenario_pe_fastq's paired library plus one long-read library (asm_flags=4) drawn from the same genome"""
    scenario_pe_fastq(d)
    g = genome(60000, 3, repeat=(400, 3))   # scenario_pe_fastq's genome
    path = os.path.join(d, "long.fq" if fastq else "long.fa")
    write_long(path, long_reads(g, n_long, min_len, max_len, seed), fastq)
    cfg = os.path.join(d, "long.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len=150\n[LIB]\navg_ins=300\nreverse_seq=0\nasm_flags=3\nrank=1\nq1={d}/pe_1.fq\nq2={d}/pe_2.fq\n"
                f"[LIB]\nasm_flags=4\nrd_len_cutoff={rd_len_cutoff}\nmap_len={map_len}\n{'q' if fastq else 'f'}={path}\n")
    return cfg


# ---------------------------------------------------------------- vectorised writers for the config-sized cases (millions of reads)
def _names(n: int, tag: bytes, width: int = 9) -> np.ndarray:
    ids = np.arange(n, dtype=np.int64)
    out = np.empty((n, len(tag) + width), dtype=np.uint8)
    out[:, :len(tag)] = np.frombuffer(tag, dtype=np.uint8)
    for d in range(width):
        out[:, len(tag) + width - 1 - d] = (ids // 10 ** d) % 10 + 48
    return out


def write_fastq_fast(path: str, reads: np.ndarray, tag: str = "r") -> None:
    n, L = reads.shape
    nm = _names(n, b"@" + tag.encode())
    rec = np.empty((n, nm.shape[1] + 1 + L + 3 + L + 1), dtype=np.uint8)
    o = nm.shape[1]
    rec[:, :o] = nm
    rec[:, o] = 10
    rec[:, o + 1:o + 1 + L] = reads
    rec[:, o + 1 + L] = 10
    rec[:, o + 2 + L] = ord("+")
    rec[:, o + 3 + L] = 10
    rec[:, o + 4 + L:o + 4 + 2 * L] = ord("I")
    rec[:, o + 4 + 2 * L] = 10
    rec.tofile(path)
    _pad_if_32k(path)


def write_fasta_fast(path: str, reads: np.ndarray, tag: str = "r") -> None:
    n, L = reads.shape
    nm = _names(n, b">" + tag.encode())
    rec = np.empty((n, nm.shape[1] + 1 + L + 1), dtype=np.uint8)
    o = nm.shape[1]
    rec[:, :o] = nm
    rec[:, o] = 10
    rec[:, o + 1:o + 1 + L] = reads
    rec[:, o + 1 + L] = 10
    rec.tofile(path)
    _pad_if_32k(path)


def config_c1(d: str, genome_len=4_600_000, coverage=30, seed=1) -> str:
    """BASELINE.json configs[0]: E. coli-sized genome, one library, 100 bp SE single-line FASTA, err 0.5 %, K=31 (SURVEY 8d C1)."""
    g = genome(genome_len, seed)
    n = genome_len * coverage // 100
    write_fasta_fast(os.path.join(d, "c1.fa"), se_reads(g, n, 100, 0.005, seed + 100), "e")
    cfg = os.path.join(d, "c1.cfg")
    write_config(cfg, 100, [{"avg_ins": 200, "files": [("f", os.path.join(d, "c1.fa"))]}])
    return cfg


def config_c2(d: str, genome_len=10_000_000, coverage=30, seed=42) -> str:
    """BASELINE.json configs[1] shape at a size the reference finishes in about a minute: 150 bp PE FASTQ q1/q2, insert 300, err 0.1 %."""
    g = genome(genome_len, seed)
    r1, r2 = pe_reads(g, genome_len * coverage // 300, 150, 300, 0.001, seed + 1)
    write_fastq_fast(os.path.join(d, "c2_1.fq"), r1, "p")
    write_fastq_fast(os.path.join(d, "c2_2.fq"), r2, "p")
    cfg = os.path.join(d, "c2.cfg")
    write_config(cfg, 150, [{"avg_ins": 300, "files": [("q1", os.path.join(d, "c2_1.fq")), ("q2", os.path.join(d, "c2_2.fq"))]}])
    return cfg


def config_c5(d: str, genome_len=20_000_000, seed=5) -> str:
    """BASELINE.json configs[4] (SURVEY 8d C5): three libraries -- rank1 avg_ins=200 q1/q2 150 bp; rank2 avg_ins=500 f1/f2 100 bp
    FASTA; rank3 avg_ins=2000 reverse_seq=1 asm_flags=3 f= + q= SE -- about 30x in total, planted repeats so the graph branches."""
    g = genome(genome_len, seed, repeat=(3000, 6))
    j = lambda n: os.path.join(d, n)
    a1, a2 = pe_reads(g, genome_len * 15 // 300, 150, 200 + 100, 0.002, seed + 1)
    write_fastq_fast(j("c5_a1.fq"), a1, "a"); write_fastq_fast(j("c5_a2.fq"), a2, "a")
    b1, b2 = pe_reads(g, genome_len * 10 // 200, 100, 500, 0.002, seed + 2)
    write_fasta_fast(j("c5_b1.fa"), b1, "b"); write_fasta_fast(j("c5_b2.fa"), b2, "b")
    write_fasta_fast(j("c5_c.fa"), se_reads(g, genome_len * 3 // 100, 100, 0.002, seed + 3), "c")
    write_fastq_fast(j("c5_d.fq"), se_reads(g, genome_len * 2 // 120, 120, 0.002, seed + 4), "d")
    cfg = j("c5.cfg")
    write_config(cfg, 150, [
        {"avg_ins": 200, "files": [("q1", j("c5_a1.fq")), ("q2", j("c5_a2.fq"))]},
        {"avg_ins": 500, "files": [("f1", j("c5_b1.fa")), ("f2", j("c5_b2.fa"))]},
        {"avg_ins": 2000, "reverse_seq": 1, "asm_flags": 3, "files": [("f", j("c5_c.fa")), ("q", j("c5_d.fq"))]},
    ])
    return cfg


# ---------------------------------------------------------------- graph motifs for the tip and edge phases
# Error-free reads on fresh random sequence, so that every link's multiplicity is exactly the number of reads that cross it.
# A "ring" is a circular backbone covered by reads of length K + c*s tiled every s bases: every ring link is crossed by exactly c
# reads and the ring has no dead end.  Branches hang off ring k-mers ("junctions"); each branch string is read `copies` times whole.
MOTIFS = ("cut", "tie", "conflict", "cascade", "isolated", "thin_orphan", "thin_multi", "lollipop", "hairpin", "figure8", "bubble",
          "ring", "large", "barrier")
_TILE = 10


class _Motifs:
    def __init__(self, K: int, seed: int):
        self.K, self.rng = K, np.random.default_rng(seed)
        self.reads: list[tuple[bytes, int]] = []       # (sequence, copies)
        self.walks: list[tuple[bytes, int, bytes]] = []  # claimed tip walks: (dead-end k-mer, linear nodes walked, k-mer it stops at)
        self.expect = {"nodes": 0, "dead_ends": 0, "junctions": 0}

    def seq(self, n: int) -> bytes:
        return _ACGT[self.rng.integers(0, 4, size=n)].tobytes()

    def other(self, *avoid) -> bytes:
        return bytes([int(self.rng.choice([b for b in b"ACGT" if b not in avoid]))])

    def ring(self, G: int, c: int) -> bytes:
        G = -(-max(G, self.K + 2) // _TILE) * _TILE
        C = self.seq(G)
        R = self.K + c * _TILE
        C2 = C * (R // G + 2)
        for j in range(0, G, _TILE):
            self.reads.append((C2[j:j + R], 1))
        self.expect["nodes"] += G
        return C

    def kmer(self, C: bytes, p: int) -> bytes:
        return (C * (self.K // len(C) + 2))[p % len(C):p % len(C) + self.K]

    def left_tip(self, C: bytes, p: int, m: int, copies: int, avoid=b"") -> bytes:
        """a branch of m linear nodes and a dead end arriving at ring k-mer p from its left"""
        J = self.kmer(C, p)
        T = self.seq(m) + self.other(C[(p - 1) % len(C)], *avoid)
        self.reads.append((T + J, copies))
        self.walks.append(((T + J)[:self.K], m, J))
        self.expect["nodes"] += m + 1
        self.expect["dead_ends"] += 1
        return T

    def right_tip(self, C: bytes, p: int, m: int, copies: int, avoid=b"") -> bytes:
        J = self.kmer(C, p)
        T = self.other(C[(p + self.K) % len(C)], *avoid) + self.seq(m)
        self.reads.append((J + T, copies))
        self.walks.append((_rc_bytes((J + T)[-self.K:]), m, _rc_bytes(J)))
        self.expect["nodes"] += m + 1
        self.expect["dead_ends"] += 1
        return T

    def tip(self, C, p, m, copies):
        return (self.left_tip if self.rng.random() < 0.5 else self.right_tip)(C, p, m, copies)


def _rc_bytes(s: bytes) -> bytes:
    return _COMP[np.frombuffer(s, dtype=np.uint8)[::-1]].tobytes()


def _motif(M: _Motifs, kind: str, i: int) -> None:
    """one instance of `kind` (i: instance number, picks the variant)"""
    K, e = M.K, M.expect
    if kind == "cut":            # chains of 2K-2 .. 2K+1 linear nodes: clipped up to 2K-1
        C = M.ring(2 * K, 3)
        M.tip(C, 0, 2 * K - 2 + i % 4, 2)
        e["junctions"] += 1
    elif kind == "tie":          # the tip's link equals the ring's (kept) or is one below (clipped)
        C = M.ring(2 * K, 3)
        M.tip(C, 0, K, 3 if i % 2 == 0 else 2)
        e["junctions"] += 1
    elif kind == "conflict":     # 2 or 3 tips into J1; J1 -> path -> J2 on a ring; after the first clip(s) J1 is linear
        ntips = 2 + i % 2
        covs = [2, 3, 4][:ntips]
        near = (i // 2) % 2 == 0        # the last tip's walk reaches J2 (else it passes 2K nodes and gives up)
        cr = sum(covs) + (i // 4) % 2   # J2: the merged branch ties with the ring or is one below it
        C = M.ring(2 * K, cr)
        J2 = M.kmer(C, 0)
        d = 1 if near else 2 * K
        J1 = M.seq(K)
        P = M.seq(d - 1) + M.other(C[-1]) if d > 1 else M.other(C[-1], J1[-1:][0])
        used = b""
        for c in covs:
            m = int(M.rng.integers(1, max(2, K - 2 - d)))
            T = M.seq(m) + M.other(*used)
            used += T[-1:]
            M.reads.append((T + J1 + P + J2, c))
            M.walks.append(((T + J1 + P + J2)[:K], m, J1))
            e["nodes"] += m + 1
        e["nodes"] += K + d              # J1 and the d + K - 1 linear nodes on to J2
        e["dead_ends"] += ntips
        e["junctions"] += 2
    elif kind == "cascade":      # A3 -> J3 <- Q3 - J2 - Q2 -> J1 <- Q1 - J0 (ring): each clip turns the next junction into a dead end
        C = M.ring(2 * K, 6)
        J0 = M.kmer(C, 0)
        J1, J2, J3 = M.seq(K), M.seq(K), M.seq(K)
        u = lambda: int(M.rng.integers(1, K // 2 + 1))
        U1 = M.other(C[K % len(C)]) + M.seq(u())
        U2 = M.seq(u())
        U3 = M.other(U2[0]) + M.seq(u())
        U2 = U2[:-1] + M.other(U1[-1]) if len(U2) > 1 else M.other(U1[-1], U3[0])
        M.reads += [(J0 + U1 + J1, 5), (J2 + U2 + J1, 4), (J2 + U3 + J3, 3)]
        m = int(M.rng.integers(1, 2 * K))
        T = M.seq(m) + M.other(U3[-1])
        M.reads.append((T + J3, 2))
        M.walks.append(((T + J3)[:K], m, J3))
        e["nodes"] += 3 * K + len(U1) + len(U2) + len(U3) - 3 + 3 + m + 1
        e["dead_ends"] += 1
        e["junctions"] += 4
    elif kind == "isolated":     # a lone path: both ends are dead ends; 2K-2 .. 2K+1 linear nodes between them
        m = 2 * K - 2 + i % 4
        S = M.seq(m + K + 1)
        M.reads.append((S, 2))
        M.walks.append((S[:K], m, _rc_bytes(S[-K:])))
        e["nodes"] += m + 2
        e["dead_ends"] += 2
    elif kind == "thin_orphan":  # a frequency-one tip whose last h nodes a second read covers: THIN stops at a non-single node
        C = M.ring(2 * K, 3)
        m = int(M.rng.integers(K // 2 + 2, 2 * K - 1))
        T = M.left_tip(C, 0, m, 1)
        h = int(M.rng.integers(1, min(m, K)))
        M.reads.append(((T + M.kmer(C, 0))[-(K + h):], 1))
        e["junctions"] += 1
    elif kind == "thin_multi":   # three frequency-one tips on each side of one ring k-mer: one THIN commit per round and junction
        C = M.ring(2 * K, 3)
        l, r = b"", b""
        for _ in range(3):
            l += M.left_tip(C, 0, int(M.rng.integers(1, 2 * K)), 1, avoid=l)[-1:]
            r += M.right_tip(C, 0, int(M.rng.integers(1, 2 * K)), 1, avoid=r)[:1]
        e["junctions"] += 1
    elif kind == "lollipop":     # a loop leaving and re-entering one junction, with a tail too long to clip
        C = M.ring(2 * K, 3)
        M.tip(C, 0, 2 * K + 3, 2)
        e["junctions"] += 1
    elif kind == "hairpin":      # J -> w -> rc(w) -> rc(J): a unipath that folds back onto itself and re-enters J by the same link
        C = M.ring(2 * K, 3)
        J = M.kmer(C, 0)
        w = M.other(C[K % len(C)]) + M.seq(int(M.rng.integers(1, 2 * K)))
        M.reads.append((J + w + _rc_bytes(J + w), 2))
        e["nodes"] += len(w) + (K - 1) // 2   # J + w + rc(J + w) has len(w) + (K + 1) / 2 distinct k-mers, J among them
        e["junctions"] += 1
    elif kind == "figure8":      # two rings through one k-mer
        J = M.seq(K)
        G = -(-2 * K // _TILE) * _TILE
        a = M.seq(G - K)
        b = M.other(a[0]) + M.seq(len(a) - 2) + M.other(a[-1])
        for x in (a, b):
            C = J + x
            R = K + 3 * _TILE
            C2 = C * (R // G + 2)
            M.reads += [(C2[j:j + R], 1) for j in range(0, G, _TILE)]
        e["nodes"] += 2 * G - 1
        e["junctions"] += 1
    elif kind == "bubble":       # J1 -> J2 along the ring (d steps) and along a bypass (t+K steps); d = 1 is a length-1 edge
        lens = [x for x in (100, 101, 200, 201) if x > K]
        d = [1, 100, 101, 200][i % 4]
        L = lens[(i // 4) % len(lens)]
        C = M.ring(d + 2 * K + 20, 3)
        J1, J2 = M.kmer(C, 0), M.kmer(C, d)
        t = L - K
        v = M.other(C[K]) + M.seq(t - 2) + M.other(C[d - 1]) if t >= 2 else M.other(C[K], C[d - 1])
        M.reads.append((J1 + v + J2, 3))
        e["nodes"] += t + K - 1
        e["junctions"] += 2
    elif kind == "barrier":      # A's clip turns X into a dead end; X's clip at Y makes Y linear; tip c, a tie at Y before, then
        C = M.ring(2 * K, 8)     # walks on to Z and is clipped there: in the same sweep only if c comes after X in iteration order
        Z = M.kmer(C, 0)
        Y, X = M.seq(K), M.seq(K)
        P = M.other(C[K % len(C)])
        Q = M.seq(int(M.rng.integers(1, K + 1)))
        mc = int(M.rng.integers(1, K - 2))
        Tc = M.other(Q[0]) + M.seq(mc)
        M.reads += [(Z + P + Y + Q + X, 3), (Z + P + Y + Tc, 4)]
        M.walks.append((_rc_bytes((Y + Tc)[-K:]), mc, _rc_bytes(Y)))
        mA = int(M.rng.integers(1, 2 * K))
        T = M.seq(mA) + M.other(Q[-1])
        M.reads.append((T + X, 2))
        M.walks.append(((T + X)[:K], mA, X))
        e["nodes"] += (K + 1) + (len(Q) + K) + (mc + 1) + (mA + 1)
        e["dead_ends"] += 2
        e["junctions"] += 3
    elif kind == "ring":         # no branch at all: no edge, no vertex
        M.ring(2 * K, 3)
    elif kind == "large":        # a long ring with a short minority tip every 12 bases: thousands of minor candidates per ring
        n = 40
        C = M.ring(n * 12, 3)
        for j in range(n):
            M.tip(C, 12 * j, 3, 2)
        e["junctions"] += n
    else:
        raise ValueError(kind)


def motif_reads(kind: str, K: int, copies: int, seed: int = 0) -> _Motifs:
    """`copies` instances of one motif on fresh random sequence; .reads, .walks and .expect describe what was built"""
    M = _Motifs(K, seed * 1000 + MOTIFS.index(kind) * 7 + K)
    for i in range(copies):
        _motif(M, kind, i)
    return M


def write_motif_scenario(d: str, kinds, K: int, copies: int, seed: int = 0) -> tuple[str, list]:
    """One FASTA library holding `copies` instances of each motif in `kinds` (reads shuffled); returns (config path, motif sets).
    The reads are checked first (check_motifs): a chance k-mer collision between instances would make a different graph."""
    sets = [motif_reads(k, K, copies, seed) for k in kinds]
    check_motifs(sets, K)
    rng = np.random.default_rng(seed + 17 * K)
    reads = [s for M in sets for s, c in M.reads for _ in range(c)]
    order = rng.permutation(len(reads))
    fa = os.path.join(d, "motif.fa")
    with open(fa, "wb") as f:
        for n, j in enumerate(order):
            f.write(b">m%d\n" % n + reads[j] + b"\n")
    _pad_if_32k(fa)
    cfg = os.path.join(d, "motif.cfg")
    write_config(cfg, max(len(r) for r in reads), [{"avg_ins": 200, "files": [("f", fa)]}])
    return cfg, sets


_CODE = {65: 0, 67: 1, 84: 2, 71: 3}             # the reference's 2-bit codes: A0 C1 T2 G3 (complement = code ^ 2)
_ORD = bytes.maketrans(b"ACTG", b"abcd")          # byte order == code order, so canonical = the smaller translated string


def _canon(k: bytes) -> tuple[bytes, bool]:
    r = _rc_bytes(k)
    return (k, True) if k.translate(_ORD) < r.translate(_ORD) else (r, False)


def debruijn(reads, K: int) -> dict:
    """The canonical k-mer graph of (sequence, copies) reads as pass 1 builds it: node -> [l[4], r[4]], counters capped at 63."""
    g: dict = {}
    for s, copies in reads:
        for j in range(len(s) - K + 1):
            k, fwd = _canon(s[j:j + K])
            prev = _CODE[s[j - 1]] if j > 0 else None
            nxt = _CODE[s[j + K]] if j + K < len(s) else None
            if not fwd:
                prev, nxt = (nxt ^ 2 if nxt is not None else None), (prev ^ 2 if prev is not None else None)
            lr = g.setdefault(k, [[0] * 4, [0] * 4])
            if prev is not None:
                lr[0][prev] = min(63, lr[0][prev] + copies)
            if nxt is not None:
                lr[1][nxt] = min(63, lr[1][nxt] + copies)
    return g


def _degree(lr):
    return sum(1 for x in lr[0] if x), sum(1 for x in lr[1] if x)


def graph_shape(g: dict) -> dict:
    shape = {"nodes": len(g), "dead_ends": 0, "junctions": 0}
    for lr in g.values():
        i, o = _degree(lr)
        if i + o == 1:
            shape["dead_ends"] += 1
        elif not (i == 1 and o == 1):
            shape["junctions"] += 1
    return shape


def tip_walk(g: dict, start: bytes, K: int) -> tuple[int, bytes]:
    """From a dead end over linear nodes: (linear nodes passed, canonical k-mer of the first non-linear node)"""
    cur, _ = _canon(start)
    i, o = _degree(g[cur])
    assert i + o == 1, f"{start!r} is not a dead end"
    ori = cur if o == 1 else _rc_bytes(cur)        # oriented so that its one link points right
    m = 0
    while True:
        k, fwd = _canon(ori)
        lr = g[k]
        if m or k != cur:
            i, o = _degree(lr)
            if not (i == 1 and o == 1):
                return m, k
            m += 1
        c = next(c for c in range(4) if lr[1][c]) if fwd else next(c for c in range(4) if lr[0][c]) ^ 2
        ori = ori[1:] + b"ACTG"[c:c + 1]


def check_motifs(sets, K: int) -> dict:
    """Asserts that the reads of the motif sets build the graph they claim: node, dead-end and junction counts, and every claimed
    tip walk's length and end node.  Returns the graph."""
    g = debruijn([r for M in sets for r in M.reads], K)
    want = {k: sum(M.expect[k] for M in sets) for k in ("nodes", "dead_ends", "junctions")}
    assert graph_shape(g) == want, (graph_shape(g), want)
    for M in sets:
        for start, m, end in M.walks:
            assert tip_walk(g, start, K) == (m, _canon(end)[0]), (start, m, end)
    return g


# ---------------------------------------------------------------- long read paths for pass 2
def figure8_long(K: int, revs: list[int], seed: int = 0) -> tuple[_Motifs, list[int]]:
    """One long read per entry of `revs`, each on its own random sequence and read twice: an entry X of 3K bases ending in G, then a
    junction k-mer J, then `revs` turns, each a loop a = A..C (4 bases) or b = G...T (5 bases) chosen at random, followed by J again.
    The loops differ in their first and last base, so J branches on both sides; X's 3K k-mers make a tip too long to clip.  The
    read's path is revs + 1 edges (the entry edge, then one loop edge per turn), so its .path record holds (revs + 1) & 255 entries:
    the reference counts a path in an unsigned char.  A path of fewer than 3 edges (revs = 1) gets no record.  Returns (the motif
    set, the expected record count of each read, None for no record).
    Reads are 4K + revs * (K + 4.5) bases on average; keep them at or below about 34,000 bases (K = 127: at most 257 turns), the
    longest the reference was seen to handle (it crashed in pass 1 on reads of 47,707 bases)."""
    M = _Motifs(K, seed * 1000 + 991 + K)
    expect = []
    for n in revs:
        J = M.seq(K)
        a = b"A" + M.seq(2) + b"C"
        b = b"G" + M.seq(3) + b"T"
        X = M.seq(3 * K - 1) + b"G"
        turns = [a if t else b for t in M.rng.integers(0, 2, size=n)]
        if n >= 2:                       # both loops at least once: J has two successors in every read
            turns[0], turns[1] = a, b
        M.reads.append((X + J + b"".join(t + J for t in turns), 2))
        M.walks.append(((X + J)[:K], 3 * K - 1, J))
        M.expect["nodes"] += 3 * K + 1 + (K + 3 if a in turns else 0) + (K + 4 if b in turns else 0)
        M.expect["dead_ends"] += 1
        M.expect["junctions"] += 1
        expect.append((n + 1) & 255 if n >= 2 else None)
    return M, expect


def write_pass2_scenario(d: str, K: int, revs: list[int], inst: int = 1, seed: int = 0, paired: bool = False, max_rd_len: int = 0,
                         n_genome: int = 0, rings: int = 0) -> tuple[str, list[int], int]:
    """`inst` figure8_long reads per entry of `revs` (each read twice), the reads of `rings` branch-free rings (each once), and
    `n_genome` reads of ragged lengths up to `max_rd_len` from a random genome, shuffled into one FASTA library; or with `paired` only
    the figure-eight reads, in an f1/f2 pair of files (the two copies of a read are mates).  max_rd_len = 0: the longest read.
    Returns (config path, the expected .path record count of every figure-eight read that gets a record, in read-stream order, the
    number of ring reads: pass 2 counts each one as deleted, since no k-mer of a ring lies in an edge)."""
    M, expect = figure8_long(K, list(revs) * inst, seed)
    R = _Motifs(K, seed * 1000 + 997 + K)
    for _ in range(rings):
        R.ring(2 * K, 3)
    check_motifs([M, R], K)
    rng = np.random.default_rng(seed + 31 * K)
    reads = [(s, e) for (s, _), e in zip(M.reads, expect)]
    mrl = max_rd_len or max(len(s) for s, _ in reads)
    assert max(len(s) for s, _ in reads) <= mrl
    j = lambda n: os.path.join(d, n)
    if paired:
        order = rng.permutation(len(reads))
        write_long(j("p2_1.fa"), [reads[i][0] for i in order], fastq=False, tag="a")
        write_long(j("p2_2.fa"), [reads[i][0] for i in order], fastq=False, tag="b")
        files = [("f1", j("p2_1.fa")), ("f2", j("p2_2.fa"))]
        counts = [reads[i][1] for i in order for _ in range(2)]
        assert not (n_genome or rings)
    else:
        reads = reads * 2
        if n_genome:
            g = genome(max(20 * mrl, 40000), seed + 7)
            lens = rng.integers(K + 1, mrl + 1, size=n_genome)
            lens[: min(4, n_genome)] = mrl                     # the full row, word for word
            reads += [(r, None) for r in long_reads_of_lengths(g, [int(x) for x in lens], seed + 8, err=0.002, n_rate=0)]
        reads += [(r, None) for r, _ in R.reads]
        order = rng.permutation(len(reads))
        write_long(j("p2.fa"), [reads[i][0] for i in order], fastq=False, tag="r")
        files = [("f", j("p2.fa"))]
        counts = [reads[i][1] for i in order]
    counts = [c for c in counts if c is not None]
    cfg = j("p2.cfg")
    write_config(cfg, mrl, [{"avg_ins": 300 if paired else 200, "files": files}])
    return cfg, counts, len(R.reads)
