"""GPU decode of records the fast path cannot handle: `N`, lower case, '.', other non-letters, CRLF, reads longer than max_rd_len,
reads shorter than K+1, and a reverse_seq library, mixed with clean records in the same chunk.  The engine fed the raw text must hold
exactly what an engine fed the already-decoded reads (plain upper-case ACGT) holds: the same reads kept, k-mer instances, coverage
histogram and node table (k-mers, links, first-occurrence ranks), and the counters must match a host decode."""
import random

import pytest

from soapdenovo2_b200 import api

pytestmark = pytest.mark.gpu

K, MAXLEN = 31, 100


@pytest.fixture(params=["direct", "aggregated"], autouse=True)
def _insert_mode(request, monkeypatch):
    monkeypatch.setenv("PGB200_SKM", "0" if request.param == "direct" else "1")


def _decode(seq: bytes, reverse: bool) -> str:
    """The general rules: the first MAXLEN characters of the line, letters and '.' kept (A0 C1 T2 G3 from (c & 6) >> 1, '.' -> A)."""
    codes = [0 if c == ord(".") else (c & 6) >> 1 for c in seq[:MAXLEN] if ord("a") <= (c | 0x20) <= ord("z") or c == ord(".")]
    if reverse:
        codes = [c ^ 2 for c in reversed(codes)]
    return "".join("ACTG"[c] for c in codes)


def _records(rng, n):
    out = []
    for i in range(n):
        kind = i % 9
        L = rng.choice([20, K, K + 1, 60, 80, 99, 100, 101, 130]) if kind == 8 else rng.randint(K + 1, MAXLEN)
        s = "".join(rng.choice("ACGT") for _ in range(L))
        if kind == 1:
            s = s.lower()
        elif kind == 2:
            s = "".join(c if rng.random() > 0.05 else "N" for c in s)
        elif kind == 3:
            s = "".join(c if rng.random() > 0.05 else "." for c in s)
        elif kind == 4:
            s = "".join(c + ("-" if rng.random() < 0.03 else "") for c in s)
        elif kind == 5:
            s = "".join(c if rng.random() > 0.3 else c.lower() for c in s)
        out.append((s.encode(), kind == 6))   # kind 6: CRLF line ends
    # long enough for the fast decode (>= K+1 bytes) but fewer than K+1 bases once the non-letters are dropped: the fix-up takes the
    # read out of "reads kept" again
    for L in (K - 1, K, K + 1):
        s = "".join(rng.choice("ACGT") for _ in range(L))
        out.append((("-" * 3 + s[:L // 2] + "*" + s[L // 2:]).encode(), False))
    return out


def _fasta(recs):
    return b"".join(b">r%d%s\n%s%s\n" % (i, b"\r" if crlf else b"", s, b"\r" if crlf else b"") for i, (s, crlf) in enumerate(recs))


def _fastq(recs):
    return b"".join(b"@r%d\n%s\n+\n%s\n" % (i, s, b"I" * len(s)) for i, (s, _) in enumerate(recs))


def _redone(err):
    line = [l for l in err.splitlines() if "decoded by the general rules" in l][-1]
    return int(line.split(",")[1].split()[0])


def test_clean_text_takes_the_fast_decode_only(capfd):
    """Upper-case ACGT reads of every length up to max_rd_len (every tail of a 4-byte group): no record goes to k_decode_fix."""
    rng = random.Random(3)
    seqs = ["".join(rng.choice("ACGT") for _ in range(L)) for L in range(1, MAXLEN + 1) for _ in range(3)]
    eng = api.PregraphEngine(K=K, P=3, initG=1, max_rd_len=MAXLEN, verbose=1)
    capfd.readouterr()
    eng.feed_text(b"".join(b">c%d\n%s\n" % (i, s.encode()) for i, s in enumerate(seqs)), fastq=False)
    eng.feed_text(b"".join(b"@c%d\n%s\n+\n%s\n" % (i, s.encode(), b"I" * len(s)) for i, s in enumerate(seqs)), fastq=True, ord_base=len(seqs))
    st = eng.finish_pass1()
    assert st.records == 2 * len(seqs)
    assert _redone(capfd.readouterr().err) == 0
    eng.close()


def test_flagged_records_decode_like_clean_ones(capfd):
    rng = random.Random(7)
    fa, fq = _records(rng, 3000), _records(rng, 2000)
    fq = [(s, False) for s, _ in fq]
    want_fa = [_decode(s, False) for s, _ in fa]
    want_fq = [_decode(s, True) for s, _ in fq]
    kept = sum(len(s) >= K + 1 for s in want_fa + want_fq)
    inst = sum(len(s) - K + 1 for s in want_fa + want_fq if len(s) >= K + 1)

    raw = api.PregraphEngine(K=K, P=3, initG=1, max_rd_len=MAXLEN, verbose=1)
    assert raw.feed_text(_fasta(fa), fastq=False, ord_base=0) == len(fa)
    assert raw.feed_text(_fastq(fq), fastq=True, ord_base=len(fa), reverse_seq=1) == len(fq)
    capfd.readouterr()
    st_raw = raw.finish_pass1()
    assert len(fa) // 9 <= _redone(capfd.readouterr().err) <= len(fa) + len(fq)   # every reverse_seq record, and the flagged ones

    clean = api.PregraphEngine(K=K, P=3, initG=1, max_rd_len=MAXLEN)
    clean.feed_text(b"".join(b">c%d\n%s\n" % (i, s.encode()) for i, s in enumerate(want_fa + want_fq)), fastq=False, ord_base=0)
    st_clean = clean.finish_pass1()

    assert (st_raw.records, st_raw.reads_kept, st_raw.instances) == (len(fa) + len(fq), kept, inst)
    assert (st_clean.reads_kept, st_clean.instances, st_clean.distinct) == (kept, inst, st_raw.distinct)
    assert raw.sweeps() == clean.sweeps()
    raw.build_layout()
    clean.build_layout()
    assert raw.dump_nodes() == clean.dump_nodes()
    raw.close()
    clean.close()
