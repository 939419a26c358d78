"""A plain-Python model of the `map` stage's contig side and read placement, written from SOAPdenovo2's behaviour so that the tests
can say what the stage must print and write for a designed input, and why:

- read_contigs: how prlContig2nodes reads `.contig` -- readseqpar's pass over fgets pieces of 4949 bytes for the stats line and the
  maximum length, then readseq1by1's pieces of 4999 bytes, each record cut at that maximum (the cut counts the '\\n'), names through
  sscanf "%s" and getID, bytes before the first '>' dropped, records shorter than K + 2 dropped.
- ContigTable: the contig k-mer table -- canonical k-mer -> (contig id, position mod 2^24, twin) of its first instance, or DELETED once
  seen twice.
- place: searchKmer and parse1read -- groups in order of first hit, `multi` from ALIGNLEN, counter2 under K < 32 / K > 32, the strict
  `>` that gives a tie to the earlier group, and the placement formulas in u32 arithmetic.
- record: recordAlldgn's `.readOnContig.gz` lines and the (len, contig, pos) heads of the `.readInGap.gz` records for read pairs.
"""
import hashlib
import struct

DELETED = "deleted"
_CODES = bytes(((c & 6) >> 1) if (65 <= c <= 90 or 97 <= c <= 122) else (0 if c == 46 else 255) for c in range(256))   # base2int, '.' -> A
_DROP = bytes(c for c in range(256) if _CODES[c] == 255)


class _Fgets:
    """fgets(str, size, fp) over a file's bytes; eof is feof after the last call"""

    def __init__(self, text):
        self.t, self.at, self.eof = text, 0, False

    def next(self, size):
        t, at = self.t, self.at
        if at == len(t):
            self.eof = True
            return None
        lim = min(len(t), at + size - 1)
        nl = t.find(b"\n", at, lim)
        end = nl + 1 if nl >= 0 else lim
        self.eof = nl < 0 and end - at < size - 1
        self.at = end
        return t[at:end].split(b"\0", 1)[0]   # strlen(str)


def _name(piece, old):
    tok = piece[1:].split()
    return tok[0] if tok else old   # sscanf "%s" with nothing to read leaves the name as it was


def read_contigs(text, K):
    """-> (stats line, [(id, base codes)] of the kept contigs, k-mer total)"""
    f, num, mx, mn, nl, n, name = _Fgets(text), -1, 10, 1000, 10, 0, b""
    while (s := f.next(4950)) is not None:   # readseqpar
        if s[:1] != b">":
            n += len(s) - 1
            continue
        if num >= 0:
            mx, mn = max(mx, n), min(mn, n)
        n, num, name = 0, num + 1, _name(s, name)
        nl = max(nl, len(name))
    mx, mn = max(mx, n), min(mn, n)
    stats = f"{num + 1} contig(s), maximum sequence length {mx}, minimum sequence length {mn}, maximum name length {nl}."
    f, name, kept = _Fgets(text), b"", []

    def record():   # readseq1by1 with gStr NULL
        nonlocal name
        codes = b""
        while (s := f.next(5000)) is not None:
            if s[:1] == b"#":
                continue
            if s[:1] == b">":
                name = _name(s, name)
                break
            codes += s[:mx - len(codes)].translate(_CODES, _DROP)
        return codes

    record()
    ordinal = 0
    while not f.eof:   # prlContig2nodes
        cid = _get_id(name)
        codes = record()
        ordinal += 1
        if len(codes) >= K + 1 and len(codes) >= K + 2:
            kept.append((cid if cid > 0 else ordinal, codes))
    return stats, kept, sum(len(c) - K + 1 for _, c in kept)


def _get_id(name):
    """getID: atoi of a name that starts with a digit, else 0"""
    if not name[:1].isdigit():
        return 0
    d = 0
    while d < len(name) and name[d:d + 1].isdigit():
        d += 1
    return int(name[:d])


def digest(codes):
    """64-bit FNV-1a of base codes, one byte each (tests/host_read_contigs.cpp prints the same)"""
    h = 1469598103934665603
    for b in codes:
        h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def _kmers(codes, K):
    """(j, canonical word, smaller) for each k-mer: smaller when the forward word is below its reverse complement"""
    mask, w, b = (1 << (2 * K)) - 1, 0, 0
    for j, c in enumerate(codes):
        w = ((w << 2) | c) & mask
        b = (b >> 2) | ((c ^ 2) << (2 * (K - 1)))
        if j >= K - 1:
            yield j - K + 1, (w if w < b else b), w < b


class ContigTable:
    def __init__(self, kept, K):
        self.K, self.t, self.seen = K, {}, {}   # seen: instances of each key
        for cid, codes in kept:
            for j, key, smaller in _kmers(codes, K):
                self.seen[key] = self.seen.get(key, 0) + 1
                if key not in self.t:
                    self.t[key] = (cid, j & 0xFFFFFF, 0 if smaller else 1)
                else:
                    self.t[key] = DELETED

    def distinct(self):
        return len(self.t)


def _i32(x):
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


class Placement:
    """parse1read's result for one read: ctg 0 when not placed; groups / deleted say why"""
    __slots__ = ("ctg", "pos", "orien", "footprint", "groups", "deleted", "tie")

    def __repr__(self):
        return (f"ctg {self.ctg} pos {self.pos} orien {self.orien} footprint {self.footprint}; groups (contig, hits) in first-hit "
                f"order {self.groups}; {self.deleted} k-mer(s) on deleted keys")


def place(codes, table, alignlen, ctg_len, bal_edge):
    """searchKmer + parse1read; ctg_len / bal_edge: .ContigIndex's length and bal_edge by contig id"""
    K, p = table.K, Placement()
    p.ctg, p.pos, p.orien, p.footprint, p.groups, p.deleted, p.tie = 0, 0, "", 0, [], 0, False
    if len(codes) < K + 1:
        return p
    groups, hits = {}, []
    for j, key, smaller in _kmers(codes, K):
        e = table.t.get(key)
        if e is DELETED:
            p.deleted += 1
        if e is None or e is DELETED:
            continue
        hits.append((j, e, smaller))
        g = groups.setdefault(e[0], [len(hits) - 1, 0])
        g[1] += 1
    multi = max(2, min(len(codes), alignlen) - K + 1)
    counter = counter2 = max_occ = 0
    best = None
    for cid, (h, flag) in groups.items():
        p.groups.append((cid, flag))
        if (K < 32 and flag >= 2) or K > 32:
            counter2 += 1
        if flag < multi:
            continue
        counter += 1
        if flag > max_occ:   # strict: a tie stays with the earlier group
            best, max_occ, p.tie = hits[h], flag, False
        elif flag == max_occ:
            p.tie = True
    if not counter:
        return p
    p.footprint = 1 if counter2 > 1 else 0
    j, (cid, npos, twin), smaller = best
    i = j + 1
    if twin == (1 if smaller else 0):
        p.orien, p.ctg = "-", cid + bal_edge[cid] - 1
        p.pos = _i32(ctg_len[cid] - npos - K - i + 1)
    else:
        p.orien, p.ctg, p.pos = "+", cid, _i32(npos - i + 1)
    return p


def contig_index(text):
    """basicContigInfo: (length, bal_edge) lists indexed by contig id"""
    lines = text.splitlines()
    n = int(lines[0].split()[1])
    length, bal_edge, k = [0] * (n + 2), [0] * (n + 2), 0
    for line in lines[2:]:
        idx, ln, bal = (int(x) for x in line.split()[:3])
        k += 1
        length[k], bal_edge[k] = ln, bal + 1
        if bal:
            k += 1
            length[k], bal_edge[k] = ln, 1 - bal
    return length, bal_edge


def record(placements, reads, ins):
    """recordAlldgn for read pairs (mates interleaved): the .readOnContig.gz lines and the (len, ctg, pos) heads of the
    .readInGap.gz records, in file order"""
    ctg = [p.ctg for p in placements]
    pos = [p.pos for p in placements]
    on, gap = [], []
    for t, p in enumerate(placements):
        rd1gap = rd2gap = False
        cid = ctg[t]
        if t % 2 == 1:
            placed, g = (t - 1, t) if ctg[t] < 1 and ctg[t - 1] > 0 else (t, t - 1) if ctg[t] > 0 and ctg[t - 1] < 1 else (None, None)
            if placed is not None:
                ctg[g], pos[g] = ctg[placed], pos[placed] + ins - len(reads[g])
                gap.append((len(reads[g]), ctg[g], pos[g]))
                rd2gap, rd1gap = g == t, g == t - 1
        if cid < 1:
            continue
        on.append(f"{t + 1}\t{cid}\t{pos[t]}\t{p.orien}")
        if t % 2 == 0:
            continue
        for r, skip in ((t - 1, rd1gap), (t, rd2gap)):
            if placements[r].footprint and not skip:
                gap.append((len(reads[r]), ctg[r], pos[r]))
    return on, gap


def read_gap_heads(raw):
    """(len, ctg, pos) of each .readInGap record: three ints, then len / 4 + 1 bytes of packed bases"""
    out, o = [], 0
    while o < len(raw):
        ln, c, ps = struct.unpack_from("<iii", raw, o)
        out.append((ln, c, ps))
        o += 12 + ln // 4 + 1
    return out


def sha(data):
    return hashlib.sha256(data).hexdigest()
