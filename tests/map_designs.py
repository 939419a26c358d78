"""Designed `map` inputs, built from seeds: `.contig` texts that reach the corners of the reference's .contig readers, a contig set
whose k-mers repeat on purpose, the reads that land on those corners, and the minimal graph files `map` reads besides `.contig`."""
import os
import random
import re

from tests import map_model, util

_COMP = str.maketrans("ACGTN", "TGCAN")


def rc(s):
    return s.translate(_COMP)[::-1]


def seq(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def wrap(s, w):
    return "\n".join(s[i:i + w] for i in range(0, len(s), w))


def bases(codes):
    return "".join("ACTG"[c] for c in codes)


def reader_cases(K=31):
    """(name, .contig bytes): the shapes of a .contig that `contig` did not write"""
    rng = random.Random(20261019)
    S = lambda n: seq(rng, n)   # noqa: E731
    cases = []
    for w in (60, 100):
        cases.append((f"wrap{w}", "".join(f">{2 * i + 1} length x cvg_1.0_tip_0\n{wrap(S(rng.randrange(200, 3000)), w)}\n"
                                          for i in range(6)).encode()))
    lens = [4948, 4949, 4950, 4998, 4999, 5000, 9898, 20000]
    for where, at in (("first", 0), ("middle", 4), ("last", len(lens))):
        ls = lens[:at] + [500000] + lens[at:]
        cases.append((f"single_line_longest_{where}", "".join(f">{2 * i + 1}\n{S(n)}\n" for i, n in enumerate(ls)).encode()))
    cases.append(("no_final_newline", f">1\n{wrap(S(700), 100)}\n>3\n{S(400)}".encode()))
    cases.append(("crlf", "".join(f">{2 * i + 1} x\r\n" + wrap(S(500), 60).replace("\n", "\r\n") + "\r\n" for i in range(4)).encode()))
    cases.append(("hash_lines", (f"# made by hand\n>1\n{S(300)}\n# a note\n{S(300)}\n>3\n#{S(6000)}\n{S(200)}\n>5\n{S(250)}\n"
                                 f"#\n").encode()))
    cases.append(("letters", (f">1\n{S(100).lower()}..NNnn{S(100)}xyzRYK{S(50)}0123-*!?{S(80)}\n>3\n"
                              f"{S(60)} {S(60)}\t{S(60)}\n").encode()))
    cases.append(("names", (f"> 12\n{S(200)}\n>\t3 x\n{S(210)}\n>abc\n{S(220)}\n>007\n{S(230)}\n>12abc\n{S(240)}\n"
                            f">5\n{S(250)}\n>5\n{S(260)}\n>ctg\n{S(270)}\n").encode()))
    cases.append(("long_headers", (f">3 {'x' * 5000}\n{S(300)}\n>5 {'ACGT' * 1260}\n{S(300)}\n>7 {'q' * 4946}\n{S(300)}\n"
                                   f">9 {'y' * 4996}\n{S(300)}\n>11\n{S(300)}\n").encode()))
    for mark in ("#", ">"):
        for off in (4949, 4999):
            line = S(off) + mark + ("9 " if mark == ">" else "") + S(3000)
            cases.append((f"{'hash' if mark == '#' else 'gt'}_at_{off}", f">1\n{S(500)}\n>3\n{line}\n>5\n{S(400)}\n".encode()))
    cases.append(("bases_before_first_header", f"{S(150)}\n{S(90)}\n>1\n{S(600)}\n>3\n{S(300)}\n".encode()))
    cases.append(("empty", b""))
    cases.append(("headers_only", b">1\n>3\n>5 x\n"))
    cases.append(("headers_only_no_final_newline", b">1\n>3\n>5"))
    cases.append(("near_cutoff", "".join(f">{2 * i + 1}\n{S(n)}\n" for i, n in enumerate((K, K + 1, K + 2, K + 3, 200))).encode()))
    return cases


def contig_index(kept, Kg, n_min=0):
    """A .ContigIndex for a set of kept contigs: ids 1..N, each its own twin (bal 0), length = contig length - graph K"""
    length = {}
    for cid, codes in kept:
        length.setdefault(cid, max(len(codes) - Kg, 1))
    n = max([n_min, *length])
    body = "".join(f"{i}\t{length.get(i, 100)}\t0\n" for i in range(1, n + 1))
    return f"Edge_num {n} {n}\nindex\tlength\treverseComplement\n{body}"


def sample_pairs(rng, kept, L, n_per=3, max_ctg=8):
    """read pairs off the kept contigs: mate 1 forward, mate 2 reverse-complement"""
    pairs = []
    for _, codes in kept[:max_ctg]:
        s = bases(codes)
        if len(s) < L:
            continue
        for _ in range(n_per):
            pairs.append((s[(p := rng.randrange(len(s) - L + 1)):p + L], rc(s[(q := rng.randrange(len(s) - L + 1)):q + L])))
    return pairs


def table_set(Kg, seed=31):
    """The designed contig set for graph K Kg: (.contig bytes, .ContigIndex text, read pairs, read length)"""
    rng = random.Random(seed + Kg)
    S = lambda n: seq(rng, n)   # noqa: E731
    entries, records, nxt = [], [], [1]

    def add(s, bal=1, name=None, entry=True):
        cid = nxt[0]
        if entry:
            entries.append((cid, max(len(s) - Kg, 1), bal))
            nxt[0] += 1 if bal == 0 else 2
        records.append((name if name is not None else str(cid), s))
        return s

    def gap():   # an id that no record names
        entries.append((nxt[0], 100, 1))
        nxt[0] += 2

    unit, half, pal, sh1, sh2, X = S(200), S(40 + Kg), S(500), S(2 * Kg), S(2 * Kg), S(900)
    c_rep = add(S(800) + unit * 3 + S(800))                    # tandem repeat: keys seen 3 times
    add(S(700) + half + rc(half) + S(700))                     # even-length palindromic segment
    add(pal + rc(pal), bal=0)                                  # a whole palindrome, its own twin
    add(S(600) + sh1 + S(600))
    add(S(500) + sh1 + S(500))                                 # a k-mer run shared on the same strand
    add(S(600) + sh2 + S(600))
    add(S(500) + rc(sh2) + S(500))                             # ... and on opposite strands
    add(X)
    add(rc(X))                                                 # a contig and its reverse complement under another id
    gap()
    P = add(S(1500))
    gap()
    Q = add(S(1500))                                           # tie partners
    add(S(1200), name="ctg_ordinal", entry=False)              # an ordinal id
    add(S(1100), name=records[3][0], entry=False)              # a duplicate id
    for n in sorted({22, 23, 26, 27, Kg + 1, Kg + 2}):
        add(S(n))                                              # around the K + 2 cutoff of each map K
    add(S(900))
    text = "".join(f">{name} length {len(s)}\n{wrap(s, 100)}\n" for name, s in records)
    n = nxt[0] - 1
    index = f"Edge_num {n} {len(entries)}\nindex\tlength\treverseComplement\n" + "".join(f"{i}\t{ln}\t{b}\n" for i, ln, b in entries)
    L = 2 * Kg + 38   # even, so that an even split is a tie, and each half holds several k-mers
    h = L // 2
    kept = [(0, [{"A": 0, "C": 1, "T": 2, "G": 3}[c] for c in s]) for _, s in records]   # sample_pairs takes base codes
    pairs = sample_pairs(rng, kept, L, n_per=4, max_ctg=len(kept))
    designed = [P[-h:] + Q[:L - h], rc(P[-h:] + Q[:L - h]),            # an even split: the earlier group keeps it
                P[-(h - 1):] + Q[:L - h], rc(P[-(h - 1):] + Q[:L - h]),   # one more hit on the later contig
                X[100:100 + L], rc(X[300:300 + L]), unit[:L // 2] + unit[:L - L // 2],   # only deleted keys
                P[-(Kg + 9):] + Q[:L - Kg - 9]]                        # two groups of several hits: the footprint
    for k in (21, 25, Kg):
        designed += [P[-k:] + Q[:L - k], rc(P[-k:] + Q[:L - k])]      # a one-hit group
        designed += [Q[200:200 + n] for n in (k, k + 1, k + 2)]       # reads of length K, K + 1, K + 2
    r = Q[400:400 + L]
    designed += [r[:20] + "N" + r[21:50] + "N" + r[51:], rc(P[700:700 + L]), c_rep[700:700 + L]]
    for i, d in enumerate(designed):
        mate = pairs[i % len(pairs)][0]
        pairs.append((d, mate) if i % 3 else (mate, d))
        if i % 4 == 0:
            pairs.append((d, S(L)))   # a mate that maps nowhere: the pair goes to .readInGap
    return text.encode(), index, pairs, L


def write_graph(d, name, contig, index, Kg, pairs, L, long_reads=False):
    """<d>/<name>.{contig,ContigIndex,preGraphBasic}, the read files and a config: (prefix, config)"""
    g = os.path.join(d, name)
    open(g + ".contig", "wb").write(contig)
    open(g + ".ContigIndex", "w").write(index)
    open(g + ".preGraphBasic", "w").write(f"VERTEX 1000 K {Kg}\n\nEDGEs 1000\n\nMaxReadLen {L} MinReadLen {L} MaxNameLen 256\n")
    r1, r2 = os.path.join(d, name + "_1.fa"), os.path.join(d, name + "_2.fa")
    with open(r1, "w") as f1, open(r2, "w") as f2:
        for i, (a, b) in enumerate(pairs):
            f1.write(f">{i}/1\n{a}\n")
            f2.write(f">{i}/2\n{b}\n")
    cfg = os.path.join(d, name + ".cfg")
    body = f"max_rd_len={L}\n[LIB]\navg_ins=300\nreverse_seq=0\nasm_flags=3\nrank=1\nf1={r1}\nf2={r2}\n"
    if long_reads:
        lr = os.path.join(d, name + "_long.fa")
        open(lr, "w").write("".join(f">{i}\n{wrap(a + b, 70)}\n" for i, (a, b) in enumerate(pairs)))
        body += f"[LIB]\nasm_flags=4\nrd_len_cutoff={4 * L}\nmap_len=35\nf={lr}\n"
    open(cfg, "w").write(body)
    return g, cfg


def ref_stats(stderr):
    """the reference's contig-side lines: (stats line, nodes allocated, k-mers in contigs)"""
    stats = re.search(r"^(\d+ contig\(s\), maximum sequence length .*)$", stderr, re.M).group(1)
    m = re.search(r"^(\d+) node\(s\) allocated, (\d+) kmer\(s\) in contigs", stderr, re.M)
    return stats, int(m.group(1)), int(m.group(2))


def predict(contig, index, pairs, K, alignlen=32, ins=300):
    """the model's view of a run: stats line, kept contigs, table, per-read placements, .readOnContig lines, .readInGap heads"""
    stats, kept, kmers = map_model.read_contigs(contig, K)
    table = map_model.ContigTable(kept, K)
    length, bal_edge = map_model.contig_index(index)
    reads = [r for p in pairs for r in p]
    code = {"A": 0, "C": 1, "T": 2, "G": 3, "N": 3}
    pl = [map_model.place([code[c] for c in r], table, alignlen, length, bal_edge) for r in reads]
    on, gap = map_model.record(pl, reads, ins)
    return dict(stats=stats, kept=kept, kmers=kmers, table=table, reads=reads, placements=pl, on=on, gap=gap)

