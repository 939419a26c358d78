"""Designed read sets for the reference's table layout, and a plain Python model of its k-mer sets.

The reference puts every k-mer instance into set crc(k-mer) % P with put_kmerset (linear probing from home = k-mer % size) and, without
-a, grows a set (encap_kmerset) whenever the check before a put finds count + 1 > threshold -- on hits too.  The layout, and with it
every output file but .kmerFreq, follows from that history.  model() replays it instance by instance in stream order (read ordinal,
then position; mates interleave as 2*pair + mate; reads shorter than K+1 contribute nothing).

Encoding: 2-bit codes A0 C1 T2 G3, first base most significant, complement = code ^ 2, canonical = min(forward, reverse complement).
Set of a key: sign_extend32(zlib.crc32(<words little-endian, most significant word first>, 0xFFFFFFFF)) mod 2^64 % P, over two words
in the 63-mer build and four in the 127-mer build.  Home: key % size (the 127-mer build's chained 32-bit modulo equals it below 2^32).

Three families of designs (SCENARIOS):
  threshold  a set ends with exactly its growth threshold of keys (793, 1588, 3177); whether a pass-1 instance of it comes after its last
             new key decides one more growth.  Contrast cases end one below and one above.
  chains     one set grows several times with its keys on a few homes modulo every size it takes, so encap_kmerset's displacement
             chains are long.
  wrap       -a 1 static sets with 2-4 homes at size-1 .. size-4 (the probe chains wrap past slot 0), later reads homed lower."""
import math
import os
import random
import struct
import zlib

import numpy as np

BASES = "ACTG"
CODE = {b: i for i, b in enumerate(BASES)}
LOAD = np.float32(0.77)


# ---------------------------------------------------------------- k-mer algebra and the reference's set geometry
def value(seq: str) -> int:
    v = 0
    for ch in seq:
        v = (v << 2) | CODE[ch]
    return v


def bases(v: int, K: int) -> str:
    return "".join(BASES[(v >> (2 * (K - 1 - i))) & 3] for i in range(K))


def revcomp(v: int, K: int) -> int:
    r = 0
    for _ in range(K):
        r = (r << 2) | ((v & 3) ^ 2)
        v >>= 2
    return r


def revcomp_seq(s: str) -> str:
    return "".join(BASES[CODE[c] ^ 2] for c in reversed(s))


def canonical(v: int, K: int) -> int:
    return min(v, revcomp(v, K))


def set_of(key: int, P: int, flavour127: bool) -> int:
    nw = 4 if flavour127 else 2
    ws = [(key >> (64 * (nw - 1 - i))) & (2**64 - 1) for i in range(nw)]
    c = zlib.crc32(struct.pack("<" + "Q" * nw, *ws), 0xFFFFFFFF)
    if c & 0x80000000:
        c -= 1 << 32
    return (c % (1 << 64)) % P


def is_prime(n: int) -> bool:
    """newhash.c's test: float square root and a strict '<', so squares of primes pass"""
    if n < 4:
        return True
    if n % 2 == 0:
        return False
    mx = int(math.sqrt(float(np.float32(n))))
    return all(n % i for i in range(3, mx, 2))


def next_prime(n: int) -> int:
    if n % 2 == 0:
        n += 1
    while not is_prime(n):
        n += 2
    return n


def threshold(size: int, lf=LOAD) -> int:
    return int(np.float32(size) * lf)


def grown_size(size: int, count: int) -> int:
    n = size
    while True:
        n = n << 1 if n < 0xFFFFFFF else n + 0xFFFFFF
        n = next_prime(n)
        if not np.float32(n) * LOAD < np.float32(count + 1):
            return n


def dynamic_sizes(n: int = 5) -> list:
    """the first n (size, threshold) pairs of a dynamic set: (1031, 793), (2063, 1588), ..."""
    out, size = [], next_prime(1024)
    for _ in range(n):
        out.append((size, threshold(size)))
        size = grown_size(size, threshold(size))
    return out


def static_size(initG: int, P: int, flavour127: bool) -> int:
    want = int(float(initG) * float(np.float32(1024.0) ** 3) / float(P) / (40 if flavour127 else 24))
    k = 1
    while k * 0xFFFFFF < want:
        k += 1
    init = k * 0xFFFFFF
    return 3 if init < 3 else next_prime(init)


# ---------------------------------------------------------------- the model: put_kmerset + encap_kmerset in stream order
class RefSet:
    def __init__(self, size, static):
        self.size, self.static = size, static
        self.mx, self.count, self.growths = threshold(size), 0, 0
        self.max_probe = self.max_chain = self.wraps = 0   # longest probe of a put, longest displacement chain of a growth, wrapped puts
        self.slot = {}   # slot -> key
        self.where = {}  # key -> slot

    def encap(self):
        if self.static:   # the reference raises the load factor of a static set and keeps filling it
            self.mx = threshold(self.size, np.float32(0.88))
            return
        n, old = grown_size(self.size, self.count), self.size
        arr, oldocc, newocc = dict(self.slot), set(self.slot), set()
        for i in range(old):   # ascending old slot, displacement chains: a re-homed key takes the place of one not moved yet
            if i not in oldocc:
                continue
            key = arr[i]
            oldocc.discard(i)
            chain = 0
            while True:
                chain += 1
                self.max_chain = max(self.max_chain, chain)
                hc = key % n
                while hc in newocc:
                    hc = hc + 1 if hc + 1 < n else 0
                newocc.add(hc)
                if hc < old and hc in oldocc:
                    key, arr[hc] = arr[hc], key
                    oldocc.discard(hc)
                else:
                    arr[hc] = key
                    break
        self.slot = {i: k for i, k in arr.items() if i in newocc}
        self.where = {k: i for i, k in self.slot.items()}
        self.size, self.mx = n, threshold(n)
        self.growths += 1

    def put(self, key, hits_grow=True):
        if key in self.where and not hits_grow:
            return
        if self.count + 1 > self.mx:
            self.encap()
        if key in self.where:
            return
        hc, probe = key % self.size, 0
        while hc in self.slot:
            hc, probe = hc + 1 if hc + 1 < self.size else 0, probe + 1
        self.max_probe = max(self.max_probe, probe)
        self.wraps += hc < key % self.size
        self.slot[hc] = key
        self.where[key] = hc
        self.count += 1


def chop(seq: str, K: int):
    """canonical keys of a read, by position (nothing for reads shorter than K+1)"""
    if len(seq) < K + 1:
        return []
    mask, out = (1 << (2 * K)) - 1, []
    f = value(seq[:K])
    r = revcomp(f, K)
    out.append(min(f, r))
    top = 2 * (K - 1)
    for ch in seq[K:]:
        c = CODE[ch]
        f = ((f << 2) | c) & mask
        r = (r >> 2) | ((c ^ 2) << top)
        out.append(min(f, r))
    return out


def model(stream, K, P, flavour127, initG=0, rule="reference"):
    """stream: reads in stream order.  rule: "reference"; "always" grows every dynamic set that ends at its threshold (the engine's
    old replay); "never" lets no hit grow a set.  Returns (the sets: RefSet with size, growths, count and probe statistics; keys in iteration order)."""
    size = static_size(initG, P, flavour127) if initG else next_prime(1024)
    sets = [RefSet(size, bool(initG)) for _ in range(P)]
    set_cache = {}
    for seq in stream:
        for key in chop(seq, K):
            s = set_cache.get(key)
            if s is None:
                s = set_cache[key] = set_of(key, P, flavour127)
            sets[s].put(key, hits_grow=rule != "never")
    if rule == "always":
        for st in sets:
            if not st.static and st.count and st.count + 1 > st.mx:
                st.encap()
    order = [st.slot[i] for st in sets for i in sorted(st.slot)]
    return sets, order


def dump_keys(dump: bytes, flavour127: bool) -> list:
    """the key column of a -T / dump_nodes table dump"""
    nw = 4 if flavour127 else 2
    rec = nw * 8 + 10
    out = []
    for i in range(0, len(dump), rec):
        ws = struct.unpack_from("<" + "Q" * nw, dump, i)
        v = 0
        for w in ws:
            v = (v << 64) | w
        out.append(v)
    return out


# ---------------------------------------------------------------- design helpers
def random_read(rng, n):
    return "".join(rng.choice(BASES) for _ in range(n))


def keys_by_construction(rng, K, want_set, P, flavour127, home, moduli, n):
    """n canonical K-mer values with value % m == home % m for every m in moduli (so the same home at each size) and set want_set"""
    M = 1
    for m in moduli:
        M *= m
    out, seen = [], set()
    top = (1 << (2 * K)) // M
    while len(out) < n:
        v = home + M * rng.randrange(top)
        if v >= 1 << (2 * K) or v in seen or v != canonical(v, K) or v == revcomp(v, K):
            continue
        if set_of(v, P, flavour127) != want_set:
            continue
        seen.add(v)
        out.append(v)
    return out


def embed(rng, key, K):
    """a read of K+1 bases whose first k-mer is the key (forward or reverse complement, at random)"""
    s = bases(key, K)
    if rng.random() < 0.5:
        return revcomp_seq(s + rng.choice(BASES))
    return s + rng.choice(BASES)


class Stream:
    """reads in stream order, with each set's distinct keys counted as they arrive"""

    def __init__(self, K, P, flavour127):
        self.K, self.P, self.f127 = K, P, flavour127
        self.reads, self.seen, self.n = [], {}, [0] * P   # key -> set, distinct keys per set

    def keys(self, seq):
        return [(j, k, self.seen[k] if k in self.seen else set_of(k, self.P, self.f127)) for j, k in enumerate(chop(seq, self.K))]

    def add(self, seq):
        for _, k, s in self.keys(seq):
            if k not in self.seen:
                self.seen[k] = s
                self.n[s] += 1
        self.reads.append(seq)

    def count(self, s):
        return self.n[s]

    def window(self, rng, pred):
        """a (K+1)-base window of an earlier read whose two keys satisfy pred(key, set)"""
        for _ in range(20000):
            r = rng.choice(self.reads)
            if len(r) < self.K + 1:
                continue
            j = rng.randrange(len(r) - self.K)
            w = r[j:j + self.K + 1]
            if all(pred(k, s) for _, k, s in self.keys(w)):
                return w
        raise RuntimeError("no window matches")


def threshold_stream(K, P, target, tail, seed, rd_len=100):
    """Fill set 0 with random reads until a read brings it to `target` keys; cut that read right after the key that does (it must be a
    reverse-complement instance for tail "rc").  Then add the tail:
      none / rc   nothing after it                       short    a read of exactly K bases: that key again (dropped by the reader)
      other       (K+1)-windows of earlier reads whose keys lie in other sets only
      cov2        a (K+1)-window holding the last key again      repeat   a window of two earlier keys of set 0, not the last
      pair_early / pair_late   (f1/f2 library) a repeat of a set-0 key as mate 2 of the pair before / of the pair whose mate 1 ends
                  with the last key; the other mate 2 slots hold other-set windows.
    Returns (stream reads, the last key)."""
    rng = random.Random(seed)
    st = Stream(K, P, False)
    last = None
    while last is None:
        r = random_read(rng, rd_len)
        need = target - st.count(0)
        new0 = []
        for j, k, s in st.keys(r):
            if s == 0 and k not in st.seen and k not in [x[1] for x in new0]:
                new0.append((j, k))
        if len(new0) < need:
            st.add(r)
            continue
        j, k = new0[need - 1]
        fwd = value(r[j:j + K])
        if j < 1 or (tail == "rc" and fwd == k):
            continue   # too short to be read once cut / a forward instance where the design wants a reverse one
        if tail.startswith("pair") and len(st.reads) % 2 == 0:
            st.add(st.window(rng, lambda key, s: s != 0))   # the cut read must be mate 1 (an even ordinal) ...
        if tail.startswith("pair"):                        # ... after the mate 2 of the pair before it
            st.add(st.window(rng, lambda key, s: s == 0) if tail == "pair_early" else st.window(rng, lambda key, s: s != 0))
        st.add(r[:j + K])
        last = k
    others = lambda key, s: s != 0
    if tail == "other":
        for _ in range(5):
            st.reads.append(st.window(rng, others))
    elif tail == "short":
        st.reads.append(bases(last, K))
    elif tail == "cov2":
        st.reads.append(st.reads[-1][-(K + 1):])
    elif tail == "repeat":
        st.reads.append(st.window(rng, lambda key, s: s == 0 and key != last))
    elif tail == "pair_early":
        st.reads.append(st.window(rng, others))
    elif tail == "pair_late":
        st.reads.append(st.window(rng, lambda key, s: s == 0 and key != last))
    return st.reads, last


def chains_stream(K, P, flavour127, seed, per_home=700, homes=4, noise=1200):
    """One set (set 0) grows three or four times with `homes` x `per_home` keys sharing `homes` homes modulo every size it takes, read
    in an order that interleaves the homes; random reads add keys in every set around them."""
    rng = random.Random(seed)
    sizes = [s for s, _ in dynamic_sizes(3)]   # the same home at 1031, 2063 and 4127 slots
    hs = [rng.randrange(1 << 20) for _ in range(homes)]
    groups = [keys_by_construction(rng, K, 0, P, flavour127, h, sizes, per_home) for h in hs]
    reads = [embed(rng, groups[i % homes][i // homes], K) for i in range(homes * per_home)]
    rd = K + 40
    noise_reads = [random_read(rng, rd) for _ in range(noise // 40)]
    for i, r in enumerate(noise_reads):
        reads.insert(rng.randrange(len(reads) + 1), r)
    return reads


def wrap_stream(K, P, flavour127, seed, per_home=(600, 500, 400, 300), want_set=0):
    """-a 1: keys of one static set on homes size-1, size-2, ... (the run of occupied slots wraps past slot 0); the reads interleave
    the homes with later keys homed lower, and a second cluster at a low home gets keys the wrap has to pass."""
    rng = random.Random(seed)
    size = static_size(1, P, flavour127)
    groups = [keys_by_construction(rng, K, want_set, P, flavour127, size - 1 - t, [size], n) for t, n in enumerate(per_home)]
    low = keys_by_construction(rng, K, want_set, P, flavour127, 5, [size], 300)
    order = []
    for i in range(max(per_home)):
        for g in groups:   # later-read keys homed lower
            if i < len(g):
                order.append(g[i])
        if i % 2 and i // 2 < len(low):
            order.append(low[i // 2])
    return [embed(rng, k, K) for k in order]


# name -> (family, K, P, flavour127, extra pregraph options, builder arguments, expected)
#   threshold: (target, tail, seed); expected = whether the set that ends at its threshold grows once more (None: contrast case)
SIZES = dynamic_sizes(5)
T1, T2, T3 = SIZES[0][1], SIZES[1][1], SIZES[2][1]
SCENARIOS = {
    "last_t1_p1": ("threshold", 31, 1, False, ("-R",), (T1, "none", 1), False),
    "last_t2_p1": ("threshold", 31, 1, False, (), (T2, "none", 2), False),
    "last_t3_p1": ("threshold", 31, 1, False, ("-R",), (T3, "none", 3), False),
    "below_t1_p1": ("threshold", 31, 1, False, (), (T1 - 1, "none", 1), None),
    "above_t1_p1": ("threshold", 31, 1, False, (), (T1 + 1, "none", 1), None),
    "below_t2_p3": ("threshold", 31, 3, False, (), (T2 - 1, "other", 4), None),
    "above_t2_p3": ("threshold", 31, 3, False, (), (T2 + 1, "other", 4), None),
    "other_t1_p3": ("threshold", 31, 3, False, ("-R",), (T1, "other", 5), False),
    "other_t3_p8": ("threshold", 31, 8, False, (), (T3, "other", 6), False),
    "rc_t2_p1": ("threshold", 31, 1, False, (), (T2, "rc", 7), False),
    "short_t1_p1": ("threshold", 31, 1, False, ("-R",), (T1, "short", 8), False),
    "pair_early_t1_p3": ("threshold", 31, 3, False, ("-R",), (T1, "pair_early", 9), False),
    "pair_early_d1_t1_p3": ("threshold", 31, 3, False, ("-d", "1"), (T1, "pair_early", 9), False),
    "pair_late_t1_p3": ("threshold", 31, 3, False, ("-R",), (T1, "pair_late", 9), True),
    "cov2_t2_p1": ("threshold", 31, 1, False, (), (T2, "cov2", 10), True),
    "repeat_t1_p3": ("threshold", 31, 3, False, ("-R",), (T1, "repeat", 11), True),
    "chains_k31_p1": ("chains", 31, 1, False, (), (21,), None),
    "chains_k63_p3": ("chains", 63, 3, False, ("-R",), (22,), None),
    "chains_k95_p2": ("chains", 95, 2, True, (), (23,), None),
    "wrap_k31_p1": ("wrap", 31, 1, False, ("-a", "1"), (31,), None),
    "wrap_k63_p3": ("wrap", 63, 3, False, ("-a", "1", "-R"), (32,), None),
    "wrap_k95_p1": ("wrap", 95, 1, True, ("-a", "1"), (33,), None),
    "wrap_k127_p3": ("wrap", 127, 3, True, ("-a", "1", "-R"), (34,), None),
}


def stream(name):
    """(reads in stream order, whether the library is an f1/f2 pair, the threshold design's last key or None)"""
    fam, K, P, f127, extra, args, _ = SCENARIOS[name]
    if fam == "threshold":
        reads, last = threshold_stream(K, P, *args)
        return reads, args[1].startswith("pair"), last
    if fam == "chains":
        return chains_stream(K, P, f127, *args), False, None
    return wrap_stream(K, P, f127, *args), False, None


def write_scenario(d, name, pad=0):
    """FASTA file(s) and config of a scenario in directory d; returns (cfg, reads in stream order).  pad: that many reads of K bases
    (shorter than K+1: records that hold no k-mer) in the middle of the stream, to spread the design over several input chunks."""
    reads, paired, _ = stream(name)
    K = SCENARIOS[name][1]
    if pad:
        mid = len(reads) // 2 & ~1
        reads = reads[:mid] + ["A" * K] * (pad & ~1) + reads[mid:]
    mrl = max(100, K + 41)
    def fasta(path, rs, tag):
        with open(path, "w") as f:
            for i, r in enumerate(rs):
                f.write(f">{tag}{i}\n{r}\n")
    if paired:
        assert len(reads) % 2 == 0
        fasta(os.path.join(d, "r1.fa"), reads[0::2], "a")
        fasta(os.path.join(d, "r2.fa"), reads[1::2], "b")
        files = [("f1", os.path.join(d, "r1.fa")), ("f2", os.path.join(d, "r2.fa"))]
    else:
        fasta(os.path.join(d, "r.fa"), reads, "r")
        files = [("f", os.path.join(d, "r.fa"))]
    cfg = os.path.join(d, "lib.cfg")
    with open(cfg, "w") as f:
        f.write(f"max_rd_len={mrl}\n[LIB]\navg_ins=200\nreverse_seq=0\nasm_flags=3\nrank=1\n")
        for k, p in files:
            f.write(f"{k}={p}\n")
    return cfg, reads
