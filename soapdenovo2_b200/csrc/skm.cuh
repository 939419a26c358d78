// skm.cuh -- super-k-mer records: the unit of the aggregated pass 1 and of the multi-GPU exchange (host + device logic; skm.cu).
//
// Why: a random update of an HBM-resident slot costs one DRAM read + one write-back whatever instruction performs it, and a
// per-instance insert (k_chop_insert, pass1.cu) pays that once per k-mer INSTANCE.
// Here all instances of a k-mer are brought together on chip first and HBM is touched once per DISTINCT k-mer:
//   1. every k-mer is assigned to a bucket by its canonical MINIMIZER (the m-mer of smallest order value among its K-m+1 m-mers,
//      strand-symmetric), so a k-mer and its reverse complement, wherever they occur, land in the same bucket;
//   2. consecutive k-mers of a read with the same bucket form a run (a super-k-mer) of at most SKM_MAX_RUN k-mers; a run becomes one
//      SELF-CONTAINED record {header, bases} of NW+2 words (32 B for K <= 63, 48 B for K <= 127: about 2 B per k-mer instance
//      instead of the 32 B {key, links, rank} tuple a per-instance exchange would ship).  Because a record carries its own bases
//      and the stream ordinal of its read, it can be aggregated on ANY GPU: bucket ranges are the unit of ownership across GPUs,
//      and the record scatter writes straight into the owner's memory (skm.cu);
//   3. one CTA per bucket aggregates {links, cov, first rank} per distinct k-mer in a shared-memory table, 32 consecutive k-mer
//      instances per warp step whatever the run boundaries, then merges each distinct k-mer into the global table once.
// The reference has no counterpart (its P threads each scan every k-mer of every read, prlHashReads.c:79-90); what has to be
// preserved is the per-k-mer result of put_kmerset/update_kmer (newhash.c:74-140, 473-528), which is a pure function of the
// multiset of instances (SURVEY.md A.3): saturating sums and a minimum, both associative and commutative.
#pragma once
#include "kmer.cuh"
#include "table.cuh"

namespace pgb {

constexpr int SKM_MAX_RUN = 32;      // k-mers per record: 1 + n + K bases must fit NW+1 words (96 bases at K=63, 160 at K=127)
constexpr int SKM_MAX_M = 15;        // minimizer length (2m bits must fit in 32)
constexpr int SKM_MAX_BUCKET_BITS = 26;
constexpr int SKM_MAX_SEGS = 128;    // segments (fed chunks, over all senders) one aggregation launch can read

struct SkmGeom {
    int K = 0, m = 0, w = 0;   // w = K - m + 1 m-mers per k-mer
    u32 mmask = 0;             // low 2m bits
    u32 n_buckets = 0;
};
inline SkmGeom make_skm_geom(int K, u32 n_buckets) {
    SkmGeom g;
    g.K = K;
    g.m = K - 2 < SKM_MAX_M ? K - 2 : SKM_MAX_M;
    if (g.m < 4) g.m = K < 4 ? K : 4;
    g.w = K - g.m + 1;
    g.mmask = g.m >= 16 ? 0xFFFFFFFFu : ((1u << (2 * g.m)) - 1u);
    g.n_buckets = n_buckets;
    return g;
}

// Order value of a canonical m-mer: a bijective 32-bit mixer (odd multiply, xor-shift, odd multiply).  The bucket of a k-mer is a
// function of the MINIMUM order value over its m-mers -- the same multiset on both strands -- so a k-mer and its reverse complement
// always agree on it; the mixer only has to make the minimum look random with respect to the sequence.
PG_HD u32 skm_fmix32(u32 x) {
    x *= 0x9E3779B1u; x ^= x >> 15; x *= 0x85EBCA6Bu;
    return x;
}
PG_HD u32 skm_order(u32 fm, u32 rm) { return skm_fmix32(fm < rm ? fm : rm); }
// minima are concentrated near 0: hash them again before the range reduction
PG_HD u32 skm_bucket(u32 minval, u32 n_buckets) {
    u32 h = (minval ^ 0x5BD1E995u) * 0x9E3779B1u;
    h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
    return (u32)(((u64)h * (u64)n_buckets) >> 32);
}
// buckets are owned in contiguous ranges: owner o holds [o * B / world, (o + 1) * B / world)
PG_HD u32 skm_owner_lo(u32 n_buckets, int world, int o) { return (u32)(((u64)n_buckets * (u64)o) / (u64)world); }
PG_HD int skm_owner_of(u32 n_buckets, int world, u32 b) {
    int o = (int)(((u64)b * (u64)world) / (u64)n_buckets);
    while (o + 1 < world && skm_owner_lo(n_buckets, world, o + 1) <= b) o++;
    while (o > 0 && skm_owner_lo(n_buckets, world, o) > b) o--;
    return o;
}

// side-buffer entry of one run (written by the counting pass, consumed by the scatter pass): bucket (26 bits) | (n - 1) << 26 | last << 31
PG_HD u32 skm_side_pack(u32 b, int n, bool last) { return b | ((u32)(n - 1) << SKM_MAX_BUCKET_BITS) | (last ? 1u << 31 : 0u); }
PG_HD u32 skm_side_bucket(u32 e) { return e & ((1u << SKM_MAX_BUCKET_BITS) - 1u); }
PG_HD int skm_side_n(u32 e) { return (int)((e >> SKM_MAX_BUCKET_BITS) & 31u) + 1; }
PG_HD bool skm_side_last(u32 e) { return (e >> 31) != 0; }

// Split one read into runs.  scratch[slot * stride] (slot < g.w) holds, per thread, the suffix minima of the previous block of w
// m-mer positions, overwritten from the front by the order values of the block being filled (slot o is written at offset o, the
// suffix minimum read at offset o is slot o + 1; the backward pass at the end of a block turns the values into suffix minima in
// place): the minimum of a window of w positions is min(suffix minimum of the previous block, running minimum of the current
// block)  (van Herk / Gil-Werman).  All threads of a warp
// are at the same position of their reads, so the once-per-block backward pass is not divergent (a per-lane rescan whenever the
// minimum leaves the window would be: some lane rescans at almost every step).  The bucket hash is only evaluated when the
// minimum changes (a few times per read).
// emit(bucket, first k-mer position, count, run ends with the last k-mer of the read).
template <class Emit>
PG_HD void skm_scan_read(const SkmGeom& g, const u64* wp, int L, u32* scratch, int stride, Emit& emit) {
    const int K = g.K, m = g.m, w = g.w;
    if (L < K + 1) return;   // reads shorter than K+1 contribute nothing (prlHashReads.c:504,642)
    u32* cur_blk = scratch;                 // raw order values of the block being filled (slots 0 .. o)
    u32* suf_blk = scratch;                 // suffix minima of the previous block (slots o + 1 .. w - 1)
    u32 fm = 0, rm = 0, pref = 0xFFFFFFFFu;
    int o = 0;                              // offset of m-mer position p inside its block
    u32* cur_p = cur_blk;                   // = cur_blk + o * stride
    const u32* suf_p = suf_blk + stride;    // = suf_blk + (o + 1) * stride
    u32 cur_b = 0, cur_min = 0;
    bool have_min = false;
    int run_start = 0, run_len = 0;
    const int rsh = 2 * (m - 1);
    u64 cur = 0;
    for (int i = 0; i < L; i++) {
        if ((i & 31) == 0) cur = wp[i >> 5];
        const u32 c = (u32)cur & 3u;
        cur >>= 2;
        fm = ((fm << 2) | c) & g.mmask;
        rm = (rm >> 2) | ((c ^ 2u) << rsh);
        if (i < m - 1) continue;
        const u32 ov = skm_order(fm, rm);
        *cur_p = ov;
        pref = ov < pref ? ov : pref;
        const int j = i - K + 1;            // k-mer position; its m-mers are the positions p-w+1 .. p
        if (j >= 0) {
            u32 minval = pref;
            if (o != w - 1) {
                const u32 sv = *suf_p;
                minval = sv < minval ? sv : minval;
            }
            bool cut = run_len == SKM_MAX_RUN;
            if (!have_min || minval != cur_min) {
                const u32 b = skm_bucket(minval, g.n_buckets);
                cut = cut || !have_min || b != cur_b;
                if (cut && run_len) { emit(cur_b, run_start, run_len, false); run_len = 0; }
                cur_b = b;
                cur_min = minval;
                have_min = true;
            } else if (cut) {
                emit(cur_b, run_start, run_len, false);
                run_len = 0;
            }
            if (run_len == 0) run_start = j;
            run_len++;
        }
        cur_p += stride;
        suf_p += stride;
        if (++o == w) {                     // block complete: its suffix minima serve the next w-1 windows
            u32 run = 0xFFFFFFFFu;
            u32* dst = cur_blk + (w - 1) * stride;
            for (int q = w - 1; q >= 0; q--, dst -= stride) {
                const u32 v = *dst;
                run = v < run ? v : run;
                *dst = run;
            }
            o = 0;
            cur_p = cur_blk;
            suf_p = suf_blk + stride;
            pref = 0xFFFFFFFFu;
        }
    }
    if (run_len) emit(cur_b, run_start, run_len, true);
}

#if defined(__CUDACC__)
// The same runs as skm_scan_read, computed by one warp per read (the partition kernels of skm.cu; tests/host_skm_warp.cu checks it
// against skm_scan_read).  The lanes take 32 consecutive positions at a time:
//   * m-mer tile T = positions 32T .. 32T+31.  Lane l builds its m-mer straight from the packed words (bases 32T+l .. are bits 2l ..
//     of words T, T+1): the reverse complement is those 2m bits XOR 0b10.., the forward m-mer their 2-bit groups reversed.  The tile's
//     order values and their prefix and suffix minima go to a per-warp ring of SKM_RING_TILES tiles in shared memory.
//   * k-mer tile t = k-mers 32t .. 32t+31; k-mer j needs the minimum over m-mer positions j .. e = j+w-1.  A window that crosses a
//     tile boundary is suffix(tile of j) + whole tiles between + prefix(tile of e); a window inside one tile (only when w <= 32) is
//     a sparse-table query over the tile (two overlapping power-of-two ranges).  Nothing is kept per thread, and the footprint does
//     not grow with w: a window spans at most ceil((31 + w) / 32) + 1 <= 5 tiles for w <= 113 (K <= 127).
//   * runs: a cut wherever the bucket changes (ballot), and every SKM_MAX_RUN k-mers since the last change, carried across tiles; the
//     lanes that start a run know its length once the next start is known, so the run that is still open at the end of a tile is
//     carried and emitted by the tile that holds the next start (or at the end of the read, with `last`).
// emit(bucket, first k-mer position, count, last, run index) is called once per run, by one lane, runs of one tile concurrently.
// Returns the number of runs (warp-uniform).  `ring` holds SKM_WARP_RING words for this warp.
constexpr int SKM_RING_TILES = 8;
constexpr int SKM_WARP_RING = 3 * SKM_RING_TILES * 32;
static_assert(SKM_MAX_RUN == 32, "forced cuts are counted modulo the tile width");
template <class Emit>
__device__ __forceinline__ int skm_warp_scan_read(const SkmGeom& g, const u64* wp, int W64, int L, u32* ring, Emit& emit) {
    const int K = g.K, m = g.m, w = g.w;
    if (L < K + 1) return 0;   // reads shorter than K+1 contribute nothing (prlHashReads.c:504,642)
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned lane_lt = (1u << lane) - 1u, lane_le = lane_lt | (1u << lane);
    const int nk = L - K + 1, nq = L - m + 1;   // k-mers, m-mer positions
    const int D = (31 + w - 1) >> 5;           // m-mer tiles ahead of the k-mer tile that its windows reach
    u32* const raw = ring;
    u32* const pre = ring + SKM_RING_TILES * 32;
    u32* const suf = pre + SKM_RING_TILES * 32;
    const u32 cmask = 0xAAAAAAAAu & g.mmask;
    auto slot = [](int T) { return (T & (SKM_RING_TILES - 1)) * 32; };
    auto fill = [&](int T) {
        if (32 * T >= nq) return;   // warp-uniform
        const u64 w0 = wp[T], w1 = T + 1 < W64 ? wp[T + 1] : 0ull;
        const int sh = 2 * lane;
        const u32 x = (u32)(sh ? (w0 >> sh) | (w1 << (64 - sh)) : w0) & g.mmask;
        u32 y = __brev(x);
        y = ((y >> 1) & 0x55555555u) | ((y << 1) & 0xAAAAAAAAu);
        const u32 ov = 32 * T + lane < nq ? skm_order(y >> (32 - 2 * m), x ^ cmask) : 0xFFFFFFFFu;
        u32 p = ov, s = ov;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 u = __shfl_up_sync(full, p, d), v = __shfl_down_sync(full, s, d);
            if (lane >= d) p = min(p, u);
            if (lane + d < 32) s = min(s, v);
        }
        raw[slot(T) + lane] = ov;
        pre[slot(T) + lane] = p;
        suf[slot(T) + lane] = s;
    };
    int len2 = 1;                               // largest power of two <= w
    while (2 * len2 <= w) len2 *= 2;
    for (int T = 0; T < D; T++) fill(T);
    u32 carry_b = 0, open_b = 0;
    int carry_seg = 0, open_start = 0, open_idx = 0, nrun = 0;
    for (int t = 0; 32 * t < nk; t++) {
        __syncwarp();
        fill(t + D);
        __syncwarp();
        const int j = 32 * t + lane;
        const bool valid = j < nk;
        const int e = j + w - 1, Te = e >> 5, le = e & 31;
        u32 mv = min(suf[slot(t) + lane], pre[slot(Te) + le]);
        for (int T = t + 1; T < Te; T++) mv = min(mv, pre[slot(T) + 31]);
        if (w <= 32) {                          // warp-uniform
            u32 sp = raw[slot(t) + lane];       // -> min over lane .. lane+len2-1 (cut at the tile end)
            for (int d = 1; d < len2; d <<= 1) {
                const u32 u = __shfl_down_sync(full, sp, d);
                if (lane + d < 32) sp = min(sp, u);
            }
            const u32 u = __shfl_sync(full, sp, (le - len2 + 1) & 31);
            if (Te == t) mv = min(sp, u);
        }
        const u32 b = skm_bucket(mv, g.n_buckets);
        u32 bprev = __shfl_up_sync(full, b, 1);
        if (lane == 0) bprev = carry_b;
        const unsigned chg = __ballot_sync(full, valid && (j == 0 || b != bprev));
        const unsigned below = chg & lane_le;
        const int seg = below ? 32 * t + 31 - __clz(below) : carry_seg;   // first k-mer of this lane's bucket stretch
        const bool st = valid && ((j - seg) & (SKM_MAX_RUN - 1)) == 0;
        const unsigned stm = __ballot_sync(full, st);
        if (stm) {
            if (nrun && lane == 0) emit(open_b, open_start, 32 * t + __ffs(stm) - 1 - open_start, false, open_idx);
            const unsigned after = stm & ~lane_le;
            if (st && after) emit(b, j, __ffs(after) - 1 - lane, false, nrun + __popc(stm & lane_lt));
            const int hs = 31 - __clz(stm);     // the tile's last run stays open
            open_b = __shfl_sync(full, b, hs);
            open_start = 32 * t + hs;
            open_idx = nrun + __popc(stm) - 1;
            nrun += __popc(stm);
        }
        carry_b = __shfl_sync(full, b, 31);
        if (chg) carry_seg = 32 * t + 31 - __clz(chg);
    }
    if (lane == 0) emit(open_b, open_start, nk - open_start, true, open_idx);
    __syncwarp();
    return nrun;
}
#endif

// bucket of ONE k-mer given as a Kmer (used by tests: every instance of a canonical k-mer must map to the same bucket)
template <int NW>
PG_HD u32 skm_bucket_of_kmer(const SkmGeom& g, const Kmer<NW>& k) {
    u32 fm = 0, rm = 0, best = 0;
    bool have = false;
    for (int t = 0; t < g.K; t++) {
        const int bit = 2 * (g.K - 1 - t);
        const u32 c = (u32)((k.w[NW - 1 - bit / 64] >> (bit % 64)) & 3);
        fm = ((fm << 2) | c) & g.mmask;
        rm = (rm >> 2) | ((c ^ 2u) << (2 * (g.m - 1)));
        if (t < g.m - 1) continue;
        const u32 o = skm_order(fm, rm);
        if (!have || o < best) { best = o; have = true; }
    }
    return skm_bucket(best, g.n_buckets);
}

// ---------------------------------------------------------------- self-contained run records
// NW+2 words.  w[0] = header, w[1..NW+1] = bases, LSB first (base index p at bit 2p):
//   base 0            the base before the run's first k-mer (read position start-1), 0 when the run starts the read
//   bases 1 .. n+K-1  the run's own bases (read positions start .. start+n+K-2)
//   base n+K          the base after the run's last k-mer, absent (0) when the run ends the read
// so k-mer t of the record (t < n) is bases t+1 .. t+K, its left neighbour base t, its right neighbour base t+K+1: one shift by 2t
// bits whatever the record.  1 + n + K <= 32 * (NW + 1) bases holds for n <= 32 at K = 63 (NW = 2) and at K = 127 (NW = 4).
//   header: n (bits 0-5, 1..32) | last-of-read (bit 6) | has_prev (bit 7) | first k-mer position (bits 8-23) | read ordinal (bits 24-63)
// The first-occurrence rank of k-mer t is (ordinal << 16) | (start + t): the same value every insert path of the engine uses.
template <int NW>
struct SkmRec {
    u64 w[NW + 2];
};
PG_HD u64 skm_rec_header(u64 ordinal, int start, int n, bool last) {
    return (ordinal << 24) | ((u64)(unsigned)start << 8) | (start > 0 ? 0x80ull : 0ull) | (last ? 0x40ull : 0ull) | (u64)(unsigned)n;
}
PG_HD int skm_rec_n(u64 h) { return (int)(h & 63); }
PG_HD bool skm_rec_last(u64 h) { return (h & 0x40) != 0; }
PG_HD bool skm_rec_has_prev(u64 h) { return (h & 0x80) != 0; }
PG_HD int skm_rec_start(u64 h) { return (int)((h >> 8) & 0xFFFF); }
PG_HD u64 skm_rec_ordinal(u64 h) { return h >> 24; }
PG_HD u64 skm_rec_rank(u64 h, int t) { return ((h >> 24) << 16) | (u64)(skm_rec_start(h) + t); }

// 64 bits of a packed read starting at bit position `bit` (may be -2: bits before the read are 0; words past W64 are 0)
PG_HD u64 skm_read_bits(const u64* wp, int W64, int bit) {
    if (bit < 0) return wp[0] << 2;   // only bit == -2 occurs
    const int wi = bit >> 6, sh = bit & 63;
    const u64 lo = wi < W64 ? wp[wi] : 0ull;
    if (!sh) return lo;
    const u64 hi = wi + 1 < W64 ? wp[wi + 1] : 0ull;
    return (lo >> sh) | (hi << (64 - sh));
}
template <int NW>
PG_HD SkmRec<NW> skm_make_rec(int K, const u64* wp, int W64, u64 ordinal, int start, int n, bool last) {
    SkmRec<NW> r;
    r.w[0] = skm_rec_header(ordinal, start, n, last);
    const int nb = n + K + (last ? 0 : 1);   // bases 0 .. nb-1 are meaningful (base 0 may be the dummy)
    const int bit0 = 2 * (start - 1);
#pragma unroll
    for (int t = 0; t < NW + 1; t++) {
        u64 v = skm_read_bits(wp, W64, bit0 + 64 * t);   // bit0 == -2 for a run that starts its read: base 0 is the dummy
        const int bits = 2 * nb - 64 * t;
        if (bits <= 0) v = 0;
        else if (bits < 64) v &= (1ull << bits) - 1ull;
        r.w[1 + t] = v;
    }
    return r;
}

// One k-mer instance: canonical k-mer + neighbour codes in the CANONICAL orientation (4 = none), SURVEY.md A.2.
// The LSB-first packing IS the base-reversed order, so the reverse complement of a k-mer is its K bases XOR 0b10..., and the
// forward k-mer is the reverse complement of that.
template <int NW>
struct SkmInst {
    Kmer<NW> canon;
    unsigned left, right;
};
// k-mer t of a record whose base words are x[0..NW] (x[i] = rec.w[1 + i]); hdr = rec.w[0]
template <int NW>
PG_HD SkmInst<NW> skm_instance_rec(const KParams<NW>& kp, u64 hdr, const u64 (&x)[NW + 1], int t) {
    const int K = kp.K;
    const int sh = 2 * t;   // 0 .. 62
    u64 y[NW + 1];          // bases t .. from bit 0
#pragma unroll
    for (int i = 0; i < NW + 1; i++) {
        const u64 hi = i + 1 < NW + 1 ? x[i + 1] : 0ull;
        y[i] = sh ? ((x[i] >> sh) | (hi << (64 - sh))) : x[i];
    }
    const unsigned pv = (t > 0 || skm_rec_has_prev(hdr)) ? (unsigned)(y[0] & 3) : 4u;
    u64 z[NW];              // bases t+1 .. from bit 0: the k-mer, then its right neighbour at bit 2K
#pragma unroll
    for (int i = 0; i < NW; i++) z[i] = (y[i] >> 2) | (y[i + 1] << 62);
    unsigned cn = 4;
    if (!(skm_rec_last(hdr) && t == skm_rec_n(hdr) - 1)) {
        const int bit = 2 * K, wi = bit >> 6;   // 2K <= 64 * NW - 2: always inside z
        u64 v = 0;
#pragma unroll
        for (int i = 0; i < NW; i++)
            if (i == wi) v = z[i];
        cn = (unsigned)((v >> (bit & 63)) & 3);
    }
    Kmer<NW> rc;
#pragma unroll
    for (int i = 0; i < NW; i++) rc.w[NW - 1 - i] = (z[i] ^ 0xAAAAAAAAAAAAAAAAull) & kp.mask.w[NW - 1 - i];
    const Kmer<NW> fwd = krc_n(rc, K);
    SkmInst<NW> r;
    const bool sm = kless(fwd, rc);          // KmerSmaller(word, bal_word); tie -> rc branch
    r.canon = sm ? fwd : rc;
    r.left = sm ? pv : (cn < 4 ? (cn ^ 2u) : 4u);
    r.right = sm ? cn : (pv < 4 ? (pv ^ 2u) : 4u);
    return r;
}

// The same instances from a record staged in shared memory (skm.cu stages a window of records at a time).  Once per record the
// aggregation writes rv[0..NW]: the record's bases 0 .. n+K-1 in REVERSE order, base n+K-1 at bit 0 and base p at bit 2(n+K-1-p)
// (the right neighbour of the last k-mer is dropped).  Forward k-mer t is then rv >> 2(n-1-t), a shift by less than 64 bits like the
// one that gives the reverse complement from the record words: no per-instance reverse complement.
template <int NW, int WS>
PG_HD void skm_rev_shift(const u64* x, u64 (&rv)[NW + 1], int bs) {
#pragma unroll
    for (int i = 0; i < NW + 1; i++) {   // word j of the reversed record is rev2bit64(x[NW - j])
        const u64 lo = i + WS <= NW ? rev2bit64(x[i + WS <= NW ? NW - i - WS : 0]) : 0ull;
        const u64 hi = i + WS + 1 <= NW ? rev2bit64(x[i + WS + 1 <= NW ? NW - i - WS - 1 : 0]) : 0ull;
        rv[i] = bs ? ((lo >> bs) | (hi << (64 - bs))) : lo;
    }
}
template <int NW>
PG_HD void skm_rec_reverse(u64 hdr, const u64* x, u64 (&rv)[NW + 1], int K) {
    // all 32(NW+1) bases reversed (base p at bit 2(32(NW+1)-1-p)), shifted right by s; 2 <= s since n + K <= 32(NW+1) - 1.  The word
    // offset goes through a switch so that every index is a constant (a dynamically indexed array lives in local memory on the GPU).
    const int s = 2 * (32 * (NW + 1) - skm_rec_n(hdr) - K), bs = s & 63;
    switch (s >> 6) {
        case 0: skm_rev_shift<NW, 0>(x, rv, bs); break;
        case 1: skm_rev_shift<NW, 1>(x, rv, bs); break;
        case 2: skm_rev_shift<NW, 2>(x, rv, bs); break;
        case 3: skm_rev_shift<NW, (NW > 2 ? 3 : 2)>(x, rv, bs); break;
        default: skm_rev_shift<NW, (NW > 2 ? 4 : 2)>(x, rv, bs); break;
    }
}
// k-mer t of a record: hdr, base words x[0..NW] (x[i] = rec.w[1 + i]) and rv[0..NW] from skm_rec_reverse.  Equals skm_instance_rec.
template <int NW>
PG_HD SkmInst<NW> skm_instance_staged(const KParams<NW>& kp, u64 hdr, const u64* x, const u64* rv, int t) {
    const int K = kp.K;
    const int sh = 2 * t;                             // 0 .. 62
    const int sf = 2 * (skm_rec_n(hdr) - 1 - t);      // 0 .. 62
    u64 y[NW + 1], v[NW + 1];                         // bases t .. from bit 0; the reversed bases from base t+K down
#pragma unroll
    for (int i = 0; i < NW + 1; i++) { y[i] = x[i]; v[i] = rv[i]; }
#pragma unroll
    for (int i = 0; i < NW + 1; i++) {
        const u64 hy = i + 1 < NW + 1 ? y[i + 1] : 0ull, hv = i + 1 < NW + 1 ? v[i + 1] : 0ull;
        y[i] = sh ? ((y[i] >> sh) | (hy << (64 - sh))) : y[i];
        v[i] = sf ? ((v[i] >> sf) | (hv << (64 - sf))) : v[i];
    }
    const unsigned pv = (t > 0 || skm_rec_has_prev(hdr)) ? (unsigned)(y[0] & 3) : 4u;
    u64 z[NW];              // bases t+1 .. from bit 0: the k-mer, then its right neighbour at bit 2K
#pragma unroll
    for (int i = 0; i < NW; i++) z[i] = (y[i] >> 2) | (y[i + 1] << 62);
    unsigned cn = 4;
    if (!(skm_rec_last(hdr) && t == skm_rec_n(hdr) - 1)) {
        const int bit = 2 * K, wi = bit >> 6;
        u64 c = 0;
#pragma unroll
        for (int i = 0; i < NW; i++)
            if (i == wi) c = z[i];
        cn = (unsigned)((c >> (bit & 63)) & 3);
    }
    Kmer<NW> rc, fwd;
#pragma unroll
    for (int i = 0; i < NW; i++) {
        rc.w[NW - 1 - i] = (z[i] ^ 0xAAAAAAAAAAAAAAAAull) & kp.mask.w[NW - 1 - i];
        fwd.w[NW - 1 - i] = v[i] & kp.mask.w[NW - 1 - i];
    }
    SkmInst<NW> r;
    const bool sm = kless(fwd, rc);          // KmerSmaller(word, bal_word); tie -> rc branch
    r.canon = sm ? fwd : rc;
    r.left = sm ? pv : (cn < 4 ? (cn ^ 2u) : 4u);
    r.right = sm ? cn : (pv < 4 ? (pv ^ 2u) : 4u);
    return r;
}

// ---------------------------------------------------------------- lane packing
// P[0..nt] = exclusive prefix sums of the k-mer counts of a tile of nt records.  Instance q of the tile belongs to the last record r
// with P[r] <= q (every record holds at least one k-mer, so P is strictly increasing); its position inside the record is q - P[r].
PG_HD int skm_pick_record(const u32* P, int nt_pow2, u32 q) {
    int lo = 0;
#pragma unroll
    for (int half = nt_pow2 >> 1; half > 0; half >>= 1)
        if (P[lo + half] <= q) lo += half;
    return lo;
}

// slot index of a k-mer inside a bucket's shared-memory table: one 64-bit multiply (the 5-multiply table_hash is only needed once
// per DISTINCT k-mer, for the global table)
template <int NW>
PG_HD u32 skm_slot_hash(const Kmer<NW>& k, int log2_slots) {
    u64 x = k.w[0];
#pragma unroll
    for (int i = 1; i < NW; i++) x = ((x << 29) | (x >> 35)) ^ k.w[i];
    x ^= x >> 31;
    x *= 0x9E3779B97F4A7C15ull;
    return (u32)(x >> (64 - log2_slots));
}

// Two partial results for the same k-mer -> the result of all their instances together.  `g` may be PAYLOAD_FRESH (slot claimed, no
// instance yet); `a` holds at least one instance.  Every instance has a neighbour on at least one side (reads are >= K+1 long), so
// cov counts instances (newhash.c:74-106, 123-140) and the fields simply add with their saturation; `single` survives only when the
// total is one instance, i.e. never when both sides are non-empty.
PG_HD u64 payload_merge(u64 g, u64 a) {
    if (g == PAYLOAD_FRESH) return a;
    u64 r = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
        unsigned l = pl_l(g, c) + pl_l(a, c), q = pl_r(g, c) + pl_r(a, c);
        r |= (u64)(l > 63 ? 63 : l) << (6 * c);
        r |= (u64)(q > 63 ? 63 : q) << (PL_R_SHIFT + 6 * c);
    }
    unsigned cv = pl_cov(g) + pl_cov(a);
    r |= (u64)(cv > 255 ? 255 : cv) << PL_COV_SHIFT;
    return r;
}

// ---------------------------------------------------------------- exchange arena (one per GPU; see skm.cu)
// Every GPU owns an arena that ALL GPUs (itself included) write run records into: `world` record regions of cap_pair records (one
// per sender, so senders never contend for space and need no coordination), a ring of segment descriptors per sender, and per
// segment the offsets of the owner's buckets inside the segment's record blob.  Everything exists twice (epoch parity): while an
// owner still aggregates epoch e, fast senders may already deliver epoch e+1 into the other half; one barrier per epoch suffices.
struct SkmSegDesc {
    u64 rec_off;     // first record of the blob, in records, inside the sender's region
    u32 n_recs;
    u32 pad;
};
struct SkmArenaGeom {
    int world = 1;
    u32 max_seg = 0;        // segments per sender per epoch
    u32 bo_max = 0;         // max buckets owned by one GPU (+1 offsets per segment)
    u64 cap_pair = 0;       // records per (sender, owner) region
    int rec_words = 0;      // NW + 2
    // byte offsets inside one epoch half
    u64 off_nseg = 0, off_ring = 0, off_segoff = 0, off_recs = 0, half_bytes = 0;
};
inline SkmArenaGeom make_skm_arena_geom(int world, u32 n_buckets, u32 max_seg, u64 cap_pair, int rec_words) {
    SkmArenaGeom a;
    a.world = world;
    a.max_seg = max_seg;
    a.bo_max = (u32)((n_buckets + (u32)world - 1) / (u32)world) + 1;
    a.cap_pair = cap_pair;
    a.rec_words = rec_words;
    auto up = [](u64 x) { return (x + 255) & ~255ull; };
    u64 o = 0;
    a.off_nseg = o;   o = up(o + (u64)world * sizeof(u32) + 64);
    a.off_ring = o;   o = up(o + (u64)world * max_seg * sizeof(SkmSegDesc));
    a.off_segoff = o; o = up(o + (u64)world * max_seg * (u64)(a.bo_max + 1) * sizeof(u32));
    a.off_recs = o;   o = up(o + (u64)world * cap_pair * (u64)rec_words * sizeof(u64));
    a.half_bytes = o;
    return a;
}
constexpr int SKM_ARENA_HALVES = 2;   // epoch parity

// the parts of epoch half `half` of an arena that starts at `base`
struct SkmArenaHalf {
    u32* nseg;          // [world] segments each sender has published
    SkmSegDesc* ring;   // [world][max_seg]
    u32* segoff;        // [world][max_seg][bo_max + 1]
    u64* recs;          // [world][cap_pair][rec_words]
};
inline SkmArenaHalf skm_arena_half(const SkmArenaGeom& g, void* base, int half) {
    char* h = static_cast<char*>(base) + (u64)half * g.half_bytes;
    return {reinterpret_cast<u32*>(h + g.off_nseg), reinterpret_cast<SkmSegDesc*>(h + g.off_ring), reinterpret_cast<u32*>(h + g.off_segoff),
            reinterpret_cast<u64*>(h + g.off_recs)};
}

}   // namespace pgb
