// deflate.cuh -- the pieces of zlib's level-6 gzip stream (deflateInit2(6, Z_DEFLATED, 31, 8, Z_DEFAULT_STRATEGY), i.e. what
// gzopen(name, "w") + gzwrite write), restated as __host__ __device__ functions.  deflate.cu runs them on the GPU in parallel;
// tests/host_deflate.cu runs them one after another on the CPU and compares the stream with Python's zlib.
//
// What the output is a function of (each item is pinned by the fuzz in tests/test_deflate_host.py):
//   hash      h(p) = ((b[p] << 10) ^ (b[p+1] << 5) ^ b[p+2]) & 0x7fff; every position with 3 bytes left is inserted
//   chain     earlier positions with the same hash, newest first; the head may be MAX_DIST back, later ones less than MAX_DIST
//   window    zlib keeps positions relative to a base that slides by 32 KB; the position at the base is NIL and never matches
//   search    max_chain 128 (32 while the pending match is >= good_length 8), nice_length 128 (clamped to the bytes left),
//             skipped while the pending match is >= max_lazy 16; a length-3 match more than TOO_FAR back is dropped
//   lazy      deflate_slow's automaton: state (match_length, match_start, match_available) at each loop top
//   blocks    a block ends after every 16383 symbols (sym_end of memLevel 8); the last block holds the rest
//   type      stored / fixed / dynamic by _tr_flush_block's byte estimates; stored only while the block start is in the window
//   trees     build_tree / gen_bitlen / gen_codes / scan_tree / send_tree / build_bl_tree with their tie-breaks and overflow fix-up
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GZ_HD __host__ __device__ __forceinline__
#else
#define GZ_HD inline
#endif

namespace gz {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int64_t i64;

constexpr int WSIZE = 32768;
constexpr int MIN_LOOKAHEAD = 262;           // MAX_MATCH + MIN_MATCH + 1
constexpr int MAX_DIST = WSIZE - MIN_LOOKAHEAD;
constexpr int MAX_MATCH = 258;
constexpr int TOO_FAR = 4096;
constexpr int NICE = 128, MAX_CHAIN = 128, GOOD = 8, MAX_LAZY = 16;
constexpr int SYM_END = 16383;               // (lit_bufsize - 1) with lit_bufsize = 1 << (8 + 6)
constexpr int L_CODES = 286, D_CODES = 30, BL_CODES = 19, HEAP_SIZE = 2 * L_CODES + 1;
constexpr int END_BLOCK = 256;

GZ_HD int clz32(u32 x) {
#ifdef __CUDA_ARCH__
    return __clz(x);
#else
    return __builtin_clz(x);
#endif
}
GZ_HD u32 hash3(u32 a, u32 b, u32 c) { return ((a << 10) ^ (b << 5) ^ c) & 0x7fff; }

// Stream offset of zlib's window base at loop top s.  fill_window slides when called (lookahead < MIN_LOOKAHEAD) with
// strstart >= WSIZE + MAX_DIST; while input remains the window is full, so the k-th slide happens at the first loop top at or
// past t_k = 32768 (k - 1) + 65275; near the end of a final stream at the first loop top past n - 262 with strstart >= 65274.
// Every loop top s counts, including the terminal one at s == n.  Not final: only loop tops below (available - 262) are asked.
GZ_HD u64 slide_base(u64 s, u64 n, bool final) {
    u64 k = s >= 65275 ? (s - 65275) / WSIZE + 1 : 0;
    if (final) {
        const u64 kfull = n >= 65536 ? (n - 65536) / WSIZE + 1 : 0;
        if (k >= kfull) {
            k = kfull;
            u64 t = (u64)WSIZE * kfull + 65274;
            if (n >= 261 && n - 261 > t) t = n - 261;
            if (t <= s) k++;
        }
    }
    return k * WSIZE;
}

// Result of longest_match at one position for both chain budgets, with best_len starting at MIN_MATCH - 1.  With best_len starting
// at prev_length instead, zlib returns the same (len, start) when len > prev_length, and otherwise a value the automaton treats the
// same way (it emits the pending match), so these two answers are all the automaton needs.  len 2 = no match.
struct Match { u16 len128, dist128, len32, dist32; };
GZ_HD u64 pack_match(Match m) { return (u64)m.len128 | (u64)m.dist128 << 16 | (u64)m.len32 << 32 | (u64)m.dist32 << 48; }
GZ_HD Match unpack_match(u64 v) { return Match{(u16)v, (u16)(v >> 16), (u16)(v >> 32), (u16)(v >> 48)}; }

// b: bytes, pv: distance to the previous position with the same hash (0: none within 32767), both indexed by position relative
// to the buffer; s: loop top (relative); ahead: bytes left from s (only its min with MAX_MATCH + 4 matters); base_rel: window base
// relative to the buffer (may be negative).
template <class Bytes, class Prev>
GZ_HD Match find_match(const Bytes& b, const Prev& pv, i64 s, i64 ahead, i64 base_rel) {
    Match r{2, 0, 2, 0};
    if (ahead < 3) return r;                       // no INSERT_STRING: hash_head stays NIL
    const u32 d0 = pv(s);
    if (d0 == 0 || d0 > (u32)MAX_DIST || s - (i64)d0 == base_rel) return r;
    const int nice = ahead < NICE ? (int)ahead : NICE;
    const int maxlen = ahead < MAX_MATCH ? (int)ahead : MAX_MATCH;   // bytes past the end never decide a result (see DESIGN §3)
    const i64 limit = s - MAX_DIST > base_rel ? s - MAX_DIST : base_rel;
    int best = 2, bestd = 0, n = 1;
    bool rec32 = false;
    i64 c = s - d0;
    const u8 s0 = b(s), s1 = b(s + 1);
    u8 e1 = s1, e0 = b(s + 2);
    for (;; n++) {
        if (b(c + best) == e0 && b(c + best - 1) == e1 && b(c) == s0 && b(c + 1) == s1) {
            int len = 2;
            while (len < maxlen && b(c + len) == b(s + len)) len++;
            if (len > best) {
                best = len;
                bestd = (int)(s - c);
                if (len >= nice) break;        // nice <= maxlen, so below best < maxlen and s + best is a real byte
                e1 = b(s + best - 1);
                e0 = b(s + best);
            }
        }
        if (n == MAX_CHAIN / 4) { r.len32 = (u16)best; r.dist32 = (u16)bestd; rec32 = true; }
        if (n == MAX_CHAIN) break;
        const u32 d = pv(c);
        if (d == 0) break;
        c -= d;
        if (c <= limit) break;
    }
    if (!rec32) { r.len32 = (u16)best; r.dist32 = (u16)bestd; }
    r.len128 = (u16)best; r.dist128 = (u16)bestd;
    if (r.len128 < 3 || (r.len128 == 3 && r.dist128 > TOO_FAR)) { r.len128 = 2; r.dist128 = 0; }
    if (r.len32 < 3 || (r.len32 == 3 && r.dist32 > TOO_FAR)) { r.len32 = 2; r.dist32 = 0; }
    return r;
}

// Automaton state at a loop top: match_length, match_start as a distance back from the loop top (0 when match_length < 3),
// match_available.  Packed for the convergence test of the speculative runs; NO_STATE marks a loop top a run never visited.
struct LazyState { u16 ml; u16 md; u8 ma; };
constexpr u32 NO_STATE = 0xffffffffu;
GZ_HD u32 pack_state(LazyState st) { return (u32)st.ma << 31 | (u32)st.ml << 16 | st.md; }
GZ_HD LazyState unpack_state(u32 v) { return LazyState{(u16)((v >> 16) & 0x7fff), (u16)v, (u8)(v >> 31)}; }
GZ_HD LazyState fresh_state() { return LazyState{2, 0, 0}; }

// One symbol as the lazy automaton emits it: a literal byte, or (length - 3, distance).  The record also keeps the byte it starts
// at and the automaton state at the next loop top, so a stream can stop after any block and resume from that state.
GZ_HD u32 sym_lit(u32 c) { return c; }
GZ_HD u32 sym_match(u32 len, u32 dist) { return 1u << 31 | (len - 3) << 16 | dist; }
GZ_HD bool sym_is_match(u32 v) { return v >> 31; }
GZ_HD u32 sym_len(u32 v) { return sym_is_match(v) ? ((v >> 16) & 0xff) + 3 : 1; }
GZ_HD u32 sym_dist(u32 v) { return v & 0xffff; }
struct Sym { u32 sym, pos, next; };   // pos: first byte (relative); next: packed state at the next loop top

// One step of deflate_slow at loop top s (s < n).  m: the match search at s.  Returns the next loop top; *emit is set when a
// symbol was tallied (at most one per step).
GZ_HD i64 lazy_step(LazyState& st, i64 s, Match m, u8 prev_byte, bool& emit, u32& sym, i64& sym_pos) {
    const u16 prev_len = st.ml, prev_md = st.md;
    u16 ml = 2, md = 0;
    if (prev_len < MAX_LAZY) {
        const bool reduced = prev_len >= GOOD;
        ml = reduced ? m.len32 : m.len128;
        md = reduced ? m.dist32 : m.dist128;
        if (ml < 3) { ml = 2; md = 0; }
    }
    if (prev_len >= 3 && ml <= prev_len) {
        emit = true;
        sym = sym_match(prev_len, prev_md - 1);   // match_start was md back from s - 1's loop top: distance (s-1) - start
        sym_pos = s - 1;
        st = fresh_state();
        return s - 1 + prev_len;
    }
    if (st.ma) { emit = true; sym = sym_lit(prev_byte); sym_pos = s - 1; }
    else emit = false;
    st.ml = ml; st.md = (u16)(ml >= 3 ? md + 1 : 0); st.ma = 1;    // stored relative to the next loop top, s + 1
    return s + 1;
}

// ---- length and distance codes (trees.c's tables, as formulas)
GZ_HD int length_code(int lc) {   // lc = length - 3
    if (lc == 255) return 28;
    if (lc < 8) return lc;
    const int n = 31 - clz32(lc);
    return 4 * (n - 1) + ((lc >> (n - 2)) & 3);
}
GZ_HD int extra_lbits(int code) { return (code < 8 || code == 28) ? 0 : (code >> 2) - 1; }
GZ_HD int base_length(int code) { return code < 8 ? code : code == 28 ? 255 : (4 + (code & 3)) << ((code >> 2) - 1); }
GZ_HD int dist_code(int d0) {     // d0 = distance - 1
    if (d0 < 4) return d0;
    const int n = 31 - clz32(d0);
    return 2 * n + ((d0 >> (n - 1)) & 1);
}
GZ_HD int extra_dbits(int code) { return code < 4 ? 0 : (code >> 1) - 1; }
GZ_HD int base_dist(int code) { return code < 4 ? code : (2 + (code & 1)) << ((code >> 1) - 1); }
GZ_HD int extra_blbits(int n) { return n == 16 ? 2 : n == 17 ? 3 : n == 18 ? 7 : 0; }
GZ_HD int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
GZ_HD int bl_order(int i) {      // {16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15}, 5 bits each
    const u64 lo = 16ull | 17ull << 5 | 18ull << 10 | 0ull << 15 | 8ull << 20 | 7ull << 25 | 9ull << 30 | 6ull << 35 | 10ull << 40 |
                   5ull << 45 | 11ull << 50 | 4ull << 55;
    const u64 hi = 12ull | 3ull << 5 | 13ull << 10 | 2ull << 15 | 14ull << 20 | 1ull << 25 | 15ull << 30;
    return i < 12 ? (int)((lo >> (5 * i)) & 31) : (int)((hi >> (5 * (i - 12))) & 31);
}
GZ_HD u32 bi_reverse(u32 code, int len) {
    u32 r = 0;
    do { r |= code & 1; code >>= 1; r <<= 1; } while (--len > 0);
    return r >> 1;
}
GZ_HD u32 static_lcode(int n) {   // reversed fixed literal/length code
    const int l = static_llen(n);
    const u32 c = n < 144 ? 0x30 + n : n < 256 ? 0x190 + (n - 144) : n < 280 ? (u32)(n - 256) : 0xc0 + (n - 280);
    return bi_reverse(c, l);
}

// ---- Huffman trees, as trees.c builds them.  Freq/Code and Dad/Len share storage in zlib; kept apart here, read in the same order.
template <int NODES>
struct Tree { u16 freq[NODES]; u16 len[NODES]; u16 dad[NODES]; u16 code[NODES]; int max_code; };
typedef Tree<HEAP_SIZE> LTree;
typedef Tree<2 * D_CODES + 1> DTree;
typedef Tree<2 * BL_CODES + 1> BLTree;
struct Heap { int heap[HEAP_SIZE]; u8 depth[HEAP_SIZE]; u16 bl_count[16], next_code[16]; int heap_len, heap_max; };
enum { K_LIT = 0, K_DIST = 1, K_BL = 2 };

GZ_HD bool smaller(const u16* f, int n, int m, const u8* depth) { return f[n] < f[m] || (f[n] == f[m] && depth[n] <= depth[m]); }
GZ_HD void pqdownheap(Heap& h, const u16* f, int k) {
    const int v = h.heap[k];
    int j = k << 1;
    while (j <= h.heap_len) {
        if (j < h.heap_len && smaller(f, h.heap[j + 1], h.heap[j], h.depth)) j++;
        if (smaller(f, v, h.heap[j], h.depth)) break;
        h.heap[k] = h.heap[j];
        k = j;
        j <<= 1;
    }
    h.heap[k] = v;
}
template <int NODES>
GZ_HD void gen_bitlen(Tree<NODES>& t, int kind, Heap& h, u64& opt_len, u64& static_len) {
    const int max_length = kind == K_BL ? 7 : 15, base = kind == K_LIT ? 257 : 0, max_code = t.max_code;
    for (int b = 0; b <= 15; b++) h.bl_count[b] = 0;
    t.len[h.heap[h.heap_max]] = 0;
    int overflow = 0, hh;
    for (hh = h.heap_max + 1; hh < HEAP_SIZE; hh++) {
        const int n = h.heap[hh];
        int bits = t.len[t.dad[n]] + 1;
        if (bits > max_length) bits = max_length, overflow++;
        t.len[n] = (u16)bits;
        if (n > max_code) continue;
        h.bl_count[bits]++;
        int xbits = 0;
        if (n >= base) xbits = kind == K_LIT ? extra_lbits(n - base) : kind == K_DIST ? extra_dbits(n) : extra_blbits(n);
        const u32 f = t.freq[n];
        opt_len += (u64)f * (u32)(bits + xbits);
        if (kind == K_LIT) static_len += (u64)f * (u32)(static_llen(n) + xbits);
        else if (kind == K_DIST) static_len += (u64)f * (u32)(5 + xbits);
    }
    if (overflow == 0) return;
    do {
        int bits = max_length - 1;
        while (h.bl_count[bits] == 0) bits--;
        h.bl_count[bits]--;
        h.bl_count[bits + 1] += 2;
        h.bl_count[max_length]--;
        overflow -= 2;
    } while (overflow > 0);
    for (int bits = max_length; bits != 0; bits--) {
        int n = h.bl_count[bits];
        while (n != 0) {
            const int m = h.heap[--hh];
            if (m > max_code) continue;
            if (t.len[m] != (u32)bits) {
                opt_len += ((u64)bits - t.len[m]) * t.freq[m];
                t.len[m] = (u16)bits;
            }
            n--;
        }
    }
}
template <int NODES>
GZ_HD void gen_codes(Tree<NODES>& t, const u16* bl_count, u16* next_code) {
    u32 code = 0;
    for (int bits = 1; bits <= 15; bits++) { code = (code + bl_count[bits - 1]) << 1; next_code[bits] = (u16)code; }
    for (int n = 0; n <= t.max_code; n++) {
        const int len = t.len[n];
        if (len == 0) continue;
        t.code[n] = (u16)bi_reverse(next_code[len]++, len);
    }
}
// t.freq[0..elems) holds the frequencies on entry.
template <int NODES>
GZ_HD void build_tree(Tree<NODES>& t, int elems, int kind, Heap& h, u64& opt_len, u64& static_len) {
    int max_code = -1, node = elems;
    h.heap_len = 0;
    h.heap_max = HEAP_SIZE;
    for (int n = 0; n < elems; n++) {
        if (t.freq[n] != 0) { h.heap[++h.heap_len] = max_code = n; h.depth[n] = 0; }
        else t.len[n] = 0;
    }
    while (h.heap_len < 2) {
        const int nd = h.heap[++h.heap_len] = (max_code < 2 ? ++max_code : 0);
        t.freq[nd] = 1;
        h.depth[nd] = 0;
        opt_len--;
        if (kind == K_LIT) static_len -= static_llen(nd);
        else if (kind == K_DIST) static_len -= 5;
    }
    t.max_code = max_code;
    for (int n = h.heap_len / 2; n >= 1; n--) pqdownheap(h, t.freq, n);
    do {
        const int n = h.heap[1];
        h.heap[1] = h.heap[h.heap_len--];
        pqdownheap(h, t.freq, 1);
        const int m = h.heap[1];
        h.heap[--h.heap_max] = n;
        h.heap[--h.heap_max] = m;
        t.freq[node] = (u16)(t.freq[n] + t.freq[m]);
        h.depth[node] = (u8)((h.depth[n] >= h.depth[m] ? h.depth[n] : h.depth[m]) + 1);
        t.dad[n] = t.dad[m] = (u16)node;
        h.heap[1] = node++;
        pqdownheap(h, t.freq, 1);
    } while (h.heap_len >= 2);
    h.heap[--h.heap_max] = h.heap[1];
    gen_bitlen(t, kind, h, opt_len, static_len);
    gen_codes(t, h.bl_count, h.next_code);
}
// scan_tree: code-length run statistics into bl.freq.  Writes the guard len[max_code + 1] = 0xffff, which send_tree reads.
template <int NODES>
GZ_HD void scan_tree(Tree<NODES>& t, BLTree& bl) {
    int prevlen = -1, nextlen = t.len[0], count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) max_count = 138, min_count = 3;
    t.len[t.max_code + 1] = 0xffff;
    for (int n = 0; n <= t.max_code; n++) {
        const int curlen = nextlen;
        nextlen = t.len[n + 1];
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) bl.freq[curlen] += (u16)count;
        else if (curlen != 0) { if (curlen != prevlen) bl.freq[curlen]++; bl.freq[16]++; }
        else if (count <= 10) bl.freq[17]++;
        else bl.freq[18]++;
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (curlen == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}
template <int NODES, class Sink>
GZ_HD void send_tree(const Tree<NODES>& t, int max_code, const BLTree& bl, Sink& out) {
    int prevlen = -1, nextlen = t.len[0], count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) max_count = 138, min_count = 3;
    for (int n = 0; n <= max_code; n++) {
        const int curlen = nextlen;
        nextlen = t.len[n + 1];
        if (++count < max_count && curlen == nextlen) continue;
        else if (count < min_count) { do { out(bl.code[curlen], bl.len[curlen]); } while (--count != 0); }
        else if (curlen != 0) {
            if (curlen != prevlen) { out(bl.code[curlen], bl.len[curlen]); count--; }
            out(bl.code[16], bl.len[16]);
            out((u32)(count - 3), 2);
        } else if (count <= 10) { out(bl.code[17], bl.len[17]); out((u32)(count - 3), 3); }
        else { out(bl.code[18], bl.len[18]); out((u32)(count - 11), 7); }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (curlen == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}

// Everything _tr_flush_block decides for one block, from its symbol frequencies.
enum { BT_STORED = 0, BT_FIXED = 1, BT_DYN = 2 };
struct BlockTrees { LTree l; DTree d; BLTree bl; Heap h; int max_blindex; u64 opt_len, static_len; };
// On entry l.freq[0..L_CODES) and d.freq[0..D_CODES) hold the counts (END_BLOCK included).  stored_ok: the block start is still in
// the window.  Returns the block type; *bits: the block's size in bits from its 3 header bits through END_BLOCK (stored: unused).
GZ_HD int plan_block(BlockTrees& t, u64 stored_len, bool stored_ok, u64* bits) {
    t.opt_len = 0; t.static_len = 0;
    build_tree(t.l, L_CODES, K_LIT, t.h, t.opt_len, t.static_len);
    build_tree(t.d, D_CODES, K_DIST, t.h, t.opt_len, t.static_len);
    for (int n = 0; n < BL_CODES; n++) t.bl.freq[n] = 0;
    scan_tree(t.l, t.bl);
    scan_tree(t.d, t.bl);
    build_tree(t.bl, BL_CODES, K_BL, t.h, t.opt_len, t.static_len);
    int mb;
    for (mb = BL_CODES - 1; mb >= 3; mb--) if (t.bl.len[bl_order(mb)] != 0) break;
    t.max_blindex = mb;
    t.opt_len += 3 * ((u64)mb + 1) + 5 + 5 + 4;
    u64 opt_lenb = (t.opt_len + 3 + 7) >> 3;
    const u64 static_lenb = (t.static_len + 3 + 7) >> 3;
    if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
    if (stored_len + 4 <= opt_lenb && stored_ok) return BT_STORED;
    if (static_lenb == opt_lenb) { *bits = 3 + t.static_len; return BT_FIXED; }
    *bits = 3 + t.opt_len;
    return BT_DYN;
}
// send_all_trees: the dynamic block's tree description (after its 3 header bits).
template <class Sink>
GZ_HD void send_all_trees(const BlockTrees& t, Sink& out) {
    const int lcodes = t.l.max_code + 1, dcodes = t.d.max_code + 1, blcodes = t.max_blindex + 1;
    out((u32)(lcodes - 257), 5);
    out((u32)(dcodes - 1), 5);
    out((u32)(blcodes - 4), 4);
    for (int rank = 0; rank < blcodes; rank++) out(t.bl.len[bl_order(rank)], 3);
    send_tree(t.l, lcodes - 1, t.bl, out);
    send_tree(t.d, dcodes - 1, t.bl, out);
}

// Bits of one symbol given the literal/length and distance code tables (code in the low 16 bits, length above).
template <class Sink>
GZ_HD void send_symbol(u32 sym, const u32* lcode, const u32* dcode, Sink& out) {
    if (!sym_is_match(sym)) { out(lcode[sym] & 0xffff, lcode[sym] >> 16); return; }
    const int lc = (int)sym_len(sym) - 3, code = length_code(lc);
    out(lcode[code + 257] & 0xffff, lcode[code + 257] >> 16);
    if (extra_lbits(code)) out((u32)(lc - base_length(code)), extra_lbits(code));
    const int d0 = (int)sym_dist(sym) - 1, dc = dist_code(d0);
    out(dcode[dc] & 0xffff, dcode[dc] >> 16);
    if (extra_dbits(dc)) out((u32)(d0 - base_dist(dc)), extra_dbits(dc));
}
GZ_HD u32 symbol_bits(u32 sym, const u32* lcode, const u32* dcode) {
    if (!sym_is_match(sym)) return lcode[sym] >> 16;
    const int lc = (int)sym_len(sym) - 3, code = length_code(lc), dc = dist_code((int)sym_dist(sym) - 1);
    return (lcode[code + 257] >> 16) + extra_lbits(code) + (dcode[dc] >> 16) + extra_dbits(dc);
}
// Code tables of a planned block: (length << 16 | reversed code) for every literal/length and distance symbol.
GZ_HD void code_tables(const BlockTrees& t, int type, u32* lcode, u32* dcode) {
    for (int n = 0; n < L_CODES; n++)   // past max_code: no code (scan_tree left its guard length there)
        lcode[n] = type == BT_FIXED ? (u32)static_llen(n) << 16 | static_lcode(n) : n > t.l.max_code ? 0 : (u32)t.l.len[n] << 16 | t.l.code[n];
    for (int n = 0; n < D_CODES; n++)
        dcode[n] = type == BT_FIXED ? 5u << 16 | bi_reverse((u32)n, 5) : n > t.d.max_code ? 0 : (u32)t.d.len[n] << 16 | t.d.code[n];
}

// ---- bit offsets: a block maps the stream's bit offset x to x + T[x mod 8] (a stored block aligns after its 3 header bits, so
// its size depends on x mod 8).  Maps compose, so the offsets of a run of blocks are a scan with this operator.
struct OffMap { u64 add[8]; };
GZ_HD OffMap off_plain(u64 bits) { OffMap m; for (int r = 0; r < 8; r++) m.add[r] = bits; return m; }
GZ_HD OffMap off_stored(u64 stored_len) {   // 3 bits, pad to a byte, LEN, NLEN, the bytes
    OffMap m;
    for (int r = 0; r < 8; r++) m.add[r] = 3 + ((8 - (r + 3) % 8) % 8) + 32 + 8 * stored_len;
    return m;
}
GZ_HD OffMap off_then(const OffMap& f, const OffMap& g) {   // f first, then g
    OffMap m;
    for (int r = 0; r < 8; r++) m.add[r] = f.add[r] + g.add[(r + f.add[r]) & 7];
    return m;
}
GZ_HD u64 off_apply(const OffMap& f, u64 x) { return x + f.add[x & 7]; }

// ---- CRC-32 (gzip's), with zlib's crc32_combine arithmetic: multiplication modulo the reflected polynomial.
constexpr u32 CRC_POLY = 0xedb88320u;
GZ_HD u32 crc_table_entry(u32 n) { u32 c = n; for (int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1; return c; }
GZ_HD u32 crc_update(u32 crc, const u32* table, const u8* p, u64 n) {   // crc: raw register (pre/post inversion done by callers)
    for (u64 i = 0; i < n; i++) crc = table[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
    return crc;
}
GZ_HD u32 multmodp(u32 a, u32 b) {
    u32 m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}
GZ_HD u32 x8nmodp(u64 n) {   // x^(8n) modulo the polynomial
    u32 p = 1u << 31, x2k = 1u << 30;   // x^0, x^1 (reflected)
    // x^(2^k) for k = 0.. by squaring; x^(8n) = product over the bits of 8n
    u64 e = n << 3;
    while (e) {
        if (e & 1) p = multmodp(x2k, p);
        x2k = multmodp(x2k, x2k);
        e >>= 1;
    }
    return p;
}
// crc of A || B from crc(A), crc(B) (finished CRCs, as zlib's crc32 returns them) and |B|.
GZ_HD u32 crc_combine(u32 crc_a, u32 crc_b, u64 len_b) { return multmodp(x8nmodp(len_b), crc_a) ^ crc_b; }

}  // namespace gz
