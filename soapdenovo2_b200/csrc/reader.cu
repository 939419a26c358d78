// reader.cu -- the map stage's line-by-line reader on the GPU: one chunk of a FASTA/FASTQ file -> 2-bit packed reads, with the rules
// of the reference's fgets readers, so that wrapped (multi-line) FASTA and FASTQ give exactly the reads the reference's `map` reads.
//
// Replaces (reference file:line, standardPregraph/):
//   readseq1by1 / read1seqfq   readseq1by1.c:50-136, 362-447   (the readers read1seqInLib calls for f=, p= and q= files)
//   the counting of read1seqInLib  readseq1by1.c:1206-1243      (*len_seq > 0 || !feof: an empty last record is not a read)
//   reverse2k                  readseq1by1.c:788-802
// Their rules, restated:
//   pieces     fgets(str, P + 1, fp) returns at most P bytes: a line of L bytes (its '\n' included) arrives as ceil(L / P) pieces, and
//              every piece is classified by its own first byte.
//   FASTA      '#' pieces are skipped anywhere; a '>' piece ends the record before it and starts the next one; every other piece is
//              appended to the current record.  Pieces before the first header are read and discarded.
//   FASTQ      pieces are skipped until one starts with '@' (the header); the next pieces are sequence until one starts with '+'; the
//              piece after that is skipped as the quality line, whatever it holds.  A state machine: seeking '@' (S0), in sequence
//              (S1), the next piece is the quality (S2).
//   truncation a sequence piece of raw length strL (every byte, '\n' and '\r' included) is cut to cutoff - n when strL + n > cutoff
//              (n: bases kept so far); letters and '.' in the kept bytes are bases, every other byte is dropped.
//   counting   a record is a read unless it is empty and the fgets that ended it reached the end of the file.
//
// Kernels, each a stream over its input:
//   k_fg_count      '\n' and NUL bytes per 2 KB tile (1 x text, 16-byte loads); the tile counts are scanned
//   k_fg_nlpos      the position of every '\n' (1 x text, 16-byte loads)
//   k_fg_pieces     one thread per line: its pieces' starts and classes (FASTA: the piece's role outright)
//   k_fq_*          FASTQ: the state before every piece, from an exclusive scan of the pieces' transition maps (3 entries of 2 bits;
//                   composition is associative) -> the piece's role.  Quality lines may start with '@' or '+', so no line-number rule
//                   can stand in for it.
//   k_fg_letters    one warp per piece, 32 bytes per step: bases in a sequence piece, and whether a base follows a dropped byte in it
//                   (1 x text); header pieces: the length of the name sscanf("%s") would copy
//   k_fg_reclen     one thread per record from two scans (header pieces -> record bounds; bases -> per-piece base prefix).  A record
//                   whose pieces hold bases before any dropped byte ("clean") has min(bases, cutoff) bases, the first that many; the
//                   truncation rule cannot reach a base past a dropped byte there.  Any other record goes on a redo list.
//   k_fg_fix_len    one warp per listed record: the truncation rule replayed piece by piece
//   k_fg_decode     one thread per output word, 32 bases from the per-piece base prefix (0.5 x text), reverse2k applied
//   k_fg_fix_decode one warp per listed record: the replay again, writing its bases
// Refused before any read is returned: a NUL byte (strlen would end the piece there, silently) and a header whose first name token is
// longer than the reference's 256-byte read_name (sscanf writes past the buffer: no output is defined for it).
//
// Chunks.  The caller cuts nothing.  A chunk that does not end the file returns the reads of every record that a later header
// completes, and the byte offset of its last header: the caller keeps the bytes from there, prepends them to its next read and calls
// again.  The next chunk therefore starts with a header piece in the seeking state, and its piece boundaries fall where the file's
// do (a header piece starts a line, or P bytes into one).  Without a header the chunk keeps its last piece.
#include "engine_impl.cuh"
#include "reader.cuh"
#include "scan.cuh"

namespace pgb {

constexpr int FG_TILE = 2048;                // bytes of text per warp tile
constexpr int FG_GROUPS = FG_TILE / 16;      // 16-byte groups per tile
constexpr int FG_ITERS = FG_GROUPS / 32;

enum : u8 { R_SKIP = 0, R_HDR = 1, R_SEQ = 2 };          // a piece's role
enum : u8 { CL_OTHER = 0, CL_AT = 1, CL_PLUS = 3 };     // FASTQ: a piece's class, before the state scan turns it into its role
enum { FG_NL = 0, FG_NUL, FG_PIECES, FG_HDR, FG_BADNAME, FG_REDO, FG_WORDS, FG_CUT, FG_TAIL, FG_SLOTS };

// bit b set <=> byte b of the 16-byte group equals the byte of `pat` (bytes past the end of the text are masked out)
__device__ __forceinline__ unsigned fg_eq_mask(const uint4& v, unsigned pat, u64 rem) {
    unsigned m = 0;
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const unsigned r = __vcmpeq4(w[k], pat) & 0x01010101u;
        m |= ((r | (r >> 7) | (r >> 14) | (r >> 21)) & 0xFu) << (4 * k);
    }
    if (rem < 16) m &= (1u << rem) - 1;
    return m;
}

__global__ void __launch_bounds__(256) k_fg_count(const uint4* __restrict__ text, u64 nbytes, u64 n_tiles, u32* __restrict__ tile_cnt, u64* slots) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n_groups = (nbytes + 15) / 16;
    unsigned nul = 0;
    for (u64 tile = warp0; tile < n_tiles; tile += nwarps) {
        unsigned cnt = 0;
#pragma unroll
        for (int it = 0; it < FG_ITERS; it++) {
            const u64 grp = tile * FG_GROUPS + it * 32 + lane;
            if (grp < n_groups) {
                const uint4 v = __ldg(text + grp);
                const u64 rem = nbytes - grp * 16;
                cnt += __popc(fg_eq_mask(v, 0x0A0A0A0Au, rem));
                nul += __popc(fg_eq_mask(v, 0u, rem));
            }
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) tile_cnt[tile] = cnt;
    }
    nul = __reduce_add_sync(0xffffffffu, nul);
    if (lane == 0 && nul) atomicAdd((unsigned long long*)&slots[FG_NUL], (unsigned long long)nul);
}

__global__ void __launch_bounds__(256) k_fg_nlpos(const uint4* __restrict__ text, u64 nbytes, u64 n_tiles, const u32* __restrict__ tile_base,
                                                  u32* __restrict__ nl) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n_groups = (nbytes + 15) / 16;
    for (u64 tile = warp0; tile < n_tiles; tile += nwarps) {
        u32 g = tile_base[tile];
#pragma unroll
        for (int it = 0; it < FG_ITERS; it++) {
            const u64 grp = tile * FG_GROUPS + it * 32 + lane;
            unsigned m = grp < n_groups ? fg_eq_mask(__ldg(text + grp), 0x0A0A0A0Au, nbytes - grp * 16) : 0u;
            const unsigned cn = __popc(m);
            unsigned inc = cn;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned v = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= d) inc += v;
            }
            u32 o = g + inc - cn;
            while (m) {
                const int b = __ffs(m) - 1;
                m &= m - 1;
                nl[o++] = (u32)(grp * 16 + b);
            }
            g += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
}

// line i = text[s, e): '\n' included, the last line possibly open
struct FgLines {
    const u32* nl;
    u64 n_nl, nbytes;
    __device__ void span(u64 i, u64& s, u64& e) const {
        s = i ? (u64)nl[i - 1] + 1 : 0;
        e = i < n_nl ? (u64)nl[i] + 1 : nbytes;
    }
};
struct FgLinePiecesIn {
    FgLines L;
    u64 P;
    __device__ u64 operator()(u64 i) const { u64 s, e; L.span(i, s, e); return (e - s + P - 1) / P; }
};

__global__ void __launch_bounds__(256) k_fg_pieces(const unsigned char* __restrict__ text, FgLines L, u64 n_lines, u32 P, const u32* __restrict__ lpb,
                                                   int fastq, u32* __restrict__ pstart, u8* __restrict__ prole) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n_lines; i += (u64)gridDim.x * blockDim.x) {
        u64 s, e;
        L.span(i, s, e);
        u32 p = lpb[i];
        for (u64 a = s; a < e; a += P, p++) {
            const unsigned char c = text[a];
            pstart[p] = (u32)a;
            prole[p] = fastq ? (c == '@' ? CL_AT : c == '+' ? CL_PLUS : CL_OTHER) : (c == '>' ? R_HDR : c == '#' ? R_SKIP : R_SEQ);
        }
        if (i == n_lines - 1) pstart[p] = (u32)L.nbytes;   // p == the piece count: pstart[np] closes the last piece
    }
}

// ---------------------------------------------------------------------------------------------- FASTQ: the state scan
// A map sends each state s in {S0, S1, S2} to map >> 2s & 3.  fq_then(a, b): first a, then b.
constexpr unsigned FQ_ID = 0x24u;   // 0 | 1 << 2 | 2 << 4
__device__ __forceinline__ unsigned fq_map(unsigned cls) {
    // '@': S0 -> S1 (a header), S1 stays (a sequence piece), S2 -> S0 (the quality);  '+': S1 -> S2;  other: S0 and S1 stay, S2 -> S0
    return cls == CL_AT ? 0x05u : cls == CL_PLUS ? 0x08u : 0x04u;
}
__device__ __forceinline__ unsigned fq_then(unsigned a, unsigned b) {
    unsigned r = 0;
#pragma unroll
    for (int s = 0; s < 3; s++) r |= ((b >> (2 * ((a >> (2 * s)) & 3u))) & 3u) << (2 * s);
    return r;
}
__device__ __forceinline__ u8 fq_role(unsigned state, unsigned cls) {
    if (state == 0) return cls == CL_AT ? R_HDR : R_SKIP;
    if (state == 1) return cls == CL_PLUS ? R_SKIP : R_SEQ;
    return R_SKIP;
}
// block-wide exclusive scan of maps (SCAN_THREADS threads); *total: the whole block's map
__device__ unsigned fq_block_scan(unsigned v, unsigned* total) {
    __shared__ unsigned s_w[SCAN_THREADS / 32], s_pre[SCAN_THREADS / 32], s_tot;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc = fq_then(o, inc);
    }
    if (lane == 31) s_w[wid] = inc;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned a = FQ_ID;
        for (int w = 0; w < SCAN_THREADS / 32; w++) { s_pre[w] = a; a = fq_then(a, s_w[w]); }
        s_tot = a;
    }
    __syncthreads();
    unsigned ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) ex = FQ_ID;
    const unsigned r = fq_then(s_pre[wid], ex);
    *total = s_tot;
    __syncthreads();
    return r;
}
// the map of SCAN_ITEMS consecutive pieces of one thread
__device__ __forceinline__ unsigned fq_thread_map(const u8* cls, u64 np, u64 first) {
    unsigned m = FQ_ID;
#pragma unroll 4
    for (int k = 0; k < SCAN_ITEMS; k++)
        if (first + k < np) m = fq_then(m, fq_map(cls[first + k]));
    return m;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_fq_tile_maps(const u8* __restrict__ cls, u64 np, u32* __restrict__ tile_map) {
    const u64 first = (u64)blockIdx.x * SCAN_TILE + (u64)threadIdx.x * SCAN_ITEMS;
    unsigned tot;
    fq_block_scan(fq_thread_map(cls, np, first), &tot);
    if (threadIdx.x == 0) tile_map[blockIdx.x] = tot;
}
// the state before every tile: one thread folds the tile maps (a few thousand per 256 MB chunk), starting in S0
__global__ void k_fq_tile_states(u32* tile_map, u64 n_tiles) {
    unsigned s = 0;
    for (u64 t = 0; t < n_tiles; t++) {
        const unsigned m = tile_map[t];
        tile_map[t] = s;
        s = (m >> (2 * s)) & 3u;
    }
}
__global__ void __launch_bounds__(SCAN_THREADS) k_fq_roles(u8* __restrict__ cls, u64 np, const u32* __restrict__ tile_state) {
    const u64 first = (u64)blockIdx.x * SCAN_TILE + (u64)threadIdx.x * SCAN_ITEMS;
    unsigned tot;
    const unsigned ex = fq_block_scan(fq_thread_map(cls, np, first), &tot);
    unsigned s = (ex >> (2 * tile_state[blockIdx.x])) & 3u;
    for (int k = 0; k < SCAN_ITEMS && first + k < np; k++) {
        const unsigned c = cls[first + k];
        cls[first + k] = fq_role(s, c);
        s = (fq_map(c) >> (2 * s)) & 3u;
    }
}

// ---------------------------------------------------------------------------------------------- records
struct FgHdrIn {
    const u8* role;
    __device__ u64 operator()(u64 i) const { return role[i] == R_HDR ? 1u : 0u; }
};
struct FgHdrOut {
    u32* hdr;
    __device__ void operator()(u64 i, u64 prefix, u64 v) const { if (v) hdr[prefix] = (u32)i; }
};

__device__ __forceinline__ bool fg_base_char(unsigned c) { return ((c | 0x20u) - 'a') < 26u || c == '.'; }
__device__ __forceinline__ unsigned fg_base_code(unsigned c) { return c == '.' ? 0u : ((c & 6u) >> 1); }
__device__ __forceinline__ bool fg_space(unsigned c) { return c == ' ' || (c >= 9u && c <= 13u); }

// val[p] = bases of sequence piece p | 1 << 32 when a base follows a dropped byte in it; 0 for every other piece
__global__ void __launch_bounds__(256) k_fg_letters(const unsigned char* __restrict__ text, const u32* __restrict__ pstart, const u8* __restrict__ role,
                                                    u64 np, u64* __restrict__ val, u64* slots) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    unsigned bad = 0;
    for (u64 p = warp0; p < np; p += nwarps) {
        const unsigned r = role[p];
        const u32 s = pstart[p], n = pstart[p + 1] - s;
        if (r == R_HDR) {   // sscanf(&str[1], "%s", name): leading white space skipped, then the token, within this piece
            if (lane == 0) {
                u32 i = 1;
                while (i < n && fg_space(text[s + i])) i++;
                u32 j = i;
                while (j < n && j - i <= (u32)FG_NAME_MAX && !fg_space(text[s + j])) j++;
                if (j - i > (u32)FG_NAME_MAX) bad++;
                val[p] = 0;
            }
            continue;
        }
        if (r != R_SEQ) { if (lane == 0) val[p] = 0; continue; }
        u32 bases = 0;
        bool dropped = false, unclean = false;
        for (u32 b = 0; b < n; b += 32) {
            const u32 i = b + lane;
            const bool in = i < n;
            const bool isb = in && fg_base_char(text[s + i]);
            const unsigned bal = __ballot_sync(0xffffffffu, isb), non = __ballot_sync(0xffffffffu, in && !isb);
            if (dropped && bal) unclean = true;
            if (non) {
                if (((u64)bal >> __ffs(non)) != 0) unclean = true;
                dropped = true;
            }
            bases += __popc(bal);
        }
        if (lane == 0) val[p] = (u64)bases | (unclean ? 1ull << 32 : 0ull);
    }
    if (bad) atomicAdd((unsigned long long*)&slots[FG_BADNAME], (unsigned long long)bad);
}

// record r: its header is piece hdr[r]; its pieces end at the next header (or at the last piece)
__device__ __forceinline__ u32 fg_rec_end(const u32* hdr, u64 n_hdr, u64 np, u64 r) { return r + 1 < n_hdr ? hdr[r + 1] : (u32)np; }

__global__ void __launch_bounds__(256) k_fg_reclen(const u32* __restrict__ hdr, u64 n_hdr, u64 n_rec, u64 np, const u64* __restrict__ pfx, u32 cutoff,
                                                   u32* __restrict__ lens, u8* __restrict__ fix, u32* __restrict__ redo, u64* slots) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < n_rec; r += (u64)gridDim.x * blockDim.x) {
        const u64 d = pfx[fg_rec_end(hdr, n_hdr, np, r)] - pfx[hdr[r]];
        if (d >> 32) {
            lens[r] = 0;
            fix[r] = 1;
            redo[atomicAdd((unsigned long long*)&slots[FG_REDO], 1ull)] = (u32)r;
        } else {
            lens[r] = min((u32)d, cutoff);
            fix[r] = 0;
        }
    }
}

// readseq1by1's loop over one record's pieces, one warp: the raw-length cut, then the bases of the kept bytes.  With out: base p
// goes to out (reverse: to len - 1 - p, complemented), out[] zeroed by the caller.  Returns the record's length (warp-uniform).
__device__ u32 fg_replay(const unsigned char* __restrict__ text, const u32* __restrict__ pstart, const u8* __restrict__ role, u32 b, u32 e, u32 cutoff,
                         int reverse, u32 len, u64* out) {
    const int lane = threadIdx.x & 31;
    u32 n = 0;
    for (u32 q = b + 1; q < e; q++) {
        if (role[q] != R_SEQ) continue;
        const u32 s = pstart[q];
        u32 strL = pstart[q + 1] - s;
        if ((u64)strL + n > cutoff) strL = cutoff - n;
        for (u32 i0 = 0; i0 < strL; i0 += 32) {
            const u32 i = i0 + lane;
            const unsigned ch = i < strL ? text[s + i] : 0u;
            const bool v = i < strL && fg_base_char(ch);
            const unsigned bal = __ballot_sync(0xffffffffu, v);
            if (out && v) {
                const u32 p = n + __popc(bal & ((1u << lane) - 1));
                const u32 oi = reverse ? len - 1 - p : p;
                atomicOr(&out[oi >> 5], (u64)(fg_base_code(ch) ^ (reverse ? 2u : 0u)) << (2 * (oi & 31)));
            }
            n += __popc(bal);
        }
    }
    return n;
}

__global__ void __launch_bounds__(256) k_fg_fix_len(const unsigned char* __restrict__ text, const u32* __restrict__ pstart, const u8* __restrict__ role,
                                                    const u32* __restrict__ hdr, u64 n_hdr, u64 np, u32 cutoff, const u32* __restrict__ redo,
                                                    const u64* slots, u32* __restrict__ lens) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n = slots[FG_REDO];
    for (u64 i = warp0; i < n; i += nwarps) {
        const u32 r = redo[i];
        const u32 len = fg_replay(text, pstart, role, hdr[r], fg_rec_end(hdr, n_hdr, np, r), cutoff, 0, 0, nullptr);
        if (lane == 0) lens[r] = len;
    }
}

__global__ void __launch_bounds__(256) k_fg_fix_decode(const unsigned char* __restrict__ text, const u32* __restrict__ pstart, const u8* __restrict__ role,
                                                       const u32* __restrict__ hdr, u64 n_hdr, u64 np, u32 cutoff, int reverse, const u32* __restrict__ redo,
                                                       const u64* slots, const u32* __restrict__ lens, const u64* __restrict__ wofs, u64* __restrict__ words) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n = slots[FG_REDO];
    for (u64 i = warp0; i < n; i += nwarps) {
        const u32 r = redo[i];
        u64* out = words + wofs[r];
        for (u64 w = lane; w < wofs[r + 1] - wofs[r]; w += 32) out[w] = 0;
        __syncwarp();
        fg_replay(text, pstart, role, hdr[r], fg_rec_end(hdr, n_hdr, np, r), cutoff, reverse, lens[r], out);
    }
}

// one thread per output word of the clean records: its record by binary search over the word offsets, its first piece by binary
// search over the base prefix (low 32 bits of pfx: the bases before each piece), then up to 32 bases
__global__ void __launch_bounds__(256) k_fg_decode(const unsigned char* __restrict__ text, const u32* __restrict__ pstart, const u32* __restrict__ hdr,
                                                   u64 n_hdr, u64 np, const u64* __restrict__ pfx, const u32* __restrict__ lens, const u8* __restrict__ fix,
                                                   const u64* __restrict__ wofs, u64 n_rec, u64 n_words, int reverse, u64* __restrict__ words) {
    for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (u64)gridDim.x * blockDim.x) {
        u64 lo = 0, hi = n_rec - 1;   // the last record with wofs[r] <= w: records without bases share their offset with the next one
        while (lo < hi) {
            const u64 mid = (lo + hi + 1) / 2;
            if (wofs[mid] <= w) lo = mid; else hi = mid - 1;
        }
        const u64 r = lo;
        if (fix[r]) continue;
        const u32 len = lens[r], i0 = (u32)(w - wofs[r]) * 32u, i1 = min(i0 + 32u, len);
        const u32 fa = reverse ? len - i1 : i0, fb = reverse ? len - i0 : i1;   // forward bases [fa, fb)
        const u32 b = hdr[r], e = fg_rec_end(hdr, n_hdr, np, r), base0 = (u32)pfx[b];
        u32 ql = b + 1, qh = e - 1;   // the last piece whose base prefix is <= fa
        while (ql < qh) {
            const u32 mid = (ql + qh + 1) / 2;
            if ((u32)pfx[mid] - base0 <= fa) ql = mid; else qh = mid - 1;
        }
        u32 q = ql, q_lo = (u32)pfx[q] - base0, q_hi = (u32)pfx[q + 1] - base0;
        u64 out = 0;
        for (u32 f = fa; f < fb; f++) {
            while (f >= q_hi) { q++; q_lo = q_hi; q_hi = (u32)pfx[q + 1] - base0; }
            const unsigned c = fg_base_code(text[pstart[q] + (f - q_lo)]);
            const u32 o = reverse ? (len - 1 - f) - i0 : f - i0;
            out |= (u64)(c ^ (reverse ? 2u : 0u)) << (2 * o);
        }
        words[w] = out;
    }
}

// where the chunk's unfinished record starts (cut), and the first record whose ending fgets reached the end of the file (tail): such a
// record is a read only when it holds bases
__global__ void k_fg_tail(const unsigned char* __restrict__ text, u64 nbytes, const u32* __restrict__ pstart, const u8* __restrict__ role,
                          const u32* __restrict__ hdr, u64 n_hdr, u64 np, u32 P, int fastq, int at_eof, u64* slots) {
    if (!at_eof) {
        slots[FG_CUT] = n_hdr ? pstart[hdr[n_hdr - 1]] : (np ? pstart[np - 1] : 0u);
        slots[FG_TAIL] = n_hdr ? n_hdr - 1 : 0;
        return;
    }
    slots[FG_CUT] = nbytes;
    if (n_hdr == 0) { slots[FG_TAIL] = 0; return; }
    // the file's last fgets ran into its end: the last piece is open and shorter than P
    const bool last_eof = text[nbytes - 1] != '\n' && pstart[np] - pstart[np - 1] < P;
    if (!fastq) {   // the last record ends at the end of the file; the one before, at a header that may be the open last piece
        slots[FG_TAIL] = (n_hdr >= 2 && hdr[n_hdr - 1] == np - 1 && last_eof) ? n_hdr - 2 : n_hdr - 1;
        return;
    }
    u64 q = hdr[n_hdr - 1] + 1;   // the last record's '+' piece, then its quality piece
    while (q < np && role[q] != R_SKIP) q++;
    const bool eof = q + 1 >= np || (q + 1 == np - 1 && last_eof);
    slots[FG_TAIL] = eof ? n_hdr - 1 : n_hdr;
}

// ---------------------------------------------------------------------------------------------- host
size_t FgetsReader::read(const unsigned char* d_text, size_t nbytes, int fastq, int piece_len, int cutoff, int reverse, bool at_eof, int n_sm,
                         cudaStream_t st, std::vector<u64>* words, std::vector<u32>* lens) {
    if (nbytes == 0) return 0;
    if (nbytes >= (1ull << 32)) throw std::runtime_error("pgb200: a text chunk must be smaller than 4 GiB (feed it in pieces)");
    if (piece_len < 1 || cutoff < 0) throw std::runtime_error("pgb200: the fgets reader needs a piece length >= 1 and a cutoff >= 0");
    const u64 P = (u64)piece_len;
    slots_.ensure(FG_SLOTS * sizeof(u64));
    u64* slots = slots_.as<u64>();
    if (!h_) h_ = make_pinned<u64>(FG_SLOTS + 2);   // made on first use, with the caller's device current
    u64* h = h_.h;
    PG_CUDA(cudaMemsetAsync(slots, 0, FG_SLOTS * sizeof(u64), st));
    scan_.ensure(scan_scratch_elems(nbytes + 2) * sizeof(u64) + 256);
    u64* tmp = scan_.as<u64>();
    const auto blocks = [&](u64 n, u64 per_block, u64 per_sm) { return (unsigned)std::max<u64>(1, std::min<u64>((n + per_block - 1) / per_block, (u64)n_sm * per_sm)); };

    // lines
    const u64 n_tiles = (nbytes + FG_TILE - 1) / FG_TILE;
    tiles_.ensure(n_tiles * sizeof(u32) * 2 + 16);
    u32* tile_cnt = tiles_.as<u32>();
    u32* tile_base = tile_cnt + n_tiles;
    const uint4* t16 = reinterpret_cast<const uint4*>(d_text);
    k_fg_count<<<blocks(n_tiles, 8, 16), 256, 0, st>>>(t16, (u64)nbytes, n_tiles, tile_cnt, slots);
    PG_CUDA(cudaGetLastError());
    device_scan(ScanU32In{tile_cnt}, ScanU32Out{tile_base}, n_tiles, tmp, slots + FG_NL, st);
    unsigned char* h_last = reinterpret_cast<unsigned char*>(h + FG_SLOTS);
    PG_CUDA(cudaMemcpyAsync(h_last, d_text + nbytes - 1, 1, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaMemcpyAsync(h, slots, FG_SLOTS * sizeof(u64), cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    if (h[FG_NUL])
        throw std::runtime_error("pgb200: the text holds a NUL byte; the reference's line reader would silently end the line there");
    const u64 n_nl = h[FG_NL], n_lines = n_nl + (*h_last != '\n' ? 1 : 0);
    nl_.ensure(n_nl * sizeof(u32) + 16);
    k_fg_nlpos<<<blocks(n_tiles, 8, 16), 256, 0, st>>>(t16, (u64)nbytes, n_tiles, tile_base, nl_.as<u32>());
    PG_CUDA(cudaGetLastError());
    const FgLines L{nl_.as<u32>(), n_nl, (u64)nbytes};
    lpb_.ensure(n_lines * sizeof(u32) + 16);
    device_scan(FgLinePiecesIn{L, P}, ScanU32Out{lpb_.as<u32>()}, n_lines, tmp, slots + FG_PIECES, st);
    PG_CUDA(cudaMemcpyAsync(h, slots, FG_SLOTS * sizeof(u64), cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));

    // pieces and their roles
    const u64 np = h[FG_PIECES];   // >= 1: the text is not empty
    pstart_.ensure((np + 1) * sizeof(u32) + 16);
    role_.ensure(np + 16);
    u32* pstart = pstart_.as<u32>();
    u8* role = role_.as<u8>();
    k_fg_pieces<<<blocks(n_lines, 256, 16), 256, 0, st>>>(d_text, L, n_lines, (u32)P, lpb_.as<u32>(), fastq, pstart, role);
    PG_CUDA(cudaGetLastError());
    if (fastq) {
        const u64 pt = (np + SCAN_TILE - 1) / SCAN_TILE;
        tiles_.ensure(std::max<u64>(n_tiles * 2, pt) * sizeof(u32) + 16);
        k_fq_tile_maps<<<(unsigned)pt, SCAN_THREADS, 0, st>>>(role, np, tiles_.as<u32>());
        k_fq_tile_states<<<1, 1, 0, st>>>(tiles_.as<u32>(), pt);
        k_fq_roles<<<(unsigned)pt, SCAN_THREADS, 0, st>>>(role, np, tiles_.as<u32>());
        PG_CUDA(cudaGetLastError());
    }
    hdr_.ensure(np * sizeof(u32) + 16);
    u32* hdr = hdr_.as<u32>();
    device_scan(FgHdrIn{role}, FgHdrOut{hdr}, np, tmp, slots + FG_HDR, st);
    val_.ensure(np * sizeof(u64) + 16);
    pfx_.ensure((np + 1) * sizeof(u64) + 16);
    u64* pfx = pfx_.as<u64>();
    k_fg_letters<<<blocks(np, 8, 16), 256, 0, st>>>(d_text, pstart, role, np, val_.as<u64>(), slots);
    PG_CUDA(cudaGetLastError());
    device_scan(ScanU64In{val_.as<u64>()}, ScanU64Out{pfx}, np, tmp, pfx + np, st);
    PG_CUDA(cudaMemcpyAsync(h, slots, FG_SLOTS * sizeof(u64), cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    if (h[FG_BADNAME])
        throw std::runtime_error("pgb200: a header's name is longer than 256 bytes; the reference would write past its read_name buffer");

    // records: lengths, word offsets, bases
    const u64 n_hdr = h[FG_HDR], n_rec = at_eof ? n_hdr : (n_hdr ? n_hdr - 1 : 0);
    lens_.ensure(n_rec * sizeof(u32) + 16);
    fix_.ensure(n_rec + 16);
    redo_.ensure(n_rec * sizeof(u32) + 16);
    wofs_.ensure((n_rec + 1) * sizeof(u64) + 16);
    u32* d_lens = lens_.as<u32>();
    u64* wofs = wofs_.as<u64>();
    if (n_rec) {
        k_fg_reclen<<<blocks(n_rec, 256, 16), 256, 0, st>>>(hdr, n_hdr, n_rec, np, pfx, (u32)cutoff, d_lens, fix_.as<u8>(), redo_.as<u32>(), slots);
        k_fg_fix_len<<<(unsigned)n_sm * 8, 256, 0, st>>>(d_text, pstart, role, hdr, n_hdr, np, (u32)cutoff, redo_.as<u32>(), slots, d_lens);
        PG_CUDA(cudaGetLastError());
    }
    device_scan(ScanWordsOfLen{d_lens}, ScanU64Out{wofs}, n_rec, tmp, wofs + n_rec, st);   // wofs[n_rec]: the word total, read as r + 1
    PG_CUDA(cudaMemcpyAsync(slots + FG_WORDS, wofs + n_rec, sizeof(u64), cudaMemcpyDeviceToDevice, st));
    k_fg_tail<<<1, 1, 0, st>>>(d_text, (u64)nbytes, pstart, role, hdr, n_hdr, np, (u32)P, fastq, at_eof ? 1 : 0, slots);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cudaMemcpyAsync(h, slots, FG_SLOTS * sizeof(u64), cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    const u64 n_words = h[FG_WORDS], cut = h[FG_CUT], tail = h[FG_TAIL];
    words_.ensure(n_words * sizeof(u64) + 16);
    if (n_words) {
        k_fg_decode<<<blocks(n_words, 256, 32), 256, 0, st>>>(d_text, pstart, hdr, n_hdr, np, pfx, d_lens, fix_.as<u8>(), wofs, n_rec, n_words, reverse,
                                                               words_.as<u64>());
        k_fg_fix_decode<<<(unsigned)n_sm * 8, 256, 0, st>>>(d_text, pstart, role, hdr, n_hdr, np, (u32)cutoff, reverse, redo_.as<u32>(), slots, d_lens, wofs,
                                                            words_.as<u64>());
        PG_CUDA(cudaGetLastError());
    }
    const size_t l0 = lens->size(), w0 = words->size();
    lens->resize(l0 + n_rec);
    words->resize(w0 + n_words);
    if (n_rec) PG_CUDA(cudaMemcpyAsync(lens->data() + l0, d_lens, n_rec * sizeof(u32), cudaMemcpyDeviceToHost, st));
    if (n_words) PG_CUDA(cudaMemcpyAsync(words->data() + w0, words_.p, n_words * sizeof(u64), cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    // read1seqInLib: a record whose last fgets reached the end of the file is a read only when it holds bases (these are the
    // chunk's last one or two records, and an empty one has no words)
    size_t n_out = l0 + n_rec;
    while (n_out > l0 + tail && (*lens)[n_out - 1] == 0) n_out--;
    lens->resize(n_out);
    return (size_t)cut;
}

}   // namespace pgb
