// deflate.cu -- a gzip writer whose files equal gzopen(path, "w") + gzwrite + gzclose's (zlib level 6), with the deflate on the GPU.
//
// zlib's deflate is one sequential loop, but its output is a function of the input text alone, and most of the work behind it is
// independent per position.  One round over a buffer of input (deflate.cuh has the rules):
//   k_hash      the hash chains: for every position, the distance to the previous one with the same hash (one warp per 64 KB tile
//               with its 32 KB of history, a shared-memory head table)
//   k_match     longest_match at every loop top, for the full and the quarter chain (one CTA per 8 KB tile, window in shared memory)
//   k_lazy_spec the lazy automaton, one thread per 4096 loop tops, each from a fresh state at its segment start
//   k_lazy_fix  every segment whose true entry state differs re-runs from it until it meets its speculative trajectory (same loop
//               top, same state), from where the symbols are the speculative ones; repeated until no exit state changes
//   k_gather    the symbols of all segments in stream order
//   k_block     one CTA per block of 16383 symbols: frequencies, the trees, the block type, the code tables, the tree header
//   (host)      the bit offset of every block: the composed offset maps of deflate.cuh (a stored block aligns)
//   k_pack      one CTA per block writes its bits at its offset (atomicOr stitches the words shared with neighbours)
//   k_crc       CRC-32 per 4 KB piece, combined on the host
// Streaming: a round runs when the buffer is full.  Not final, it writes every complete block and carries the input from the next
// block's first byte (and the 32 KB before it), the automaton state there and the partial output byte; the carry is at most one
// block's input plus the window, so memory is bounded by the buffer whatever the file size.
#include "cuda_owner.h"
#include "deflate.cuh"
#include "deflate.h"

#include <cuda_runtime.h>
#include <zlib.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

namespace gz {

constexpr int HTILE = 65536;           // positions per k_hash warp
constexpr int MTILE = 8192;            // loop tops per k_match CTA
constexpr int MTHREADS = 512;
constexpr int SEG = 4096;              // loop tops per automaton segment
constexpr int HDR_WORDS = 160;         // a dynamic block's tree description fits in 160 words (at most 14 + 57 + 316 * 14 bits)
constexpr int CRC_PIECE = 4096;
constexpr size_t DEFAULT_CHUNK = 32ull << 20;
constexpr size_t MIN_CHUNK = 5ull << 20;   // > 16383 * 258: every full round completes at least one block
constexpr size_t CARRY = 8ull << 20;       // >= one block's input + the window + the undecided tail

// ---- hash chains
__global__ void __launch_bounds__(32) k_hash(const u8* __restrict__ b, i64 nhash, u16* __restrict__ pv) {
    extern __shared__ u32 head[];   // 32768: position - h0 + 1 of the newest insert per hash (0: none)
    const int lane = threadIdx.x;
    const i64 t0 = (i64)blockIdx.x * HTILE, t1 = min(t0 + HTILE, nhash), h0 = max(t0 - (i64)WSIZE, (i64)0);
    for (int i = lane; i < 32768; i += 32) head[i] = 0;
    __syncwarp();
    for (i64 p0 = h0; p0 < t1; p0 += 32) {
        const i64 p = p0 + lane;
        const bool ok = p < t1;
        const u32 h = ok ? hash3(b[p], b[p + 1], b[p + 2]) : 0x10000u + lane;
        const u32 grp = __match_any_sync(0xffffffffu, h);
        const u32 lower = grp & ((1u << lane) - 1);
        u32 d = 0;
        if (ok) {
            if (lower) d = lane - (31 - __clz(lower));
            else if (const u32 q = head[h]) { const i64 dd = p - (h0 + q - 1); d = dd < WSIZE ? (u32)dd : 0; }
            if (p >= t0) pv[p] = (u16)d;
        }
        __syncwarp();
        if (ok && (grp >> lane) == 1u) head[h] = (u32)(p - h0 + 1);
        __syncwarp();
    }
}

// ---- longest_match at every loop top in [lt0, lt1)
struct Round {
    const u8* b;        // buffer
    u64 buf0;           // stream offset of b[0]
    i64 avail;          // bytes in the buffer
    int final;
    i64 r0;             // first loop top (relative)
    i64 nlt;            // loop tops [r0, r0 + nlt): final includes the terminal one at avail
    i64 lmatch;         // loop tops below lmatch have a match search
};
__device__ __forceinline__ i64 base_rel(const Round& R, i64 s) {
    return (i64)slide_base(R.buf0 + (u64)s, R.buf0 + (u64)R.avail, R.final) - (i64)R.buf0;
}
__global__ void __launch_bounds__(MTHREADS) k_match(Round R, const u16* __restrict__ pv, u64* __restrict__ mt) {
    extern __shared__ __align__(16) u8 sm[];
    const i64 t0 = R.r0 + (i64)blockIdx.x * MTILE, t1 = min(t0 + MTILE, R.lmatch);
    const i64 lo = max(t0 - (i64)WSIZE, (i64)0), hi = min(t1 + MAX_MATCH + 4, R.avail);
    u16* spv = (u16*)sm;
    u8* sb = sm + 2 * (size_t)(t1 - lo);
    for (i64 i = lo + threadIdx.x; i < t1; i += blockDim.x) spv[i - lo] = pv[i];
    for (i64 i = lo + threadIdx.x; i < hi; i += blockDim.x) sb[i - lo] = R.b[i];
    __syncthreads();
    auto B = [&](i64 i) { return sb[i - lo]; };
    auto P = [&](i64 i) { return (u32)spv[i - lo]; };
    for (i64 s = t0 + threadIdx.x; s < t1; s += blockDim.x) {
        const i64 ahead = R.final ? R.avail - s : (i64)MAX_MATCH + 4;
        mt[s - R.r0] = pack_match(find_match(B, P, s, ahead, base_rel(R, s)));
    }
}

// ---- the lazy automaton
__device__ __forceinline__ i64 auto_step(const Round& R, const u64* mt, LazyState& st, i64 s, bool& emit, Sym& out) {
    if (R.final && s == R.avail) {   // the loop ends: the pending literal, if any
        emit = st.ma;
        if (emit) out = Sym{sym_lit(R.b[s - 1]), (u32)(s - 1), 0};
        st = fresh_state();
        return s + 1;
    }
    u32 sym;
    i64 pos;
    const i64 nx = lazy_step(st, s, unpack_match(mt[s - R.r0]), s ? R.b[s - 1] : 0, emit, sym, pos);
    if (emit) out = Sym{sym, (u32)pos, pack_state(st)};
    return nx;
}
__device__ __forceinline__ u64 pack_exit(i64 s, LazyState st) { return (u64)pack_state(st) << 32 | (u32)s; }

struct Segs {
    u32* state_at;   // per loop top (index s - r0): the speculative state there, NO_STATE if not visited
    u16* symidx_at;  // per loop top: speculative symbols of its segment before that step
    Sym* spec;       // SEG per segment
    Sym* pre;        // SEG per segment: the re-run's symbols before it met the speculative trajectory
    u32 *nspec, *npre, *skip;
    u64 *spec_exit, *entry, *exitA, *exitB;
    int* changed;
    i64 nseg;
};
__global__ void k_lazy_spec(Round R, const u64* __restrict__ mt, Segs G, u32 st0) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G.nseg) return;
    const i64 s0 = R.r0 + i * SEG, s1 = min(s0 + SEG, R.r0 + R.nlt);
    LazyState st = i == 0 ? unpack_state(st0) : fresh_state();
    G.entry[i] = pack_exit(s0, st);
    u32 k = 0;
    i64 s = s0;
    while (s < s1) {
        G.state_at[s - R.r0] = pack_state(st);
        G.symidx_at[s - R.r0] = (u16)k;
        bool emit;
        Sym y;
        s = auto_step(R, mt, st, s, emit, y);
        if (emit) G.spec[i * SEG + k++] = y;
    }
    G.nspec[i] = k;
    G.npre[i] = 0;
    G.skip[i] = 0;
    G.spec_exit[i] = G.exitA[i] = pack_exit(s, st);
}
__global__ void k_lazy_fix(Round R, const u64* __restrict__ mt, Segs G, const u64* __restrict__ ein, u64* __restrict__ eout) {
    const i64 i = (i64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G.nseg) return;
    if (i == 0 || ein[i - 1] == G.entry[i]) { eout[i] = ein[i]; return; }
    const u64 e = ein[i - 1];
    G.entry[i] = e;
    const i64 s1 = min(R.r0 + (i + 1) * SEG, R.r0 + R.nlt);
    i64 s = (u32)e;
    LazyState st = unpack_state((u32)(e >> 32));
    u32 k = 0;
    u64 x;
    for (;;) {
        if (s >= s1) { G.skip[i] = G.nspec[i]; x = pack_exit(s, st); break; }
        if (G.state_at[s - R.r0] == pack_state(st)) { G.skip[i] = G.symidx_at[s - R.r0]; x = G.spec_exit[i]; break; }
        bool emit;
        Sym y;
        s = auto_step(R, mt, st, s, emit, y);
        if (emit) G.pre[i * SEG + k++] = y;
    }
    G.npre[i] = k;
    eout[i] = x;
    if (x != ein[i]) *G.changed = 1;
}
__global__ void k_gather(Segs G, const u32* __restrict__ offs, Sym* __restrict__ syms) {
    const i64 i = blockIdx.x;
    const u32 np = G.npre[i], sk = G.skip[i], ns = G.nspec[i], o = offs[i];
    for (u32 j = threadIdx.x; j < np; j += blockDim.x) syms[o + j] = G.pre[i * SEG + j];
    for (u32 j = threadIdx.x; j < ns - sk; j += blockDim.x) syms[o + np + j] = G.spec[i * SEG + sk + j];
}

// ---- blocks
struct BlockOut { u32 type, hbits, stored_len, first; u64 nbits; };
struct Blocks {
    const Sym* syms;
    u64 nsyms;
    int nblocks;        // blocks this round
    int last_final;     // the round's last block is the stream's last
    BlockOut* info;
    u32* lcode;         // L_CODES per block
    u32* dcode;         // D_CODES per block
    u32* hdr;           // HDR_WORDS per block
};
struct HdrSink {
    u32* w;
    u32 pos;
    __device__ void operator()(u32 v, int n) {
        w[pos >> 5] |= v << (pos & 31);
        if ((pos & 31) + n > 32) w[(pos >> 5) + 1] |= v >> (32 - (pos & 31));
        pos += n;
    }
};
__global__ void __launch_bounds__(256) k_block(Round R, Blocks K) {
    __shared__ BlockTrees t;
    __shared__ u32 cl[L_CODES], cd[D_CODES];
    const int k = blockIdx.x;
    const u64 a0 = (u64)k * SYM_END, a1 = min(a0 + SYM_END, K.nsyms);
    for (int n = threadIdx.x; n < L_CODES; n += blockDim.x) cl[n] = 0;
    for (int n = threadIdx.x; n < D_CODES; n += blockDim.x) cd[n] = 0;
    __syncthreads();
    for (u64 j = a0 + threadIdx.x; j < a1; j += blockDim.x) {
        const u32 v = K.syms[j].sym;
        if (!sym_is_match(v)) atomicAdd(&cl[v], 1u);
        else { atomicAdd(&cl[257 + length_code((int)sym_len(v) - 3)], 1u); atomicAdd(&cd[dist_code((int)sym_dist(v) - 1)], 1u); }
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int n = 0; n < L_CODES; n++) t.l.freq[n] = (u16)cl[n];
    for (int n = 0; n < D_CODES; n++) t.d.freq[n] = (u16)cd[n];
    t.l.freq[END_BLOCK] = 1;
    const bool last = K.last_final && k == K.nblocks - 1;
    const u64 N = R.buf0 + (u64)R.avail;
    const u64 first = a1 > a0 ? R.buf0 + K.syms[a0].pos : N;
    const Sym& y = K.syms[a1 > a0 ? a1 - 1 : a0];
    const u64 end = last ? N : R.buf0 + y.pos + sym_len(y.sym);
    const u64 flush_top = last ? N : R.buf0 + y.pos + 1;
    const bool stored_ok = first >= slide_base(flush_top, N, R.final);
    u64 nbits = 0;
    const int type = plan_block(t, end - first, stored_ok, &nbits);
    BlockOut o{(u32)type, 0, (u32)(end - first), (u32)(first - R.buf0), nbits};
    if (type != BT_STORED) {
        code_tables(t, type, K.lcode + (size_t)k * L_CODES, K.dcode + (size_t)k * D_CODES);
        if (type == BT_DYN) {
            HdrSink hs{K.hdr + (size_t)k * HDR_WORDS, 0};
            send_all_trees(t, hs);
            o.hbits = hs.pos;
        }
    }
    K.info[k] = o;
}

__device__ __forceinline__ void put_bits(u32* out, u64 pos, u32 v, int n) {
    if (n == 0) return;
    const int sh = (int)(pos & 31);
    atomicOr(&out[pos >> 5], v << sh);
    if (sh + n > 32) atomicOr(&out[(pos >> 5) + 1], v >> (32 - sh));
}
struct OutSink {
    u32* out;
    u64 pos;
    __device__ void operator()(u32 v, int n) { put_bits(out, pos, v, n); pos += n; }
};
__global__ void __launch_bounds__(256) k_pack(Round R, Blocks K, const u64* __restrict__ offs, u32* __restrict__ out) {
    __shared__ u32 lc[L_CODES], dc[D_CODES];
    __shared__ u64 part[256];
    const int k = blockIdx.x;
    const BlockOut o = K.info[k];
    const u64 off = offs[k];
    const bool last = K.last_final && k == K.nblocks - 1;
    if (o.type == BT_STORED) {
        const u64 a = (off + 3 + 7) & ~7ull;
        if (threadIdx.x == 0) { put_bits(out, off, (u32)last, 3); put_bits(out, a, o.stored_len & 0xffff, 16); put_bits(out, a + 16, ~o.stored_len & 0xffff, 16); }
        for (u32 i = threadIdx.x; i < o.stored_len; i += blockDim.x) put_bits(out, a + 32 + 8ull * i, R.b[o.first + i], 8);
        return;
    }
    for (int n = threadIdx.x; n < L_CODES; n += blockDim.x) lc[n] = K.lcode[(size_t)k * L_CODES + n];
    for (int n = threadIdx.x; n < D_CODES; n += blockDim.x) dc[n] = K.dcode[(size_t)k * D_CODES + n];
    if (threadIdx.x == 0) put_bits(out, off, o.type << 1 | (u32)last, 3);
    for (u32 w = threadIdx.x; w * 32 < o.hbits; w += blockDim.x)
        put_bits(out, off + 3 + 32ull * w, K.hdr[(size_t)k * HDR_WORDS + w], (int)min(32u, o.hbits - 32 * w));
    __syncthreads();
    const u64 a0 = (u64)k * SYM_END, a1 = min(a0 + SYM_END, K.nsyms), cnt = a1 - a0;
    const u64 per = (cnt + blockDim.x - 1) / blockDim.x;
    const u64 j0 = a0 + min(cnt, per * threadIdx.x), j1 = a0 + min(cnt, per * (threadIdx.x + 1));
    u64 mine = 0;
    for (u64 j = j0; j < j1; j++) mine += symbol_bits(K.syms[j].sym, lc, dc);
    part[threadIdx.x] = mine;
    __syncthreads();
    for (int d = 1; d < (int)blockDim.x; d <<= 1) {   // inclusive scan
        const u64 v = threadIdx.x >= (unsigned)d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    OutSink os{out, off + 3 + o.hbits + part[threadIdx.x] - mine};
    for (u64 j = j0; j < j1; j++) send_symbol(K.syms[j].sym, lc, dc, os);
    if (threadIdx.x == blockDim.x - 1) os(lc[END_BLOCK] & 0xffff, lc[END_BLOCK] >> 16);
}

// ---- CRC-32 per piece
__global__ void k_crc(const u8* __restrict__ b, i64 n, u32* __restrict__ crcs) {
    __shared__ u32 table[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) table[i] = crc_table_entry(i);
    __syncthreads();
    const i64 p = (i64)blockIdx.x * blockDim.x + threadIdx.x, s = p * CRC_PIECE;
    if (s >= n) return;
    crcs[p] = ~crc_update(~0u, table, b + s, (u64)min((i64)CRC_PIECE, n - s));
}

// ---- the writer
class GpuGzFile : public GzFile {
public:
    GpuGzFile(const std::string& path, int device, size_t chunk, std::vector<u8>* mem = nullptr) : dev_(device), mem_(mem) {
        if (!mem_) {
            f_ = fopen(path.c_str(), "wb");
            if (!f_) throw std::runtime_error("Cannot open " + path);
        }
        chunk_ = std::max(chunk ? chunk : DEFAULT_CHUNK, MIN_CHUNK);
        cap_ = chunk_ + CARRY;
        const pgb::DeviceScope on(dev_);
        Owners d;   // declared after the scope: released with the device current when a step below throws
        d.st = pgb::make_stream();
        for (pgb::DevBuf& b : d.buf) b.alloc(cap_ + 64);
        d.changed.alloc(sizeof(int));
        d.crcs.alloc((cap_ / CRC_PIECE + 2) * sizeof(u32));
        PG_CUDA(cudaFuncSetAttribute(k_hash, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768 * 4));
        PG_CUDA(cudaFuncSetAttribute(k_match, cudaFuncAttributeMaxDynamicSharedMemorySize, match_smem()));
        d_ = std::move(d);
        G_.changed = d_.changed.as<int>();
        x8_piece_ = x8nmodp(CRC_PIECE);
        const u8 hdr[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};   // no name, no time, xfl 0, OS_CODE 3 (Unix)
        emit(hdr, 10);
    }
    ~GpuGzFile() override {
        try { if (!closed_) close(); } catch (...) {}
        const pgb::DeviceScope on(dev_);
        d_ = Owners{};   // the owners leave with this temporary, inside the scope
        if (f_) fclose(f_);
    }
    void write(const void* p, size_t n, bool on_device) override {
        if (closed_) throw std::runtime_error("gpu gzip: write after close");
        const pgb::DeviceScope on(dev_);
        const u8* q = (const u8*)p;
        while (n) {
            const size_t take = std::min(n, cap_ - (size_t)avail_);
            PG_CUDA(cudaMemcpyAsync(d_.buf[cur_].as<u8>() + avail_, q, take, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, d_.st));
            PG_CUDA(cudaStreamSynchronize(d_.st));   // the caller may reuse its buffer when write returns
            avail_ += (i64)take;
            total_ += take;
            q += take;
            n -= take;
            if ((size_t)avail_ == cap_) round(false);
        }
    }
    void close() override {
        if (closed_) return;
        closed_ = true;
        const pgb::DeviceScope on(dev_);
        round(true);
        if (nbits_pend_) { const u8 c = (u8)pend_; emit(&c, 1); }
        u8 tr[8];
        for (int i = 0; i < 4; i++) { tr[i] = (u8)(crc_ >> (8 * i)); tr[4 + i] = (u8)(total_ >> (8 * i)); }
        emit(tr, 8);
        if (f_) {
            const int e = fclose(f_);
            f_ = nullptr;
            if (e) throw std::runtime_error("gpu gzip: close failed");
        }
    }

private:
    // The per-position work arrays, sized for a round over n bytes (the first full round sets the size for good; a small file
    // allocates only what it needs).
    void ensure_work(size_t n) {
        n = std::max(n, (size_t)1 << 16);
        if (n <= work_) return;
        const i64 nseg = (i64)(n / SEG) + 2;
        nblk_max_ = (int)(n / SYM_END) + 3;
        d_.pv.alloc(n * sizeof(u16));
        d_.mt.alloc(n * sizeof(u64));
        d_.state_at.alloc((n + 2) * sizeof(u32));
        d_.symidx_at.alloc((n + 2) * sizeof(u16));
        d_.spec.alloc((size_t)nseg * SEG * sizeof(Sym));
        d_.pre.alloc((size_t)nseg * SEG * sizeof(Sym));
        d_.syms.alloc((n + 2) * sizeof(Sym));
        d_.segw.alloc((size_t)nseg * 4 * sizeof(u32));
        d_.sege.alloc((size_t)nseg * 5 * sizeof(u64));
        d_.binfo.alloc(nblk_max_ * sizeof(BlockOut));
        d_.lcode.alloc((size_t)nblk_max_ * L_CODES * sizeof(u32));
        d_.dcode.alloc((size_t)nblk_max_ * D_CODES * sizeof(u32));
        d_.hdr.alloc((size_t)nblk_max_ * HDR_WORDS * sizeof(u32));
        d_.boffs.alloc(nblk_max_ * sizeof(u64));
        d_.out.alloc((2 * n + (1 << 20)) / 4 * sizeof(u32));
        G_.state_at = d_.state_at.as<u32>(); G_.symidx_at = d_.symidx_at.as<u16>(); G_.spec = d_.spec.as<Sym>(); G_.pre = d_.pre.as<Sym>();
        G_.nspec = d_.segw.as<u32>(); G_.npre = G_.nspec + nseg; G_.skip = G_.nspec + 2 * nseg; soffs_ = G_.nspec + 3 * nseg;
        G_.spec_exit = d_.sege.as<u64>(); G_.entry = G_.spec_exit + nseg; G_.exitA = G_.spec_exit + 2 * nseg; G_.exitB = G_.spec_exit + 3 * nseg;
        work_ = n;   // last: a round after a failed allocation allocates again
    }
    static size_t match_smem() { return (size_t)(MTILE + WSIZE) * 2 + MTILE + WSIZE + MAX_MATCH + 8; }
    void emit(const void* p, size_t n) {
        if (mem_) mem_->insert(mem_->end(), (const u8*)p, (const u8*)p + n);
        else if (n && fwrite(p, 1, n, f_) != n) throw std::runtime_error("gpu gzip: short write");
    }
    void round(bool final) {
        ensure_work((size_t)avail_);
        Round R{d_.buf[cur_].as<u8>(), buf0_, avail_, final, (i64)(r0_ - buf0_), 0, 0};
        // CRC of the bytes this buffer holds for the first time
        if (avail_ > crc_from_) {
            const i64 n = avail_ - crc_from_, np = (n + CRC_PIECE - 1) / CRC_PIECE;
            k_crc<<<(unsigned)((np + 127) / 128), 128, 0, d_.st>>>(R.b + crc_from_, n, d_.crcs.as<u32>());
            std::vector<u32> c(np);
            PG_CUDA(cudaMemcpyAsync(c.data(), d_.crcs.p, np * sizeof(u32), cudaMemcpyDeviceToHost, d_.st));
            PG_CUDA(cudaStreamSynchronize(d_.st));
            for (i64 i = 0; i < np; i++) {
                const u64 len = (u64)std::min((i64)CRC_PIECE, n - i * CRC_PIECE);
                crc_ = crc_any_ ? multmodp(len == CRC_PIECE ? x8_piece_ : x8nmodp(len), crc_) ^ c[i] : c[i];
                crc_any_ = true;
            }
            crc_from_ = avail_;
        }
        R.lmatch = final ? avail_ : avail_ - MIN_LOOKAHEAD;
        R.nlt = (final ? avail_ + 1 : R.lmatch) - R.r0;
        const i64 nhash = avail_ - 2;
        if (nhash > 0) k_hash<<<(unsigned)((nhash + HTILE - 1) / HTILE), 32, 32768 * 4, d_.st>>>(R.b, nhash, d_.pv.as<u16>());
        if (R.lmatch > R.r0)
            k_match<<<(unsigned)((R.lmatch - R.r0 + MTILE - 1) / MTILE), MTHREADS, match_smem(), d_.st>>>(R, d_.pv.as<u16>(), d_.mt.as<u64>());
        G_.nseg = (R.nlt + SEG - 1) / SEG;
        PG_CUDA(cudaMemsetAsync(G_.state_at, 0xff, (size_t)R.nlt * sizeof(u32), d_.st));
        const unsigned sg = (unsigned)((G_.nseg + 127) / 128);
        k_lazy_spec<<<sg, 128, 0, d_.st>>>(R, d_.mt.as<u64>(), G_, pack_state(st0_));
        for (int pass = 0;; pass++) {
            PG_CUDA(cudaMemsetAsync(G_.changed, 0, sizeof(int), d_.st));
            k_lazy_fix<<<sg, 128, 0, d_.st>>>(R, d_.mt.as<u64>(), G_, G_.exitA, G_.exitB);
            int ch = 0;
            PG_CUDA(cudaMemcpyAsync(&ch, G_.changed, sizeof(int), cudaMemcpyDeviceToHost, d_.st));
            PG_CUDA(cudaStreamSynchronize(d_.st));
            std::swap(G_.exitA, G_.exitB);
            if (!ch) break;
        }
        // symbol counts -> offsets
        std::vector<u32> w((size_t)G_.nseg * 3);
        PG_CUDA(cudaMemcpyAsync(w.data(), G_.nspec, G_.nseg * sizeof(u32), cudaMemcpyDeviceToHost, d_.st));
        PG_CUDA(cudaMemcpyAsync(w.data() + G_.nseg, G_.npre, G_.nseg * sizeof(u32), cudaMemcpyDeviceToHost, d_.st));
        PG_CUDA(cudaMemcpyAsync(w.data() + 2 * G_.nseg, G_.skip, G_.nseg * sizeof(u32), cudaMemcpyDeviceToHost, d_.st));
        PG_CUDA(cudaStreamSynchronize(d_.st));
        std::vector<u32> offs(G_.nseg);
        u64 T = 0;
        for (i64 i = 0; i < G_.nseg; i++) { offs[i] = (u32)T; T += w[G_.nseg + i] + w[i] - w[2 * G_.nseg + i]; }
        PG_CUDA(cudaMemcpyAsync(soffs_, offs.data(), G_.nseg * sizeof(u32), cudaMemcpyHostToDevice, d_.st));
        k_gather<<<(unsigned)G_.nseg, 256, 0, d_.st>>>(G_, soffs_, d_.syms.as<Sym>());
        // blocks: final -- all, an empty last block when an in-loop flush took the last symbol; not final -- the complete ones
        if (!final) {
            if (T < (u64)SYM_END) throw std::runtime_error("gpu gzip: a full buffer holds no complete block");
            T -= T % SYM_END;
        }
        Sym lastsym{0, 0, 0};
        if (T) PG_CUDA(cudaMemcpyAsync(&lastsym, d_.syms.as<Sym>() + T - 1, sizeof(Sym), cudaMemcpyDeviceToHost, d_.st));
        PG_CUDA(cudaStreamSynchronize(d_.st));
        int nb = (int)(T / SYM_END + (T % SYM_END != 0));
        if (final && T % SYM_END == 0 && !(T && !sym_is_match(lastsym.sym) && (i64)lastsym.pos == avail_ - 1)) nb++;
        if (nb > nblk_max_) throw std::runtime_error("gpu gzip: block table overflow");
        Blocks K{d_.syms.as<Sym>(), T, nb, final, d_.binfo.as<BlockOut>(), d_.lcode.as<u32>(), d_.dcode.as<u32>(), d_.hdr.as<u32>()};
        if (nb) {
            PG_CUDA(cudaMemsetAsync(d_.hdr.p, 0, (size_t)nb * HDR_WORDS * sizeof(u32), d_.st));
            k_block<<<nb, 256, 0, d_.st>>>(R, K);
        }
        std::vector<BlockOut> info(nb);
        if (nb) PG_CUDA(cudaMemcpyAsync(info.data(), d_.binfo.p, nb * sizeof(BlockOut), cudaMemcpyDeviceToHost, d_.st));
        PG_CUDA(cudaStreamSynchronize(d_.st));
        std::vector<u64> boffs(nb);
        u64 bit = (u64)nbits_pend_;
        for (int k = 0; k < nb; k++) {
            boffs[k] = bit;
            bit = off_apply(info[k].type == BT_STORED ? off_stored(info[k].stored_len) : off_plain(info[k].nbits), bit);
        }
        if (final) bit = (bit + 7) & ~7ull;   // bi_windup after the last block
        const size_t words = (size_t)(bit / 32 + 2);
        if (words * sizeof(u32) > d_.out.bytes) throw std::runtime_error("gpu gzip: output buffer overflow");
        PG_CUDA(cudaMemsetAsync(d_.out.p, 0, words * sizeof(u32), d_.st));
        if (nbits_pend_) PG_CUDA(cudaMemcpyAsync(d_.out.p, &pend_, sizeof(u32), cudaMemcpyHostToDevice, d_.st));
        if (nb) {
            PG_CUDA(cudaMemcpyAsync(d_.boffs.p, boffs.data(), nb * sizeof(u64), cudaMemcpyHostToDevice, d_.st));
            k_pack<<<nb, 256, 0, d_.st>>>(R, K, d_.boffs.as<u64>(), d_.out.as<u32>());
        }
        PG_CUDA(cudaGetLastError());
        std::vector<u8> ob(words * 4);
        PG_CUDA(cudaMemcpyAsync(ob.data(), d_.out.p, words * 4, cudaMemcpyDeviceToHost, d_.st));
        PG_CUDA(cudaStreamSynchronize(d_.st));
        emit(ob.data(), bit / 8);
        nbits_pend_ = (int)(bit & 7);
        pend_ = nbits_pend_ ? ob[bit / 8] : 0;
        if (final) return;
        // carry: from the first byte of the next block, its 32 KB of history, the automaton state at the next loop top
        const u32 len = sym_len(lastsym.sym);
        const u64 bstart = buf0_ + lastsym.pos + len;
        r0_ = buf0_ + lastsym.pos + (sym_is_match(lastsym.sym) ? len : 2);
        st0_ = sym_is_match(lastsym.sym) ? fresh_state() : unpack_state(lastsym.next);
        const u64 nb0 = bstart > (u64)WSIZE ? bstart - WSIZE : 0;
        const i64 keep = avail_ - (i64)(nb0 - buf0_);
        PG_CUDA(cudaMemcpyAsync(d_.buf[cur_ ^ 1].p, R.b + (nb0 - buf0_), keep, cudaMemcpyDeviceToDevice, d_.st));
        PG_CUDA(cudaStreamSynchronize(d_.st));
        cur_ ^= 1;
        crc_from_ -= (i64)(nb0 - buf0_);
        buf0_ = nb0;
        avail_ = keep;
    }

    int dev_;
    std::vector<u8>* mem_;
    FILE* f_ = nullptr;
    size_t chunk_, cap_, work_ = 0;
    int nblk_max_ = 0;
    // The stream and device memory, released with the writer's device current: ~GpuGzFile resets them inside its DeviceScope.
    struct Owners {
        pgb::Stream st;
        pgb::DevBuf buf[2], changed, crcs;
        pgb::DevBuf pv, mt, state_at, symidx_at, spec, pre, syms, segw, sege, binfo, lcode, dcode, hdr, boffs, out;   // ensure_work
    } d_;
    int cur_ = 0;
    Segs G_{};   // views into d_, as are soffs_ and the kernels' other pointer arguments
    u32* soffs_ = nullptr;
    u32 x8_piece_;
    // stream state
    u64 buf0_ = 0;          // stream offset of the buffer's first byte
    i64 avail_ = 0;
    u64 r0_ = 0;            // next loop top
    LazyState st0_ = fresh_state();
    u64 total_ = 0;
    i64 crc_from_ = 0;      // buffer position from which bytes have not entered the CRC
    u32 crc_ = 0;
    bool crc_any_ = false;
    u32 pend_ = 0;          // the partial last output byte
    int nbits_pend_ = 0;
    bool closed_ = false;
};

class HostGzFile : public GzFile {
public:
    explicit HostGzFile(const std::string& path) : name_(path) {
        f_ = gzopen(path.c_str(), "w");
        if (!f_) throw std::runtime_error("Cannot open " + path);
    }
    ~HostGzFile() override { if (f_) gzclose(f_); }
    void write(const void* p, size_t n, bool on_device) override {
        std::vector<u8> h;
        if (on_device) {
            h.resize(n);
            PG_CUDA(cudaMemcpy(h.data(), p, n, cudaMemcpyDeviceToHost));
            p = h.data();
        }
        size_t off = 0;
        while (off < n) {
            const size_t k = std::min<size_t>(n - off, 1u << 30);
            if (gzwrite(f_, (const char*)p + off, (unsigned)k) != (int)k) throw std::runtime_error("gzwrite failed on " + name_);
            off += k;
        }
    }
    void close() override {
        if (!f_) return;
        const int e = gzclose(f_);
        f_ = nullptr;
        if (e != Z_OK) throw std::runtime_error("gzclose failed on " + name_);
    }

private:
    std::string name_;
    gzFile f_;
};

// The probe the writer is checked on before first use: several blocks, window slides, a stored block (random bytes), runs that make
// 258-byte matches, DNA and map-shaped text.  ~420 KB.
static std::vector<u8> probe_text() {
    std::vector<u8> t;
    u64 x = 0x9e3779b97f4a7c15ull;
    auto rnd = [&] { x ^= x << 13; x ^= x >> 7; x ^= x << 17; return x; };
    char line[64];
    for (int i = 0; i < 6000; i++) {
        const int n = snprintf(line, sizeof line, "%d\t%u\t%u\t%c\n", i + 1, (unsigned)(rnd() % 40000), (unsigned)(rnd() % 5000), rnd() & 1 ? '+' : '-');
        t.insert(t.end(), line, line + n);
    }
    for (int i = 0; i < 120000; i++) t.push_back("ACGT"[rnd() & 3]);
    for (int i = 0; i < 70000; i++) t.push_back((u8)rnd());
    t.insert(t.end(), 40000, 'N');
    for (int r = 0; r < 3000; r++) t.insert(t.end(), (size_t)(rnd() % 40 + 1), "ACGTN"[rnd() % 5]);
    for (int i = 0; i < 60000; i++) t.push_back("ACGT"[rnd() & 3]);
    return t;
}
static std::vector<u8> zlib_gzip(const std::vector<u8>& in) {
    z_stream z{};
    if (deflateInit2(&z, 6, Z_DEFLATED, 31, 8, Z_DEFAULT_STRATEGY) != Z_OK) return {};
    std::vector<u8> out(deflateBound(&z, in.size()) + 64);
    z.next_in = (Bytef*)in.data();
    z.avail_in = (uInt)in.size();
    z.next_out = out.data();
    z.avail_out = (uInt)out.size();
    const int rc = deflate(&z, Z_FINISH);
    out.resize(z.total_out);
    deflateEnd(&z);
    return rc == Z_STREAM_END ? out : std::vector<u8>{};
}

}  // namespace gz

static bool verbose() { const char* v = getenv("PGB200_VERBOSE"); return v && *v && strcmp(v, "0"); }

bool gz_gpu_matches_zlib(int device) {
    static std::mutex mu;
    static int state = -1;   // for the process's first device
    std::lock_guard<std::mutex> lk(mu);
    if (state >= 0) return state == 1;
    const std::vector<gz::u8> probe = gz::probe_text(), want = gz::zlib_gzip(probe);
    std::vector<gz::u8> got;
    try {
        gz::GpuGzFile w("", device, 0, &got);
        w.write(probe.data(), probe.size(), false);
        w.close();
    } catch (const std::exception& ex) {
        if (verbose()) fprintf(stderr, "[pgb200] gzip: the GPU writer failed on the probe (%s); writing .gz files with zlib\n", ex.what());
        state = 0;
        return false;
    }
    state = got == want ? 1 : 0;
    if (!state && verbose())
        fprintf(stderr, "[pgb200] gzip: this zlib (%s) writes other level-6 bytes than the GPU writer reproduces; writing .gz files with zlib\n",
                zlibVersion());
    return state == 1;
}

GzFile* gz_open_gpu(const std::string& path, int device, size_t chunk) { return new gz::GpuGzFile(path, device, chunk); }
GzFile* gz_open_host(const std::string& path) { return new gz::HostGzFile(path); }
GzFile* gz_open(const std::string& path, int device) {
    const char* m = getenv("PGB200_GZ");
    if (m && !strcmp(m, "host")) return gz_open_host(path);
    if (m && *m && strcmp(m, "gpu")) throw std::runtime_error(std::string("PGB200_GZ must be gpu or host, not ") + m);
    if (!gz_gpu_matches_zlib(device)) return gz_open_host(path);
    size_t chunk = 0;
    if (const char* c = getenv("PGB200_GZ_CHUNK_MB")) chunk = (size_t)atoll(c) << 20;
    // a GPU whose memory the stage has filled cannot hold the writer's buffers (about 60 bytes per byte of a round): zlib writes
    size_t free_b = 0, total_b = 0;
    const pgb::DeviceScope on(device);
    const bool room = cudaMemGetInfo(&free_b, &total_b) == cudaSuccess &&
                      free_b > 64 * (std::max(chunk ? chunk : gz::DEFAULT_CHUNK, gz::MIN_CHUNK) + gz::CARRY) + (256ull << 20);
    if (!room) {
        if (verbose()) fprintf(stderr, "[pgb200] gzip: %zu MB free on GPU %d is too little for the writer; %s is written with zlib\n", free_b >> 20, device, path.c_str());
        return gz_open_host(path);
    }
    return gz_open_gpu(path, device, chunk);
}
