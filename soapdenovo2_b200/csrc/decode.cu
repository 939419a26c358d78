// decode.cu -- K1: FASTA/FASTQ text -> 2-bit packed reads, entirely on the GPU, plus feed_text (the per-chunk driver of pass 1).
//
// Replaces (reference file:line, standardPregraph/):
//   readseqInBuf / readseqfq (readseq1by1.c:138-209, 279-360): record scan of a text buffer, base decoding, truncation
//   reverse2k (readseq1by1.c:788-802): whole-read reverse complement for reverse_seq libraries
// The text is read 2.5 times, every time with coalesced 16-byte loads:
//   k_nl_count    newlines per 2 KB tile                               (1 x text)
//   k_line_index  line number of every newline from the scanned tile counts -> start/end of every sequence line; checks that
//                 header lines start with '>' / '@' and FASTQ separator lines with '+'          (1 x text)
//   k_decode_fast one thread per 32-base output word: 36 bytes of text -> 64 packed bits with SIMD-in-register byte arithmetic
//                 (0.5 x text); it also adds up the read statistics.  A record that needs the general rules (a byte that is not a
//                 letter inside the line) is appended once to a redo list; k_decode_fix, on a small fixed grid, redoes just the
//                 listed records (every record of a reverse_seq library), one warp per record, and corrects their statistics.  On
//                 clean text the list is empty and k_decode_fix returns at once.
// Base code = (ch & 6) >> 1 for letters (A0 C1 T2 G3, N->3), '.' -> 0, every other byte is dropped; only the first
// min(linelen, maxlen) characters of the sequence line are considered (readseq1by1.c:177-200).  Output: LSB-first 2-bit packing,
// W64 words per read, zero past the read's end.
#include "engine_impl.cuh"
#include "scan.cuh"

namespace pgb {

constexpr int NL_TILE = 2048;              // bytes of text per warp tile
constexpr int NL_GROUPS = NL_TILE / 16;    // 16-byte groups per tile
constexpr int NL_ITERS = NL_GROUPS / 32;

// bit b set <=> byte b of the 16-byte group is '\n' (bytes past the end of the text are masked out)
__device__ __forceinline__ unsigned nl_mask16(const uint4* __restrict__ text, u64 nbytes, u64 grp) {
    const uint4 v = __ldg(text + grp);
    unsigned m = 0;
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const unsigned r = __vcmpeq4(w[k], 0x0A0A0A0Au) & 0x01010101u;   // exact per-byte compare
        m |= ((r | (r >> 7) | (r >> 14) | (r >> 21)) & 0xFu) << (4 * k);
    }
    const u64 rem = nbytes - grp * 16;
    if (rem < 16) m &= (1u << rem) - 1;
    return m;
}

__global__ void __launch_bounds__(256) k_nl_count(const uint4* __restrict__ text, u64 nbytes, u64 n_tiles, u32* __restrict__ tile_cnt) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n_groups = (nbytes + 15) / 16;
    for (u64 tile = warp0; tile < n_tiles; tile += nwarps) {
        unsigned cnt = 0;
#pragma unroll
        for (int it = 0; it < NL_ITERS; it++) {
            const u64 grp = tile * NL_GROUPS + it * 32 + lane;
            if ((grp + 1) * 16 <= nbytes) {   // a whole group: every equal byte is 0xFF in the compare result, 8 set bits
                const uint4 v = __ldg(text + grp);
                cnt += (__popc(__vcmpeq4(v.x, 0x0A0A0A0Au)) + __popc(__vcmpeq4(v.y, 0x0A0A0A0Au)) + __popc(__vcmpeq4(v.z, 0x0A0A0A0Au)) +
                        __popc(__vcmpeq4(v.w, 0x0A0A0A0Au))) >> 3;
            } else if (grp < n_groups) cnt += __popc(nl_mask16(text, nbytes, grp));
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) tile_cnt[tile] = cnt;
    }
}

// newline number g (0-based) at byte `pos`: it ends line g and line g+1 starts at pos+1.  Records are lpr = 1 << lshift lines long:
// line 0 of a record is its header, line 1 its sequence, FASTQ line 2 the '+' separator.
struct LineIndexCtx {
    const unsigned char* bytes;
    u64 nbytes, n_rec;
    u32* seq_start;
    u32* seq_end;
    int lshift;
    unsigned lmask;
    unsigned char hdr;
};
__device__ __forceinline__ unsigned line_index_one(const LineIndexCtx& c, u64 pos, u64 g) {
    unsigned bad = 0;
    if (((unsigned)g & c.lmask) == 1u) {
        const u64 r = g >> c.lshift;
        if (r < c.n_rec) c.seq_end[r] = (u32)pos;
    }
    const u64 g1 = g + 1;
    const unsigned ph = (unsigned)g1 & c.lmask;
    if (ph == 1u) {
        const u64 r = g1 >> c.lshift;
        if (r < c.n_rec) c.seq_start[r] = (u32)(pos + 1);
    } else if (pos + 1 < c.nbytes) {
        if (ph == 0u) { if ((g1 >> c.lshift) < c.n_rec && c.bytes[pos + 1] != c.hdr) bad++; }
        else if (ph == 2u && c.bytes[pos + 1] != '+') bad++;     // only reached for FASTQ (lmask == 3)
    }
    return bad;
}

// One warp per 2 KB tile.  A lane finds 0.2 newlines per 16-byte group on FASTQ text, so the newlines of a tile are first compacted
// into a per-warp queue (their order = their global line numbers) and then handled 32 at a time, all lanes busy.
constexpr int LI_QUEUE = 160, LI_BURST = 64;
__global__ void __launch_bounds__(256) k_line_index(const uint4* __restrict__ text, u64 nbytes, u64 n_tiles, const u32* __restrict__ tile_base, int lshift,
                                                    u64 n_rec, u32* __restrict__ seq_start, u32* __restrict__ seq_end, u64* counters) {
    __shared__ u32 s_q[8][LI_QUEUE];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n_groups = (nbytes + 15) / 16;
    LineIndexCtx c{reinterpret_cast<const unsigned char*>(text), nbytes, n_rec, seq_start, seq_end, lshift, (1u << lshift) - 1u, (unsigned char)(lshift == 2 ? '@' : '>')};
    u32* q = s_q[wib];
    unsigned bad = 0;
    if (warp0 == 0 && lane == 0 && nbytes && c.bytes[0] != c.hdr) bad++;
    for (u64 tile = warp0; tile < n_tiles; tile += nwarps) {
        u64 gq = tile_base[tile];     // global line number of the first queued newline
        unsigned qn = 0;              // queued newlines (warp-uniform)
        const u64 tile_byte0 = tile * NL_TILE;
        unsigned m[NL_ITERS];
#pragma unroll
        for (int it = 0; it < NL_ITERS; it++) {
            const u64 grp = tile * NL_GROUPS + it * 32 + lane;
            m[it] = grp < n_groups ? nl_mask16(text, nbytes, grp) : 0u;
        }
#pragma unroll
        for (int it = 0; it < NL_ITERS; it++) {
            const unsigned cn = __popc(m[it]);
            unsigned inc = cn;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned v = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= d) inc += v;
            }
            const unsigned total = __shfl_sync(0xffffffffu, inc, 31);
            const unsigned off0 = (unsigned)(it * 512 + lane * 16);   // byte offset of this lane's group inside the tile
            unsigned mm = m[it];
            if (total > (unsigned)LI_BURST) {
                // pathological text (a newline every few bytes): drain the queue, then let every lane walk its own bits
                __syncwarp();
                for (unsigned i = lane; i < qn; i += 32) bad += line_index_one(c, tile_byte0 + q[i], gq + i);
                gq += qn;
                qn = 0;
                u64 g = gq + (inc - cn);
                while (mm) {
                    const int b = __ffs(mm) - 1;
                    mm &= mm - 1;
                    bad += line_index_one(c, tile_byte0 + off0 + b, g++);
                }
                gq += total;
                __syncwarp();
                continue;
            }
            unsigned slot = qn + (inc - cn);
            while (mm) {
                const int b = __ffs(mm) - 1;
                mm &= mm - 1;
                q[slot++] = off0 + b;
            }
            qn += total;
            if (qn > (unsigned)(LI_QUEUE - LI_BURST) || it == NL_ITERS - 1) {
                __syncwarp();
                for (unsigned i = lane; i < qn; i += 32) bad += line_index_one(c, tile_byte0 + q[i], gq + i);
                gq += qn;
                qn = 0;
                __syncwarp();
            }
        }
    }
    if (bad) atomicAdd(&counters[C_BADFMT], (u64)bad);
}

// 4 text bytes -> 0xFF in every byte that is a letter or '.'
__device__ __forceinline__ unsigned base_char_mask4(unsigned v, unsigned& dot) {
    const unsigned t = v | 0x20202020u;
    dot = __vcmpeq4(v, 0x2E2E2E2Eu);
    return (__vcmpgeu4(t, 0x61616161u) & __vcmpleu4(t, 0x7A7A7A7Au)) | dot;
}

// "kmer(s) in reads" / reads kept of a read of n bases: reads shorter than K+1 are skipped (prlHashReads.c:504,642)
__device__ __forceinline__ u64 read_instances(int n, int K) { return n >= K + 1 ? (u64)(n - K + 1) : 0ull; }

// Sum of v over the CTA, added to *dst with one global atomic (every thread of the CTA calls it)
__device__ __forceinline__ void cta_add_u64(u64 v, u64* dst) {
    __shared__ u64 s_sum;
    if (threadIdx.x == 0) s_sum = 0;
    __syncthreads();
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd((unsigned long long*)&s_sum, (unsigned long long)v);
    __syncthreads();
    if (threadIdx.x == 0 && s_sum) atomicAdd((unsigned long long*)dst, (unsigned long long)s_sum);
}

// Every record is counted here with the length of its fast decode; a record the fast rules cannot handle is appended (once) to the
// redo list, and k_decode_fix corrects the counters of just those records.
__global__ void __launch_bounds__(256) k_decode_fast(const unsigned char* __restrict__ text, u64 nbytes, const u32* __restrict__ seq_start,
                                                     const u32* __restrict__ seq_end, u64 n_rec, int maxlen, int K, int W64, u64* __restrict__ words,
                                                     u32* __restrict__ lens, u32* __restrict__ flag, u32* __restrict__ redo, u32* n_redo, u64* counters) {
    const u64 total = n_rec * (u64)W64;
    u64 inst = 0, kept = 0;
    for (u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (u64)gridDim.x * blockDim.x) {
        const u64 r = idx / (unsigned)W64;
        const int w = (int)(idx - r * (unsigned)W64);
        const u32 s = seq_start[r], e = seq_end[r];
        const int raw = e > s ? (int)min(e - s, 0x7fffffffu) : 0;
        int use = raw < maxlen ? raw : maxlen;
        if (raw > 0 && raw <= maxlen && text[e - 1] == '\r') use = raw - 1;   // CRLF: the '\r' would be dropped as a non-letter
        if (w == 0) {
            lens[r] = (u32)use;
            const u64 n = read_instances(use, K);
            inst += n;
            kept += n ? 1 : 0;
        }
        int cnt = use - 32 * w;
        if (cnt <= 0) { words[idx] = 0ull; continue; }
        if (cnt > 32) cnt = 32;
        const u64 a = (u64)s + 32ull * w, a4 = a & ~3ull;
        const int sh = (int)(a & 3) * 8;
        unsigned t[9];
#pragma unroll
        for (int i = 0; i < 9; i++) {
            const u64 off = a4 + 4ull * i;
            t[i] = (off < nbytes && 4 * i < sh / 8 + cnt) ? __ldg(reinterpret_cast<const unsigned*>(text + off)) : 0u;
        }
        u64 out = 0;
        bool clean = true;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const unsigned v = __funnelshift_r(t[i], t[i + 1], sh);
            int nb = cnt - 4 * i;
            nb = nb < 0 ? 0 : (nb > 4 ? 4 : nb);
            const unsigned need = (unsigned)((1ull << (8 * nb)) - 1ull);   // nb in 0..4: a 64-bit shift is defined for all of them
            unsigned dot;
            const unsigned ok = base_char_mask4(v, dot);
            clean = clean && ((ok & need) == need);
            const unsigned codes = ((v >> 1) & 0x03030303u) & ~dot & need;
            out |= (u64)((codes * 0x01041040u) >> 24) << (8 * i);   // 4 two-bit codes, one per byte -> one byte
        }
        if (!clean && atomicOr(&flag[r], 1u) == 0u) redo[atomicAdd(n_redo, 1u)] = (u32)r;
        words[idx] = out;
    }
    cta_add_u64(inst, &counters[C_INSTANCES]);
    cta_add_u64(kept, &counters[C_KEPT]);
}

__device__ __forceinline__ bool is_base_char(unsigned c) { return ((c | 0x20u) - 'a') < 26u || c == '.'; }
__device__ __forceinline__ unsigned base_code(unsigned c) { return c == '.' ? 0u : ((c & 6u) >> 1); }

// general rules, one warp per record: drop every byte that is not a letter or '.', optional whole-read reverse complement; returns the
// read's length (warp-uniform)
__device__ int decode_record_warp(const unsigned char* __restrict__ text, u32 s, u32 e, int maxlen, int reverse, int W64, u64* out, u32* len_out) {
    const int lane = threadIdx.x & 31;
    const int raw = e > s ? (int)min(e - s, 0x7fffffffu) : 0;
    const int use = raw < maxlen ? raw : maxlen;
    int n = 0;
    for (int b = 0; b < use; b += 32) {
        const int i = b + lane;
        const bool v = i < use && is_base_char(text[s + i]);
        n += __popc(__ballot_sync(0xffffffffu, v));
    }
    for (int w = lane; w < W64; w += 32) out[w] = 0;
    __syncwarp();
    int pos0 = 0;
    for (int b = 0; b < use; b += 32) {
        const int i = b + lane;
        const unsigned ch = i < use ? text[s + i] : 0;
        const bool v = i < use && is_base_char(ch);
        const unsigned bal = __ballot_sync(0xffffffffu, v);
        if (v) {
            const int p = pos0 + __popc(bal & ((1u << lane) - 1));
            const int oi = reverse ? n - 1 - p : p;
            const u64 c = base_code(ch) ^ (reverse ? 2u : 0u);
            atomicOr(&out[oi >> 5], c << (2 * (oi & 31)));
        }
        pos0 += __popc(bal);
    }
    if (lane == 0) *len_out = (u32)n;
    __syncwarp();
    return n;
}

// Redo the records on the redo list (every record when reverse != 0), one warp per record, and replace what k_decode_fast counted for
// each of them by what it really holds.  A small fixed grid: on clean text the list is empty and every warp leaves at once.
__global__ void __launch_bounds__(256) k_decode_fix(const unsigned char* __restrict__ text, const u32* __restrict__ seq_start, const u32* __restrict__ seq_end,
                                                    u64 n_rec, int maxlen, int reverse, int K, int W64, u64* __restrict__ words, u32* __restrict__ lens,
                                                    const u32* __restrict__ redo, const u32* __restrict__ n_redo, u64* counters) {
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 n = reverse ? n_rec : (u64)*n_redo;
    if (n == 0) return;   // grid-uniform
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd((unsigned long long*)&counters[C_REDO], (unsigned long long)n);
    u64 inst = 0, kept = 0;   // deltas, modulo 2^64
    for (u64 i = warp0; i < n; i += nwarps) {
        const u64 rr = reverse ? i : (u64)redo[i];
        const int before = (int)lens[rr];
        __syncwarp();
        const int after = decode_record_warp(text, seq_start[rr], seq_end[rr], maxlen, reverse, W64, words + rr * (u64)W64, lens + rr);
        if (lane == 0) {
            inst += read_instances(after, K) - read_instances(before, K);
            kept += (u64)(read_instances(after, K) ? 1 : 0) - (u64)(read_instances(before, K) ? 1 : 0);
        }
    }
    cta_add_u64(inst, &counters[C_INSTANCES]);
    cta_add_u64(kept, &counters[C_KEPT]);
}

// ------------------------------------------------------------------------------------------------ the decode of one text chunk
void check_format(const u64* h_cnt) {
    if (h_cnt[C_BADFMT])
        throw std::runtime_error("pgb200: input is not single-line FASTA / 4-line FASTQ (a header line does not start with '>' / '@', or a FASTQ "
                                 "separator line does not start with '+'); multi-line FASTA is not supported");
}

DecodeLines decode_lines(const unsigned char* d_text, size_t nbytes, int fastq, int n_sm, DevBuf& scan_buf, DevBuf& line_buf, u64* d_cnt, u64* h_cnt,
                         cudaStream_t sd) {
    const int lshift = fastq ? 2 : 1, lpr = 1 << lshift;
    const u64 n_tiles = (nbytes + NL_TILE - 1) / NL_TILE;
    scan_buf.ensure((2 * n_tiles + 16) * sizeof(u32) + scan_scratch_elems(n_tiles) * sizeof(u64) + 256);
    u32* tile_cnt = scan_buf.template as<u32>();
    u32* tile_base = tile_cnt + n_tiles + 8;
    u64* scan_tmp = reinterpret_cast<u64*>((reinterpret_cast<uintptr_t>(tile_base + n_tiles + 8) + 255) & ~(uintptr_t)255);
    const uint4* t16 = reinterpret_cast<const uint4*>(d_text);
    const unsigned nl_blocks = (unsigned)std::min<u64>((n_tiles + 7) / 8, (u64)n_sm * 16);
    k_nl_count<<<nl_blocks, 256, 0, sd>>>(t16, (u64)nbytes, n_tiles, tile_cnt);
    PG_CUDA(cudaGetLastError());
    device_scan(ScanU32In{tile_cnt}, ScanU32Out{tile_base}, n_tiles, scan_tmp, d_cnt + C_MISC0, sd);
    unsigned char* h_last = reinterpret_cast<unsigned char*>(h_cnt + C_COUNT);
    PG_CUDA(cudaMemcpyAsync(h_last, d_text + nbytes - 1, 1, cudaMemcpyDeviceToHost, sd));
    PG_CUDA(cudaMemcpyAsync(h_cnt, d_cnt, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, sd));
    PG_CUDA(cudaStreamSynchronize(sd));
    check_format(h_cnt);
    const u64 n_lines = h_cnt[C_MISC0];
    // a final line without '\n' still counts (the reference's FASTQ path tolerates it; its FASTA path does not)
    const bool open_tail = *h_last != '\n';
    DecodeLines L{nullptr, nullptr, nullptr, nullptr, nullptr, (n_lines + (open_tail ? 1 : 0)) / lpr};
    if ((n_lines + (open_tail ? 1 : 0)) % lpr != 0)
        throw std::runtime_error("pgb200: text chunk does not hold whole FASTA/FASTQ records (line count not a multiple of 2/4)");
    const u64 n_rec = L.n_rec;
    if (n_rec == 0) return L;
    line_buf.ensure((4 * n_rec + 1) * sizeof(u32) + 256);
    L.seq_start = line_buf.template as<u32>();
    L.seq_end = L.seq_start + n_rec;
    L.n_redo = L.seq_end + n_rec;
    L.flag = L.n_redo + 1;
    L.redo = L.flag + n_rec;
    PG_CUDA(cudaMemsetAsync(L.n_redo, 0, (n_rec + 1) * sizeof(u32), sd));   // the count and the flags
    if (open_tail) PG_CUDA(cudaMemsetAsync(L.seq_end, 0, n_rec * sizeof(u32), sd));   // FASTQ: the open line is the quality line
    k_line_index<<<nl_blocks, 256, 0, sd>>>(t16, (u64)nbytes, n_tiles, tile_base, lshift, n_rec, L.seq_start, L.seq_end, d_cnt);
    PG_CUDA(cudaGetLastError());
    if (open_tail && !fastq) {
        const u32 e = (u32)nbytes;
        PG_CUDA(cudaMemcpyAsync(L.seq_end + n_rec - 1, &e, sizeof e, cudaMemcpyHostToDevice, sd));
        PG_CUDA(cudaStreamSynchronize(sd));
    }
    return L;
}

void decode_records(const unsigned char* d_text, size_t nbytes, const DecodeLines& L, int maxlen, int reverse, int K, int W64, int n_sm, u64* words,
                    u32* lens, u64* d_cnt, cudaStream_t sd) {
    const u64 n_rec = L.n_rec, total = n_rec * (u64)W64;
    k_decode_fast<<<(unsigned)std::min<u64>((total + 255) / 256, (u64)n_sm * 64), 256, 0, sd>>>(d_text, (u64)nbytes, L.seq_start, L.seq_end, n_rec, maxlen, K,
                                                                                            W64, words, lens, L.flag, L.redo, L.n_redo, d_cnt);
    PG_CUDA(cudaGetLastError());
    k_decode_fix<<<(unsigned)std::min<u64>((n_rec + 7) / 8, (u64)n_sm * 8), 256, 0, sd>>>(d_text, L.seq_start, L.seq_end, n_rec, maxlen, reverse, K, W64,
                                                                                    words, lens, L.redo, L.n_redo, d_cnt);
    PG_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ feed_text
template <int NW>
void EngineT<NW>::check_format_counter() { check_format(h_cnt_); }

template <int NW>
void EngineT<NW>::feed_text(const char* text, size_t nbytes, bool on_device, int fastq, uint64_t ord_base, uint64_t ord_stride,
                            int reverse_seq, int maxlen) {
    double t_a = host_now(), t_b = 0, t_c = 0, t_e = 0;
    last_records_ = 0;
    if (nbytes == 0) return;
    if (nbytes >= (1ull << 32)) throw std::runtime_error("pgb200: a text chunk must be smaller than 4 GiB (feed it in pieces)");
    PG_CUDA(cudaSetDevice(prm_.device));
    // Which insert: several GPUs -> records (the only exchange format).  One GPU: text that is already in HBM -> aggregated (one HBM
    // update per DISTINCT k-mer); text that arrives over PCIe -> per-instance inserts, which run at the DRAM update rate but can hide
    // under the H2D copies, whereas the aggregation can only finish after the last chunk (aggregating mid-stream multiplies the HBM
    // updates).  PGB200_SKM=0|1 forces one of them.
    const bool use_skm = prm_.world > 1 || skm_mode_ > 0 || (skm_mode_ < 0 && on_device);
    cudaStream_t sd = use_skm ? st_dec_ : st_;   // the per-instance insert needs exact counters per chunk: one stream
    if (!use_skm) clear_table_if_dirty();        // the inserts need an empty table: its clear runs beside this chunk's decode
    const unsigned char* d_text = nullptr;
    const bool host_src = !on_device;
    if (host_src) {
        // H2D on its own stream into the buffer the previous chunk is NOT using: the copy overlaps the previous chunks' kernels
        DevBuf& tb = text_bufs_[text_flip_];
        text_flip_ ^= 1;
        tb.ensure(nbytes + 16);
        PG_CUDA(cudaMemcpyAsync(tb.p, text, nbytes, cudaMemcpyHostToDevice, st_copy_));
        PG_CUDA(cudaEventRecord(ev_copy_, st_copy_));
        PG_CUDA(cudaStreamWaitEvent(sd, ev_copy_, 0));
        d_text = tb.template as<unsigned char>();
    }
    if (ev_head_ - ev_tail_ >= (unsigned)EV_RING) settle_oldest();
    const Event* ev = ev_ring_[ev_head_ % EV_RING];
    PG_CUDA(cudaEventRecord(ev[0], sd));
    if (on_device) {
        d_text = reinterpret_cast<const unsigned char*>(text);
        if ((uintptr_t)text & 15) {   // the line index reads 16-byte groups: realign with one device-to-device copy
            DevBuf& tb = text_bufs_[text_flip_];
            text_flip_ ^= 1;
            tb.ensure(nbytes + 16);
            PG_CUDA(cudaMemcpyAsync(tb.p, text, nbytes, cudaMemcpyDeviceToDevice, sd));
            d_text = tb.template as<unsigned char>();
        }
    }
    if (maxlen > prm_.max_rd_len) maxlen = prm_.max_rd_len;
    // ONE host sync per chunk, of the decode stream: line count, last byte, and the counters as they are
    const DecodeLines L = decode_lines(d_text, nbytes, fastq, n_sm_, scan_buf_, line_buf_, d_cnt_, h_cnt_, sd);
    const u64 n_rec = L.n_rec;
    const u64 have_distinct = h_cnt_[C_DISTINCT];
    if (n_rec == 0) return;
    t_b = host_now();

    ReadChunk ch;
    ch.n_rec = n_rec;
    ch.ord_base = ord_base;
    ch.ord_stride = ord_stride;
    ch.words = reinterpret_cast<u64*>(arena_alloc(n_rec * (u64)W64_ * sizeof(u64)));
    ch.len = reinterpret_cast<u32*>(arena_alloc(n_rec * sizeof(u32)));
    chunks_.push_back(ch);
    t_c = host_now();
    decode_records(d_text, nbytes, L, maxlen, reverse_seq, prm_.K, W64_, n_sm_, ch.words, ch.len, d_cnt_, sd);
    PG_CUDA(cudaEventRecord(ev[1], sd));
    if (use_skm) {
        PG_CUDA(cudaEventRecord(ev_dec_done_, sd));
        skm_make_room(n_rec, host_src);            // may launch the aggregation of what the arena holds (timed by itself)
        PG_CUDA(cudaStreamWaitEvent(st_, ev_dec_done_, 0));
        PG_CUDA(cudaEventRecord(ev[2], st_));
        skm_feed_chunk(chunks_.size() - 1);
    } else {
        PG_CUDA(cudaEventRecord(ev[2], st_));
        // per-instance inserts: table capacity for the worst case of this chunk (host-side bound; growth itself syncs when it happens)
        const int per_read = maxlen - prm_.K + 1;
        ensure_table_bound(have_distinct, per_read > 0 ? n_rec * (u64)per_read : 0);
        chop_insert_chunk(ch);
    }
    PG_CUDA(cudaEventRecord(ev[3], st_));
    ev_head_++;
    if (host_src) PG_CUDA(cudaEventSynchronize(ev_copy_));   // the caller may reuse its host buffer; the kernels keep running
    p1_.launches += 8;   // newline count, 3 scan launches, line index, 2 decode launches (+ the insert side, counted there)
    last_records_ = n_rec;
    total_records_ += n_rec;
    t_e = host_now();
    if (prm_.verbose >= 2)
        fprintf(stderr, "[pgb200] chunk %zu: %llu rec, host ms: count %.2f alloc %.2f launch %.2f\n", chunks_.size(), (unsigned long long)n_rec, t_b - t_a, t_c - t_b,
                t_e - t_c);
}

template <int NW>
void EngineT<NW>::settle_oldest() {
    if (ev_tail_ == ev_head_) return;
    const Event* ev = ev_ring_[ev_tail_ % EV_RING];
    PG_CUDA(cudaEventSynchronize(ev[1]));
    PG_CUDA(cudaEventSynchronize(ev[3]));
    float ms;
    PG_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1])); p1_.ms_decode += ms;
    PG_CUDA(cudaEventElapsedTime(&ms, ev[2], ev[3])); p1_.ms_insert += ms;
    ev_tail_++;
}
template <int NW>
void EngineT<NW>::settle_timing() {
    while (ev_tail_ != ev_head_) settle_oldest();
}

template void EngineT<2>::feed_text(const char*, size_t, bool, int, uint64_t, uint64_t, int, int);
template void EngineT<4>::feed_text(const char*, size_t, bool, int, uint64_t, uint64_t, int, int);
template void EngineT<2>::settle_timing(); template void EngineT<4>::settle_timing();
template void EngineT<2>::settle_oldest(); template void EngineT<4>::settle_oldest();
template void EngineT<2>::check_format_counter(); template void EngineT<4>::check_format_counter();

}   // namespace pgb
