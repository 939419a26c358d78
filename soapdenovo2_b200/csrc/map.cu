// map.cu -- the GPU half of the `map` stage: the contig k-mer table and the read-to-contig placement.
//
// Replaces (reference file:line, standardPregraph/):
//   prlContig2nodes / chopKmer4read / singleKmer   prlHashCtg.c:129-155, 185-256, 325-467   -> k_map_contigs
//   chopKmer4read / searchKmer / parse1read        prlRead2Ctg.c:153-361                    -> k_map_reads
// Text decoding is pass 1's (decode_lines / decode_records, decode.cu); the host (map_stage.cpp) parses .contig, builds the batches
// and restates recordAlldgn.
//
// Contig table.  Every canonical k-mer of every kept contig is inserted into a Table<NW> with the claim protocol of pass 1.  The
// claimer stores the payload {contig id (bits 0..31), position mod 2^24 (bits 32..55, the reference's 24-bit r_links field), twin
// (bits 56..57)}; every instance, the claimer's included, adds 1 to `aux`, which starts at ~0 (the table's memset state).  So after
// the launch aux == 0 exactly when the key occurred once.  The reference stores the fields of the FIRST instance and sets `deleted`
// on every further one: a key seen twice is deleted whatever the order, and a key seen once has only one instance to store.  The
// result is therefore a pure function of the multiset of instances -- exact under any interleaving of the threads.
//
// Reads.  One thread per read rolls the forward and reverse-complement k-mers, does one read-only lookup per k-mer (K <= 63: one
// 32 B sector holds key, payload and count) and writes the hit, or 0, to its own span of a per-batch scratch array -- the reference's
// nodeBuffer.  The same thread then runs parse1read over that span, in the reference's own order: groups by contig id in order of
// first occurrence (later members are cleared as they are counted), `counter2` / `counter` / the strict `>` that gives a tie to the
// earlier group.  Per-read state is a handful of registers whatever the read length, so no read spills; the span lives in global
// memory (8 B per k-mer, at most 100 M k-mers per batch, the reference's buffer_size).
//
// Long reads (prlLongRead2Ctg, prlRead2Ctg.c:1080-1298).  A batch holds 100 M / (longReadLen - K + 1) reads -- 20 000 at a 5 kbp
// cutoff -- so one thread per read would leave most of the GPU idle, each thread doing thousands of dependent lookups.  k_map_long
// gives each read one CTA: the threads take contiguous slices of at least MAP_SEG k-mers, build the slice's first forward / reverse-
// complement pair and roll from there, look each k-mer up with map_lookup and write the hit to the span as k_map_reads does.  Each
// hit is also counted in a shared-memory group table keyed by contig id; parse1read's result is a function of the groups' (count,
// first index) alone, and the table stays exact past its size by grouping the leftover ids in further rounds (map_group.cuh has
// the argument).  The reads are stored at their own packed length, located by word offsets.
#include "engine_impl.cuh"
#include "map.h"
#include "map_group.cuh"
#include <algorithm>
#include <cstdlib>

#pragma GCC visibility push(hidden)
namespace pgb {

constexpr int MAP_SEG = 64;   // contig k-mers per thread of k_map_contigs; the least k-mers per thread of k_map_long
constexpr int MAP_LONG_THREADS = 128;

struct CtgSeg {
    u64 base;      // global base index of the segment's first k-mer
    u32 ctg_id;
    u32 pos0;      // index of that k-mer on its contig
    u32 n;         // k-mers in the segment
    u32 pad;
};

// prevKmer with the new base or-ed into every word under a select: kprev's `if (i == top_word)` is compiled into a dynamically
// indexed store, which puts the k-mer in local memory once per base
template <int NW>
PG_D Kmer<NW> kprev_reg(const Kmer<NW>& a, unsigned c, const KParams<NW>& p) {
    Kmer<NW> r = kshr2(a);
#pragma unroll
    for (int i = 0; i < NW; i++) r.w[i] |= i == p.top_word ? (u64)c << p.top_shift : 0ull;
    return r;
}

template <int NW>
struct KPair { Kmer<NW> f, rc; };
template <int NW>
PG_D KPair<NW> first_kmer(const u64* __restrict__ w, u64 b, const KParams<NW>& kp) {
    KPair<NW> k{kzero<NW>(), kzero<NW>()};
    for (int i = 0; i < kp.K; i++) {
        const u64 p = b + i;
        const unsigned c = (unsigned)(w[p >> 5] >> (2 * (p & 31))) & 3u;
        k.f = knext(k.f, c, kp);
        k.rc = kprev_reg(k.rc, c ^ 2u, kp);
    }
    return k;
}

// the canonical k-mer, selected word by word so that both candidates stay in registers (a select of a whole Kmer by reference puts
// them in local memory)
template <int NW>
PG_D Kmer<NW> kcanon(const Kmer<NW>& f, const Kmer<NW>& rc, bool smaller) {
    Kmer<NW> c;
#pragma unroll
    for (int i = 0; i < NW; i++) c.w[i] = smaller ? f.w[i] : rc.w[i];
    return c;
}

template <int NW>
__global__ void __launch_bounds__(256) k_map_contigs(Table<NW> t, KParams<NW> kp, const u64* __restrict__ bases, const CtgSeg* __restrict__ segs, u64 n_seg,
                                                     u64* __restrict__ n_claimed) {
    u64 mine = 0;
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += (u64)gridDim.x * blockDim.x) {
        const CtgSeg g = segs[s];
        const KPair<NW> k0 = first_kmer(bases, g.base, kp);
        Kmer<NW> f = k0.f, rc = k0.rc;
        for (u32 j = 0; j < g.n; j++) {
            if (j) {
                const u64 p = g.base + j + kp.K - 1;
                const unsigned c = (unsigned)(bases[p >> 5] >> (2 * (p & 31))) & 3u;
                f = knext(f, c, kp);
                rc = kprev_reg(rc, c ^ 2u, kp);
            }
            const bool smaller = kless(f, rc);
            bool claimed;
            const u64 idx = table_find_or_claim(t, kcanon(f, rc, smaller), &claimed);
            Slot<NW>* sl = t.slots + idx;
            if (claimed) { sl->payload = (u64)g.ctg_id | ((u64)((g.pos0 + j) & 0xFFFFFFu) << 32) | ((u64)(smaller ? 0 : 1) << 56); mine++; }
            atomicAdd(&sl->aux, 1ull);
        }
    }
    if (mine) atomicAdd(n_claimed, mine);
}

// payload | HIT_VALID of a key that occurred once, else 0
template <int NW>
PG_D u64 map_lookup(const Table<NW>& t, const Kmer<NW>& k) {
    if constexpr (NW == 2) {
        u64 idx = table_hash(k) & t.mask;
        for (;;) {
            const U256 v = ld256(t.slots + idx);
            if (v.a == k.w[0] && v.b == k.w[1]) return v.d == 0 ? (v.c | HIT_VALID) : 0ull;
            if (v.a == EMPTY64 && v.b == EMPTY64) return 0ull;
            idx = (idx + 1) & t.mask;
        }
    } else {
        const u64 idx = table_find(t, k);
        if (idx == ~0ull) return 0ull;
        const U128 v = ldcg128(&t.slots[idx].payload);
        return v.b == 0 ? (v.a | HIT_VALID) : 0ull;
    }
}

template <int NW>
__global__ void __launch_bounds__(128) k_map_reads(Table<NW> t, KParams<NW> kp, const u64* __restrict__ words, const u32* __restrict__ lens,
                                                   const u64* __restrict__ kofs, u64 n_reads, int W64, int alignlen, u64* __restrict__ hits,
                                                   MapHit* __restrict__ out) {
    const int K = kp.K;
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += (u64)gridDim.x * blockDim.x) {
        const int len = (int)lens[r];
        const u64* w = words + r * (u64)W64;
        u64* h = hits + kofs[r];
        const int nk = len >= K + 1 ? len - K + 1 : 0;   // chopKmer4read returns early below K+1 (the span is empty)
        if (nk > 0) {
            const KPair<NW> k0 = first_kmer(w, 0, kp);
            Kmer<NW> f = k0.f, rc = k0.rc;
            for (int j = 0; j < nk; j++) {
                if (j) {
                    const int p = j + K - 1;
                    const unsigned c = (unsigned)(w[p >> 5] >> (2 * (p & 31))) & 3u;
                    f = knext(f, c, kp);
                    rc = kprev_reg(rc, c ^ 2u, kp);
                }
                const bool smaller = kless(f, rc);
                const u64 v = map_lookup(t, kcanon(f, rc, smaller));
                h[j] = v ? v | ((u64)smaller << HIT_SMALLER_SHIFT) : 0ull;
            }
        }
        // parse1read
        const int alldgn = len > alignlen ? alignlen : len;
        const int multi = alldgn - K + 1 < 2 ? 2 : alldgn - K + 1;
        int counter = 0, counter2 = 0, max_occ = 0, best_j = 0;
        u64 best = 0;
        for (int j = 0; j < nk; j++) {
            const u64 v = h[j];
            if (!v) continue;
            int flag = 1;
            for (int s = j + 1; s < nk; s++) {
                const u64 u = h[s];
                if (u && (u32)u == (u32)v) { flag++; h[s] = 0; }
            }
            if ((K < 32 && flag >= 2) || K > 32) counter2++;
            if (flag < multi) continue;
            counter++;
            if (flag > max_occ) { best_j = j; max_occ = flag; best = v; }
        }
        MapHit o{0u, 0, 0, 0u};
        if (counter) {
            const unsigned twin = (unsigned)(best >> 56) & 3u, smaller = (unsigned)(best >> HIT_SMALLER_SHIFT) & 1u;
            o.ctg = (u32)best;
            o.node_pos = (int)((best >> 32) & 0xFFFFFFu);
            o.i = best_j + 1;
            o.flags = MAP_PLACED | (twin == smaller ? MAP_MINUS : 0u) | (counter2 > 1 ? MAP_FOOTPRINT : 0u);
        }
        out[r] = o;
    }
}

// one CTA per read (grid-stride over the batch); read r is words[wofs[r] ...], its hits go to hits[kofs[r] ...]
template <int NW>
__global__ void __launch_bounds__(MAP_LONG_THREADS) k_map_long(Table<NW> t, KParams<NW> kp, const u64* __restrict__ words, const u64* __restrict__ wofs,
                                                               const u32* __restrict__ lens, const u64* __restrict__ kofs, u64 n_reads, int alignlen,
                                                               u32 n_groups, u64* __restrict__ hits, MapHit* __restrict__ out) {
    __shared__ u32 s_id[MAP_GROUPS], s_cnt[MAP_GROUPS], s_first[MAP_GROUPS];
    __shared__ GroupAcc s_acc;
    __shared__ int s_pending;
    const int K = kp.K, tid = threadIdx.x, nthr = blockDim.x;
    const GroupTab g{s_id, s_cnt, s_first, n_groups};
    for (u64 r = blockIdx.x; r < n_reads; r += gridDim.x) {
        const int len = (int)lens[r];
        const u64* w = words + wofs[r];
        u64* h = hits + kofs[r];
        const u32 nk = len >= K + 1 ? (u32)(len - K + 1) : 0u;   // chopKmer4read returns early below K+1 (the span is empty)
        group_clear(g, tid, nthr);
        if (tid == 0) { s_acc = GroupAcc{0u, 0u, 0ull}; s_pending = 0; }
        __syncthreads();
        // this thread's slice: [j0, j1), at least MAP_SEG k-mers unless the read has fewer
        const u32 per = max((u32)MAP_SEG, (nk + nthr - 1) / nthr);
        const u32 j0 = min(nk, (u32)tid * per), j1 = min(nk, j0 + per);
        if (j0 < j1) {
            const KPair<NW> k0 = first_kmer(w, j0, kp);
            Kmer<NW> f = k0.f, rc = k0.rc;
            for (u32 j = j0; j < j1; j++) {
                if (j > j0) {
                    const u32 p = j + K - 1;
                    const unsigned c = (unsigned)(w[p >> 5] >> (2 * (p & 31))) & 3u;
                    f = knext(f, c, kp);
                    rc = kprev_reg(rc, c ^ 2u, kp);
                }
                const bool smaller = kless(f, rc);
                const u64 v = map_lookup(t, kcanon(f, rc, smaller));
                h[j] = v ? v | ((u64)smaller << HIT_SMALLER_SHIFT) : 0ull;
                if (v) group_add_hit(h, j, g, &s_pending);
            }
        }
        // parse1read: fold the groups; ids left over when the table is full are grouped in further rounds
        const int alldgn = len > alignlen ? alignlen : len;
        const u32 multi = (u32)(alldgn - K + 1 < 2 ? 2 : alldgn - K + 1);
        for (;;) {
            __syncthreads();
            group_fold(g, K, multi, tid, nthr, &s_acc);
            const int more = s_pending;   // no thread writes it between the barriers around this read
            __syncthreads();
            if (!more) break;
            group_clear(g, tid, nthr);
            if (tid == 0) s_pending = 0;
            __syncthreads();
            group_round(h, nk, g, tid, nthr, &s_pending);
        }
        if (tid == 0) {
            const GroupAcc a = s_acc;
            MapHit o{0u, 0, 0, 0u};
            if (a.counter) {
                const u32 bj = group_best_j(a);
                const u64 best = h[bj];
                const unsigned twin = (unsigned)(best >> 56) & 3u, smaller = (unsigned)(best >> HIT_SMALLER_SHIFT) & 1u;
                o.ctg = (u32)best;
                o.node_pos = (int)((best >> 32) & 0xFFFFFFu);
                o.i = (int)bj + 1;
                o.flags = MAP_PLACED | (twin == smaller ? MAP_MINUS : 0u) | (a.counter2 > 1 ? MAP_FOOTPRINT : 0u);
            }
            out[r] = o;
        }
        __syncthreads();   // s_acc is read before the next read resets it
    }
}

// strided decode output (stride words per read) -> packed at each read's own length, read r at ofs[r]
__global__ void __launch_bounds__(256) k_pack_reads(const u64* __restrict__ in, int stride, const u32* __restrict__ lens, const u64* __restrict__ ofs,
                                                    u64 n, u64* __restrict__ packed) {
    const int lane = threadIdx.x & 31;
    for (u64 r = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((u64)gridDim.x * blockDim.x) >> 5) {
        const u32 nw = (lens[r] + 31) / 32;
        for (u32 i = lane; i < nw; i += 32) packed[ofs[r] + i] = in[r * (u64)stride + i];
    }
}

template <int NW>
class MapEngineT : public IMapEngine {
public:
    MapEngineT(int K, int device, int max_rd_len) : K_(K), device_(device) {
        kp_ = make_kparams<NW>(K);
        W64_ = std::max(1, (max_rd_len + 31) / 32);
        PG_CUDA(cudaSetDevice(device));
        PG_CUDA(cudaDeviceGetAttribute(&n_sm_, cudaDevAttrMultiProcessorCount, device));
        PG_CUDA(cudaStreamCreateWithFlags(&st_.h, cudaStreamNonBlocking));
        PG_CUDA(cudaEventCreate(&ev_[0].h)); PG_CUDA(cudaEventCreate(&ev_[1].h));
        PG_CUDA(cudaHostAlloc(&h_cnt_.h, (C_COUNT + 2) * sizeof(u64), cudaHostAllocDefault));
        cnt_.alloc(C_COUNT * sizeof(u64));
        PG_CUDA(cudaMemsetAsync(cnt_.p, 0, C_COUNT * sizeof(u64), st_));
    }
    ~MapEngineT() override { if (st_) cudaStreamSynchronize(st_); }
    int words_per_read() const override { return W64_; }

    void hash_contigs(const u64* packed, u64 n_bases, const u64* ctg_off, const u32* ctg_id, u64 n_ctg, u64* distinct) override {
        std::vector<CtgSeg> segs;
        u64 n_kmers = 0;
        for (u64 c = 0; c < n_ctg; c++) {
            const u64 n = ctg_off[c + 1] - ctg_off[c] - (u64)K_ + 1;
            n_kmers += n;
            for (u64 j = 0; j < n; j += MAP_SEG) segs.push_back({ctg_off[c] + j, ctg_id[c], (u32)j, (u32)std::min<u64>(MAP_SEG, n - j), 0u});
        }
        const u64 cap = next_pow2(std::max<u64>(1024, n_kmers * 2));
        tab_buf_.alloc(cap * sizeof(Slot<NW>));
        PG_CUDA(cudaMemsetAsync(tab_buf_.p, 0xFF, cap * sizeof(Slot<NW>), st_));
        tab_ = Table<NW>{tab_buf_.as<Slot<NW>>(), cap - 1};
        DevBuf d_bases, d_segs;
        d_bases.alloc((n_bases + 31) / 32 * sizeof(u64) + 8);
        d_segs.alloc(segs.size() * sizeof(CtgSeg));
        PG_CUDA(cudaMemcpyAsync(d_bases.p, packed, (n_bases + 31) / 32 * sizeof(u64), cudaMemcpyHostToDevice, st_));
        if (!segs.empty()) PG_CUDA(cudaMemcpyAsync(d_segs.p, segs.data(), segs.size() * sizeof(CtgSeg), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaEventRecord(ev_[0], st_));
        if (!segs.empty()) {
            k_map_contigs<NW><<<(unsigned)std::min<u64>((segs.size() + 255) / 256, (u64)n_sm_ * 8), 256, 0, st_>>>(tab_, kp_, d_bases.as<u64>(), d_segs.as<CtgSeg>(),
                                                                                                             (u64)segs.size(), cnt_.as<u64>() + C_DISTINCT);
            PG_CUDA(cudaGetLastError());
        }
        PG_CUDA(cudaEventRecord(ev_[1], st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        ms_hash_ += ms;
        PG_CUDA(cudaMemcpy(h_cnt_, cnt_.p, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost));
        *distinct = h_cnt_[C_DISTINCT];
    }

    void decode_text(const char* text, size_t nbytes, int fastq, int reverse, int maxlen, int stride, std::vector<u64>* words,
                     std::vector<u32>* lens) override {
        if (nbytes == 0) return;
        if (nbytes >= (1ull << 32)) throw std::runtime_error("pgb200: a text chunk must be smaller than 4 GiB (feed it in pieces)");
        PG_CUDA(cudaSetDevice(device_));
        text_buf_.ensure(nbytes + 16);
        PG_CUDA(cudaMemcpyAsync(text_buf_.p, text, nbytes, cudaMemcpyHostToDevice, st_));
        const unsigned char* d_text = text_buf_.as<unsigned char>();
        PG_CUDA(cudaEventRecord(ev_[0], st_));
        const DecodeLines L = decode_lines(d_text, nbytes, fastq, n_sm_, scan_buf_, line_buf_, cnt_.as<u64>(), h_cnt_, st_);
        if (L.n_rec == 0) return;
        const u64 n = L.n_rec;
        const int S = stride > 0 ? stride : std::max(1, (maxlen + 31) / 32);   // the decode's stride: room for maxlen bases
        read_words_.ensure(n * S * sizeof(u64));
        read_lens_.ensure(n * sizeof(u32));
        decode_records(d_text, nbytes, L, maxlen, reverse, K_, S, n_sm_, read_words_.as<u64>(), read_lens_.as<u32>(), cnt_.as<u64>(), st_);
        if (stride > 0) PG_CUDA(cudaEventRecord(ev_[1], st_));
        const size_t w0 = words->size(), l0 = lens->size();
        lens->resize(l0 + n);
        PG_CUDA(cudaMemcpyAsync(lens->data() + l0, read_lens_.p, n * sizeof(u32), cudaMemcpyDeviceToHost, st_));
        // the line index of THIS chunk flags malformed records (decode_lines checked the counters before it ran)
        PG_CUDA(cudaMemcpyAsync(h_cnt_, cnt_.p, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, st_));
        u64 n_words = n * S;
        const u64* src = read_words_.as<u64>();
        if (stride <= 0) {   // packed: each read at its own length, ceil(len / 32) words
            PG_CUDA(cudaStreamSynchronize(st_));
            check_format(h_cnt_);
            std::vector<u64> ofs(n);
            n_words = 0;
            for (u64 r = 0; r < n; r++) { ofs[r] = n_words; n_words += ((*lens)[l0 + r] + 31) / 32; }
            pack_ofs_.ensure(n * sizeof(u64));
            pack_words_.ensure(n_words * sizeof(u64) + 8);
            PG_CUDA(cudaMemcpyAsync(pack_ofs_.p, ofs.data(), n * sizeof(u64), cudaMemcpyHostToDevice, st_));
            k_pack_reads<<<(unsigned)std::min<u64>((n + 7) / 8, (u64)n_sm_ * 16), 256, 0, st_>>>(src, S, read_lens_.as<u32>(), pack_ofs_.as<u64>(), n,
                                                                                                 pack_words_.as<u64>());
            PG_CUDA(cudaGetLastError());
            PG_CUDA(cudaEventRecord(ev_[1], st_));
            src = pack_words_.as<u64>();
        }
        words->resize(w0 + n_words);
        PG_CUDA(cudaMemcpyAsync(words->data() + w0, src, n_words * sizeof(u64), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        check_format(h_cnt_);
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        ms_decode_ += ms;
    }

    void map_batch(const u64* words, const u32* lens, u64 n, int alignlen, MapHit* out) override {
        PG_CUDA(cudaSetDevice(device_));
        std::vector<u64> kofs(n + 1);
        u64 k = 0;
        for (u64 r = 0; r < n; r++) { kofs[r] = k; if ((int)lens[r] >= K_ + 1) k += lens[r] - K_ + 1; }
        kofs[n] = k;
        batch_words_.ensure(n * W64_ * sizeof(u64));
        batch_lens_.ensure(n * sizeof(u32) + 4);
        batch_kofs_.ensure((n + 1) * sizeof(u64));
        hits_.ensure(k * sizeof(u64) + 8);
        out_.ensure(n * sizeof(MapHit) + 16);
        PG_CUDA(cudaMemcpyAsync(batch_words_.p, words, n * W64_ * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_lens_.p, lens, n * sizeof(u32), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_kofs_.p, kofs.data(), (n + 1) * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaEventRecord(ev_[0], st_));
        if (n) {
            k_map_reads<NW><<<(unsigned)std::min<u64>((n + 127) / 128, (u64)n_sm_ * 16), 128, 0, st_>>>(tab_, kp_, batch_words_.as<u64>(), batch_lens_.as<u32>(),
                                                                                                   batch_kofs_.as<u64>(), n, W64_, alignlen, hits_.as<u64>(),
                                                                                                   out_.as<MapHit>());
            PG_CUDA(cudaGetLastError());
        }
        PG_CUDA(cudaEventRecord(ev_[1], st_));
        PG_CUDA(cudaMemcpyAsync(out, out_.p, n * sizeof(MapHit), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        ms_scan_ += ms;
    }

    void map_long_batch(const u64* words, u64 n_words, const u64* wofs, const u32* lens, u64 n, int alignlen, MapHit* out) override {
        PG_CUDA(cudaSetDevice(device_));
        std::vector<u64> kofs(n + 1);
        u64 k = 0;
        for (u64 r = 0; r < n; r++) { kofs[r] = k; if ((int)lens[r] >= K_ + 1) k += lens[r] - K_ + 1; }
        kofs[n] = k;
        batch_words_.ensure(n_words * sizeof(u64) + 8);
        batch_wofs_.ensure(n * sizeof(u64) + 8);
        batch_lens_.ensure(n * sizeof(u32) + 4);
        batch_kofs_.ensure((n + 1) * sizeof(u64));
        hits_.ensure(k * sizeof(u64) + 8);
        out_.ensure(n * sizeof(MapHit) + 16);
        PG_CUDA(cudaMemcpyAsync(batch_words_.p, words, n_words * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_wofs_.p, wofs, n * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_lens_.p, lens, n * sizeof(u32), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_kofs_.p, kofs.data(), (n + 1) * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaEventRecord(ev_[0], st_));
        if (n) {
            k_map_long<NW><<<(unsigned)std::min<u64>(n, (u64)n_sm_ * 16), MAP_LONG_THREADS, 0, st_>>>(tab_, kp_, batch_words_.as<u64>(), batch_wofs_.as<u64>(),
                                                                                                       batch_lens_.as<u32>(), batch_kofs_.as<u64>(), n, alignlen,
                                                                                                       n_groups_, hits_.as<u64>(), out_.as<MapHit>());
            PG_CUDA(cudaGetLastError());
        }
        PG_CUDA(cudaEventRecord(ev_[1], st_));
        PG_CUDA(cudaMemcpyAsync(out, out_.p, n * sizeof(MapHit), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        ms_long_ += ms;
        lookups_long_ += k;
    }
    void times(MapTimes* t) const override { *t = MapTimes{ms_hash_, ms_decode_, ms_scan_, ms_long_, lookups_long_}; }

private:
    int K_, device_, W64_ = 1, n_sm_ = 0;
    // group slots of k_map_long; PGB200_MAP_GROUPS lowers it (1..MAP_GROUPS) so that a test can force the overflow rounds
    u32 n_groups_ = getenv("PGB200_MAP_GROUPS") ? (u32)std::min<long>(std::max<long>(1, atol(getenv("PGB200_MAP_GROUPS"))), (long)MAP_GROUPS) : MAP_GROUPS;
    KParams<NW> kp_;
    Stream st_;
    Event ev_[2];
    Pinned<u64> h_cnt_;
    DevBuf cnt_, tab_buf_, text_buf_, scan_buf_, line_buf_, read_words_, read_lens_, pack_ofs_, pack_words_, batch_words_, batch_wofs_, batch_lens_,
        batch_kofs_, hits_, out_;
    Table<NW> tab_{nullptr, 0};
    double ms_hash_ = 0, ms_decode_ = 0, ms_scan_ = 0, ms_long_ = 0;
    u64 lookups_long_ = 0;
};

IMapEngine* make_map_engine(int K, int device, int max_rd_len) {
    if (K <= 63) return new MapEngineT<2>(K, device, max_rd_len);
    return new MapEngineT<4>(K, device, max_rd_len);
}

}   // namespace pgb
#pragma GCC visibility pop
