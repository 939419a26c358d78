// map.cu -- the GPU half of the `map` stage: the contig k-mer table and the read-to-contig placement.
//
// Replaces (reference file:line, standardPregraph/):
//   prlContig2nodes / chopKmer4read / singleKmer   prlHashCtg.c:129-155, 185-256, 325-467   -> k_map_contigs
//   chopKmer4read / searchKmer / parse1read        prlRead2Ctg.c:153-361                    -> k_map_reads
// Text decoding is pass 1's (decode_lines / decode_records, decode.cu, then k_pack_reads), or the fgets reader (reader.cu) that reads
// wrapped records as the reference's map stage does; the host (map_stage.cpp) parses .contig, builds the batches and restates
// recordAlldgn.  Both readers return, and both read kernels take, one layout: each read packed 2 bits per base at its own length,
// ceil(len / 32) words, located by word offsets.  k_map_contigs, k_map_reads and k_map_long share one k-mer step (kmer_at: roll,
// canonical; read_hit adds the lookup) and the two read kernels one placement (map_hit).
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
// the argument).
#include "engine_impl.cuh"
#include "map.h"
#include "map_group.cuh"
#include "reader.cuh"
#include "scan.cuh"
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

// The canonical form of k-mer j of the bases at w (bases b + j .. b + j + K - 1).  k holds k-mer j - 1 and is rolled on by one base,
// except at the first k-mer j0 of a loop, which first_kmer built.  *smaller: the forward k-mer is the smaller (isSmaller).
template <int NW>
PG_D Kmer<NW> kmer_at(const u64* __restrict__ w, u32 b, u32 j, u32 j0, KPair<NW>& k, const KParams<NW>& kp, bool* smaller) {
    if (j > j0) {
        const u32 p = b + j + kp.K - 1;
        const unsigned c = (unsigned)(w[p >> 5] >> (2 * (p & 31))) & 3u;
        k.f = knext(k.f, c, kp);
        k.rc = kprev_reg(k.rc, c ^ 2u, kp);
    }
    *smaller = kless(k.f, k.rc);
    return kcanon(k.f, k.rc, *smaller);
}

template <int NW>
__global__ void __launch_bounds__(256) k_map_contigs(Table<NW> t, KParams<NW> kp, const u64* __restrict__ bases, const CtgSeg* __restrict__ segs, u64 n_seg,
                                                     u64* __restrict__ n_claimed) {
    u64 mine = 0;
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += (u64)gridDim.x * blockDim.x) {
        const CtgSeg g = segs[s];
        KPair<NW> k = first_kmer(bases, g.base, kp);
        for (u32 j = 0; j < g.n; j++) {
            bool smaller, claimed;
            const u64 idx = table_find_or_claim(t, kmer_at(bases + (g.base >> 5), (u32)(g.base & 31), j, 0u, k, kp, &smaller), &claimed);
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

// the span entry of read k-mer j (kmer_at's rolling): its contig's payload | HIT_VALID with isSmaller at HIT_SMALLER_SHIFT, or 0
template <int NW>
PG_D u64 read_hit(const Table<NW>& t, const u64* __restrict__ w, u32 j, u32 j0, KPair<NW>& k, const KParams<NW>& kp) {
    bool smaller;
    const u64 v = map_lookup(t, kmer_at(w, 0u, j, j0, k, kp, &smaller));
    return v ? v | ((u64)smaller << HIT_SMALLER_SHIFT) : 0ull;
}

// parse1read's placement from the winning group's first hit `best`, at index best_j of the read
PG_D MapHit map_hit(u64 best, u32 best_j, u32 counter2) {
    const unsigned twin = (unsigned)(best >> 56) & 3u, smaller = (unsigned)(best >> HIT_SMALLER_SHIFT) & 1u;
    return MapHit{(u32)best, (int)((best >> 32) & 0xFFFFFFu), (int)best_j + 1,
                  MAP_PLACED | (twin == smaller ? MAP_MINUS : 0u) | (counter2 > 1 ? MAP_FOOTPRINT : 0u)};
}

// A read's two offsets in one word, so that a thread holds one value for both (k_map_reads keeps 32 registers at NW = 2): its first
// word in the batch's words (bits 32..63) and its first hit in the batch's span (bits 0..31).  A batch holds 100 M / (L - K + 1) reads
// of at most L bases, L >= K: at most 100 M k-mers and 4 x 100 M words, so both fit (map_batch checks).
PG_D const u64* read_words(const u64* words, u64 o) { return words + (o >> 32); }
PG_D u64* read_hits(u64* hits, u64 o) { return hits + (u32)o; }

// one thread per read (grid-stride over the batch); read r's words and hits are at ofs[r]
template <int NW>
__global__ void __launch_bounds__(128) k_map_reads(Table<NW> t, KParams<NW> kp, const u64* __restrict__ words, const u64* __restrict__ ofs,
                                                   const u32* __restrict__ lens, u64 n_reads, int alignlen,
                                                   u64* __restrict__ hits, MapHit* __restrict__ out) {
    const int K = kp.K;
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += (u64)gridDim.x * blockDim.x) {
        const int len = (int)lens[r];
        const u64* w = read_words(words, ofs[r]);
        u64* h = read_hits(hits, ofs[r]);
        const int nk = len >= K + 1 ? len - K + 1 : 0;   // chopKmer4read returns early below K+1 (the span is empty)
        if (nk > 0) {
            KPair<NW> k = first_kmer(w, 0, kp);
            for (int j = 0; j < nk; j++) h[j] = read_hit(t, w, (u32)j, 0u, k, kp);
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
        out[r] = counter ? map_hit(best, (u32)best_j, (u32)counter2) : MapHit{0u, 0, 0, 0u};
    }
}

// one CTA per read (grid-stride over the batch); read r's words and hits are at ofs[r]
template <int NW>
__global__ void __launch_bounds__(MAP_LONG_THREADS) k_map_long(Table<NW> t, KParams<NW> kp, const u64* __restrict__ words, const u64* __restrict__ ofs,
                                                               const u32* __restrict__ lens, u64 n_reads, int alignlen,
                                                               u32 n_groups, u64* __restrict__ hits, MapHit* __restrict__ out) {
    __shared__ u32 s_id[MAP_GROUPS], s_cnt[MAP_GROUPS], s_first[MAP_GROUPS];
    __shared__ GroupAcc s_acc;
    __shared__ int s_pending;
    const int K = kp.K, tid = threadIdx.x, nthr = blockDim.x;
    const GroupTab g{s_id, s_cnt, s_first, n_groups};
    for (u64 r = blockIdx.x; r < n_reads; r += gridDim.x) {
        const int len = (int)lens[r];
        const u64* w = read_words(words, ofs[r]);
        u64* h = read_hits(hits, ofs[r]);
        const u32 nk = len >= K + 1 ? (u32)(len - K + 1) : 0u;   // chopKmer4read returns early below K+1 (the span is empty)
        group_clear(g, tid, nthr);
        if (tid == 0) { s_acc = GroupAcc{0u, 0u, 0ull}; s_pending = 0; }
        __syncthreads();
        // this thread's slice: [j0, j1), at least MAP_SEG k-mers unless the read has fewer
        const u32 per = max((u32)MAP_SEG, (nk + nthr - 1) / nthr);
        const u32 j0 = min(nk, (u32)tid * per), j1 = min(nk, j0 + per);
        if (j0 < j1) {
            KPair<NW> k = first_kmer(w, j0, kp);
            for (u32 j = j0; j < j1; j++) {
                const u64 v = read_hit(t, w, j, j0, k, kp);
                h[j] = v;
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
            const u32 bj = group_best_j(a);
            out[r] = a.counter ? map_hit(h[bj], bj, a.counter2) : MapHit{0u, 0, 0, 0u};
        }
        __syncthreads();   // s_acc is read before the next read resets it
    }
}

// strided decode output (stride words per read) -> packed at each read's own length, read r at ofs[r]; one thread per input word
__global__ void __launch_bounds__(256) k_pack_reads(const u64* __restrict__ in, int stride, const u32* __restrict__ lens, const u64* __restrict__ ofs,
                                                    u64 n, u64* __restrict__ packed) {
    const u64 total = n * (u64)stride;
    for (u64 idx = (u64)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (u64)gridDim.x * blockDim.x) {
        const u64 r = idx / (unsigned)stride;
        const u32 w = (u32)(idx - r * (unsigned)stride);
        if (w < (lens[r] + 31) / 32) packed[ofs[r] + w] = in[idx];
    }
}

template <int NW>
class MapEngineT : public IMapEngine {
public:
    MapEngineT(int K, int device) : K_(K), device_(device) {
        kp_ = make_kparams<NW>(K);
        PG_CUDA(cudaSetDevice(device));
        PG_CUDA(cudaDeviceGetAttribute(&n_sm_, cudaDevAttrMultiProcessorCount, device));
        st_ = make_stream();
        for (Event& e : ev_) e = make_event();
        h_cnt_ = make_pinned<u64>(C_COUNT + 2);
        cnt_.alloc(C_COUNT * sizeof(u64));
        PG_CUDA(cudaMemsetAsync(cnt_.p, 0, C_COUNT * sizeof(u64), st_));
    }
    ~MapEngineT() override { if (st_) cudaStreamSynchronize(st_); }

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

    void decode_text(const char* text, size_t nbytes, int fastq, int reverse, int maxlen, std::vector<u64>* words, std::vector<u32>* lens) override {
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
        const int S = std::max(1, (maxlen + 31) / 32);   // the decode's stride: room for maxlen bases
        read_words_.ensure(n * S * sizeof(u64));
        read_lens_.ensure(n * sizeof(u32));
        decode_records(d_text, nbytes, L, maxlen, reverse, K_, S, n_sm_, read_words_.as<u64>(), read_lens_.as<u32>(), cnt_.as<u64>(), st_);
        // each read packed at its own length, ceil(len / 32) words, at the exclusive scan of those counts; pack_ofs_[n]: the total
        pack_ofs_.ensure((n + 1) * sizeof(u64));
        pack_scan_.ensure(scan_scratch_elems(n) * sizeof(u64));
        pack_words_.ensure(n * S * sizeof(u64));
        u64* ofs = pack_ofs_.as<u64>();
        device_scan(ScanWordsOfLen{read_lens_.as<u32>()}, ScanU64Out{ofs}, n, pack_scan_.as<u64>(), ofs + n, st_);
        k_pack_reads<<<(unsigned)std::min<u64>((n * S + 255) / 256, (u64)n_sm_ * 64), 256, 0, st_>>>(read_words_.as<u64>(), S, read_lens_.as<u32>(), ofs, n,
                                                                                             pack_words_.as<u64>());
        PG_CUDA(cudaGetLastError());
        PG_CUDA(cudaEventRecord(ev_[1], st_));
        const size_t w0 = words->size(), l0 = lens->size();
        lens->resize(l0 + n);
        PG_CUDA(cudaMemcpyAsync(lens->data() + l0, read_lens_.p, n * sizeof(u32), cudaMemcpyDeviceToHost, st_));
        // the line index of THIS chunk flags malformed records (decode_lines checked the counters before it ran)
        PG_CUDA(cudaMemcpyAsync(h_cnt_, cnt_.p, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaMemcpyAsync(h_cnt_ + C_COUNT + 1, ofs + n, sizeof(u64), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        check_format(h_cnt_);
        const u64 n_words = h_cnt_[C_COUNT + 1];
        words->resize(w0 + n_words);
        PG_CUDA(cudaMemcpyAsync(words->data() + w0, pack_words_.p, n_words * sizeof(u64), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        ms_decode_ += ms;
    }

    size_t read_text(const char* text, size_t nbytes, int fastq, int piece_len, int cutoff, int reverse, bool at_eof, std::vector<u64>* words,
                     std::vector<u32>* lens) override {
        if (nbytes == 0) return 0;
        PG_CUDA(cudaSetDevice(device_));
        text_buf_.ensure(nbytes + 16);
        PG_CUDA(cudaMemcpyAsync(text_buf_.p, text, nbytes, cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaEventRecord(ev_[0], st_));
        const size_t cut = reader_.read(text_buf_.as<unsigned char>(), nbytes, fastq, piece_len, cutoff, reverse, at_eof, n_sm_, st_, words, lens);
        PG_CUDA(cudaEventRecord(ev_[1], st_));
        PG_CUDA(cudaEventSynchronize(ev_[1]));
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        ms_decode_ += ms;
        return cut;
    }

    void map_batch(const u64* words, u64 n_words, const u64* wofs, const u32* lens, u64 n, int alignlen, bool per_read_cta, MapHit* out) override {
        PG_CUDA(cudaSetDevice(device_));
        std::vector<u64> ofs(n);   // read_words / read_hits
        u64 k = 0;
        for (u64 r = 0; r < n; r++) { ofs[r] = wofs[r] << 32 | k; if ((int)lens[r] >= K_ + 1) k += lens[r] - K_ + 1; }
        if (n_words >> 32 || k >> 32) throw std::runtime_error("pgb200: a map batch holds 2^32 words or k-mers");
        batch_words_.ensure(n_words * sizeof(u64) + 8);
        batch_ofs_.ensure(n * sizeof(u64) + 8);
        batch_lens_.ensure(n * sizeof(u32) + 4);
        hits_.ensure(k * sizeof(u64) + 8);
        out_.ensure(n * sizeof(MapHit) + 16);
        PG_CUDA(cudaMemcpyAsync(batch_words_.p, words, n_words * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_ofs_.p, ofs.data(), n * sizeof(u64), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaMemcpyAsync(batch_lens_.p, lens, n * sizeof(u32), cudaMemcpyHostToDevice, st_));
        PG_CUDA(cudaEventRecord(ev_[0], st_));
        if (n) {
            if (per_read_cta)
                k_map_long<NW><<<(unsigned)std::min<u64>(n, (u64)n_sm_ * 16), MAP_LONG_THREADS, 0, st_>>>(tab_, kp_, batch_words_.as<u64>(), batch_ofs_.as<u64>(),
                                                                                                           batch_lens_.as<u32>(), n, alignlen,
                                                                                                           n_groups_, hits_.as<u64>(), out_.as<MapHit>());
            else
                k_map_reads<NW><<<(unsigned)std::min<u64>((n + 127) / 128, (u64)n_sm_ * 16), 128, 0, st_>>>(tab_, kp_, batch_words_.as<u64>(), batch_ofs_.as<u64>(),
                                                                                                       batch_lens_.as<u32>(), n, alignlen,
                                                                                                       hits_.as<u64>(), out_.as<MapHit>());
            PG_CUDA(cudaGetLastError());
        }
        PG_CUDA(cudaEventRecord(ev_[1], st_));
        PG_CUDA(cudaMemcpyAsync(out, out_.p, n * sizeof(MapHit), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
        float ms;
        PG_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
        if (per_read_cta) {
            ms_long_ += ms;
            lookups_long_ += k;
        } else ms_scan_ += ms;
    }
    void times(MapTimes* t) const override { *t = MapTimes{ms_hash_, ms_decode_, ms_scan_, ms_long_, lookups_long_}; }

private:
    int K_, device_, n_sm_ = 0;
    // group slots of k_map_long; PGB200_MAP_GROUPS lowers it (1..MAP_GROUPS) so that a test can force the overflow rounds
    u32 n_groups_ = getenv("PGB200_MAP_GROUPS") ? (u32)std::min<long>(std::max<long>(1, atol(getenv("PGB200_MAP_GROUPS"))), (long)MAP_GROUPS) : MAP_GROUPS;
    KParams<NW> kp_;
    Stream st_;
    Event ev_[2];
    Pinned<u64> h_cnt_;
    DevBuf cnt_, tab_buf_, text_buf_, scan_buf_, line_buf_, read_words_, read_lens_, pack_ofs_, pack_scan_, pack_words_, batch_words_, batch_ofs_,
        batch_lens_, hits_, out_;
    Table<NW> tab_{nullptr, 0};
    FgetsReader reader_;
    double ms_hash_ = 0, ms_decode_ = 0, ms_scan_ = 0, ms_long_ = 0;
    u64 lookups_long_ = 0;
};

IMapEngine* make_map_engine(int K, int device) {
    if (K <= 63) return new MapEngineT<2>(K, device);
    return new MapEngineT<4>(K, device);
}

}   // namespace pgb
#pragma GCC visibility pop
