// skm.cu -- aggregated pass 1 (the default insert path, and the ONLY one across GPUs), the exchange: super-k-mer partition per chunk,
// run records scattered straight into the memory of the GPU that owns their bucket.  The aggregation of each bucket is skm_apply.cu,
// the region build of the table table_build.cu.  Logic shared with the host tests lives in skm.cuh.
//
//   feed_text(chunk):  k_skm_count    minimizers of every read -> runs, run count per bucket, runs kept in a side buffer
//                      device_scan    bucket counts -> offsets of the chunk's bucket-major record blob
//                      k_skm_publish  reserves room for the blob in every owner's arena (sender-private region: no coordination),
//                                     writes the segment descriptor and the owner's slice of the offsets INTO THE OWNER'S MEMORY
//                      k_skm_scatter  one lane per run: builds the self-contained records and stores each one at its final position
//                                     in its owner's arena: plain stores for the local GPU, NVLink peer stores (CUDA IPC / peer access mappings)
//                                     for the others.  Partition and "all-to-all" are the same kernel; no library collective, no
//                                     staging buffer, no second pass over the records.
// Replaces, for the same result, chopKmer4read + the owner filter + put_kmerset (prlHashReads.c:163-259, 79-90; newhash.c:473-528).
#include "engine_impl.cuh"
#include "skm.cuh"
#include "scan.cuh"

namespace pgb {

constexpr int SKM_PART_THREADS = 128;
constexpr int SKM_SIDE_RUNS = 16;

// ------------------------------------------------------------------------------------------------ partition: count
struct CountEmit {
    u32* cnt;
    u32* side;
    int nrun;
    __device__ __forceinline__ void operator()(u32 b, int, int n, bool last) {
        atomicAdd(&cnt[b], 1u);
        if (nrun < SKM_SIDE_RUNS) side[nrun] = skm_side_pack(b, n, last);
        nrun++;
    }
};

// One thread per read.  (The warp routine of k_skm_rescan, skm_warp_scan_read, makes the same runs but issues about three times the
// instructions per read at 150 bases: 27.6 against 9.6 ms per step on H100, DESIGN.md §5.)
__global__ void __launch_bounds__(SKM_PART_THREADS) k_skm_count(SkmGeom g, const u64* __restrict__ words, const u32* __restrict__ lens, u64 n_rec, int W64,
                                                               u32* cnt, u32* side, u8* nruns) {
    extern __shared__ u32 s_ring[];   // [g.w][blockDim.x]: one column per thread, bank = thread -> conflict-free
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < n_rec; r += (u64)gridDim.x * blockDim.x) {
        CountEmit e{cnt, side + r * SKM_SIDE_RUNS, 0};
        skm_scan_read(g, words + r * (u64)W64, (int)lens[r], s_ring + threadIdx.x, (int)blockDim.x, e);
        nruns[r] = e.nrun <= SKM_SIDE_RUNS ? (u8)e.nrun : (u8)255;
    }
}

// ------------------------------------------------------------------------------------------------ partition: publish + scatter
struct SkmSendArgs {
    u32 n_buckets;
    int world, rank;
    int own_shift;            // >= 0: owner(b) = b >> own_shift (power-of-two split), else the generic range search
    u32 seg_idx, max_seg, bo_stride;
    u64 cap_pair, epoch;
    const u32* segoff;        // [B] exclusive offsets of this chunk's blob (bucket-major), *total = record count
    const u64* total;
    u64* cursor;              // [world] records this GPU has already placed in owner o's region this epoch
    u64* dst_delta;           // [world] out: position of record i of bucket b = dst_delta[o] + segoff[b] + i   (mod 2^64)
    u32* dst_ok;              // [world] out: 0 = the blob does not fit owner o's region (error raised, records dropped)
    // this epoch's half of every owner's arena, as mapped into this process
    u32* peer_nseg[SKM_MAXW];
    SkmSegDesc* peer_ring[SKM_MAXW];
    u32* peer_segoff[SKM_MAXW];
    u64* peer_recs[SKM_MAXW];   // start of THIS sender's region in owner o's arena
    u64* counters;
};
// the exchange's device-side scratch (one per engine)
struct SkmScratch {
    u64 cursor[SKM_MAXW], dst_delta[SKM_MAXW];   // SkmSendArgs::cursor, dst_delta
    u32 dst_ok[SKM_MAXW];                        // SkmSendArgs::dst_ok
    u64 blob_total;                              // records of the chunk's blob (SkmSendArgs::total)
};
__device__ __forceinline__ int skm_owner(const SkmSendArgs& a, u32 b) {
    return a.own_shift >= 0 ? (int)(b >> a.own_shift) : skm_owner_of(a.n_buckets, a.world, b);
}
__device__ __forceinline__ u32 skm_segoff_at(const SkmSendArgs& a, u32 b) { return b < a.n_buckets ? a.segoff[b] : (u32)*a.total; }

__global__ void __launch_bounds__(256) k_skm_publish(SkmSendArgs a) {
    if (blockIdx.x == 0 && (int)threadIdx.x < a.world) {
        const int o = threadIdx.x;
        const u32 lo = skm_owner_lo(a.n_buckets, a.world, o), hi = o + 1 < a.world ? skm_owner_lo(a.n_buckets, a.world, o + 1) : a.n_buckets;
        const u32 first = skm_segoff_at(a, lo), n = skm_segoff_at(a, hi) - first;
        const u64 base = a.cursor[o];
        const bool fits = base + n <= a.cap_pair;
        if (!fits) atomicAdd(&a.counters[C_XERR], 1ull);
        a.dst_ok[o] = fits ? 1u : 0u;
        a.dst_delta[o] = base - (u64)first;
        if (fits) a.cursor[o] = base + n;
        SkmSegDesc d;
        d.rec_off = base;
        d.n_recs = fits ? n : 0u;
        d.pad = 0;
        a.peer_ring[o][(u64)a.rank * a.max_seg + a.seg_idx] = d;
        a.peer_nseg[o][a.rank] = a.seg_idx + 1;
        atomicMax((unsigned long long*)&a.counters[C_XUSED], (unsigned long long)(fits ? base + n : base));   // fullest region (host-side room checks)
        if (o == 0) {
            __threadfence();
            a.counters[C_XEPOCH] = a.epoch;
            atomicAdd((unsigned long long*)&a.counters[C_XSEGS], 1ull);
        }
    }
    // the owner's slice of the offsets, relative to the blob: entry (b - lo) for its buckets, plus the end entry
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < (u64)a.n_buckets + a.world; i += (u64)gridDim.x * blockDim.x) {
        int o;
        u32 b;
        if (i < a.n_buckets) { b = (u32)i; o = skm_owner(a, b); }
        else { o = (int)(i - a.n_buckets); b = o + 1 < a.world ? skm_owner_lo(a.n_buckets, a.world, o + 1) : a.n_buckets; }   // end entry of owner o
        const u32 lo = skm_owner_lo(a.n_buckets, a.world, o);
        const u32 first = skm_segoff_at(a, lo);
        a.peer_segoff[o][((u64)a.rank * a.max_seg + a.seg_idx) * a.bo_stride + (b - lo)] = skm_segoff_at(a, b) - first;
    }
}

template <int NW>
__device__ __forceinline__ void skm_store_rec(u64* dst, const SkmRec<NW>& r) {
    if (NW == 2) {
        st256(dst, r.w[0], r.w[1], r.w[2], r.w[3]);                       // 32-byte records are 32-byte aligned
    } else {
        // 48-byte records: 16-byte aligned only
#pragma unroll
        for (int p = 0; p < (NW + 2) / 2; p++) {
            uint4 v;
            v.x = (unsigned)r.w[2 * p]; v.y = (unsigned)(r.w[2 * p] >> 32);
            v.z = (unsigned)r.w[2 * p + 1]; v.w = (unsigned)(r.w[2 * p + 1] >> 32);
            reinterpret_cast<uint4*>(dst)[p] = v;
        }
    }
}
template <int NW>
__device__ __forceinline__ void skm_emit_rec(const SkmSendArgs& a, u32* cursor_b, int K, const u64* wp, int W64, u64 ordinal, u32 b, int start, int n, bool last) {
    const u32 i = atomicAdd(&cursor_b[b], 1u);
    const int o = skm_owner(a, b);
    if (!a.dst_ok[o]) return;
    const u64 idx = a.dst_delta[o] + (u64)a.segoff[b] + i;
    const SkmRec<NW> r = skm_make_rec<NW>(K, wp, W64, ordinal, start, n, last);
    skm_store_rec<NW>(a.peer_recs[o] + idx * (NW + 2), r);
}

// one lane per run: a warp takes two reads, a half-warp per read and one side-row entry per lane, so the side rows load coalesced and
// every run of the warp has its cursor atomic and its record store in flight at once.  A run starts where the runs before it in its
// row end (prefix over the half-warp).  The runs come from the side buffer: no minimizer work here.
template <int NW>
__global__ void __launch_bounds__(256) k_skm_scatter(SkmSendArgs a, int K, const u64* __restrict__ words, u64 n_rec, int W64, u64 ord_base, u64 ord_stride,
                                                     const u32* __restrict__ side, const u8* __restrict__ nruns, u32* cursor_b) {
    static_assert(SKM_SIDE_RUNS == 16, "a half-warp holds one side row");
    const int lane = threadIdx.x & 31, slot = lane & 15;
    const u64 n_pairs = (n_rec + 1) / 2;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 p = warp0; p < n_pairs; p += nwarps) {
        const u64 r = 2 * p + (lane >> 4);
        int nr = r < n_rec ? (int)nruns[r] : 0;
        if (nr == 255) nr = 0;   // more runs than the side row holds: k_skm_rescan
        const bool act = slot < nr;
        const u32 e = act ? __ldg(side + r * SKM_SIDE_RUNS + slot) : 0u;
        const int n = act ? skm_side_n(e) : 0;
        int inc = n;
#pragma unroll
        for (int d = 1; d < 16; d <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, d, 16);
            if (slot >= d) inc += v;
        }
        if (act) skm_emit_rec<NW>(a, cursor_b, K, words + r * (u64)W64, W64, ord_base + r * ord_stride, skm_side_bucket(e), inc - n, n, skm_side_last(e));
    }
}

// reads with more than SKM_SIDE_RUNS runs (rare): full re-scan of just those reads
template <int NW>
struct RescanEmit {
    const SkmSendArgs& a;
    u32* cursor_b;
    int K;
    const u64* wp;
    int W64;
    u64 ordinal;
    __device__ __forceinline__ void operator()(u32 b, int s, int n, bool last, int) const { skm_emit_rec<NW>(a, cursor_b, K, wp, W64, ordinal, b, s, n, last); }
};
// the lanes of a warp check 32 reads at a time; the warp re-scans each flagged one (skm_warp_scan_read)
template <int NW>
__global__ void __launch_bounds__(SKM_PART_THREADS) k_skm_rescan(SkmSendArgs a, SkmGeom g, const u64* __restrict__ words, const u32* __restrict__ lens, u64 n_rec,
                                                                int W64, u64 ord_base, u64 ord_stride, const u8* __restrict__ nruns, u32* cursor_b) {
    __shared__ u32 s_ring[SKM_PART_THREADS / 32][SKM_WARP_RING];
    const int lane = threadIdx.x & 31;
    const u64 warp0 = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 r0 = warp0 * 32; r0 < n_rec; r0 += nwarps * 32) {
        unsigned todo = __ballot_sync(0xffffffffu, r0 + lane < n_rec && nruns[r0 + lane] == 255);
        while (todo) {
            const u64 r = r0 + (__ffs(todo) - 1);
            todo &= todo - 1;
            const u64* wp = words + r * (u64)W64;
            const RescanEmit<NW> e{a, cursor_b, g.K, wp, W64, ord_base + r * ord_stride};
            skm_warp_scan_read(g, wp, W64, (int)lens[r], s_ring[threadIdx.x >> 5], e);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
template <int NW>
void EngineT<NW>::skm_init() {
    if (skm_geom_.n_buckets) return;
    const int world = prm_.world > 1 ? prm_.world : 1;
    if (world > SKM_MAXW) throw std::runtime_error("pgb200: at most 16 GPUs");
    u64 est = 0;   // expected number of distinct k-mers on THIS GPU
    if (prm_.table_slots) est = prm_.table_slots / 2;
    else if (prm_.initG) est = (u64)((double)prm_.P * (double)ref_static_set_size(prm_.initG, prm_.P, prm_.flavour127 != 0) * 0.77) / world;
    u64 Bo = est ? next_pow2((est + SKM_SLOTS / 2 - 1) / (SKM_SLOTS / 2)) : (1ull << 16);   // half a shared-memory table per bucket on average
    if (Bo < 1024) Bo = 1024;
    u64 B = Bo * world;
    if (const char* e = getenv("PGB200_SKM_BUCKETS")) B = strtoull(e, nullptr, 0);
    if (B < (u64)world) B = world;
    if (B > (1ull << SKM_MAX_BUCKET_BITS)) B = 1ull << SKM_MAX_BUCKET_BITS;   // the side buffer packs the bucket in 26 bits
    skm_geom_ = make_skm_geom(prm_.K, (u32)B);
    skm_own_lo_ = skm_owner_lo((u32)B, world, prm_.rank);
    skm_own_hi_ = prm_.rank + 1 < world ? skm_owner_lo((u32)B, world, prm_.rank + 1) : (u32)B;
    skm_own_shift_ = -1;
    if ((B & (B - 1)) == 0 && (world & (world - 1)) == 0 && B >= (u64)world) {
        int s = 0;
        while (((u64)world << s) < B) s++;
        skm_own_shift_ = s;
    }
    skm_cnt_.alloc((B + 1) * sizeof(u32));
    skm_segoff_.alloc((B + 1) * sizeof(u32));
    skm_cursor_.alloc((B + 1) * sizeof(u32));
    skm_scan_.alloc(scan_scratch_elems(B) * sizeof(u64) + 256);
    skm_scratch_.alloc(sizeof(SkmScratch));
    PG_CUDA(cudaMemsetAsync(skm_scratch_.p, 0, sizeof(SkmScratch), st_));
    for (DevBuf& d : skm_deferred_) d.alloc((size_t)(skm_own_hi_ - skm_own_lo_ + 1) * sizeof(u32));
    if (skm_geom_.w > SKM_RING_TILES * 32 - 63) throw std::runtime_error("pgb200: minimizer window too long for the partition kernels");
    skm_part_threads_ = SKM_PART_THREADS;
    while ((size_t)skm_part_threads_ * skm_geom_.w * sizeof(u32) > 160 * 1024 && skm_part_threads_ > 32) skm_part_threads_ /= 2;
    const size_t ring = (size_t)skm_part_threads_ * skm_geom_.w * sizeof(u32);
    if (ring > 48 * 1024) PG_CUDA(cudaFuncSetAttribute(k_skm_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring));
    if (prm_.verbose) fprintf(stderr, "[pgb200] aggregated pass 1: %u buckets (%u owned by GPU %d of %d), minimizer length %d, window %d\n", skm_geom_.n_buckets,
                              skm_own_hi_ - skm_own_lo_, prm_.rank, world, skm_geom_.m, skm_geom_.w);
}

// ---- the exchange arena
template <int NW>
void EngineT<NW>::xchg_setup(uint64_t cap_records) {
    skm_init();
    const int world = prm_.world > 1 ? prm_.world : 1;
    if (xa_buf_.p) throw std::runtime_error("pgb200: exchange arena already set up");
    if (!cap_records) {   // default: a fifth of the free HBM, at most 32 GB, split into the two epoch halves
        create_table_if_needed();
        size_t free_b = 0, total_b = 0;
        PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
        u64 bytes = std::min<u64>((u64)free_b / 5, 32ull << 30);
        if (const char* e = getenv("PGB200_SKM_ARENA_MB")) bytes = strtoull(e, nullptr, 0) << 20;
        cap_records = bytes / ((NW + 2) * sizeof(u64)) / 2;
    }
    u64 cap_pair = cap_records / world;
    if (cap_pair < 4096) cap_pair = 4096;
    u32 max_seg = (u32)(SKM_MAX_SEGS / world);   // an aggregation launch reads at most SKM_MAX_SEGS segments over all senders
    if (const char* e = getenv("PGB200_SKM_MAX_SEG")) max_seg = (u32)atoi(e);
    if (max_seg < 1) max_seg = 1;
    if (max_seg > (u32)SKM_MAX_SEGS) max_seg = SKM_MAX_SEGS;
    xa_geom_ = make_skm_arena_geom(world, skm_geom_.n_buckets, max_seg, cap_pair, NW + 2);
    xa_buf_.alloc(xa_geom_.half_bytes * SKM_ARENA_HALVES);   // an epoch is aggregated (asynchronously) while the next one is being delivered
    for (int h = 0; h < SKM_ARENA_HALVES; h++)
        PG_CUDA(cudaMemsetAsync(skm_arena_half(xa_geom_, xa_buf_.p, h).nseg, 0, xa_geom_.off_recs - xa_geom_.off_nseg, st_));   // nseg, ring, offsets
    sync();
    xa_peer_.assign(world, nullptr);
    xa_peer_[prm_.rank] = xa_buf_.p;
    xa_send_epoch_ = 0;
    xa_seg_idx_ = 0;
    xa_flushed_epoch_ = 0;
    xa_reads_cum_.assign(1, 0);
    if (prm_.verbose) fprintf(stderr, "[pgb200] exchange arena: %d x %.2f GB (%llu records per sender, %u segments per sender and epoch)\n", SKM_ARENA_HALVES,
                              xa_geom_.half_bytes / 1e9, (unsigned long long)cap_pair, max_seg);
}
template <int NW>
void EngineT<NW>::xchg_export(void* handle64) {
    if (!xa_buf_.p) throw std::runtime_error("pgb200: xchg_export before xchg_setup");
    cudaIpcMemHandle_t h;
    PG_CUDA(cudaIpcGetMemHandle(&h, xa_buf_.p));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle64, &h, 64);
}
template <int NW>
void EngineT<NW>::xchg_import(int peer, const void* handle64) {
    if (peer < 0 || peer >= (int)xa_peer_.size() || peer == prm_.rank) throw std::runtime_error("pgb200: xchg_import: bad peer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    void* p = nullptr;
    PG_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    xa_peer_[peer] = p;
    xa_ipc_opened_.emplace_back(p);
}
template <int NW>
void EngineT<NW>::xchg_import_ptr(int peer, int peer_device, void* base) {
    if (peer < 0 || peer >= (int)xa_peer_.size() || peer == prm_.rank) throw std::runtime_error("pgb200: xchg_import_ptr: bad peer");
    PG_CUDA(cudaSetDevice(prm_.device));
    int can = 0;
    PG_CUDA(cudaDeviceCanAccessPeer(&can, prm_.device, peer_device));
    if (!can) throw std::runtime_error("pgb200: GPUs cannot access each other's memory (no peer access)");
    cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) PG_CUDA(e);
    cudaGetLastError();
    xa_peer_[peer] = base;
}
template <int NW>
void* EngineT<NW>::xchg_base() { return xa_buf_.p; }

template <int NW>
void EngineT<NW>::xchg_default_setup() {
    if (xa_buf_.p) return;
    if (prm_.world > 1) throw std::runtime_error("pgb200: multi-GPU engines need pgb200_xchg_setup + xchg_import before the first chunk");
    xchg_setup(0);
}

// Upper estimate of the fullest arena region's fill once a chunk of n_rec more reads has been partitioned.  What the host knows
// (C_XUSED after C_XSEGS segments of epoch C_XEPOCH) lags behind the stream; the chunks it does not know yet are assumed to make
// twice the records per read seen so far in this epoch -- before anything has been seen: four times a run every w/4 k-mers, runs being
// about w/3 long on random sequence -- and never more than one record per k-mer.  An estimate that turns out too low is caught on the
// device: k_skm_publish refuses the blob and raises C_XERR (an error, not a wrong result).
template <int NW>
u64 EngineT<NW>::skm_room_estimate(u64 n_rec) {
    const u64 per_read_worst = (u64)std::max(1, prm_.max_rd_len - prm_.K + 1);
    const bool current = h_cnt_[C_XEPOCH] == xa_send_epoch_ + 1;
    u64 segs_done = current ? h_cnt_[C_XSEGS] : 0, used = current ? h_cnt_[C_XUSED] : 0;
    if (xa_reads_cum_.empty()) xa_reads_cum_.push_back(0);
    if (segs_done >= xa_reads_cum_.size()) segs_done = xa_reads_cum_.size() - 1;
    const u64 reads_done = xa_reads_cum_[segs_done], reads_fed = xa_reads_cum_.back();
    u64 per_read = 4 * (per_read_worst / (u64)std::max(1, skm_geom_.w / 4) + 1);
    if (reads_done) per_read = std::max<u64>(1, (2 * used * (u64)xa_geom_.world + reads_done - 1) / reads_done);   // `used` is ONE region's fill
    per_read = std::min(per_read, per_read_worst);
    return used + ((reads_fed - reads_done + n_rec) * per_read + xa_geom_.world - 1) / xa_geom_.world;
}

// Room for the next chunk's records and segment (called OUTSIDE the caller's per-chunk event bracket: an aggregation times itself).
// Single GPU: decided here; the aggregation launch is asynchronous (it is ordered behind the scatter kernels by the stream, and
// the next chunks go to the other arena half).  Several GPUs: the caller fences + flushes all GPUs collectively (pgb200_xchg_room).
template <int NW>
void EngineT<NW>::skm_make_room(u64 n_rec, bool host_text) {
    skm_init();
    xchg_default_setup();
    if (xa_geom_.world == 1) {
        // Host text arrives at PCIe speed and leaves the GPU idle most of the time: whenever the insert stream has drained and at least
        // two chunks are waiting, they are aggregated right away, so that only the last couple of chunks remain for pgb200_finish_pass1.
        // Device-resident text is fed faster than it is partitioned: the stream never drains and everything is aggregated once, unless
        // the arena really fills up.
        // PGB200_SKM_FLUSH_EVERY=n forces a fixed cadence (0: only when the arena is full).
        bool early = false;
        if (skm_flush_every_ > 0) early = xa_seg_idx_ >= (u32)skm_flush_every_;
        else if (skm_flush_every_ < 0 && host_text && xa_seg_idx_ >= 2) {
            early = cudaStreamQuery(st_) == cudaSuccess;
            if (!early) cudaGetLastError();   // cudaErrorNotReady is not an error; do not leave it for the next launch check
        }
        bool full = xa_seg_idx_ >= xa_geom_.max_seg || skm_room_estimate(n_rec) > xa_geom_.cap_pair;
        if (full && !early && xa_seg_idx_ < xa_geom_.max_seg && !(h_cnt_[C_XEPOCH] == xa_send_epoch_ + 1 && h_cnt_[C_XSEGS] >= xa_seg_idx_)) {
            // The estimate ran on counters that lag the partition stream (at worst on the first-chunk guess, several times the records
            // a read really makes).  A flush costs a pass over every owned bucket and a merge per distinct k-mer per flush, so wait for
            // the chunks already queued (this chunk's decode keeps running on its own stream) and decide on what they really made.
            read_counters_on(st_);
            full = skm_room_estimate(n_rec) > xa_geom_.cap_pair;
        }
        if ((full || early) && xa_seg_idx_ > 0) {
            skm_close_epoch(false);
            skm_flush();
        }
    } else if (xa_seg_idx_ >= xa_geom_.max_seg) {
        throw std::runtime_error("pgb200: too many chunks in one exchange epoch: call pgb200_xchg_fence + pgb200_flush (on all GPUs) more often");
    }
}

// several GPUs: the coordinator asks before it feeds the next chunk
template <int NW>
bool EngineT<NW>::xchg_room(uint64_t n_rec) {
    if (!xa_buf_.p) return true;
    return xa_seg_idx_ < xa_geom_.max_seg && skm_room_estimate(n_rec) <= xa_geom_.cap_pair;
}

// partition the chunk just decoded and deliver its records (inside the caller's "insert" event bracket)
template <int NW>
void EngineT<NW>::skm_feed_chunk(size_t ci) {
    const ReadChunk& ch = chunks_[ci];
    const u32 B = skm_geom_.n_buckets;
    const int world = xa_geom_.world;
    PG_CUDA(cudaMemsetAsync(skm_cnt_.p, 0, (B + 1) * sizeof(u32), st_));
    PG_CUDA(cudaMemsetAsync(skm_cursor_.p, 0, (B + 1) * sizeof(u32), st_));
    constexpr int part_warps = SKM_PART_THREADS / 32;
    skm_side_.ensure(ch.n_rec * (SKM_SIDE_RUNS * sizeof(u32) + 1) + 256);
    u32* side = skm_side_.template as<u32>();
    u8* nruns = reinterpret_cast<u8*>(side + ch.n_rec * SKM_SIDE_RUNS);
    const size_t ring = (size_t)skm_part_threads_ * skm_geom_.w * sizeof(u32);
    k_skm_count<<<(unsigned)std::min<u64>((ch.n_rec + skm_part_threads_ - 1) / skm_part_threads_, (u64)n_sm_ * 16), skm_part_threads_, ring, st_>>>(skm_geom_, ch.words, ch.len, ch.n_rec, W64_, skm_cnt_.template as<u32>(), side, nruns);
    PG_CUDA(cudaGetLastError());
    SkmScratch* sc = skm_scratch_.template as<SkmScratch>();
    device_scan(ScanU32In{skm_cnt_.template as<u32>()}, ScanU32Out{skm_segoff_.template as<u32>()}, (u64)B, skm_scan_.template as<u64>(),
                &sc->blob_total, st_);
    SkmSendArgs a;
    a.n_buckets = B;
    a.world = world;
    a.rank = prm_.rank;
    a.own_shift = skm_own_shift_;
    a.seg_idx = xa_seg_idx_;
    a.epoch = xa_send_epoch_ + 1;   // 0 = nothing published yet
    a.max_seg = xa_geom_.max_seg;
    a.bo_stride = xa_geom_.bo_max + 1;
    a.cap_pair = xa_geom_.cap_pair;
    a.segoff = skm_segoff_.template as<u32>();
    a.total = &sc->blob_total;
    a.cursor = sc->cursor;
    a.dst_delta = sc->dst_delta;
    a.dst_ok = sc->dst_ok;
    const int half = (int)(xa_send_epoch_ % SKM_ARENA_HALVES);
    for (int o = 0; o < world; o++) {
        if (!xa_peer_[o]) throw std::runtime_error("pgb200: exchange peer not imported");
        const SkmArenaHalf h = skm_arena_half(xa_geom_, xa_peer_[o], half);
        a.peer_nseg[o] = h.nseg;
        a.peer_ring[o] = h.ring;
        a.peer_segoff[o] = h.segoff;
        a.peer_recs[o] = h.recs + (u64)prm_.rank * xa_geom_.cap_pair * (NW + 2);
    }
    a.counters = d_cnt_;
    k_skm_publish<<<(unsigned)std::min<u64>(((u64)B + world + 255) / 256, (u64)n_sm_ * 8), 256, 0, st_>>>(a);
    PG_CUDA(cudaGetLastError());
    u32* cursor_b = skm_cursor_.template as<u32>();
    k_skm_scatter<NW><<<(unsigned)std::min<u64>((ch.n_rec + 15) / 16, (u64)n_sm_ * 16), 256, 0, st_>>>(a, prm_.K, ch.words, ch.n_rec, W64_, ch.ord_base, ch.ord_stride, side, nruns, cursor_b);
    PG_CUDA(cudaGetLastError());
    k_skm_rescan<NW><<<(unsigned)std::min<u64>((ch.n_rec + 32 * part_warps - 1) / (32 * part_warps), (u64)n_sm_ * 16), SKM_PART_THREADS, 0, st_>>>(a, skm_geom_, ch.words, ch.len, ch.n_rec, W64_, ch.ord_base, ch.ord_stride, nruns, cursor_b);
    PG_CUDA(cudaGetLastError());
    if (xa_reads_cum_.empty()) xa_reads_cum_.push_back(0);
    xa_reads_cum_.push_back(xa_reads_cum_.back() + ch.n_rec);
    xa_seg_idx_++;
    xa_dirty_ = true;
    p1_.launches += 7;
}

// Close the current exchange epoch: the chunks fed from now on go to the other arena half.
//   hard (pgb200_xchg_fence; several GPUs: before the caller's barrier): waits until every record this GPU produced has reached its
//        owner, books the chunk timings, raises decode / arena errors;
//   soft (single GPU, mid-stream): nothing to wait for -- the aggregation launch is stream-ordered behind the scatter kernels.
// Either way the previous aggregation (it read the half that is about to be written again) is completed first.
template <int NW>
void EngineT<NW>::skm_close_epoch(bool hard) {
    if (hard) {
        settle_timing();
        read_counters();
        check_format_counter();
        if (h_cnt_[C_XERR])
            throw std::runtime_error("pgb200: exchange arena overflow (records of a chunk did not fit their owner's region, or too many segments): "
                                     "raise the arena capacity (pgb200_xchg_setup / PGB200_SKM_ARENA_MB) or flush more often");
    }
    if (!xa_buf_.p) return;
    skm_flush_complete();
    if (xa_dirty_ || prm_.world > 1) {
        xa_send_epoch_++;
        xa_seg_idx_ = 0;
        xa_reads_cum_.assign(1, 0);
        xa_dirty_ = false;
        PG_CUDA(cudaMemsetAsync(skm_scratch_.template as<SkmScratch>()->cursor, 0, sizeof(SkmScratch::cursor), st_));
        PG_CUDA(cudaMemsetAsync(d_cnt_ + C_XUSED, 0, sizeof(u64), st_));
        PG_CUDA(cudaMemsetAsync(d_cnt_ + C_XSEGS, 0, sizeof(u64), st_));
    }
}
template <int NW>
void EngineT<NW>::skm_fence() { skm_close_epoch(true); }

template <int NW>
void EngineT<NW>::skm_reset() {
    // single GPU: nothing of the arena survives a reset; several GPUs: the epochs keep alternating (peers may already deliver)
    if (!xa_buf_.p) return;
    sync();
    skm_flush_complete();
    if (prm_.world <= 1 && (xa_dirty_ || xa_flushed_epoch_ != xa_send_epoch_)) {
        skm_close_epoch(false);
        for (int h = 0; h < SKM_ARENA_HALVES; h++)
            PG_CUDA(cudaMemsetAsync(skm_arena_half(xa_geom_, xa_buf_.p, h).nseg, 0, sizeof(u32), st_));
        xa_flushed_epoch_ = xa_send_epoch_;
    }
}

#define PGB_INST(NW)                                                         \
    template void EngineT<NW>::skm_init();                                   \
    template void EngineT<NW>::xchg_setup(uint64_t);                         \
    template void EngineT<NW>::xchg_export(void*);                           \
    template void EngineT<NW>::xchg_import(int, const void*);                \
    template void EngineT<NW>::xchg_import_ptr(int, int, void*);             \
    template void* EngineT<NW>::xchg_base();                                 \
    template void EngineT<NW>::xchg_default_setup();                         \
    template void EngineT<NW>::skm_feed_chunk(size_t);                       \
    template void EngineT<NW>::skm_make_room(u64, bool);                     \
    template bool EngineT<NW>::xchg_room(uint64_t);                          \
    template void EngineT<NW>::skm_fence();                                  \
    template void EngineT<NW>::skm_close_epoch(bool);                        \
    template u64 EngineT<NW>::skm_room_estimate(u64);                        \
    template void EngineT<NW>::skm_reset();
PGB_INST(2)
PGB_INST(4)

}   // namespace pgb
