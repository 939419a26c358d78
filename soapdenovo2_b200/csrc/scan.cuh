// scan.cuh -- device-wide exclusive prefix sum with fused input/output functors (hand-written, no CUB).
//
// Used for: newline -> line index (decode.cu), occupancy -> position in reference iteration order (layout.cu),
// per-edge text lengths / edge ids (edges.cu), per-read record offsets (pass2.cu).
// Three launches per level: tile sums -> (recursive) scan of the tile sums -> rescan tiles with their base.
// A tile is SCAN_THREADS x SCAN_ITEMS consecutive elements; thread t owns items [t*ITEMS, (t+1)*ITEMS) so a tile needs one
// block-wide scan (the per-thread runs are contiguous 256 B pieces for 16-byte elements: sector-efficient streaming).
#pragma once
#include "kmer.cuh"
#include <cuda_runtime.h>

namespace pgb {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// block-wide exclusive scan of one value per thread; returns exclusive prefix, *total = block sum
__device__ __forceinline__ u64 block_exclusive_scan(u64 v, u64* total) {
    __shared__ u64 warp_sums[SCAN_THREADS / 32];
    __shared__ u64 block_total;
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    u64 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        u64 n = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += n;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        u64 ws = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
        u64 wi = ws;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            u64 n = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += n;
        }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = wi - ws;
        if (lane == SCAN_THREADS / 32 - 1) block_total = wi;
    }
    __syncthreads();
    u64 r = warp_sums[wid] + inc - v;
    *total = block_total;
    __syncthreads();
    return r;
}

// Each thread owns SCAN_ITEMS CONSECUTIVE elements of the tile (one block-wide scan per tile instead of one per strip).
template <class In>
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tile_sums(In in, u64 n, u64* sums) {
    u64 first = (u64)blockIdx.x * SCAN_TILE + (u64)threadIdx.x * SCAN_ITEMS;
    u64 acc = 0;
#pragma unroll 4
    for (int s = 0; s < SCAN_ITEMS; s++) {
        u64 i = first + s;
        if (i < n) acc += in(i);
    }
    u64 tot;
    block_exclusive_scan(acc, &tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

template <class In, class Out>
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_apply(In in, Out out, u64 n, const u64* tile_base) {
    u64 first = (u64)blockIdx.x * SCAN_TILE + (u64)threadIdx.x * SCAN_ITEMS;
    u64 v[SCAN_ITEMS];
    u64 acc = 0;
#pragma unroll
    for (int s = 0; s < SCAN_ITEMS; s++) {
        u64 i = first + s;
        u64 x = i < n ? in(i) : 0;
        v[s] = x;
        acc += x;
    }
    u64 tot;
    u64 running = tile_base[blockIdx.x] + block_exclusive_scan(acc, &tot);
#pragma unroll
    for (int s = 0; s < SCAN_ITEMS; s++) {
        u64 i = first + s;
        if (i < n) out(i, running, v[s]);
        running += v[s];
    }
}

// single-block in-place exclusive scan of a small u64 array (the tile sums)
static __global__ void __launch_bounds__(SCAN_THREADS) k_scan_small(u64* a, u64 n, u64* total_out) {
    u64 running = 0;
    for (u64 b = 0; b < n; b += SCAN_THREADS) {
        u64 i = b + threadIdx.x;
        u64 v = i < n ? a[i] : 0, tot;
        u64 ex = block_exclusive_scan(v, &tot);
        if (i < n) a[i] = running + ex;
        running += tot;
    }
    if (threadIdx.x == 0 && total_out) *total_out = running;
}

struct ScanU64In {
    const u64* a;
    __device__ u64 operator()(u64 i) const { return a[i]; }
};
struct ScanU64Out {
    u64* a;
    __device__ void operator()(u64 i, u64 prefix, u64) const { a[i] = prefix; }
};

// scratch: caller-provided device buffer of at least scan_scratch_elems(n) u64.
static inline u64 scan_scratch_elems(u64 n) {
    u64 t1 = n / SCAN_TILE + 2, t2 = t1 / SCAN_TILE + 2;
    return t1 + t2 + 8;
}

// Exclusive scan of in(i), i in [0,n); out(i, prefix, value) is called for every i; *d_total (device) gets the sum.
template <class In, class Out>
void device_scan(In in, Out out, u64 n, u64* scratch, u64* d_total, cudaStream_t st) {
    if (n == 0) { cudaMemsetAsync(d_total, 0, sizeof(u64), st); return; }
    u64 tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    u64* sums = scratch;
    k_scan_tile_sums<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(in, n, sums);
    if (tiles <= (u64)SCAN_TILE * 64) {
        k_scan_small<<<1, SCAN_THREADS, 0, st>>>(sums, tiles, d_total);
    } else {
        // second level: more than 4096 x 262144 elements.  The layout scans the reference's set geometry, which -a sizes from the
        // memory the user names, so any -a large enough reaches it (-p 8 -a 21 in the 63-mer build)
        u64* sums2 = scratch + tiles + 1;
        device_scan(ScanU64In{sums}, ScanU64Out{sums}, tiles, sums2, d_total, st);
    }
    k_scan_apply<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(in, out, n, sums);
}

// Split form for the case "total first, then (after the caller has sized its outputs) the prefixes": phase 1 leaves the scanned
// tile bases in `scratch`, phase 2 reuses them -- the input is read twice in total instead of four times.
template <class In>
void device_scan_total(In in, u64 n, u64* scratch, u64* d_total, cudaStream_t st) {
    if (n == 0) { cudaMemsetAsync(d_total, 0, sizeof(u64), st); return; }
    u64 tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    k_scan_tile_sums<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(in, n, scratch);
    if (tiles <= (u64)SCAN_TILE * 64) k_scan_small<<<1, SCAN_THREADS, 0, st>>>(scratch, tiles, d_total);
    else device_scan(ScanU64In{scratch}, ScanU64Out{scratch}, tiles, scratch + tiles + 1, d_total, st);
}
template <class In, class Out>
void device_scan_finish(In in, Out out, u64 n, const u64* scratch, cudaStream_t st) {
    if (n == 0) return;
    u64 tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    k_scan_apply<<<(unsigned)tiles, SCAN_THREADS, 0, st>>>(in, out, n, scratch);
}

}   // namespace pgb
