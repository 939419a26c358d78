// GPU harness for device_scan (scan.cuh): every input is a function of the index alone, so scans of more than 2^32 elements need no
// input memory, and every output is checked on the device against the input's closed-form prefix.  Prints one line per scan:
//   scan <input> <entry> <n> <tiles> <bad> <first_bad> <visits> <total> <want_total> <canary_ok>
// tests/test_gpu_scan.py runs it once and asserts on the numbers.
#include "../soapdenovo2_b200/csrc/scan.cuh"
#include <cstdio>
#include <cstdlib>
#include <vector>
using namespace pgb;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(2); } } while (0)

struct Ones {
    __device__ u64 operator()(u64) const { return 1; }
    __device__ u64 prefix(u64 i) const { return i; }
};
struct Mod7 {
    __device__ u64 operator()(u64 i) const { return i % 7; }
    __device__ u64 prefix(u64 i) const { const u64 r = i % 7; return 21 * (i / 7) + r * (r - 1) / 2; }
};
struct Zeros {
    __device__ u64 operator()(u64) const { return 0; }
    __device__ u64 prefix(u64) const { return 0; }
};
// Occupancy-like sparse input: 1 where a hash of (i mod PER) falls below a threshold (about 60 % of the slots, in irregular runs).
// PER is not a multiple of the tile, so tile sums differ from tile to tile; pre[] (host-built) gives the prefix within one period.
constexpr u64 PER = 40961;
constexpr u64 THR = 0x9999999999999999ull;
struct Sparse {
    const u32* pre;   // [PER + 1]
    __device__ u64 operator()(u64 i) const { return mix64(i % PER) < THR ? 1 : 0; }
    __device__ u64 prefix(u64 i) const { return (i / PER) * pre[PER] + pre[i % PER]; }
};

struct Counters { u64 bad, first, visits[64]; };

template <class F>
struct Check {
    F f;
    Counters* c;
    __device__ void operator()(u64 i, u64 prefix, u64 v) const {
        if (prefix != f.prefix(i) || v != f(i)) { atomicAdd(&c->bad, 1ull); atomicMin(&c->first, i); }
        const unsigned m = __activemask();   // one count per warp and call: every index must be visited exactly once
        if ((threadIdx.x & 31) == (unsigned)(__ffs(m) - 1)) atomicAdd(&c->visits[blockIdx.x & 63], (u64)__popc(m));
    }
};

constexpr u64 CANARY = 4096;
constexpr unsigned char CANARY_BYTE = 0xA5;

template <class F>
static void one(const char* name, F f, u64 want_total, u64 n, bool split, Counters* d_c, u64* d_total) {
    const u64 elems = scan_scratch_elems(n);
    u64* scratch;
    CK(cudaMalloc(&scratch, (elems + CANARY) * sizeof(u64)));
    CK(cudaMemset(scratch, 0x3C, elems * sizeof(u64)));
    CK(cudaMemset(scratch + elems, CANARY_BYTE, CANARY * sizeof(u64)));
    Counters h0{};
    h0.first = ~0ull;
    CK(cudaMemcpy(d_c, &h0, sizeof(Counters), cudaMemcpyHostToDevice));
    CK(cudaMemset(d_total, 0x5A, sizeof(u64)));   // garbage: the scan must overwrite it, also for n = 0
    const Check<F> out{f, d_c};
    if (split) {
        device_scan_total(f, n, scratch, d_total, 0);
        device_scan_finish(f, out, n, scratch, 0);
    } else {
        device_scan(f, out, n, scratch, d_total, 0);
    }
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    Counters h;
    u64 total;
    CK(cudaMemcpy(&h, d_c, sizeof(Counters), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&total, d_total, sizeof(u64), cudaMemcpyDeviceToHost));
    std::vector<unsigned char> can(CANARY * sizeof(u64));
    CK(cudaMemcpy(can.data(), scratch + elems, can.size(), cudaMemcpyDeviceToHost));
    bool canary_ok = true;
    for (unsigned char b : can) canary_ok &= b == CANARY_BYTE;
    CK(cudaFree(scratch));
    u64 visits = 0;
    for (u64 v : h.visits) visits += v;
    printf("scan %s %s %llu %llu %llu %lld %llu %llu %llu %d\n", name, split ? "split" : "whole", (unsigned long long)n,
           (unsigned long long)((n + SCAN_TILE - 1) / SCAN_TILE), (unsigned long long)h.bad, h.first == ~0ull ? -1ll : (long long)h.first,
           (unsigned long long)visits, (unsigned long long)total, (unsigned long long)want_total, canary_ok ? 1 : 0);
    fflush(stdout);
}

int main() {
    std::vector<u32> pre(PER + 1, 0);
    for (u64 i = 0; i < PER; i++) pre[i + 1] = pre[i] + (mix64(i) < THR ? 1u : 0u);
    u32* d_pre;
    CK(cudaMalloc(&d_pre, pre.size() * sizeof(u32)));
    CK(cudaMemcpy(d_pre, pre.data(), pre.size() * sizeof(u32), cudaMemcpyHostToDevice));
    Counters* d_c;
    u64* d_total;
    CK(cudaMalloc(&d_c, sizeof(Counters)));
    CK(cudaMalloc(&d_total, sizeof(u64)));

    const u64 one_level = (u64)SCAN_TILE * SCAN_TILE * 64;   // the largest input whose tile sums fit one k_scan_small
    const u64 sizes[] = {0, 1, 15, 16, 17, 4095, 4096, 4097, one_level - 1, one_level, one_level + 1, (1ull << 32) - 1, (1ull << 32) + 4097};
    for (u64 n : sizes) {
        const u64 r7 = n % 7;
        const u64 sp = (n / PER) * pre[PER] + pre[n % PER];
        for (int split = 0; split < 2; split++) {
            one("ones", Ones{}, n, n, split, d_c, d_total);
            one("mod7", Mod7{}, 21 * (n / 7) + r7 * (r7 - 1) / 2, n, split, d_c, d_total);
            one("zeros", Zeros{}, 0, n, split, d_c, d_total);
            one("sparse", Sparse{d_pre}, sp, n, split, d_c, d_total);
        }
    }
    CK(cudaFree(d_pre));
    CK(cudaFree(d_c));
    CK(cudaFree(d_total));
    return 0;
}
