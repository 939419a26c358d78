// GPU check of the warp partition of the aggregated pass 1 (skm_warp_scan_read, soapdenovo2_b200/csrc/skm.cuh) against its host
// definition skm_scan_read, compiled for sm_90a by tests/test_skm_warp.py.  For every odd K from 13 to 127 and n_buckets 1, 2, 3 and
// 65536 (few buckets: the forced cuts every SKM_MAX_RUN k-mers dominate), reads of every length class -- shorter than K+1, K+1, at and
// around multiples of 32, hundreds of bases (far more than SKM_SIDE_RUNS runs) -- with random bases, homopolymers and low-complexity
// repeats: every run (bucket, start, length, last, order) and the run count must be the same.
#include "../soapdenovo2_b200/csrc/skm.cuh"
#include <cstdio>
#include <cstring>
#include <vector>
using namespace pgb;

constexpr int MAXL = 700;
constexpr int W64 = (MAXL + 31) / 32;

struct Run {
    u32 b;
    int start, n, last;
};

struct DevEmit {
    Run* out;
    __device__ void operator()(u32 b, int s, int n, bool last, int idx) const { out[idx] = Run{b, s, n, last ? 1 : 0}; }
};

__global__ void k_warp_runs(SkmGeom g, const u64* words, const int* lens, int n_reads, Run* runs, int* nruns) {
    __shared__ u32 s_ring[4][SKM_WARP_RING];
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int r = warp; r < n_reads; r += nwarps) {
        const DevEmit e{runs + (size_t)r * MAXL};
        const int n = skm_warp_scan_read(g, words + (size_t)r * W64, W64, lens[r], s_ring[threadIdx.x >> 5], e);
        if ((threadIdx.x & 31) == 0) nruns[r] = n;
    }
}

struct HostEmit {
    std::vector<Run>* v;
    void operator()(u32 b, int s, int n, bool last) { v->push_back(Run{b, s, n, last ? 1 : 0}); }
};

static u64 rng_state = 0x9E3779B97F4A7C15ull;
static u64 rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); return 2; } } while (0)

int main() {
    std::vector<int> lens_all;
    std::vector<u64> words_all;
    long total_err = 0;
    u64* d_words = nullptr;
    int *d_lens = nullptr, *d_nruns = nullptr;
    Run* d_runs = nullptr;
    const int max_reads = 4096;
    CK(cudaMalloc(&d_words, sizeof(u64) * W64 * max_reads));
    CK(cudaMalloc(&d_lens, sizeof(int) * max_reads));
    CK(cudaMalloc(&d_nruns, sizeof(int) * max_reads));
    CK(cudaMalloc(&d_runs, sizeof(Run) * (size_t)MAXL * max_reads));
    for (int K = 13; K <= 127; K += 2) {
        // read lengths: below K+1, K+1, around multiples of 32, long
        std::vector<int> Ls = {1, K - 1, K, K + 1, K + 2, K + 31, K + 32, K + 33, 150, 200, 299, 300, 513, MAXL};
        for (int q = 32; q <= 320; q += 32)
            for (int d = -1; d <= 1; d++) Ls.push_back(q + d);
        std::vector<int> lens;
        std::vector<u64> words;
        for (int L : Ls)
            for (int kind = 0; kind < 8; kind++) {
                if (L < 1 || L > MAXL) continue;
                std::vector<u64> wv(W64, 0);
                const int period = 1 + (int)(rnd() % 6);
                u32 motif[8];
                for (int i = 0; i < 8; i++) motif[i] = (u32)(rnd() & 3);
                for (int i = 0; i < L; i++) {
                    u32 c;
                    if (kind == 0 || kind == 1) c = (u32)(rnd() & 3);                 // random
                    else if (kind == 2) c = motif[0];                               // homopolymer
                    else if (kind == 3) c = motif[i % period];                      // short tandem repeat
                    else if (kind == 4) c = (i / 40) & 1 ? motif[i % period] : (u32)(rnd() & 3);   // repeats between random stretches
                    else if (kind == 5) c = (rnd() % 10) ? motif[0] : (u32)(rnd() & 3);            // homopolymer with errors
                    else c = (u32)(rnd() & 3);
                    wv[i >> 5] |= (u64)c << (2 * (i & 31));
                }
                lens.push_back(L);
                words.insert(words.end(), wv.begin(), wv.end());
            }
        const int n_reads = (int)lens.size();
        if (n_reads > max_reads) { printf("too many reads\n"); return 2; }
        long err = 0, runs_checked = 0;
        for (u32 nb : {1u, 2u, 3u, 65536u}) {
            const SkmGeom g = make_skm_geom(K, nb);
            CK(cudaMemcpy(d_words, words.data(), sizeof(u64) * words.size(), cudaMemcpyHostToDevice));
            CK(cudaMemcpy(d_lens, lens.data(), sizeof(int) * n_reads, cudaMemcpyHostToDevice));
            CK(cudaMemset(d_runs, 0xFF, sizeof(Run) * (size_t)MAXL * n_reads));
            k_warp_runs<<<64, 128>>>(g, d_words, d_lens, n_reads, d_runs, d_nruns);
            CK(cudaGetLastError());
            CK(cudaDeviceSynchronize());
            std::vector<int> nr(n_reads);
            std::vector<Run> got((size_t)MAXL * n_reads);
            CK(cudaMemcpy(nr.data(), d_nruns, sizeof(int) * n_reads, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(got.data(), d_runs, sizeof(Run) * got.size(), cudaMemcpyDeviceToHost));
            std::vector<u32> scratch(g.w);
            for (int r = 0; r < n_reads; r++) {
                std::vector<Run> want;
                HostEmit he{&want};
                skm_scan_read(g, words.data() + (size_t)r * W64, lens[r], scratch.data(), 1, he);
                bool ok = nr[r] == (int)want.size();
                for (size_t i = 0; ok && i < want.size(); i++) {
                    const Run& a = got[(size_t)r * MAXL + i];
                    ok = a.b == want[i].b && a.start == want[i].start && a.n == want[i].n && a.last == want[i].last;
                }
                runs_checked += (long)want.size();
                if (!ok) {
                    if (err < 5) printf("MISMATCH K=%d buckets=%u read=%d L=%d runs %d vs %zu\n", K, nb, r, lens[r], nr[r], want.size());
                    err++;
                }
            }
        }
        printf("K=%d reads=%d runs=%ld errors=%ld\n", K, n_reads, runs_checked, err);
        total_err += err;
    }
    printf(total_err ? "FAILED\n" : "ALL OK\n");
    return total_err ? 1 : 0;
}
