// chop.cuh -- K2: roll the canonical k-mer along one 2-bit packed read (chopKmer4read, prlHashReads.c:163-259).
// sink(canon, left, right, j) is called for every k-mer position j; left/right are the neighbour base codes in the
// CANONICAL orientation (4 = none), SURVEY.md A.2.
#pragma once
#include "kmer.cuh"

namespace pgb {

template <int NW, class Sink>
__device__ __forceinline__ void chop_read(const KParams<NW>& kp, const u64* __restrict__ wp, int L, Sink& sink) {
    const int K = kp.K;
    Kmer<NW> fwd = kzero<NW>(), rc = kzero<NW>();
    u64 cur = wp[0];
    unsigned c = (unsigned)(cur & 3);          // base i
    for (int i = 0; i < L; i++) {
        // look ahead one base (needed as the right neighbour of the k-mer ending at i)
        unsigned cn = 4;
        if (i + 1 < L) {
            if (((i + 1) & 31) == 0) cur = wp[(i + 1) >> 5];
            cn = (unsigned)((cur >> (2 * ((i + 1) & 31))) & 3);
        }
        unsigned dropped = kfirst(fwd, kp);    // base j-1 (valid when j >= 1)
        fwd = knext(fwd, c, kp);
        rc = kprev(rc, c ^ 2u, kp);
        int j = i - K + 1;
        if (j >= 0) {
            unsigned pv = j > 0 ? dropped : 4u;
            bool sm = kless(fwd, rc);          // KmerSmaller(word, bal_word); tie -> rc branch
            unsigned left = sm ? pv : (cn < 4 ? (cn ^ 2u) : 4u);
            unsigned right = sm ? cn : (pv < 4 ? (pv ^ 2u) : 4u);
            sink(sm ? fwd : rc, left, right, j);
        }
        c = cn;
    }
}


#if defined(__CUDACC__)
// ---------------------------------------------------------------- TMA staging of a tile of packed reads
// A block's 256 reads are one contiguous run of the read store (256 x W64 x 8 B, e.g. 10 KB at 150 bp): one elected thread
// arms an mbarrier with the byte count and issues a single bulk tensor-less TMA copy (cp.async.bulk -> SASS UBLKCP.S.G);
// every thread then rolls its read out of shared memory instead of issuing strided 8-byte global loads.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u64* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, unsigned bytes, u64* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(u64* bar, unsigned parity) {
    asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(
                     smem_u32(bar)),
                 "r"(parity)
                 : "memory");
}
// an arrival that expects no bytes (a stage with nothing to copy)
__device__ __forceinline__ void mbar_arrive(u64* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// The other direction: a bulk copy from shared to global memory (SASS UBLKCP.G.S), tracked in the issuing thread's bulk async-groups.
// Generic-proxy writes of the source must be ordered before it by fence.proxy.async.shared::cta in every writing thread, then a barrier.
__device__ __forceinline__ void tma_bulk_s2g(void* dst, const void* src, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// until at most N of this thread's committed groups still read their source (the older ones' shared memory may be written again)
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// until every committed group has completed (its global writes are done)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
#endif

}   // namespace pgb
