// table_build.cu -- aggregated pass 1, the region build of the k-mer table.
// The table of a launch into an empty table is a pure function of its aggregates, and its slot positions are private to the engine (any
// valid linear-probing placement will do): so it is built like a partitioned hash build.  Each region (RS slots) is made in shared
// memory: fill with EMPTY, find or claim each entry of the bin (the region's own table memory, written by k_skm_apply<NW, true>) by
// linear probing WITHOUT wrap-around and merge its partials, sweep every occupied slot, write the region out whole, empty slots
// included.  Every partial of a key lands in the same bin, and slots never empty again, so a key is either entirely in the region --
// final, and swept here -- or all its probes run off the region's end: a carry, appended to the remnant list and merged by
// k_merge_remnants once every region is written.
// What bounds the build is the memory traffic each SM keeps in flight, not issue: so a CTA is a pipeline over its regions (grid-stride),
// with every byte of a bin and of a region moved by bulk copies.  While it builds region i, the bin of region i+1 arrives in the other
// stage (one cp.async.bulk, complete on that stage's mbarrier) and region i-1 leaves from the other region buffer (one bulk store):
// two region buffers of RS slots and two stages of 256 entries.  A bin holds at most RS entries (bin_store); one larger than its stage
// arrives in pieces.  The end-of-pass sweeps -- delow, linear flag, coverage histogram (thread_delow / thread_mark / freqStat,
// prlHashReads.c:953-1132) -- are applied to every entry as its region is written.
#include "engine_impl.cuh"
#include "table_build.cuh"
#include "chop.cuh"

namespace pgb {

constexpr int TB_THREADS = 256;   // one coverage-histogram bin per thread (SweepTally)
constexpr int TB_REGION_LOG2 = 9;           // 512 slots: 16 KB regions at K <= 63 (4 CTAs per SM), 32 KB above (2 CTAs per SM)
constexpr u32 TB_STAGE_SLOTS = 256;         // entries per stage; a bin of more arrives in pieces
__host__ __device__ constexpr u32 tb_stage_slots(u32 region_slots) { return region_slots < TB_STAGE_SLOTS ? region_slots : TB_STAGE_SLOTS; }

struct TableBuildArgs {
    BinArgs bins;
    int sweep, D;     // apply the end-of-pass sweeps (PendingFlush::sweep), delow threshold
    u64* hist;        // [256] coverage histogram of the swept entries
    u64* counters;    // C_DISTINCT += keys built; C_CARRY, C_BIN_OVF; C_LINEAR, C_REMOVED; C_SPILLKEYS (k_merge_remnants)
    u64* spill_list;  // k_merge_remnants: slots of the keys it claimed, swept from this list afterwards (k_sweep_list)
    u64 spill_cap;
};

// Dynamic shared memory: region buffers 0 and 1 (RS slots each), then stages 0 and 1 (SE slots each).  Region i of the CTA uses buffer
// and stage i & 1.
template <int NW>
__global__ void __launch_bounds__(TB_THREADS) k_table_build(Table<NW> tab, TableBuildArgs a) {
    constexpr int SW = (int)sizeof(Slot<NW>) / 8;   // words per slot
    extern __shared__ __align__(128) u64 s_buf[];
    __shared__ SweepTally s_sw;
    __shared__ u64 s_bar[2];   // stage s is full
    __shared__ u32 s_n[2];     // entries in the bin that stage s takes
    __shared__ unsigned s_new;
    const int tid = threadIdx.x;
    const u32 RS = 1u << a.bins.region_log2, SE = tb_stage_slots(RS);
    const u32 RW = RS * SW;   // words per region buffer
    const u64 n_regions = (tab.mask + 1) >> a.bins.region_log2;
    // a bin overflow leaves partials of some keys on the remnant list, merged after the build: then nothing may be swept here
    const bool sweep = a.sweep && ldcg64(&a.counters[C_BIN_OVF]) == 0;
    // one thread moves the bins in: m entries from src into stage s, or an arrival without bytes when there are none
    auto piece_in = [&](const Slot<NW>* src, u32 m, int s) {
        if (m) {
            mbar_expect_tx(&s_bar[s], m * (u32)sizeof(Slot<NW>));
            tma_bulk_g2s(s_buf + 2 * RW + s * SE * SW, src, m * (u32)sizeof(Slot<NW>), &s_bar[s]);
        } else {
            mbar_arrive(&s_bar[s]);
        }
    };
    auto bin_in = [&](u64 r, u32 cursor, int s) {
        const u32 n = min(cursor, RS);
        s_n[s] = n;
        piece_in(tab.slots + (r << a.bins.region_log2), min(n, SE), s);
    };
    s_sw.clear();
    u32 c_next = 0;   // thread 0: the cursor of the bin after the one in flight, read one region ahead of its use
    if (tid == 0) {
        s_new = 0;
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        bin_in(blockIdx.x, a.bins.cursor[blockIdx.x], 0);   // (the grid has no more CTAs than regions)
        if (blockIdx.x + gridDim.x < n_regions) c_next = a.bins.cursor[blockIdx.x + gridDim.x];
    }
    unsigned lin = 0, rem = 0, my_new = 0;
    u32 it = 0, phase = 0;   // bit s: the parity of the next wait on stage s
    for (u64 r = blockIdx.x; r < n_regions; r += gridDim.x, it++) {
        const int b = it & 1;
        u64* const reg = s_buf + b * RW;
        const u64* const stage = s_buf + 2 * RW + b * SE * SW;
        Slot<NW>* const g = tab.slots + (r << a.bins.region_log2);
        // the other stage was read by region it-1 (fence.proxy.async and the barrier at its end): the next bin goes there
        if (tid == 0 && r + gridDim.x < n_regions) {
            bin_in(r + gridDim.x, c_next, b ^ 1);
            if (r + 2ull * gridDim.x < n_regions) c_next = a.bins.cursor[r + 2ull * gridDim.x];
        }
        // this buffer's store (region it-2) has finished reading it: waited for before region it-1's store was issued
        for (u32 i = tid; i < RW / 2; i += TB_THREADS) reinterpret_cast<uint4*>(reg)[i] = make_uint4(~0u, ~0u, ~0u, ~0u);
        __syncthreads();   // the region is EMPTY; s_n[b] is written
        const u32 n = s_n[b];
        for (u32 p0 = 0;;) {
            mbar_wait(&s_bar[b], (phase >> b) & 1u);
            phase ^= 1u << b;
            const u32 m = min(n - p0, SE);
            for (u32 i = tid; i < m; i += TB_THREADS) {
                const u64* const e = stage + (u64)i * SW;
                Kmer<NW> k;
#pragma unroll
                for (int w = 0; w < NW; w++) k.w[w] = e[w];
                const u64 pay = e[NW], rank = e[NW + 1];
                // into the region by linear probing WITHOUT wrap-around from the key's home slot: a claim writes {payload, rank} before it
                // publishes the key (a new key), a match merges its partial; a carry when every probe runs off the region's end
                u32 j = (u32)(table_hash(k) & (RS - 1));
                if (smem_find_or_claim<NW, false>(reg, SW, 1, RS, k, j, [] { return true; },
                                                  [&](u32 j) {
                                                      volatile u64* const ks = reg + (u64)j * SW;
                                                      ks[NW] = pay;
                                                      ks[NW + 1] = rank;
                                                  },
                                                  [&](u32 j, bool claimed) {
                                                      u64* const sl = reg + (u64)j * SW;
                                                      if (claimed) my_new++;
                                                      else slot_merge(sl + NW, sl + NW + 1, ((volatile u64*)sl)[NW], pay, rank);
                                                  }))
                    continue;
                const u64 c = atomicAdd(&a.counters[C_CARRY], 1ull);   // a carry
                if (c < a.bins.remnant_cap) slot_store(reinterpret_cast<Slot<NW>*>(a.bins.remnant) + c, k, pay, rank);
            }
            p0 += SE;
            if (p0 >= n) break;
            // a bin larger than the stage: its next piece into the same stage, once every thread has read this one
            fence_proxy_async_smem();
            __syncthreads();
            if (tid == 0) piece_in(g + p0, min(n - p0, SE), b);
        }
        __syncthreads();   // every entry is placed
        if (sweep)
            for (u32 j = tid; j < RS; j += TB_THREADS) {
                u64* const sl = reg + (u64)j * SW;
                if (!(sl[0] == EMPTY64 && sl[1] == EMPTY64)) sl[NW] = sweep_payload(sl[NW], a.D, rem, lin, s_sw.hist);
            }
        // this thread's writes of the region and reads of the stage come before the bulk copies that read or overwrite them
        fence_proxy_async_smem();
        if (tid == 0) bulk_wait_read<0>();   // region it-1's store no longer reads the other buffer, which region it+1 fills
        __syncthreads();
        if (tid == 0) {
            tma_bulk_s2g(g, reg, RS * (u32)sizeof(Slot<NW>));
            bulk_commit();
        }
    }
    if (tid == 0) bulk_wait_all();   // the region stores read shared memory until they complete, and the CTA's table is written
    if (my_new) atomicAdd(&s_new, my_new);
    s_sw.flush(lin, rem, a.hist, &a.counters[C_LINEAR], &a.counters[C_REMOVED]);   // (synchronises the CTA first)
    if (tid == 0 && s_new) atomicAdd(&a.counters[C_DISTINCT], (u64)s_new);
}

// The remnant list (bin overflow, then carries) into the finished table with the CAS protocol: a carry's probe continues into the next
// regions, and a key placed into an empty slot breaks no other key's probe path.  Several entries may hold partials of one key, so a
// claim merges into the empty slot's {PAYLOAD_FRESH, ~0} like any other writer instead of storing.
template <int NW>
__global__ void __launch_bounds__(256) k_merge_remnants(Table<NW> tab, TableBuildArgs a) {
    __shared__ unsigned s_new;
    if (threadIdx.x == 0) s_new = 0;
    __syncthreads();
    const u64 n = min(ldcg64(&a.counters[C_CARRY]), a.bins.remnant_cap);
    const Slot<NW>* const list = reinterpret_cast<const Slot<NW>*>(a.bins.remnant);
    unsigned my_new = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        Kmer<NW> k;
        u64 pay, rank;
        slot_load(list + i, k, pay, rank);
        bool claimed;
        const u64 idx = table_merge<false>(tab, k, pay, rank, &claimed);
        if (claimed) {
            my_new++;
            const u64 sn = atomicAdd((unsigned long long*)&a.counters[C_SPILLKEYS], 1ull);
            if (sn < a.spill_cap) a.spill_list[sn] = idx;
        }
    }
    if (my_new) atomicAdd(&s_new, my_new);
    __syncthreads();
    if (threadIdx.x == 0 && s_new) atomicAdd(&a.counters[C_DISTINCT], (u64)s_new);
}

// ------------------------------------------------------------------------------------------------ host side
template <int NW>
BinArgs EngineT<NW>::bin_args() const {
    return BinArgs{bin_cursor_.template as<u32>(), carry_buf_.p, carry_cap_, region_log2_};
}

// Before a region-mode aggregation launch: the region size, empty bins, room for the remnant list, and cleared build counters
template <int NW>
void EngineT<NW>::table_build_prepare() {
    int rl = TB_REGION_LOG2;
    if (const char* e = getenv("PGB200_TABLE_REGION")) {   // slots per region (a power of two; tests use tiny regions for carries)
        const u64 v = strtoull(e, nullptr, 0);
        if (v < 1 || (v & (v - 1)) || v > (1ull << rl)) throw std::runtime_error("pgb200: PGB200_TABLE_REGION must be a power of two up to the default region size");
        rl = __builtin_ctzll(v);
    }
    while ((1ull << rl) > cap_) rl--;
    region_log2_ = rl;
    bin_cursor_.ensure((cap_ >> rl) * sizeof(u32));
    carry_cap_ = std::max<u64>(cap_ / 64, 1ull << 16);
    if (const char* e = getenv("PGB200_TABLE_REMNANT_CAP")) carry_cap_ = strtoull(e, nullptr, 0);
    carry_buf_.ensure(carry_cap_ * sizeof(Slot<NW>));
    hist_buf_.ensure(256 * sizeof(u64));
    spill_list_.ensure(SPILL_CAP * sizeof(u64));
    PG_CUDA(cudaMemsetAsync(bin_cursor_.p, 0, (cap_ >> rl) * sizeof(u32), st_));
    PG_CUDA(cudaMemsetAsync(d_cnt_ + C_SPILLKEYS, 0, sizeof(u64), st_));
    PG_CUDA(cudaMemsetAsync(d_cnt_ + C_CARRY, 0, 2 * sizeof(u64), st_));   // C_CARRY, C_BIN_OVF
    PG_CUDA(cudaMemsetAsync(hist_buf_.p, 0, 256 * sizeof(u64), st_));
    PG_CUDA(cudaMemsetAsync(d_cnt_ + C_LINEAR, 0, 2 * sizeof(u64), st_));
}

// k_table_build + k_merge_remnants behind the region-mode aggregation launch (inside its timing events)
template <int NW>
void EngineT<NW>::table_build_launch() {
    TableBuildArgs b;
    b.bins = bin_args();
    b.sweep = flush_.sweep ? 1 : 0;
    b.D = (int)(signed char)prm_.D;   // deLowKmer is a `char` (inc/global.h:67)
    b.hist = hist_buf_.template as<u64>();
    b.counters = d_cnt_;
    b.spill_list = spill_list_.template as<u64>();
    b.spill_cap = SPILL_CAP;
    const size_t smem = 2 * sizeof(Slot<NW>) * ((1ull << region_log2_) + tb_stage_slots(1u << region_log2_));   // two region buffers, two stages
    PG_CUDA(cudaFuncSetAttribute(k_table_build<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    PG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_table_build<NW>, TB_THREADS, smem));
    if (per_sm < 1) per_sm = 1;
    k_table_build<NW><<<(unsigned)std::min<u64>(cap_ >> region_log2_, (u64)n_sm_ * per_sm), TB_THREADS, smem, st_>>>(tab_, b);
    PG_CUDA(cudaGetLastError());
    k_merge_remnants<NW><<<n_sm_ * 4, 256, 0, st_>>>(tab_, b);
    PG_CUDA(cudaGetLastError());
    table_dirty_ = false;   // every slot is written
    p1_.launches += 2;
}

// After the launch has completed: its outcome.  A bin overflow leaves the build's sweeps undone (k_table_build); returns true when
// the remnant list was full, i.e. entries were dropped and the launch must run again in merge mode.
template <int NW>
bool EngineT<NW>::table_build_redo() {
    u64 rc[2];   // C_CARRY, C_BIN_OVF
    PG_CUDA(cudaMemcpy(rc, d_cnt_ + C_CARRY, sizeof rc, cudaMemcpyDeviceToHost));
    const bool redo = rc[0] > carry_cap_;
    if (prm_.verbose)
        fprintf(stderr, "[pgb200] region build: %llu regions of %u slots, bin overflow %llu, carries %llu, remnant list %llu of %llu%s\n",
                (unsigned long long)(cap_ >> region_log2_), 1u << region_log2_, (unsigned long long)rc[1], (unsigned long long)(rc[0] - rc[1]),
                (unsigned long long)rc[0], (unsigned long long)carry_cap_, redo ? ": full, the launch runs again in merge mode" : "");
    if (rc[1] && pass_sweeps_ == PassSweeps::Fused) pass_sweeps_ = PassSweeps::Plain;   // the build swept nothing (k_table_build)
    return redo;
}

#define PGB_INST(NW)                                      \
    template BinArgs EngineT<NW>::bin_args() const;       \
    template void EngineT<NW>::table_build_prepare();     \
    template void EngineT<NW>::table_build_launch();      \
    template bool EngineT<NW>::table_build_redo();
PGB_INST(2)
PGB_INST(4)

}   // namespace pgb
