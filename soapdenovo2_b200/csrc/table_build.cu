// table_build.cu -- aggregated pass 1, the region build of the k-mer table.
// The table of a launch into an empty table is a pure function of its aggregates, and its slot positions are private to the engine (any
// valid linear-probing placement will do): so it is built like a partitioned hash build.  One CTA per region (grid-stride): fill the
// region in shared memory with EMPTY, read the bin's entries (the region's own table memory, written by k_skm_apply<NW, true>), find or
// claim each key by linear probing WITHOUT wrap-around and merge its partials, sweep every occupied slot, write the region out whole,
// empty slots included.  Every partial of a key lands in the same bin, and slots never empty again, so a key is either entirely in the
// region -- final, and swept here -- or all its probes run off the region's end: a carry, appended to the remnant list and merged by
// k_merge_remnants once every region is written.  Regions of 64 KB let 3 CTAs share an SM (one region's fill, read, probe and
// write-back overlap another's); a bin holds 2048 (K <= 63) or 1024 slots' worth of entries, twice the expected fill at 0.85 load.
// The end-of-pass sweeps -- delow, linear flag, coverage histogram (thread_delow / thread_mark / freqStat, prlHashReads.c:953-1132) --
// are applied to every entry as its region is written.
#include "engine_impl.cuh"
#include "table_build.cuh"

namespace pgb {

constexpr int TB_THREADS = 256;   // one coverage-histogram bin per thread (SweepTally)
constexpr int TB_REGION_BYTES = 64 * 1024;
template <int NW>
constexpr int tb_region_log2() { return __builtin_ctz(TB_REGION_BYTES / (int)sizeof(Slot<NW>)); }

struct TableBuildArgs {
    BinArgs bins;
    int sweep, D;     // apply the end-of-pass sweeps (PendingFlush::sweep), delow threshold
    u64* hist;        // [256] coverage histogram of the swept entries
    u64* counters;    // C_DISTINCT += keys built; C_CARRY, C_BIN_OVF; C_LINEAR, C_REMOVED; C_SPILLKEYS (k_merge_remnants)
    u64* spill_list;  // k_merge_remnants: slots of the keys it claimed, swept from this list afterwards (k_sweep_list)
    u64 spill_cap;
};

template <int NW>
__global__ void __launch_bounds__(TB_THREADS) k_table_build(Table<NW> tab, TableBuildArgs a) {
    constexpr int SW = (int)sizeof(Slot<NW>) / 8;   // words per slot
    extern __shared__ __align__(16) u64 s_reg[];    // [RS] slots in table format
    __shared__ SweepTally s_sw;
    __shared__ unsigned s_new;
    const int tid = threadIdx.x;
    const u32 RS = 1u << a.bins.region_log2;
    const u64 n_regions = (tab.mask + 1) >> a.bins.region_log2;
    // a bin overflow leaves partials of some keys on the remnant list, merged after the build: then nothing may be swept here
    const bool sweep = a.sweep && ldcg64(&a.counters[C_BIN_OVF]) == 0;
    s_sw.clear();
    if (tid == 0) s_new = 0;
    unsigned lin = 0, rem = 0, my_new = 0;
    for (u64 r = blockIdx.x; r < n_regions; r += gridDim.x) {
        __syncthreads();   // the previous region is written out
        for (u32 i = tid; i < RS * SW / 2; i += TB_THREADS) reinterpret_cast<uint4*>(s_reg)[i] = make_uint4(~0u, ~0u, ~0u, ~0u);
        __syncthreads();
        Slot<NW>* const g = tab.slots + (r << a.bins.region_log2);
        const u32 n = min(a.bins.cursor[r], RS);
        for (u32 i = tid; i < n; i += TB_THREADS) {
            Kmer<NW> k;
            u64 pay, rank;
            slot_load(g + i, k, pay, rank);
            // into the region by linear probing WITHOUT wrap-around from the key's home slot: a claim writes {payload, rank} before it
            // publishes the key (a new key), a match merges its partial; a carry when every probe runs off the region's end
            u32 j = (u32)(table_hash(k) & (RS - 1));
            if (smem_find_or_claim<NW, false>(s_reg, SW, 1, RS, k, j, [] { return true; },
                                              [&](u32 j) {
                                                  volatile u64* const ks = s_reg + (u64)j * SW;
                                                  ks[NW] = pay;
                                                  ks[NW + 1] = rank;
                                              },
                                              [&](u32 j, bool claimed) {
                                                  u64* const sl = s_reg + (u64)j * SW;
                                                  if (claimed) my_new++;
                                                  else slot_merge(sl + NW, sl + NW + 1, ((volatile u64*)sl)[NW], pay, rank);
                                              }))
                continue;
            const u64 c = atomicAdd(&a.counters[C_CARRY], 1ull);   // a carry
            if (c < a.bins.remnant_cap) slot_store(reinterpret_cast<Slot<NW>*>(a.bins.remnant) + c, k, pay, rank);
        }
        __syncthreads();   // every entry of the bin is read and placed: its table memory may be overwritten
        if (sweep)
            for (u32 j = tid; j < RS; j += TB_THREADS) {
                u64* const sl = s_reg + (u64)j * SW;
                if (!(sl[0] == EMPTY64 && sl[1] == EMPTY64)) sl[NW] = sweep_payload(sl[NW], a.D, rem, lin, s_sw.hist);
            }
        __syncthreads();
        for (u32 i = tid; i < RS * SW / 2; i += TB_THREADS) stcg128(reinterpret_cast<U128*>(g) + i, reinterpret_cast<const U128*>(s_reg)[i]);
    }
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
    int rl = tb_region_log2<NW>();
    if (const char* e = getenv("PGB200_TABLE_REGION")) {   // slots per region (a power of two; tests use tiny regions for carries)
        const u64 v = strtoull(e, nullptr, 0);
        if (v < 1 || (v & (v - 1)) || v > (1ull << rl)) throw std::runtime_error("pgb200: PGB200_TABLE_REGION must be a power of two up to the 64 KB region");
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
    const size_t smem = sizeof(Slot<NW>) << region_log2_;
    PG_CUDA(cudaFuncSetAttribute(k_table_build<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, TB_REGION_BYTES));
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
