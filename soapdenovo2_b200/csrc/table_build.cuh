// table_build.cuh -- the one contract between the bucket aggregation (skm_apply.cu) and the region build (table_build.cu): where a
// region-mode aggregation launch stores its aggregates.
#pragma once
#include "engine_impl.cuh"

namespace pgb {

// Region mode: an aggregate of key k goes to its bin, the table memory of its home region (table_hash(k) & mask) >> region_log2, at
// the position one atomicAdd on the bin's cursor hands out.  Past the bin's capacity (the region's slot count) it goes to the remnant
// list, which k_merge_remnants merges after the build; past the list's capacity it is counted only, and the host builds the pass again
// in merge mode (skm_flush_complete).
struct BinArgs {
    u32* cursor;      // [regions]
    void* remnant;    // Slot<NW>[cap]
    u64 remnant_cap;
    int region_log2;
};
template <int NW>
__device__ __forceinline__ void bin_store(const Table<NW>& t, const BinArgs& b, u64* counters, const Kmer<NW>& k, u64 pay, u64 rank) {
    const u64 bin = (table_hash(k) & t.mask) >> b.region_log2;
    const u32 at = atomicAdd(&b.cursor[bin], 1u);
    Slot<NW>* s;
    if (at < (1u << b.region_log2)) {
        s = t.slots + (bin << b.region_log2) + at;
    } else {
        atomicAdd(&counters[C_BIN_OVF], 1ull);
        const u64 j = atomicAdd(&counters[C_CARRY], 1ull);
        if (j >= b.remnant_cap) return;
        s = reinterpret_cast<Slot<NW>*>(b.remnant) + j;
    }
    slot_store(s, k, pay, rank);
}

}   // namespace pgb
