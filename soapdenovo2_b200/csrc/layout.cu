// layout.cu -- K3b: rebuild the REFERENCE's table layout, i.e. the iteration order "set 0 slot 0..size-1, set 1 ..."
// that defines vertex order, edge ids, tip-clipping order and therefore every output file except .kmerFreq
// (SURVEY.md facts 1-2, A.4-A.5).
//
// Reference behaviour being reproduced (standardPregraph/):
//   * set of a k-mer       = crc(kmer) % P                               prlHashReads.c:83, hashFunction.c:155-158
//   * home slot in the set = kmer % prime size (or modular())            newhash.c:490-492 / 36-47
//   * slot                 = first free slot from home at insertion time, insertion order = first occurrence in the read stream
//                            (FCFS linear probing)                        newhash.c:473-528
// FCFS linear probing == priority linear probing with priority = first-occurrence rank, and that is order-independent:
// every distinct k-mer walks from its home slot doing atomicMin(slot, rank); whoever holds the larger rank moves on
// (carrying the displaced rank if it won).  The fixed point is exactly the sequential layout.  Ranks are unique
// (read ordinal << 16 | position), so the 64-bit slot word needs no payload; a second pass lets every k-mer find its
// own rank again, a third turns the rank table into "position -> ktab slot", and one scan compacts it into order[].
#include "engine_impl.cuh"
#include "scan.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <thread>

namespace pgb {

struct RefGeom {
    const u64* set_size;   // [P]
    const u64* set_base;   // [P]
    int P;
    bool flavour127;
};

template <int NW>
__global__ void __launch_bounds__(256) k_count_sets(Table<NW> tab, int P, u64* set_count) {
    __shared__ unsigned s_cnt[256];
    s_cnt[threadIdx.x] = 0;
    __syncthreads();
    u64 n = tab.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const Slot<NW>* s = tab.slots + i;
        if (!slot_occupied(s)) continue;
        atomicAdd(&s_cnt[crc_hash(slot_key(s)) % (u64)P], 1u);
    }
    __syncthreads();
    if ((int)threadIdx.x < P && s_cnt[threadIdx.x]) atomicAdd(&set_count[threadIdx.x], (u64)s_cnt[threadIdx.x]);
}

template <int NW>
__global__ void __launch_bounds__(256) k_layout_place(Table<NW> tab, RefGeom g, u64* R) {
    u64 n = tab.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const Slot<NW>* s = tab.slots + i;
        if (!slot_occupied(s)) continue;
        Kmer<NW> k = slot_key(s);
        int set = (int)(crc_hash(k) % (u64)g.P);
        u64 size = g.set_size[set];
        u64* base = R + g.set_base[set];
        u64 pos = ref_home(k, size, g.flavour127);
        u64 r = s->aux;   // first-occurrence rank
        for (;;) {
            u64 old = atomicMin(&base[pos], r);
            if (old == EMPTY64) break;       // took a free slot
            if (old > r) r = old;            // displaced a later arrival: carry it on
            if (++pos == size) pos = 0;
        }
    }
}

template <int NW>
__global__ void __launch_bounds__(256) k_layout_resolve(Table<NW> tab, RefGeom g, const u64* R, u64* gpos_out) {
    u64 n = tab.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const Slot<NW>* s = tab.slots + i;
        if (!slot_occupied(s)) { continue; }
        Kmer<NW> k = slot_key(s);
        int set = (int)(crc_hash(k) % (u64)g.P);
        u64 size = g.set_size[set];
        const u64* base = R + g.set_base[set];
        u64 pos = ref_home(k, size, g.flavour127);
        u64 r = s->aux;
        while (base[pos] != r) { if (++pos == size) pos = 0; }
        gpos_out[i] = g.set_base[set] + pos;
    }
}

template <int NW>
__global__ void __launch_bounds__(256) k_layout_fill(Table<NW> tab, const u64* gpos, u64* R) {
    u64 n = tab.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        if (!slot_occupied(tab.slots + i)) continue;
        R[gpos[i]] = i;   // every resolve has finished (kernel boundary): the rank is no longer needed
    }
}

struct OccIn {
    const u64* R;
    __device__ u64 operator()(u64 i) const { return R[i] != EMPTY64; }
};
template <int NW>
struct OrderOut {
    const u64* R;
    u64* order;
    Slot<NW>* slots;
    __device__ void operator()(u64 i, u64 prefix, u64 v) const {
        if (!v) return;
        u64 slot = R[i];
        order[prefix] = slot;
        slots[slot].aux = prefix;   // aux now = index in reference iteration order
    }
};

// ---------------------------------------------------------------- f1: dynamic tables (no -a): growth-history replay
// Without -a the reference's sets start at 1031 slots and grow (encap_kmerset, newhash.c:340-455): new prime size, array
// realloc'ed IN PLACE, entries re-inserted in ascending old-slot order with displacement chains.  The final layout therefore
// depends on the whole growth history.  The history is a function of the keys' first-occurrence order alone (growth k happens
// when the set holds exactly its first max_k distinct keys), so it can be replayed after the fact: the GPU sorts the distinct
// k-mers by (set, rank) (library radix sort: plumbing outside the metric) and each set is replayed by one host thread with
// the same put / grow rules.  Cost O(distinct); only runs when -a is absent.
template <int NW>
__global__ void __launch_bounds__(256) k_replay_keys(Table<NW> tab, int P, u64* sort_key, u64* sort_val, u64* cursor) {
    u64 n = tab.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const Slot<NW>* s = tab.slots + i;
        if (!slot_occupied(s)) continue;
        u64 set = crc_hash(slot_key(s)) % (u64)P;
        u64 p = atomicAdd(cursor, 1ull);
        sort_key[p] = (set << 56) | (s->aux & ((1ull << 56) - 1));   // rank < 2^56 (read ordinal < 2^40)
        sort_val[p] = i;
    }
}
template <int NW>
__global__ void __launch_bounds__(256) k_gather_keys(Table<NW> tab, const u64* slots_sorted, u64 n, u64* keys_out) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        Kmer<NW> k = slot_key(tab.slots + slots_sorted[i]);
        for (int w = 0; w < NW; w++) keys_out[i * NW + w] = k.w[w];
    }
}
__global__ void __launch_bounds__(256) k_fill_R(const u64* slots_sorted, const u64* gpos, u64 n, u64* R) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) R[gpos[i]] = slots_sorted[i];
}

// one reference set, replayed on the host: keys[0..n) in first-occurrence order; returns the final size and pos[i]
template <int NW>
static u64 replay_one_set(const u64* keys, u64 n, bool flavour127, std::vector<u32>& slot /* out: index+1 per slot */) {
    u64 size = ref_next_prime(1024);
    const float lf = 0.77f;
    u64 mx = (u64)(size * lf), count = 0;
    slot.assign(size, 0);
    auto home = [&](u64 idx, u64 sz) {
        Kmer<NW> k;
        for (int w = 0; w < NW; w++) k.w[w] = keys[idx * NW + w];
        return ref_home(k, sz, flavour127);
    };
    std::vector<unsigned char> oldocc, newocc;
    auto grow = [&]() {   // encap_kmerset, dynamic branch (newhash.c:368-452)
        u64 nn = size;
        do { if (nn < 0xFFFFFFFULL) nn <<= 1; else nn += 0xFFFFFFULL; nn = ref_next_prime(nn); } while (nn * lf < count + 1);
        u64 old = size;
        oldocc.assign(old, 0);
        for (u64 j = 0; j < old; j++) oldocc[j] = slot[j] != 0;
        slot.resize(nn, 0);
        newocc.assign(nn, 0);
        size = nn;
        mx = (u64)(nn * lf);
        for (u64 j = 0; j < old; j++) {
            if (!oldocc[j]) continue;
            u32 key = slot[j];
            oldocc[j] = 0;
            for (;;) {
                u64 hc = home(key - 1, nn);
                while (newocc[hc]) { if (++hc == nn) hc = 0; }
                newocc[hc] = 1;
                if (hc < old && oldocc[hc]) { std::swap(key, slot[hc]); oldocc[hc] = 0; }
                else { slot[hc] = key; break; }
            }
        }
        for (u64 j = 0; j < old; j++) if (!newocc[j]) slot[j] = 0;
    };
    for (u64 i = 0; i < n; i++) {
        if (count + 1 > mx) grow();   // checked on EVERY put, before probing (newhash.c:477-480)
        u64 hc = home(i, size);
        while (slot[hc]) { if (++hc == size) hc = 0; }
        slot[hc] = (u32)(i + 1);
        count++;
    }
    // the check also fires on hits: a set that ends exactly at its threshold grows at its next (repeat) instance, which
    // exists unless the set's last new k-mer is also its very last instance in the read stream (not tracked; assumed)
    if (n && count + 1 > mx) grow();
    return size;
}

template <int NW>
void EngineT<NW>::build_layout() {
    const int P = prm_.P;
    if (P < 1 || P > 255) throw std::runtime_error("pgb200: -p must be in 1..255 (reference thread ids are unsigned char)");
    settle_timing();
    read_counters();
    n_nodes_ = h_cnt_[C_DISTINCT];
    std::vector<u64> set_size(P), set_base(P);
    DevBuf d_geom;
    d_geom.alloc(3 * P * sizeof(u64));
    u64* d_size = d_geom.template as<u64>();
    u64* d_base = d_size + P;
    u64* d_count = d_base + P;
    PG_CUDA(cudaMemsetAsync(d_count, 0, P * sizeof(u64), st_));
    k_count_sets<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, P, d_count);
    PG_CUDA(cudaGetLastError());
    std::vector<u64> cnt(P);
    PG_CUDA(cudaMemcpyAsync(cnt.data(), d_count, P * sizeof(u64), cudaMemcpyDeviceToHost, st_));
    sync();
    if (prm_.initG) {
        u64 sz = ref_static_set_size(prm_.initG, P, prm_.flavour127 != 0);
        for (int i = 0; i < P; i++) {
            set_size[i] = sz;
            if (cnt[i] >= sz) throw std::runtime_error("pgb200: -a too small: a reference set would overflow (the reference spins forever here)");
        }
    } else {
        // Dynamic growth: replay every set's growth history (see above)
        for (int i = 0; i < P; i++)
            if (cnt[i] >= 0xFFFFFFF0ull) throw std::runtime_error("pgb200: a dynamic reference set would exceed 2^32 entries; use -a");
        const u64 N = n_nodes_;
        DevBuf kb, vb, kb2, vb2, curb, tmpb, keysb;
        kb.alloc((N + 1) * sizeof(u64)); vb.alloc((N + 1) * sizeof(u64)); kb2.alloc((N + 1) * sizeof(u64)); vb2.alloc((N + 1) * sizeof(u64));
        curb.alloc(sizeof(u64));
        PG_CUDA(cudaMemsetAsync(curb.p, 0, sizeof(u64), st_));
        k_replay_keys<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, P, kb.template as<u64>(), vb.template as<u64>(), curb.template as<u64>());
        PG_CUDA(cudaGetLastError());
        size_t tmp_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, kb.template as<u64>(), kb2.template as<u64>(), vb.template as<u64>(), vb2.template as<u64>(), N, 0, 64, st_);
        tmpb.alloc(tmp_bytes);
        cub::DeviceRadixSort::SortPairs(tmpb.p, tmp_bytes, kb.template as<u64>(), kb2.template as<u64>(), vb.template as<u64>(), vb2.template as<u64>(), N, 0, 64, st_);
        keysb.alloc((N + 1) * NW * sizeof(u64));
        k_gather_keys<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, vb2.template as<u64>(), N, keysb.template as<u64>());
        PG_CUDA(cudaGetLastError());
        std::vector<u64> h_keys(N * NW + 1);
        PG_CUDA(cudaMemcpyAsync(h_keys.data(), keysb.p, N * NW * sizeof(u64), cudaMemcpyDeviceToHost, st_));
        sync();
        std::vector<u64> first(P + 1, 0);
        for (int i = 0; i < P; i++) first[i + 1] = first[i] + cnt[i];
        std::vector<std::vector<u32>> slots(P);
        {
            std::vector<std::thread> th;
            const bool f127 = prm_.flavour127 != 0;
            for (int i = 0; i < P; i++)
                th.emplace_back([&, i]() { set_size[i] = replay_one_set<NW>(h_keys.data() + first[i] * NW, cnt[i], f127, slots[i]); });
            for (auto& t : th) t.join();
        }
        u64 total = 0;
        for (int i = 0; i < P; i++) { set_base[i] = total; total += set_size[i]; }
        std::vector<u64> h_gpos(N + 1);
        for (int i = 0; i < P; i++)
            for (u64 j = 0; j < set_size[i]; j++)
                if (slots[i][j]) h_gpos[first[i] + slots[i][j] - 1] = set_base[i] + j;
        DevBuf gposb, Rb, scratch;
        gposb.alloc((N + 1) * sizeof(u64));
        PG_CUDA(cudaMemcpyAsync(gposb.p, h_gpos.data(), N * sizeof(u64), cudaMemcpyHostToDevice, st_));
        Rb.alloc(total * sizeof(u64));
        PG_CUDA(cudaMemsetAsync(Rb.p, 0xFF, total * sizeof(u64), st_));
        k_fill_R<<<n_sm_ * 8, 256, 0, st_>>>(vb2.template as<u64>(), gposb.template as<u64>(), N, Rb.template as<u64>());
        PG_CUDA(cudaGetLastError());
        order_buf_.alloc((N + 1) * sizeof(u64));
        scratch.alloc(scan_scratch_elems(total) * sizeof(u64));
        device_scan(OccIn{Rb.template as<u64>()}, OrderOut<NW>{Rb.template as<u64>(), order_buf_.template as<u64>(), tab_.slots}, total,
                    scratch.template as<u64>(), d_cnt_ + C_MISC0, st_);
        read_counters();
        if (h_cnt_[C_MISC0] != N) throw std::runtime_error("pgb200: internal error: dynamic layout replay lost k-mers");
        return;
    }
    u64 total = 0;
    for (int i = 0; i < P; i++) { set_base[i] = total; total += set_size[i]; }
    if (prm_.verbose)
        fprintf(stderr, "[pgb200] layout: %llu reference slots in %d sets, %llu scan tiles\n", (unsigned long long)total, P,
                (unsigned long long)((total + SCAN_TILE - 1) / SCAN_TILE));
    PG_CUDA(cudaMemcpyAsync(d_size, set_size.data(), P * sizeof(u64), cudaMemcpyHostToDevice, st_));
    PG_CUDA(cudaMemcpyAsync(d_base, set_base.data(), P * sizeof(u64), cudaMemcpyHostToDevice, st_));

    DevBuf Rb, gposb, scratch;
    Rb.alloc(total * sizeof(u64));
    gposb.alloc(cap_ * sizeof(u64));
    PG_CUDA(cudaMemsetAsync(Rb.p, 0xFF, total * sizeof(u64), st_));
    u64* R = Rb.template as<u64>();
    RefGeom g{d_size, d_base, P, prm_.flavour127 != 0};
    k_layout_place<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, g, R);
    k_layout_resolve<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, g, R, gposb.template as<u64>());
    k_layout_fill<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, gposb.template as<u64>(), R);
    PG_CUDA(cudaGetLastError());
    order_buf_.alloc((n_nodes_ + 1) * sizeof(u64));
    scratch.alloc(scan_scratch_elems(total) * sizeof(u64));
    device_scan(OccIn{R}, OrderOut<NW>{R, order_buf_.template as<u64>(), tab_.slots}, total, scratch.template as<u64>(), d_cnt_ + C_MISC0, st_);
    read_counters();
    if (h_cnt_[C_MISC0] != n_nodes_) throw std::runtime_error("pgb200: internal error: layout lost k-mers");
}

// ---------------------------------------------------------------- parity dump (record format documented in include/pregraph_b200.h)
template <int NW>
__global__ void k_dump_nodes(Table<NW> tab, const u64* order, u64 n, int out_words, unsigned char* out) {
    const int rec = out_words * 8 + 10;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const Slot<NW>* s = tab.slots + order[i];
        Kmer<NW> k = slot_key(s);
        u64 p = s->payload;
        unsigned char* o = out + i * rec;
        for (int w = 0; w < out_words; w++) {
            int src = w - (out_words - NW);
            u64 v = src >= 0 ? k.w[src] : 0ull;
            for (int b = 0; b < 8; b++) o[w * 8 + b] = (unsigned char)(v >> (8 * b));
        }
        o += out_words * 8;
        for (int c = 0; c < 4; c++) { o[c] = (unsigned char)pl_l(p, c); o[4 + c] = (unsigned char)pl_r(p, c); }
        o[8] = (unsigned char)pl_cov(p);
        o[9] = (unsigned char)(((p & PL_SINGLE) ? 1 : 0) | ((p & PL_LINEAR) ? 2 : 0) | ((p & PL_DELETED) ? 4 : 0));
    }
}

template <int NW>
void EngineT<NW>::dump_nodes(void* host_out) {
    if (!order_buf_.p) throw std::runtime_error("pgb200: dump_nodes before build_layout");
    const int out_words = prm_.flavour127 ? 4 : 2;
    const size_t rec = out_words * 8 + 10;
    DevBuf d;
    d.alloc(n_nodes_ * rec);
    k_dump_nodes<NW><<<n_sm_ * 4, 256, 0, st_>>>(tab_, order_buf_.template as<u64>(), n_nodes_, out_words, d.template as<unsigned char>());
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cudaMemcpyAsync(host_out, d.p, n_nodes_ * rec, cudaMemcpyDeviceToHost, st_));
    sync();
}

template void EngineT<2>::build_layout();
template void EngineT<4>::build_layout();
template void EngineT<2>::dump_nodes(void*);
template void EngineT<4>::dump_nodes(void*);

}   // namespace pgb
