// table.cuh -- the GPU-resident open-addressing k-mer table ("ktab").
//
// Replaces the reference's KmerSet (standardPregraph/newhash.c, inc/newhash.h:77-113) on the hot path:
//   reference                                       here
//   P prime-sized sets, one thread per set          ONE power-of-two table in HBM, every thread inserts anywhere
//   2-bit flag array + 24/40 B kmer_t               32 B (K<=63) / 64 B (K<=127) sector-aligned slots, no flag array
//   put_kmerset: probe, memset+init | update        128-bit atomicCAS claim of the key (table_probe), then a 64-bit CAS loop on
//   (newhash.c:473-528, 74-140)                     payload (saturating link/coverage counters, payload_fold) + a 64-bit atomicMin
//                                                   on the rank (min first-seen rank, rank_min)
// The payload word has EXACTLY the reference's kmer_t bit layout (newhash.h:77-102) so that later phases and the
// parity dump can use it verbatim:
//   bits  0..23  l_links (4 x 6 bit, index = base code)   bits 24..31  cov (8 bit, saturates at 255)
//   bits 32..55  r_links (4 x 6 bit)                      bit 56 linear, 57 deleted, 58 checked, 59 single,
//   bits 60..61  twin                                     bits 62..63 inEdge
// `aux` holds, in turn: the first-occurrence rank (pass 1) -> the position in reference iteration order (after layout)
// Slot position in ktab is private to the engine; the reference's FCFS layout is rebuilt from the ranks (layout.cu).
#pragma once
#include "kmer.cuh"

namespace pgb {

struct alignas(16) U128 {
    u64 a, b;
};

constexpr u64 EMPTY64 = ~0ull;
constexpr u64 PAYLOAD_FRESH = ~0ull;          // memset(0xFF) state: "key claimed but no instance applied yet"
constexpr u64 BUSY_BIT = 1ull << 63;           // NW==4 claim protocol (w[0] uses at most 62 bits for K <= 127)

constexpr int PL_COV_SHIFT = 24;
constexpr int PL_R_SHIFT = 32;
constexpr u64 PL_LINEAR = 1ull << 56;
constexpr u64 PL_DELETED = 1ull << 57;
constexpr u64 PL_CHECKED = 1ull << 58;
constexpr u64 PL_SINGLE = 1ull << 59;
constexpr int PL_TWIN_SHIFT = 60;
constexpr int PL_INEDGE_SHIFT = 62;
constexpr u64 PL_LLINKS_MASK = 0xFFFFFFull;
constexpr u64 PL_RLINKS_MASK = 0xFFFFFFull << 32;

PG_HD unsigned pl_l(u64 p, int c) { return (unsigned)((p >> (6 * c)) & 63); }
PG_HD unsigned pl_r(u64 p, int c) { return (unsigned)((p >> (PL_R_SHIFT + 6 * c)) & 63); }
PG_HD unsigned pl_cov(u64 p) { return (unsigned)((p >> PL_COV_SHIFT) & 255); }
PG_HD int pl_nl(u64 p) { return (pl_l(p, 0) > 0) + (pl_l(p, 1) > 0) + (pl_l(p, 2) > 0) + (pl_l(p, 3) > 0); }
PG_HD int pl_nr(u64 p) { return (pl_r(p, 0) > 0) + (pl_r(p, 1) > 0) + (pl_r(p, 2) > 0) + (pl_r(p, 3) > 0); }
PG_HD int pl_first_l(u64 p) { for (int c = 0; c < 4; c++) if (pl_l(p, c)) return c; return 4; }
PG_HD int pl_first_r(u64 p) { for (int c = 0; c < 4; c++) if (pl_r(p, c)) return c; return 4; }
PG_HD u64 pl_clear_l(u64 p, int c) { return p & ~(63ull << (6 * c)); }
PG_HD u64 pl_clear_r(u64 p, int c) { return p & ~(63ull << (PL_R_SHIFT + 6 * c)); }
PG_HD unsigned pl_twin(u64 p) { return (unsigned)((p >> PL_TWIN_SHIFT) & 3); }
PG_HD unsigned pl_inedge(u64 p) { return (unsigned)((p >> PL_INEDGE_SHIFT) & 3); }

// One instance applied to a payload word: set_new_kmer (newhash.c:123-140) when fresh, else update_kmer (:74-106)
// + `single = 0` (newhash.c:509).  left/right are base codes 0..3 or 4 (= none).  Branch-free on the update path (the lanes of a
// warp hold different neighbours and different counters): one increment word, with the increments of saturated fields removed.
PG_HD u64 payload_apply(u64 p, unsigned left, unsigned right) {
    const u64 il = left < 4 ? 1ull << (6 * left) : 0ull;
    const u64 ir = right < 4 ? 1ull << (PL_R_SHIFT + 6 * right) : 0ull;
    if (p == PAYLOAD_FRESH) return (1ull << PL_COV_SHIFT) | PL_SINGLE | il | ir;
    const u64 ml = il * 63ull, mr = ir * 63ull, mc = 255ull << PL_COV_SHIFT;      // the fields the increments land in
    u64 inc = ((p & ml) == ml ? 0ull : il) | ((p & mr) == mr ? 0ull : ir);
    if ((il | ir) != 0ull && (p & mc) != mc) inc |= 1ull << PL_COV_SHIFT;
    return (p + inc) & ~PL_SINGLE;
}
// c identical instances applied at once: equals c calls of payload_apply (c >= 1), and IS payload_apply when c == 1.  The aggregation
// applies each k-mer of a record that occurs c times in its bucket this way (skm_apply.cu).
PG_HD u64 payload_apply_n(u64 p, unsigned left, unsigned right, unsigned c) {
    if (c == 1) return payload_apply(p, left, right);
    if (p == PAYLOAD_FRESH) { p = payload_apply(p, left, right); c--; }
    c = c > 255 ? 255u : c;
    if (left < 4) {
        const int sh = 6 * (int)left;
        const unsigned v = (unsigned)((p >> sh) & 63) + c;
        p = (p & ~(63ull << sh)) | ((u64)(v > 63 ? 63 : v) << sh);
    }
    if (right < 4) {
        const int sh = PL_R_SHIFT + 6 * (int)right;
        const unsigned v = (unsigned)((p >> sh) & 63) + c;
        p = (p & ~(63ull << sh)) | ((u64)(v > 63 ? 63 : v) << sh);
    }
    if (left < 4 || right < 4) {
        const unsigned v = pl_cov(p) + c;
        p = (p & ~(255ull << PL_COV_SHIFT)) | ((u64)(v > 255 ? 255 : v) << PL_COV_SHIFT);
    }
    return p & ~PL_SINGLE;
}

// Two partial results for the same k-mer -> the result of all their instances together.  `g` may be PAYLOAD_FRESH (slot claimed, no
// instance yet); `a` holds at least one instance.  Every instance has a neighbour on at least one side (reads are >= K+1 long), so
// cov counts instances (newhash.c:74-106, 123-140) and the fields simply add with their saturation; `single` survives only when the
// total is one instance, i.e. never when both sides are non-empty.
PG_HD u64 payload_merge(u64 g, u64 a) {
    if (g == PAYLOAD_FRESH) return a;
    u64 r = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
        unsigned l = pl_l(g, c) + pl_l(a, c), q = pl_r(g, c) + pl_r(a, c);
        r |= (u64)(l > 63 ? 63 : l) << (6 * c);
        r |= (u64)(q > 63 ? 63 : q) << (PL_R_SHIFT + 6 * c);
    }
    unsigned cv = pl_cov(g) + pl_cov(a);
    r |= (u64)(cv > 255 ? 255 : cv) << PL_COV_SHIFT;
    return r;
}

// The per-entry sweeps of pass 1's end (K4): delow (thread_delow: zero every link counter <= D, deleted = 1 if nothing is left), mark
// (thread_mark: linear = 1 iff exactly one non-zero left and one non-zero right link, NO deleted check there), histogram of cov.
// Used by k_sweep (pass1.cu) and, fused, by the region build (table_build.cu).  The linear flag is recomputed, not inherited.
#if defined(__CUDACC__)
__device__ __forceinline__ u64 sweep_payload(u64 p, int D, unsigned& rem, unsigned& lin, unsigned* s_hist) {
    p &= ~PL_LINEAR;
    if (D > 0) {
#pragma unroll
        for (int c = 0; c < 4; c++) {
            unsigned l = pl_l(p, c), r = pl_r(p, c);
            if (l > 0 && l <= (unsigned)D) p = pl_clear_l(p, c);
            if (r > 0 && r <= (unsigned)D) p = pl_clear_r(p, c);
        }
        if ((p & PL_LLINKS_MASK) == 0 && (p & PL_RLINKS_MASK) == 0) { p |= PL_DELETED; rem++; }
    }
    atomicAdd(&s_hist[pl_cov(p)], 1u);
    if (pl_nl(p) == 1 && pl_nr(p) == 1) { p |= PL_LINEAR; lin++; }
    return p;
}

// What the CTAs that call sweep_payload gather in shared memory (256 threads: one histogram bin each)
struct SweepTally {
    unsigned hist[256], lin, rem;
    __device__ __forceinline__ void clear() {   // the caller synchronises before the first sweep_payload
        hist[threadIdx.x] = 0;
        if (threadIdx.x == 0) { lin = 0; rem = 0; }
    }
    // every thread of the CTA, with its own linear / removed counts: the CTA's tally goes to global memory
    __device__ __forceinline__ void flush(unsigned my_lin, unsigned my_rem, u64* g_hist, u64* g_linear, u64* g_removed) {
        if (my_lin) atomicAdd(&lin, my_lin);
        if (my_rem) atomicAdd(&rem, my_rem);
        __syncthreads();
        if (hist[threadIdx.x]) atomicAdd(&g_hist[threadIdx.x], (u64)hist[threadIdx.x]);
        if (threadIdx.x == 0) {
            if (lin) atomicAdd(g_linear, (u64)lin);
            if (rem) atomicAdd(g_removed, (u64)rem);
        }
    }
};
#endif

template <int NW>
struct Slot;
template <>
struct alignas(32) Slot<2> {
    u64 key[2];
    u64 payload;
    u64 aux;
};
template <>
struct alignas(64) Slot<4> {
    u64 key[4];
    u64 payload;
    u64 aux;
    u64 pad[2];
};

template <int NW>
struct Table {
    Slot<NW>* slots;
    u64 mask;   // capacity - 1 (capacity is a power of two)
};

#if defined(__CUDACC__)

// Table loads are STRONG (relaxed, gpu scope): a weak ld.global may legally be hoisted out of a polling loop by ptxas
// (observed: the publish-wait below was turned into a single load, producing duplicate 256-bit keys on the GPU).
PG_D U128 ldcg128(const void* p) {
    U128 r;
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%2];" : "=l"(r.a), "=l"(r.b) : "l"(p) : "memory");
    return r;
}
struct alignas(32) U256 {
    u64 a, b, c, d;
};
// one 32-byte sector: key + payload + aux of a K<=63 slot.  sm_90 has no 256-bit global load, so the sector arrives as two 128-bit
// loads issued back to back (both in flight together, one sector).  The halves are not one atomic read: a stale payload only makes
// the CAS in slot_apply retry, a stale rank only issues an atomicMin that is not needed.
PG_D U256 ld256(const void* p) {
    U256 r;
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0,%1}, [%4];\n\t"
                 "ld.relaxed.gpu.global.v2.u64 {%2,%3}, [%4+16];"
                 : "=l"(r.a), "=l"(r.b), "=l"(r.c), "=l"(r.d) : "l"(p) : "memory");
    return r;
}
PG_D u64 ldcg64(const void* p) {
    u64 r;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
    return r;
}
PG_D u64 ldacq64(const void* p) {
    u64 r;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
    return r;
}
PG_D void stcg128(void* p, U128 v) { asm volatile("st.global.cg.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(v.a), "l"(v.b) : "memory"); }
// A record goes out with as few stores as possible: over NVLink every store is a packet.  sm_90's widest global store is 128 bits, so
// a 32-byte record is two 16-byte stores to the same sector.
PG_D void st256(u64* dst, u64 a, u64 b, u64 c, u64 d) {
    asm volatile("st.global.v2.u64 [%0], {%1,%2};\n\t"
                 "st.global.v2.u64 [%0+16], {%3,%4};" ::"l"(dst), "l"(a), "l"(b), "l"(c), "l"(d) : "memory");
}

// One whole slot {key, payload, rank} with 16-byte stores (fire and forget)
template <int NW>
PG_D void slot_store(Slot<NW>* s, const Kmer<NW>& k, u64 pay, u64 rank) {
    u64* d = reinterpret_cast<u64*>(s);
    if (NW == 2) {
        st256(d, k.w[0], k.w[1], pay, rank);
    } else {
        stcg128(d, U128{k.w[0], k.w[1]});
        stcg128(d + 2, U128{k.w[2], k.w[3]});
        stcg128(d + 4, U128{pay, rank});
    }
}
template <int NW>
PG_D void slot_load(const Slot<NW>* s, Kmer<NW>& k, u64& pay, u64& rank) {
    if constexpr (NW == 2) {
        const U256 v = ld256(s);
        k.w[0] = v.a; k.w[1] = v.b; pay = v.c; rank = v.d;
    } else {
        const U128 x = ldcg128(&s->key[0]), y = ldcg128(&s->key[2]), z = ldcg128(&s->payload);
        k.w[0] = x.a; k.w[1] = x.b; k.w[2] = y.a; k.w[3] = y.b; pay = z.a; rank = z.b;
    }
}

// The one linear probe of the global table, from the key's home slot.  CLAIM (find-or-claim): an empty slot is claimed for the key, and
// *claimed tells whether this call claimed it.  Else (find, in a frozen table): an empty slot ends the probe and the call returns ~0, the
// key is absent (search_kmerset, newhash.c:277-318).  ENTRY (find-or-claim at K <= 63): each probe reads the whole 32 B sector (ld256),
// and *entry receives the {payload, rank} that arrived with the key, or {PAYLOAD_FRESH, ~0} (the memset state) after a claim: a hit
// needs no second read.
template <bool CLAIM, bool ENTRY = false, int NW>
PG_D u64 table_probe(const Table<NW>& t, const Kmer<NW>& k, bool* claimed = nullptr, U128* entry = nullptr) {
    static_assert(!ENTRY || (CLAIM && NW == 2), "a 256-bit key's {payload, rank} is in the next sector");
    u64 idx = table_hash(k) & t.mask;
    if (CLAIM) *claimed = false;
    for (;;) {
        Slot<NW>* s = t.slots + idx;
        if constexpr (NW == 2) {
            // 128-bit keys: one 128-bit CAS claims the key
            U128 key, ent;
            if constexpr (ENTRY) {
                const U256 v = ld256(s);
                key = U128{v.a, v.b};
                ent = U128{v.c, v.d};
            } else {
                key = ldcg128(s->key);
            }
            if (!CLAIM && key.a == EMPTY64 && key.b == EMPTY64) return ~0ull;
            if (key.a == k.w[0] && key.b == k.w[1]) {
                if constexpr (ENTRY) *entry = ent;
                return idx;
            }
            if (CLAIM && key.a == EMPTY64 && key.b == EMPTY64) {
                const U128 old = atomicCAS(reinterpret_cast<U128*>(s->key), U128{EMPTY64, EMPTY64}, U128{k.w[0], k.w[1]});   // ATOMG.E.CAS.128
                if (old.a == EMPTY64 && old.b == EMPTY64) {
                    *claimed = true;
                    if (ENTRY) *entry = U128{PAYLOAD_FRESH, EMPTY64};
                    return idx;
                }
                if (old.a == k.w[0] && old.b == k.w[1]) {
                    if (ENTRY) *entry = ldcg128(&s->payload);
                    return idx;
                }
            }
        } else {
            // 256-bit keys: claim {w0|BUSY, w1} with one 128-bit CAS, publish {w2,w3}, then clear BUSY.  A reader only has to wait when
            // the upper halves match (i.e. it is very likely looking at its own key being published).  The claim in shared memory
            // (smem_find_or_claim) takes the same steps with one 64-bit CAS on w0.  A frozen table holds no BUSY bit.
            U128 hi = ldcg128(&s->key[0]);
            if (hi.a == EMPTY64 && hi.b == EMPTY64) {
                if (!CLAIM) return ~0ull;
                const U128 old = atomicCAS(reinterpret_cast<U128*>(&s->key[0]), U128{EMPTY64, EMPTY64}, U128{k.w[0] | BUSY_BIT, k.w[1]});
                if (old.a == EMPTY64 && old.b == EMPTY64) {
                    stcg128(&s->key[2], U128{k.w[2], k.w[3]});
                    // publish with a release store (orders the lower half before it) instead of __threadfence() + exchange: the fence
                    // compiles to MEMBAR.SC + CCTL.IVALL, paid by every new 256-bit key (a third of the instances at K=127)
                    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(&s->key[0]), "l"(k.w[0]) : "memory");
                    *claimed = true;
                    return idx;
                }
                hi = old;
            }
            if ((CLAIM ? hi.a & ~BUSY_BIT : hi.a) == k.w[0] && hi.b == k.w[1]) {
                // wait (acquire) until the lower half has been published, then compare it
                if (CLAIM)
                    do { hi.a = ldacq64(&s->key[0]); } while (hi.a & BUSY_BIT);
                const U128 lo = ldcg128(&s->key[2]);
                if (hi.a == k.w[0] && lo.a == k.w[2] && lo.b == k.w[3]) return idx;
            }
        }
        idx = (idx + 1) & t.mask;
    }
}
// Find-or-claim the slot of key k.  Returns the slot index; *claimed = true if this call inserted the key.
template <int NW>
PG_D u64 table_find_or_claim(const Table<NW>& t, const Kmer<NW>& k, bool* claimed) { return table_probe<true>(t, k, claimed); }
// Read-only lookup (frozen table).  Returns slot index or ~0 when absent.
template <int NW>
PG_D u64 table_find(const Table<NW>& t, const Kmer<NW>& k) { return table_probe<false>(t, k); }

// The updates of a slot's {payload, aux} words, in the global table or in a table in shared memory.  EVERY writer of these words
// (per-instance insert, aggregation, spills, region build, merges) uses the same two 64-bit atomics: atomics of different widths on
// overlapping words are not guaranteed to be atomic with respect to each other.  Order-independent: the final {payload, rank} is a
// pure function of the multiset of instances (SURVEY.md A.3).
// The payload word, whose value was `cur` when read: a 64-bit CAS loop folds `step` into it (payload_apply_n: instances;
// payload_merge: a partial aggregate).  A step that changes nothing (saturated) is read-only.
template <class Step>
PG_D void payload_fold(u64* pay, u64 cur, Step step) {
    for (;;) {
        const u64 nxt = step(cur);
        if (nxt == cur) break;
        const u64 old = atomicCAS(pay, cur, nxt);
        if (old == cur) break;
        cur = old;
    }
}
// The first-occurrence rank: atomicMin, issued only when `earlier` (the rank is below the one read with the payload, where one was read)
PG_D void rank_min(u64* rnk, u64 rank, bool earlier = true) {
    if (earlier) atomicMin(rnk, rank);
}
// A partial aggregate into an entry whose payload word was `cur` when read
PG_D void slot_merge(u64* pay, u64* rnk, u64 cur, u64 agg, u64 rank) {
    payload_fold(pay, cur, [agg](u64 p) { return payload_merge(p, agg); });
    rank_min(rnk, rank);
}

// Fused find-or-claim + apply for one k-mer instance (c identical instances).  Returns true if this call inserted the key.
template <int NW>
PG_D bool table_insert(const Table<NW>& t, const Kmer<NW>& k, unsigned left, unsigned right, u64 rank, unsigned c = 1) {
    bool claimed;
    U128 cur;
    Slot<NW>* s = t.slots + table_probe<true, NW == 2>(t, k, &claimed, &cur);
    if (NW != 2) cur = claimed ? U128{PAYLOAD_FRESH, EMPTY64} : ldcg128(&s->payload);
    payload_fold(&s->payload, cur.a, [=](u64 p) { return payload_apply_n(p, left, right, c); });
    rank_min(&s->aux, rank, rank < cur.b);
    return claimed;
}

// One aggregate {agg, rank} of key k into the global table.  Returns the slot index; *claimed = true if this call inserted the key.
// SOLE (the aggregation's merge mode): a k-mer lives in exactly one bucket and a bucket is aggregated by one CTA at a time, so when this
// call CLAIMS the slot nobody else can be touching its {payload, aux} words: they are written with one plain 16-byte store (probe load
// -> claim CAS -> store: two dependent memory round trips per new key).  Else (the region build's remnant list) several entries may
// hold partials of one key, so a claim merges into the empty slot's {PAYLOAD_FRESH, ~0} like any other writer.  A key that already
// exists is merged with slot_merge.
template <bool SOLE, int NW>
PG_D u64 table_merge(const Table<NW>& t, const Kmer<NW>& k, u64 agg, u64 rank, bool* claimed) {
    const u64 idx = table_find_or_claim(t, k, claimed);
    Slot<NW>* s = t.slots + idx;
    if (SOLE && *claimed) stcg128(&s->payload, U128{agg, rank});
    else slot_merge(&s->payload, &s->aux, *claimed ? PAYLOAD_FRESH : ldcg64(&s->payload), agg, rank);
    return idx;
}

// Find or claim key k in a table in SHARED memory by linear probing from slot `idx` (left at the key's slot).  Key word w of slot j is
// key[j * slot_stride + w * word_stride].  WRAP: the probe wraps around at slot n and gives up after n probes; else it gives up at
// slot n.  Claim: CAS(w0, EMPTY -> w0|BUSY), write the other key words, `fill(j)` (what else the claimer writes before it publishes),
// fence, store w0.  A thread that meets a BUSY w0 whose other bits match waits for the publication (independent thread scheduling: the
// claimer makes progress even inside the same warp).  `room()` is read before each claim: false makes the call give up (a claim limit).
// Returns false when the call gave up; else it has called done(j, claimed) with the key's slot j.
template <int NW, bool WRAP, class Room, class Fill, class Done>
PG_D bool smem_find_or_claim(u64* key, u32 slot_stride, u32 word_stride, u32 n, const Kmer<NW>& k, u32& idx, Room room, Fill fill, Done done) {
    for (u32 probe = 0; WRAP ? probe < n : idx < n; probe++) {
        u64* const sl = key + (u64)idx * slot_stride;
        volatile u64* const ks = sl;
        u64 k0 = ks[0];
        if (k0 == EMPTY64) {
            if (!room()) return false;
            k0 = atomicCAS(sl, EMPTY64, k.w[0] | BUSY_BIT);
            if (k0 == EMPTY64) {
#pragma unroll
                for (int w = 1; w < NW; w++) ks[w * word_stride] = k.w[w];
                fill(idx);
                __threadfence_block();
                ks[0] = k.w[0];
                done(idx, true);
                return true;
            }
        }
        if ((k0 & ~BUSY_BIT) == k.w[0]) {
            while (k0 & BUSY_BIT) k0 = ks[0];
            bool same = true;
#pragma unroll
            for (int w = 1; w < NW; w++) same = same && ks[w * word_stride] == k.w[w];
            if (same) {
                done(idx, false);
                return true;
            }
        }
        idx = WRAP && idx + 1 == n ? 0u : idx + 1;
    }
    return false;
}

template <int NW>
PG_D Kmer<NW> slot_key(const Slot<NW>* s) {
    Kmer<NW> k;
#pragma unroll
    for (int i = 0; i < NW; i++) k.w[i] = s->key[i];
    if (NW == 4) k.w[0] &= ~BUSY_BIT;
    return k;
}
template <int NW>
PG_D bool slot_occupied(const Slot<NW>* s) { return !(s->key[0] == EMPTY64 && s->key[1] == EMPTY64); }

#endif   // __CUDACC__

}   // namespace pgb
