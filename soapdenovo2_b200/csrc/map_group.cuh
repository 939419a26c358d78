// map_group.cuh -- parse1read (prlRead2Ctg.c:260-361) over one read's hit span as k_map_long's CTA computes it (map.cu): a group
// table keyed by contig id, filled by every thread of the CTA, then folded into the three values parse1read's result depends on.
// Host code (tests/host_map_group.cu) compiles the same functions; there the atomics are plain read-modify-writes, and running the
// CTA's threads one after another inside each phase is one of the interleavings the kernel allows.
//
// Why a grouping gives parse1read's result.  parse1read visits the groups of equal contig id in order of first occurrence.  For a
// group of `flag` hits whose first hit is j:
//   counter2 += (K < 32 && flag >= 2) || K > 32,    counter += flag >= multi,
//   and the group wins when flag >= multi and flag > maxOcc (strict), so among the qualifying groups the largest flag wins, and a
//   tie goes to the group visited first: the one with the smallest first j.
// The reported hit is span[first j of the winner].  So (count, first j) per group determines the result, in any visiting order:
// the fold takes sums for counter / counter2 and the max of (count << 32 | ~first j) for the winner.
//
// Overflow.  The table holds `n` groups.  A hit whose contig finds neither its own slot nor a free one is marked HIT_PENDING in the
// span and left for a later round.  Keys are never removed within a round, so an id that fails once fails for the rest of the round
// (every slot its probe passed holds another id, and the table is full): each id is either counted whole in a round or left whole
// for a later one.  The rounds' groups are disjoint, and sums and maxima merge across them.  Each round places at least one new id.
#pragma once

#if defined(__CUDACC__)
#define MG_HD __host__ __device__ __forceinline__
#else
#define MG_HD inline
#endif

namespace pgb {

typedef unsigned long long u64;
typedef unsigned int u32;

constexpr u64 HIT_VALID = 1ull << 63;     // a hit: payload {contig id 0..31, position 32..55, twin 56..57} | smaller << 58
constexpr u64 HIT_PENDING = 1ull << 62;   // not grouped yet (overflow round)
constexpr int HIT_SMALLER_SHIFT = 58;
constexpr u32 GROUP_EMPTY = 0;            // contig ids are >= 1 (atoi(name) > 0 or an ordinal from 1)
constexpr u32 MAP_GROUPS = 1024;          // group slots of one CTA (12 KB of shared memory)

struct GroupTab {
    u32* id;
    u32* cnt;
    u32* first;
    u32 n;   // slots in use, 1..MAP_GROUPS
};
// counter, counter2 and the winner's key (count << 32 | ~first j; 0 = no qualifying group)
struct GroupAcc {
    u32 counter, counter2;
    u64 best;
};

MG_HD u32 mg_cas(u32* p, u32 cmp, u32 v) {
#ifdef __CUDA_ARCH__
    return atomicCAS(p, cmp, v);
#else
    const u32 old = *p;
    if (old == cmp) *p = v;
    return old;
#endif
}
MG_HD void mg_add(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;
#endif
}
MG_HD void mg_min(u32* p, u32 v) {
#ifdef __CUDA_ARCH__
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
MG_HD void mg_max64(u64* p, u64 v) {
#ifdef __CUDA_ARCH__
    atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}

MG_HD void group_clear(const GroupTab& t, int tid, int nthr) {
    for (u32 s = (u32)tid; s < t.n; s += (u32)nthr) { t.id[s] = GROUP_EMPTY; t.cnt[s] = 0; t.first[s] = ~0u; }
}

// count hit j of contig `id` in its group; false when the table holds neither `id` nor a free slot
MG_HD bool group_add(const GroupTab& t, u32 id, u32 j) {
    u32 s = (u32)(((u64)(id * 0x9E3779B1u) * t.n) >> 32);
    for (u32 probe = 0; probe < t.n; probe++) {
        const u32 old = mg_cas(t.id + s, GROUP_EMPTY, id);
        if (old == GROUP_EMPTY || old == id) {
            mg_add(t.cnt + s, 1u);
            mg_min(t.first + s, j);
            return true;
        }
        if (++s == t.n) s = 0;
    }
    return false;
}

// the first round, hit by hit as the scan makes them: h[j] is a hit (HIT_VALID set)
MG_HD void group_add_hit(u64* h, u32 j, const GroupTab& t, int* pending) {
    const u64 v = h[j];
    if (!group_add(t, (u32)v, j)) { h[j] = v | HIT_PENDING; *pending = 1; }
}

// a later round: the pending hits of the span, strided over the CTA
MG_HD void group_round(u64* h, u32 nk, const GroupTab& t, int tid, int nthr, int* pending) {
    for (u32 j = (u32)tid; j < nk; j += (u32)nthr) {
        const u64 v = h[j];
        if (!(v & HIT_PENDING)) continue;
        if (group_add(t, (u32)v, j)) h[j] = v & ~HIT_PENDING;
        else *pending = 1;
    }
}

// this thread's slots into acc
MG_HD void group_fold(const GroupTab& t, int K, u32 multi, int tid, int nthr, GroupAcc* acc) {
    u32 c1 = 0, c2 = 0;
    u64 best = 0;
    for (u32 s = (u32)tid; s < t.n; s += (u32)nthr) {
        if (t.id[s] == GROUP_EMPTY) continue;
        const u32 c = t.cnt[s];
        if ((K < 32 && c >= 2) || K > 32) c2++;
        if (c < multi) continue;
        c1++;
        const u64 key = (u64)c << 32 | (u64)(~t.first[s]);
        if (key > best) best = key;
    }
    if (c1) mg_add(&acc->counter, c1);
    if (c2) mg_add(&acc->counter2, c2);
    if (best) mg_max64(&acc->best, best);
}

MG_HD u32 group_best_j(const GroupAcc& a) { return ~(u32)a.best; }

}   // namespace pgb
