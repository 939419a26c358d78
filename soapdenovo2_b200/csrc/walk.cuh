// walk.cuh -- the unipath walk of tip clipping (tips.cu) and edge emission (edges.cu): from one link of a node, through linear
// nodes (one link on each side), to the first node that is not linear.
//
// Reference (standardPregraph/): clipTipFromNode cutTipPreGraph.c:43-346, startEdgeFromNode / stringBeads node2edge.c:86-352,
// dislink2prevUncertain node2edge.c (the terminal's link back along the walk).
#pragma once
#include "table.cuh"

namespace pgb {

// A link of a node: (side << 2) | base.  Side 0 holds the right links r[base] (the base that follows the node's k-mer), side 1 the
// left links l[base] (the base that follows its reverse complement).  Edge starts are numbered with the same three bits (edges.cu).
PG_HD int link_shift(unsigned link) { return ((link & 4u) ? 0 : PL_R_SHIFT) + 6 * (int)(link & 3u); }
PG_HD unsigned link_count(u64 p, unsigned link) { return (unsigned)(p >> link_shift(link)) & 63u; }
PG_HD u64 link_clear(u64 p, unsigned link) { return p & ~(63ull << link_shift(link)); }

enum WalkStep { WALK_GO, WALK_STOP, WALK_GIVE_UP };     // a visitor's answer at a linear node
enum WalkStatus { WALK_REACHED, WALK_GAVE_UP, WALK_MISS };

template <int NW>
struct WalkEnd {
    int status;
    u32 length;     // nodes read after the start, the terminal included
    Kmer<NW> frm;   // the start node, read along the walk
    // WALK_REACHED only:
    u64 slot;       // the terminal node
    int sm;         // the terminal's k-mer read along the walk is its canonical form
    Kmer<NW> to;    // the terminal, read along the walk
    Kmer<NW> pre;   // the node before the terminal, read along the walk
    unsigned rev;   // the terminal's link back to `pre`
};

// Walk from node `start` through its link `link`.  visit(i, slot, sm, k-mer read along the walk, payload) is called at the i-th node
// after the start (i = 1, 2, ...) while that node is linear: WALK_GO steps on, WALK_STOP makes the node the terminal, WALK_GIVE_UP ends
// the walk without one.  The first node that is not linear is the terminal.  A k-mer the table does not hold ends the walk with
// WALK_MISS.  A node is read along the walk in its canonical orientation when the k-mer is not larger than its reverse complement.
template <int NW, class Visit>
__device__ __forceinline__ WalkEnd<NW> unipath_walk(const Table<NW>& tab, const KParams<NW>& kp, u64 start, unsigned link, Visit& visit) {
    WalkEnd<NW> e;
    const Kmer<NW> key = slot_key(tab.slots + start);
    e.frm = (link & 4u) ? krc_n(key, kp.K) : key;
    e.length = 0;
    Kmer<NW> pre = e.frm;   // apart from e: kfirst indexes it dynamically, which would put all of e in local memory
    Kmer<NW> ori = knext(e.frm, (link & 4u) ? (link & 3u) ^ 2u : link & 3u, kp);
    for (;;) {
        const Kmer<NW> rc = krc_n(ori, kp.K);
        const int sm = !kless(rc, ori);
        const u64 os = table_find(tab, kcanon(ori, rc, sm));
        if (os == ~0ull) { e.status = WALK_MISS; return e; }
        e.length++;
        const u64 po = tab.slots[os].payload;
        const int step = (po & PL_LINEAR) ? visit(e.length, os, sm, ori, po) : WALK_STOP;
        if (step == WALK_GIVE_UP) { e.status = WALK_GAVE_UP; return e; }
        if (step == WALK_STOP) {
            const unsigned c = kfirst(pre, kp);
            e.status = WALK_REACHED; e.slot = os; e.sm = sm; e.to = ori; e.pre = pre;
            e.rev = sm ? 4u | c : c ^ 2u;
            return e;
        }
        pre = ori;
        ori = knext(ori, sm ? (unsigned)pl_first_r(po) : (unsigned)pl_first_l(po) ^ 2u, kp);
    }
}

}   // namespace pgb
