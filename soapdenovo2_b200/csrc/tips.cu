// tips.cu -- K5: tip clipping on the k-mer graph, bit-exact with the reference's SEQUENTIAL mutate-while-iterating
// loops, but executed in parallel on the GPU.
//
// Reference (standardPregraph/cutTipPreGraph.c):
//   clipTipFromNode :43-346   walk from a dead-end node (in=0,out=1 | in=1,out=0) over linear nodes (<= 2K of them) to the
//                             first non-linear node `out`; THIN pass: stop at the first non-single node instead.
//                             out is a dead end too  -> delete both ends ("isolated")
//                             THIN                   -> delete start, unlink at out, out.linear = 0
//                             else if the tip's link at out is weaker than out's strongest link on that side
//                                                    -> delete start, unlink, out.linear = 1 if out became 1-in-1-out
//   removeSingleTips :363-399 one sweep in iteration order over `!linear && !deleted && single` nodes, THIN = 1 (only when -d 0)
//   removeMinorTips  :414-488 sweeps in iteration order over `!linear && !deleted` nodes until a sweep clips nothing
//   thread_mark      :532-564 re-mark 1-in-1-out nodes linear (skips deleted / already linear)
// The walk itself is walk.cuh's, shared with the edges.
//
// Why this can be parallel and still exact:
//   THIN pass.  Chain nodes are linear AND single and are never written; start nodes are single dead ends whose only link
//   is never cleared.  Hence every walk, its end node `out` and the link it would clear are independent of the processing
//   order.  Only the per-junction sequence matters (isolated-or-not depends on how many links `out` still has), so the
//   candidates are resolved in rounds: a candidate commits when it holds the minimum iteration index on both `out` and
//   its own start node; at most one arrival per link => <= 9 rounds.
//   Minor pass.  Walks are NOT static (out.linear = 1 merges chains).  Speculate a window of pending candidates on the
//   current state; a candidate is dirty if any node it read was written by a pending clip with a smaller iteration
//   index; commit exactly the prefix below the first dirty candidate (and below any node that a committed clip turns
//   into a NEW dead end further down the sweep).  The first pending candidate is always clean => progress, and every
//   committed candidate saw precisely the state the sequential loop would have shown it.
#include "engine_impl.cuh"
#include "scan.cuh"
#include "walk.cuh"
#include <algorithm>

namespace pgb {

struct TipRec {
    u64 n1_slot;
    u64 out_slot;
    u32 code;     // bits 0..2: the link to clear at out (walk.cuh); 8 makes out linear, 16 makes it a dead end, 32 no out (THIN)
    u32 state;    // THIN: 0 pending, 1 done.   minor: decision 0 none / 1 clip / 2 isolated
};

// A tip starts at a dead end, (in, out) = (0, 1) or (1, 0), and leaves through its only link; ~0u: not a dead end
__device__ __forceinline__ unsigned tip_link(u64 p) {
    if (pl_nl(p) == 0 && pl_nr(p) == 1) return (unsigned)pl_first_r(p);
    if (pl_nl(p) == 1 && pl_nr(p) == 0) return 4u | (unsigned)pl_first_l(p);
    return ~0u;
}

// clipTipFromNode's walk: the THIN pass stops at the first linear node that is not single, and a walk gives up when its count of
// nodes (the start included) passes `cut`.  read(slot) sees each linear node the walk reads.
template <class Read>
struct TipVisit {
    int cut;
    bool thin;
    Read read;
    template <int NW>
    __device__ int operator()(u32 i, u64 slot, int, const Kmer<NW>&, u64 po) {
        read(slot);
        if (thin && !(po & PL_SINGLE)) return WALK_STOP;
        return (int)i + 1 > cut ? WALK_GIVE_UP : WALK_GO;
    }
};

struct NoVisit {
    __device__ void operator()(u64) const {}
};

// ---------------------------------------------------------------- candidate lists (compaction in iteration order)
template <int NW>
struct CandIn {
    const Slot<NW>* slots;
    const u64* order;
    bool thin;
    __device__ u64 operator()(u64 i) const {
        u64 p = slots[order[i]].payload;
        if (p & (PL_LINEAR | PL_DELETED)) return 0;
        if (thin && !(p & PL_SINGLE)) return 0;
        int in = pl_nl(p), on = pl_nr(p);
        return (in + on == 1) ? 1 : 0;   // dead end: (0,1) or (1,0); everything else returns 0 from clipTipFromNode at once
    }
};
struct CandOut {
    u64* list;
    __device__ void operator()(u64 i, u64 prefix, u64 v) const { if (v) list[prefix] = i; }
};

// ---------------------------------------------------------------- THIN pass
template <int NW>
__global__ void __launch_bounds__(256) k_thin_walk(Table<NW> tab, KParams<NW> kp, const u64* order, const u64* cand, u64 n, int cut, TipRec* rec, u64* err) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 s1 = order[cand[i]];
        TipRec r;
        r.n1_slot = s1; r.out_slot = 0;
        r.code = 32u;   // no `out` node (too long, or not a tip): nothing to do, and k_thin_unmark must not follow out_slot
        r.state = 1u;
        const unsigned link = tip_link(tab.slots[s1].payload);
        if (link != ~0u) {
            TipVisit<NoVisit> tv{cut, true, NoVisit()};
            WalkEnd<NW> w = unipath_walk(tab, kp, s1, link, tv);
            if (w.status == WALK_REACHED) { r.out_slot = w.slot; r.code = w.rev; r.state = 0u; }
            if (w.status == WALK_MISS) atomicAdd(err, 1ull);
        }
        rec[i] = r;
    }
}
template <int NW>
__global__ void __launch_bounds__(256) k_thin_mark(Table<NW> tab, const u64* cand, u64 n, const TipRec* rec, u64* mark) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        if (rec[i].state) continue;
        u64 me = cand[i];
        atomicMin(&mark[tab.slots[rec[i].out_slot].aux], me);
        atomicMin(&mark[me], me);
    }
}
template <int NW>
__global__ void __launch_bounds__(256) k_thin_commit(Table<NW> tab, const u64* cand, u64 n, TipRec* rec, const u64* mark, u64* counters) {
    unsigned tips = 0, pending = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        if (rec[i].state) continue;
        u64 me = cand[i];
        Slot<NW>* out = tab.slots + rec[i].out_slot;
        Slot<NW>* n1 = tab.slots + rec[i].n1_slot;
        if (mark[out->aux] != me || mark[me] != me) { pending++; continue; }
        rec[i].state = 1;
        if (n1->payload & PL_DELETED) continue;     // deleted by the other end of an isolated path earlier in the sweep
        u64 po = out->payload;
        tips++;
        n1->payload |= PL_DELETED;
        if (pl_nl(po) + pl_nr(po) == 1) { out->payload = po | PL_DELETED; continue; }
        out->payload = link_clear(po, rec[i].code & 7u) & ~PL_LINEAR;
    }
    if (tips) atomicAdd(&counters[C_MISC0], (u64)tips);
    if (pending) atomicAdd(&counters[C_MISC1], (u64)pending);
}
template <int NW>
__global__ void __launch_bounds__(256) k_thin_unmark(Table<NW> tab, const u64* cand, u64 n, const TipRec* rec, u64* mark) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        if (rec[i].code & 32u) continue;   // never marked anything (its out_slot is 0: following it reads slot 0's aux, ~0 when that slot is empty)
        mark[tab.slots[rec[i].out_slot].aux] = EMPTY64;
        mark[cand[i]] = EMPTY64;
    }
}

// ---------------------------------------------------------------- re-mark linear nodes (thread_mark, cutTipPreGraph.c:532-564)
template <int NW>
__global__ void __launch_bounds__(256) k_remark(Table<NW> tab, u64* counters) {
    unsigned c = 0;
    u64 n = tab.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        Slot<NW>* s = tab.slots + i;
        if (!slot_occupied(s)) continue;
        u64 p = s->payload;
        if (p & (PL_DELETED | PL_LINEAR)) continue;
        if (pl_nl(p) == 1 && pl_nr(p) == 1) { s->payload = p | PL_LINEAR; c++; }
    }
    if (c) atomicAdd(&counters[C_MISC0], (u64)c);
}

// ---------------------------------------------------------------- minor pass
// decision of candidate `s1` on the current (read-only) state
template <int NW>
struct MinorDecision {
    int decision;      // 0 none, 1 clip (unlink), 2 isolated
    u64 out_slot;
    u32 code;
    bool makes_linear;
    bool makes_deadend;
};
template <int NW, class Visit>
__device__ MinorDecision<NW> minor_decide(const Table<NW>& tab, const KParams<NW>& kp, u64 s1, int cut, Visit visit, u64* err) {
    MinorDecision<NW> d;
    d.decision = 0; d.out_slot = 0; d.code = 0; d.makes_linear = false; d.makes_deadend = false;
    u64 p1 = tab.slots[s1].payload;
    visit(s1);
    if (p1 & (PL_LINEAR | PL_DELETED)) return d;   // no longer a candidate at its turn
    const unsigned link = tip_link(p1);
    if (link == ~0u) return d;
    TipVisit<Visit> tv{cut, false, visit};
    WalkEnd<NW> w = unipath_walk(tab, kp, s1, link, tv);
    if (w.status == WALK_MISS) { atomicAdd(err, 1ull); return d; }
    if (w.status == WALK_GAVE_UP) return d;
    visit(w.slot);
    d.out_slot = w.slot;
    u64 po = tab.slots[w.slot].payload;
    if (pl_nl(po) + pl_nr(po) == 1) { d.decision = 2; return d; }
    unsigned mx = 0;
    for (unsigned c = 0; c < 4; c++) mx = max(mx, link_count(po, (w.rev & 4u) | c));
    d.code = w.rev;
    if (link_count(po, w.rev) < mx) {
        d.decision = 1;
        u64 pn = link_clear(po, w.rev);
        int in = pl_nl(pn), on = pl_nr(pn);
        d.makes_linear = (in == 1 && on == 1);
        // out turns into a NEW dead end that the same sweep will visit if it lies further down the iteration order
        d.makes_deadend = !d.makes_linear && (in + on == 1) && !(pn & (PL_DELETED));
    }
    return d;
}

template <int NW>
struct MarkVisit {
    const Slot<NW>* slots;
    const u64* mark;
    u64 me;
    bool* dirty;
    __device__ void operator()(u64 slot) const {
        if (mark[slots[slot].aux] < me) *dirty = true;
    }
};

// phase A: decide on the current state, publish the nodes a clip would WRITE
template <int NW>
__global__ void __launch_bounds__(128) k_minor_decide(Table<NW> tab, KParams<NW> kp, const u64* order, const u64* win, u64 n, int cut, TipRec* rec, u64* mark, u64* err) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 me = win[i];
        u64 s1 = order[me];
        MinorDecision<NW> d = minor_decide(tab, kp, s1, cut, NoVisit(), err);
        TipRec r;
        r.n1_slot = s1; r.out_slot = d.out_slot; r.code = d.code | (d.makes_linear ? 8u : 0u) | (d.makes_deadend ? 16u : 0u); r.state = (u32)d.decision;
        rec[i] = r;
        if (d.decision) {
            atomicMin(&mark[tab.slots[d.out_slot].aux], me);
            atomicMin(&mark[me], me);
        }
    }
}
// phase B: dirty detection (re-walk, compare marks) + barrier of clean clips; reduces into ctl[0] = min dirty ord, ctl[1] = min barrier
template <int NW>
__global__ void __launch_bounds__(128) k_minor_check(Table<NW> tab, KParams<NW> kp, const u64* order, const u64* win, u64 n, int cut, const TipRec* rec, const u64* mark, u64* ctl, u64* err) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 me = win[i];
        bool dirty = false;
        MarkVisit<NW> mv{tab.slots, mark, me, &dirty};
        minor_decide(tab, kp, order[me], cut, mv, err);
        if (dirty) { atomicMin(&ctl[0], me); continue; }
        if (rec[i].state == 1 && (rec[i].code & 16u)) {
            u64 b = tab.slots[rec[i].out_slot].aux;
            if (b > me) atomicMin(&ctl[1], b);
        }
    }
}
// phase C: commit everything below the frontier; collect new dead ends; clear marks
template <int NW>
__global__ void __launch_bounds__(128) k_minor_commit(Table<NW> tab, const u64* win, u64 n, const TipRec* rec, u64* mark, u64 frontier, u64* extra, u64* ctl) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 me = win[i];
        TipRec r = rec[i];
        if (r.state) { mark[tab.slots[r.out_slot].aux] = EMPTY64; mark[me] = EMPTY64; }
        if (me >= frontier) {
            u64 k = atomicAdd(&ctl[3], 1ull);   // stays pending
            extra[k] = me;
            continue;
        }
        if (!r.state) continue;
        Slot<NW>* out = tab.slots + r.out_slot;
        Slot<NW>* n1 = tab.slots + r.n1_slot;
        atomicAdd(&ctl[2], 1ull);              // tip_c++ / flag++
        n1->payload |= PL_DELETED;
        if (r.state == 2) { out->payload |= PL_DELETED; continue; }
        u64 po = link_clear(out->payload, r.code & 7u);
        if (r.code & 8u) po |= PL_LINEAR;
        out->payload = po;
        if (r.code & 16u) {
            u64 b = out->aux;
            if (b > me) { u64 k = atomicAdd(&ctl[3], 1ull); extra[k] = b; }   // visited later in this very sweep
        }
    }
}

template <int NW>
void EngineT<NW>::remove_tips(TipStats* st) {
    if (!order_buf_.p) throw std::runtime_error("pgb200: remove_tips before build_layout");
    const int cut = 2 * prm_.K;
    const int D = (int)(signed char)prm_.D;
    const u64 N = n_nodes_;
    u64* order = order_buf_.template as<u64>();
    DevBuf markb, candb, recb, scratch, ctlb, errb;
    markb.alloc((N + 1) * sizeof(u64));
    PG_CUDA(cudaMemsetAsync(markb.p, 0xFF, (N + 1) * sizeof(u64), st_));
    candb.alloc((N + 1) * sizeof(u64));
    scratch.alloc(scan_scratch_elems(N) * sizeof(u64));
    errb.alloc(sizeof(u64));
    PG_CUDA(cudaMemsetAsync(errb.p, 0, sizeof(u64), st_));
    u64* mark = markb.template as<u64>();
    u64* cand = candb.template as<u64>();
    u64* err = errb.template as<u64>();
    auto check_err = [&]() {
        u64 e;
        PG_CUDA(cudaMemcpyAsync(&e, err, sizeof e, cudaMemcpyDeviceToHost, st_));
        sync();
        if (e) throw std::runtime_error("pgb200: tip walk fell off the k-mer table (the reference exits here too: 'Kmer ... is not found')");
    };
    auto remark = [&]() -> u64 {
        PG_CUDA(cudaMemsetAsync(d_cnt_ + C_MISC0, 0, sizeof(u64), st_));
        k_remark<NW><<<n_sm_ * 8, 256, 0, st_>>>(tab_, d_cnt_);
        PG_CUDA(cudaGetLastError());
        read_counters();
        return h_cnt_[C_MISC0];
    };
    auto build_cands = [&](bool thin) -> u64 {
        device_scan(CandIn<NW>{tab_.slots, order, thin}, CandOut{cand}, N, scratch.template as<u64>(), d_cnt_ + C_MISC2, st_);
        read_counters();
        return h_cnt_[C_MISC2];
    };

    if (D == 0) {   // pregraph.c:106-113
        u64 nc = build_cands(true);
        if (nc) {
            recb.alloc(nc * sizeof(TipRec));
            TipRec* rec = recb.template as<TipRec>();
            unsigned blocks = (unsigned)std::min<u64>((nc + 255) / 256, (u64)n_sm_ * 16);
            k_thin_walk<NW><<<blocks, 256, 0, st_>>>(tab_, kp_, order, cand, nc, cut, rec, err);
            PG_CUDA(cudaGetLastError());
            check_err();
            PG_CUDA(cudaMemsetAsync(d_cnt_ + C_MISC0, 0, sizeof(u64), st_));
            for (int round = 0;; round++) {
                PG_CUDA(cudaMemsetAsync(d_cnt_ + C_MISC1, 0, sizeof(u64), st_));
                k_thin_mark<NW><<<blocks, 256, 0, st_>>>(tab_, cand, nc, rec, mark);
                k_thin_commit<NW><<<blocks, 256, 0, st_>>>(tab_, cand, nc, rec, mark, d_cnt_);
                k_thin_unmark<NW><<<blocks, 256, 0, st_>>>(tab_, cand, nc, rec, mark);
                PG_CUDA(cudaGetLastError());
                read_counters();
                st->rounds++;
                st->thin_rounds++;
                if (h_cnt_[C_MISC1] == 0) break;
                if (round > 64) throw std::runtime_error("pgb200: THIN tip resolution did not converge");
            }
            st->single_tips = h_cnt_[C_MISC0];
        }
        st->single_relinear = remark();
    }

    // ---- removeMinorTips: sweeps until nothing is clipped
    ctlb.alloc(8 * sizeof(u64));
    u64* ctl = ctlb.template as<u64>();
    DevBuf winb, win2b;
    u64 total_minor = 0;
    // PGB200_TIP_WINDOW=n: every window takes n list entries (no adaptation).  The result is the same at any n; n = 1..3 cut every
    // conflict across windows, so that tests reach the dirty / barrier / re-queue paths on small graphs.
    const u64 fixed_window = getenv("PGB200_TIP_WINDOW") ? (u64)std::max(1L, atol(getenv("PGB200_TIP_WINDOW"))) : 0;
    for (int sweep = 0;; sweep++) {
        u64 nc = build_cands(false);
        u64 clipped = 0;
        if (nc) {
            // pending candidates: a static sorted list (cand[lo..nc)) plus a small unsorted "extra" set
            std::vector<u64> h_extra;
            u64 lo = 0;
            u64 Wn = fixed_window ? fixed_window : 4096;
            std::vector<u64> h_cand;   // fetched lazily in pieces
            while (lo < nc || !h_extra.empty()) {
                // window = next Wn list entries + every extra below the window end
                u64 take = std::min<u64>(Wn, nc - lo);
                u64 wend = EMPTY64;     // ord of the first list candidate beyond the window
                if (lo + take < nc) PG_CUDA(cudaMemcpyAsync(&wend, cand + lo + take, sizeof(u64), cudaMemcpyDeviceToHost, st_));
                sync();
                std::vector<u64> ex_in, ex_out;
                for (u64 e : h_extra) (e < wend ? ex_in : ex_out).push_back(e);
                u64 nwin = take + ex_in.size();
                winb.ensure((nwin + 1) * sizeof(u64));
                win2b.ensure((2 * nwin + 16) * sizeof(u64));
                recb.ensure((nwin + 1) * sizeof(TipRec));
                u64* win = winb.template as<u64>();
                if (take) PG_CUDA(cudaMemcpyAsync(win, cand + lo, take * sizeof(u64), cudaMemcpyDeviceToDevice, st_));
                if (!ex_in.empty()) PG_CUDA(cudaMemcpyAsync(win + take, ex_in.data(), ex_in.size() * sizeof(u64), cudaMemcpyHostToDevice, st_));
                u64 init[4] = {EMPTY64, EMPTY64, 0, 0};
                PG_CUDA(cudaMemcpyAsync(ctl, init, sizeof init, cudaMemcpyHostToDevice, st_));
                TipRec* rec = recb.template as<TipRec>();
                unsigned blocks = (unsigned)std::min<u64>((nwin + 127) / 128, (u64)n_sm_ * 16);
                k_minor_decide<NW><<<blocks, 128, 0, st_>>>(tab_, kp_, order, win, nwin, cut, rec, mark, err);
                k_minor_check<NW><<<blocks, 128, 0, st_>>>(tab_, kp_, order, win, nwin, cut, rec, mark, ctl, err);
                PG_CUDA(cudaGetLastError());
                u64 h_ctl[4];
                PG_CUDA(cudaMemcpyAsync(h_ctl, ctl, sizeof h_ctl, cudaMemcpyDeviceToHost, st_));
                sync();
                u64 frontier = std::min(std::min(h_ctl[0], h_ctl[1]), wend);
                k_minor_commit<NW><<<blocks, 128, 0, st_>>>(tab_, win, nwin, rec, mark, frontier, win2b.template as<u64>(), ctl);
                PG_CUDA(cudaGetLastError());
                PG_CUDA(cudaMemcpyAsync(h_ctl, ctl, sizeof h_ctl, cudaMemcpyDeviceToHost, st_));
                sync();
                clipped += h_ctl[2];
                st->rounds++;
                st->minor_windows++;
                if (frontier < wend) {
                    if (frontier == h_ctl[0]) st->dirty_frontiers++;
                    else st->barrier_frontiers++;
                }
                const u64 survivors_extra = (u64)std::count_if(ex_in.begin(), ex_in.end(), [&](u64 e) { return e >= frontier; });
                // survivors of the window (ord >= frontier) + new dead ends
                std::vector<u64> back(h_ctl[3]);
                if (h_ctl[3]) PG_CUDA(cudaMemcpyAsync(back.data(), win2b.p, h_ctl[3] * sizeof(u64), cudaMemcpyDeviceToHost, st_));
                sync();
                // list entries that stay pending are re-read from the list itself: advance `lo` to the first entry >= frontier
                // (entries of the window that are >= frontier came back in `back` too; drop those that belong to the list)
                u64 committed_list = 0;
                if (take) {
                    std::vector<u64> wl(take);
                    PG_CUDA(cudaMemcpyAsync(wl.data(), cand + lo, take * sizeof(u64), cudaMemcpyDeviceToHost, st_));
                    sync();
                    committed_list = std::lower_bound(wl.begin(), wl.end(), frontier) - wl.begin();
                    // list members that came back are exactly wl[committed_list..take): remove them from `back`
                    std::vector<u64> keep;
                    for (u64 e : back) if (!std::binary_search(wl.begin() + committed_list, wl.end(), e)) keep.push_back(e);
                    back.swap(keep);
                }
                lo += committed_list;
                st->requeued += back.size();
                st->deadends_ahead += back.size() - survivors_extra;
                if (prm_.verbose) {   // committed clips that made a new dead end, ahead or behind (rec and win are still those of this window)
                    std::vector<TipRec> hr(nwin);
                    std::vector<u64> hw(nwin);
                    PG_CUDA(cudaMemcpyAsync(hr.data(), rec, nwin * sizeof(TipRec), cudaMemcpyDeviceToHost, st_));
                    PG_CUDA(cudaMemcpyAsync(hw.data(), win, nwin * sizeof(u64), cudaMemcpyDeviceToHost, st_));
                    sync();
                    u64 made = 0;
                    for (u64 i = 0; i < nwin; i++) made += hw[i] < frontier && hr[i].state == 1 && (hr[i].code & 16u);
                    st->deadends_behind += made - (back.size() - survivors_extra);
                }
                h_extra = ex_out;
                for (u64 e : back) h_extra.push_back(e);
                // adapt the window to the observed commit run length
                u64 done = committed_list;
                if (!fixed_window) Wn = std::min<u64>(1u << 18, std::max<u64>(1024, done * 2));
                if (st->rounds > (1ull << 26)) throw std::runtime_error("pgb200: minor tip sweeps did not converge");
            }
        }
        check_err();
        st->minor_cycles.push_back(clipped);
        total_minor += clipped;
        if (!clipped) break;
    }
    st->minor_tips = total_minor;
    st->minor_relinear = remark();
    if (prm_.verbose)
        fprintf(stderr, "[pgb200] remove_tips: %llu THIN round(s), %llu minor window(s), %llu dirty frontier(s), %llu barrier frontier(s), "
                "%llu re-queued, %llu new dead end(s) queued ahead, %llu behind\n", (unsigned long long)st->thin_rounds,
                (unsigned long long)st->minor_windows, (unsigned long long)st->dirty_frontiers, (unsigned long long)st->barrier_frontiers,
                (unsigned long long)st->requeued, (unsigned long long)st->deadends_ahead, (unsigned long long)st->deadends_behind);
}

template void EngineT<2>::remove_tips(TipStats*);
template void EngineT<4>::remove_tips(TipStats*);

}   // namespace pgb
