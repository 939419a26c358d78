// edges.cu -- K6: unipath compaction (k-mer graph -> edges), edge ids, .edge text, (K+1)-mer patch table, vertices.
//
// Reference (standardPregraph/): make_edge node2edge.c:366-411, startEdgeFromNode :237-352, stringBeads :86-218,
// check_iden_kmerList :624-649, merge_linearV2 :430-609, output_1edge output_pregraph.c:88-110, output_vertex :50-86.
//
// The reference walks sequentially: for every non-linear, non-deleted node in iteration order, for every non-zero right
// link (base 0..3) then left link, follow linear nodes to the next non-linear node, emit the edge, number it, and CLEAR
// the link at both ends -- which is what stops the same unipath from being emitted again from its other end.
// Parallel, exact restatement used here:
//   start      := (node, side, base); key(start) = iteration index * 8 + side * 4 + base   (the sequential visiting order)
//   every start is walked independently (one thread each); rev(start) := the link the walk would clear at its far end
//   a start is emitted iff no EMITTED start with a smaller key has it as its rev()   (resolved in rounds; with symmetric
//   links that is simply "the smaller key of each {start, rev(start)} pair", and start == rev(start) is a palindrome)
//   edge id   := 1 + exclusive prefix over emitted starts of (1 + bal_edge)      (edge_c += bal_edge reserves the twin)
//   text      := prefix sum of per-edge text lengths, then every edge writes its own record
// Interior nodes get {edgeId overlaid on l_links|cov, twin, inEdge} exactly like the reference's union (newhash.h:83-102).
// The walk is walk.cuh's, shared with tip clipping; a start's (side, base) is its link there, and rev(start) the walk's `rev`.
#include "engine_impl.cuh"
#include "scan.cuh"
#include "patch.cuh"
#include "walk.cuh"
#include <algorithm>

namespace pgb {

struct EdgeRec {
    u64 rev_id;
    u64 symbol;
    u32 length;
    u32 hdr_len;
    u32 text_len;
    u32 status;   // 0 unknown, 1 emitted, 2 suppressed
};

// ---------------------------------------------------------------- formatting helpers
__device__ __forceinline__ int dec_len(u64 v) { int n = 1; while (v >= 10) { v /= 10; n++; } return n; }
__device__ __forceinline__ int hex_len(u64 v) { return v ? (64 - __clzll((long long)v) + 3) / 4 : 1; }
__device__ __forceinline__ char* put_dec(char* p, u64 v) { int n = dec_len(v); for (int i = n - 1; i >= 0; i--) { p[i] = '0' + (char)(v % 10); v /= 10; } return p + n; }
__device__ __forceinline__ char* put_hex(char* p, u64 v) { int n = hex_len(v); for (int i = n - 1; i >= 0; i--) { unsigned d = v & 15; p[i] = d < 10 ? '0' + d : 'a' + d - 10; v >>= 4; } return p + n; }
__device__ __forceinline__ char* put_str(char* p, const char* s) { while (*s) *p++ = *s++; return p; }
template <int NW>
__device__ int kmer_hex_len(const Kmer<NW>& k, int out_words) {   // "%llx %llx[ %llx %llx]"
    int n = out_words - 1;
    for (int w = 0; w < out_words; w++) n += hex_len(kout_word(k, w, out_words));
    return n;
}
template <int NW>
__device__ char* put_kmer_hex(char* p, const Kmer<NW>& k, int out_words) {
    for (int w = 0; w < out_words; w++) { if (w) *p++ = ' '; p = put_hex(p, kout_word(k, w, out_words)); }
    return p;
}
__device__ __forceinline__ u32 edge_cvg(u64 symbol, u32 length) {   // node2edge.c:585-592 (integer division first)
    if (length <= 1) return 0;
    u64 v = symbol / (length - 1) * 10;
    return v > 16000 ? 16000u : (u32)v;
}

// ---------------------------------------------------------------- start enumeration
template <int NW>
struct StartIn {
    const Slot<NW>* slots;
    const u64* order;
    __device__ u64 operator()(u64 i) const {
        u64 p = slots[order[i]].payload;
        if (p & (PL_LINEAR | PL_DELETED)) return 0;
        return (u64)(pl_nl(p) + pl_nr(p));
    }
};
template <int NW>
struct StartOut {
    const Slot<NW>* slots;
    const u64* order;
    u64* starts;
    __device__ void operator()(u64 i, u64 prefix, u64 v) const {
        if (!v) return;
        u64 p = slots[order[i]].payload;
        u64 k = prefix;
        for (int c = 0; c < 4; c++) if (pl_r(p, c)) starts[k++] = i * 8 + c;        // right links first ...
        for (int c = 0; c < 4; c++) if (pl_l(p, c)) starts[k++] = i * 8 + 4 + c;    // ... then left links
    }
};

__device__ __forceinline__ u64 bsearch_u64(const u64* a, u64 n, u64 key) {   // index of key in sorted a, or ~0
    u64 lo = 0, hi = n;
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (a[mid] < key) lo = mid + 1; else hi = mid; }
    return (lo < n && a[lo] == key) ? lo : ~0ull;
}

struct SymbolVisit {
    u64 symbol;
    template <int NW>
    __device__ int operator()(u32, u64, int, const Kmer<NW>&, u64 po) {
        symbol += pl_l(po, 0) + pl_l(po, 1) + pl_l(po, 2) + pl_l(po, 3);
        return WALK_GO;
    }
};

template <int NW>
__global__ void __launch_bounds__(128) k_edge_walk(Table<NW> tab, KParams<NW> kp, const u64* order, const u64* starts, u64 S, int out_words, EdgeRec* rec, u64* err) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < S; j += (u64)gridDim.x * blockDim.x) {
        u64 sid = starts[j];
        SymbolVisit sv{0};
        WalkEnd<NW> end = unipath_walk(tab, kp, order[sid >> 3], (unsigned)(sid & 7), sv);
        EdgeRec r;
        r.status = 0; r.symbol = sv.symbol; r.length = end.length; r.rev_id = EMPTY64; r.hdr_len = 0; r.text_len = 0;
        if (end.status != WALK_REACHED) { atomicAdd(err, 1ull); rec[j] = r; continue; }
        const Slot<NW>* T = tab.slots + end.slot;
        if (!(T->payload & PL_DELETED)) r.rev_id = T->aux * 8 + end.rev;   // the start at the far end that walks this path back
        u32 cvg = edge_cvg(sv.symbol, end.length);
        // ">length %d,%llx %llx,%llx %llx,cvg %d, %d\n"
        r.hdr_len = 8 + dec_len(end.length) + 1 + kmer_hex_len(end.frm, out_words) + 1 + kmer_hex_len(end.to, out_words) + 1 + 4 + dec_len(cvg) + 2 + 1 + 1;
        r.text_len = r.hdr_len + end.length + (end.length + 99) / 100;
        rec[j] = r;
    }
}

__global__ void __launch_bounds__(256) k_edge_claim(const u64* starts, u64 S, const EdgeRec* rec, u64* claim) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < S; j += (u64)gridDim.x * blockDim.x) {
        if (rec[j].status == 2) continue;
        u64 r = rec[j].rev_id, me = starts[j];
        if (r == EMPTY64 || !(me < r)) continue;
        u64 t = bsearch_u64(starts, S, r);
        if (t != ~0ull) atomicMin(&claim[t], me);
    }
}
__global__ void __launch_bounds__(256) k_edge_resolve(const u64* starts, u64 S, EdgeRec* rec, const u64* claim, u64* unresolved) {
    unsigned left = 0;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < S; j += (u64)gridDim.x * blockDim.x) {
        if (rec[j].status) continue;
        u64 c = claim[j];
        if (c == EMPTY64) { rec[j].status = 1; continue; }
        u64 t = bsearch_u64(starts, S, c);
        u32 ts = *((volatile u32*)&rec[t].status);
        if (ts == 1) rec[j].status = 2; else left++;
    }
    if (left) atomicAdd(unresolved, (u64)left);
}

struct IdIn {
    const u64* starts;
    const EdgeRec* rec;
    __device__ u64 operator()(u64 j) const { return rec[j].status == 1 ? (rec[j].rev_id == starts[j] ? 1ull : 2ull) : 0ull; }
};
struct TextIn {
    const EdgeRec* rec;
    __device__ u64 operator()(u64 j) const { return rec[j].status == 1 ? (u64)rec[j].text_len : 0ull; }
};
struct Len1In {
    const EdgeRec* rec;
    __device__ u64 operator()(u64 j) const { return rec[j].status == 1 && rec[j].length == 1; }
};
struct EmIn {
    const EdgeRec* rec;
    __device__ u64 operator()(u64 j) const { return rec[j].status == 1; }
};
struct EmNoRevIn {   // emitted starts whose far end is a deleted node (nothing to claim)
    const EdgeRec* rec;
    __device__ u64 operator()(u64 j) const { return rec[j].status == 1 && rec[j].rev_id == EMPTY64; }
};

template <int NW>
struct EmitVisit {
    char* seq;           // start of the sequence part of this edge's text
    Slot<NW>* slots;
    u32 eid, bal;
    __device__ void put_base(u32 i, unsigned code) {   // i = 1-based node number == 1-based base number
        u32 c = i - 1;
        seq[c + c / 100] = "ACTG"[code];
        if (i % 100 == 0) seq[c + c / 100 + 1] = '\n';
    }
    __device__ int operator()(u32 i, u64 slot, int sm, const Kmer<NW>& ori, u64 po) {
        put_base(i, klast(ori));
        // a node met twice inside one path keeps the values of its FIRST occurrence (the reference assigns back to front)
        if (pl_inedge(po)) return WALK_GO;
        // The reference overlays edgeId on l_links|cov (union, newhash.h:83-88).  Here the id goes to `aux` (the iteration
        // index is no longer needed for a linear node) so that the link fields stay intact while other walks still read them.
        u64 twin = sm ? (u64)(bal + 1) : (u64)(1 - bal);
        slots[slot].aux = sm ? eid : eid + bal;
        slots[slot].payload = (po & ~(3ull << PL_TWIN_SHIFT)) | (twin << PL_TWIN_SHIFT) | (1ull << PL_INEDGE_SHIFT);
        return WALK_GO;
    }
};

template <int NW>
__global__ void __launch_bounds__(128) k_edge_emit(Table<NW> tab, KParams<NW> kp, const u64* order, const u64* starts, u64 S, const EdgeRec* rec,
                                                   const u64* id_prefix, const u64* text_prefix, int out_words, char* text,
                                                   PatchSlot<NW>* patch, u64 patch_mask, bool quirk128, u64* err) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < S; j += (u64)gridDim.x * blockDim.x) {
        if (rec[j].status != 1) continue;
        u64 sid = starts[j];
        EdgeRec r = rec[j];
        u32 bal = r.rev_id == sid ? 0u : 1u;
        u32 eid = (u32)(id_prefix[j] + 1);
        char* base = text + text_prefix[j];
        EmitVisit<NW> ev{base + r.hdr_len, tab.slots, eid, bal};
        u64 e_slot = order[sid >> 3];
        WalkEnd<NW> end = unipath_walk(tab, kp, e_slot, (unsigned)(sid & 7), ev);
        if (end.status != WALK_REACHED || end.length != r.length) { atomicAdd(err, 1ull); continue; }
        ev.put_base(end.length, klast(end.to));
        if (end.length % 100 != 0) { u32 c = end.length - 1; ev.seq[c + c / 100 + 1] = '\n'; }
        // header
        char* p = base;
        p = put_str(p, ">length "); p = put_dec(p, end.length); *p++ = ',';
        p = put_kmer_hex(p, end.frm, out_words); *p++ = ',';
        p = put_kmer_hex(p, end.to, out_words); *p++ = ',';
        p = put_str(p, "cvg "); p = put_dec(p, edge_cvg(r.symbol, end.length)); *p++ = ','; *p++ = ' ';
        p = put_dec(p, bal); *p++ = '\n';
        if ((u32)(p - base) != r.hdr_len) atomicAdd(err, 1ull);
        // unlink both ends (dislink2nextUncertain(first) / dislink2prevUncertain(last)); other edges touch the same words
        atomicAnd(&tab.slots[e_slot].payload, ~(63ull << link_shift((unsigned)(sid & 7))));
        atomicAnd(&tab.slots[end.slot].payload, ~(63ull << link_shift(end.rev)));
        if (end.length == 1) {   // (K+1)-mer patch entry, node2edge.c:481-541
            Kmer<NW> wp = kshl2(end.frm);
            wp.w[NW - 1] |= klast(end.to);
            Kmer<NW> bwp = krc_ref(wp, kp.K + 1, quirk128);
            if (kless(wp, bwp)) patch_insert(patch, patch_mask, wp, PATCH_VALID | ((u64)(bal + 1) << 32) | eid);
            else patch_insert(patch, patch_mask, bwp, PATCH_VALID | ((u64)(1 - bal) << 32) | (u64)(eid + bal));
        }
    }
}

template <int NW>
void EngineT<NW>::build_edges(EdgeStats* st, std::string* edge_text) {
    if (!order_buf_.p) throw std::runtime_error("pgb200: build_edges before build_layout");
    const u64 N = n_nodes_;
    u64* order = order_buf_.template as<u64>();
    DevBuf scratch, startsb, recb, claimb, idb, txb, errb, textb;
    scratch.alloc(scan_scratch_elems(N) * sizeof(u64));
    errb.alloc(2 * sizeof(u64));
    PG_CUDA(cudaMemsetAsync(errb.p, 0, 2 * sizeof(u64), st_));
    u64* err = errb.template as<u64>();
    // starts
    device_scan_total(StartIn<NW>{tab_.slots, order}, N, scratch.template as<u64>(), d_cnt_ + C_MISC0, st_);
    read_counters();
    const u64 S = h_cnt_[C_MISC0];
    startsb.alloc((S + 1) * sizeof(u64));
    u64* starts = startsb.template as<u64>();
    device_scan_finish(StartIn<NW>{tab_.slots, order}, StartOut<NW>{tab_.slots, order, starts}, N, scratch.template as<u64>(), st_);
    recb.alloc((S + 1) * sizeof(EdgeRec));
    EdgeRec* rec = recb.template as<EdgeRec>();
    unsigned blocks = (unsigned)std::min<u64>((S + 127) / 128 + 1, (u64)n_sm_ * 16);
    k_edge_walk<NW><<<blocks, 128, 0, st_>>>(tab_, kp_, order, starts, S, out_words(), rec, err);
    PG_CUDA(cudaGetLastError());
    // who emits: rounds of claim / resolve
    claimb.alloc((S + 1) * sizeof(u64));
    u64* claim = claimb.template as<u64>();
    int rounds = 0;
    for (int round = 0;; round++) {
        rounds = round + 1;
        PG_CUDA(cudaMemsetAsync(claim, 0xFF, (S + 1) * sizeof(u64), st_));
        PG_CUDA(cudaMemsetAsync(err + 1, 0, sizeof(u64), st_));
        k_edge_claim<<<blocks, 256, 0, st_>>>(starts, S, rec, claim);
        k_edge_resolve<<<blocks, 256, 0, st_>>>(starts, S, rec, claim, err + 1);
        PG_CUDA(cudaGetLastError());
        u64 h[2];
        PG_CUDA(cudaMemcpyAsync(h, err, sizeof h, cudaMemcpyDeviceToHost, st_));
        sync();
        if (h[0]) throw std::runtime_error("pgb200: edge walk fell off the k-mer table");
        if (!h[1]) break;
        if (round > 1000) throw std::runtime_error("pgb200: edge ownership did not converge");
    }
    // edge ids, text offsets, length-1 edges
    idb.alloc((S + 1) * sizeof(u64));
    txb.alloc((S + 1) * sizeof(u64));
    DevBuf scr2;
    scr2.alloc(scan_scratch_elems(S) * sizeof(u64));
    device_scan(IdIn{starts, rec}, ScanU64Out{idb.template as<u64>()}, S, scr2.template as<u64>(), d_cnt_ + C_MISC0, st_);
    device_scan(TextIn{rec}, ScanU64Out{txb.template as<u64>()}, S, scr2.template as<u64>(), d_cnt_ + C_MISC1, st_);
    device_scan_total(Len1In{rec}, S, scr2.template as<u64>(), d_cnt_ + C_MISC2, st_);
    read_counters();
    const u64 num_ed = h_cnt_[C_MISC0], text_bytes = h_cnt_[C_MISC1], n_len1 = h_cnt_[C_MISC2];
    if (num_ed >= 0xFFFFFFFFull) throw std::runtime_error("pgb200: more than 2^32 edges (the reference's ids are 32-bit)");
    // patch table
    u64 pcap = 1024;
    while (pcap < 2 * n_len1 + 64) pcap <<= 1;
    patch_buf_.alloc(pcap * sizeof(PatchSlot<NW>));
    PG_CUDA(cudaMemsetAsync(patch_buf_.p, 0, pcap * sizeof(PatchSlot<NW>), st_));
    patch_mask_ = pcap - 1;
    textb.alloc(text_bytes + 16);
    k_edge_emit<NW><<<blocks, 128, 0, st_>>>(tab_, kp_, order, starts, S, rec, idb.template as<u64>(), txb.template as<u64>(), out_words(),
                                             textb.template as<char>(), patch_buf_.template as<PatchSlot<NW>>(), patch_mask_, quirk128(), err);
    PG_CUDA(cudaGetLastError());
    edge_text->resize(text_bytes);
    if (text_bytes) PG_CUDA(cudaMemcpyAsync(&(*edge_text)[0], textb.p, text_bytes, cudaMemcpyDeviceToHost, st_));
    u64 h0;
    PG_CUDA(cudaMemcpyAsync(&h0, err, sizeof h0, cudaMemcpyDeviceToHost, st_));
    sync();
    if (h0) throw std::runtime_error("pgb200: edge emission inconsistency");
    // number of emitted records = starts with status 1
    num_ed_ = num_ed;
    st->num_ed = num_ed;
    st->extra_nodes = n_len1;
    // emitted = num_ed - (number of non-palindromic emitted) ; count directly
    {
        device_scan_total(EmIn{rec}, S, scr2.template as<u64>(), d_cnt_ + C_MISC0, st_);
        read_counters();
        st->edges = h_cnt_[C_MISC0];
    }
    if (prm_.verbose) {
        device_scan_total(EmNoRevIn{rec}, S, scr2.template as<u64>(), d_cnt_ + C_MISC0, st_);
        read_counters();
        fprintf(stderr, "[pgb200] build_edges: %llu start(s), %d claim/resolve round(s), %llu emitted start(s) without a reverse start\n",
                (unsigned long long)S, rounds, (unsigned long long)h_cnt_[C_MISC0]);
    }
}

// ---------------------------------------------------------------- vertices (output_vertex, output_pregraph.c:31-86)
template <int NW>
struct VertIn {
    const Slot<NW>* slots;
    const u64* order;
    __device__ u64 operator()(u64 i) const { return (slots[order[i]].payload & (PL_LINEAR | PL_DELETED)) ? 0 : 1; }
};
template <int NW>
struct VertOut {
    const Slot<NW>* slots;
    const u64* order;
    Kmer<NW>* out;
    __device__ void operator()(u64 i, u64 prefix, u64 v) const {
        if (v) out[prefix] = slot_key(slots + order[i]);
    }
};

template <int NW>
void EngineT<NW>::vertices(std::string* vertex_text, uint64_t* n_vertex) {
    const u64 N = n_nodes_;
    u64* order = order_buf_.template as<u64>();
    DevBuf scratch, outb;
    scratch.alloc(scan_scratch_elems(N) * sizeof(u64));
    device_scan_total(VertIn<NW>{tab_.slots, order}, N, scratch.template as<u64>(), d_cnt_ + C_MISC0, st_);
    read_counters();
    u64 nv = h_cnt_[C_MISC0];
    outb.alloc((nv + 1) * sizeof(Kmer<NW>));
    device_scan_finish(VertIn<NW>{tab_.slots, order}, VertOut<NW>{tab_.slots, order, outb.template as<Kmer<NW>>()}, N, scratch.template as<u64>(), st_);
    std::vector<Kmer<NW>> h(nv + 1);
    if (nv) PG_CUDA(cudaMemcpyAsync(h.data(), outb.p, nv * sizeof(Kmer<NW>), cudaMemcpyDeviceToHost, st_));
    sync();
    const int out_words = this->out_words();
    std::string& s = *vertex_text;
    s.clear();
    s.reserve(nv * (out_words * 17 + 1) + 16);
    char b[96];
    for (u64 i = 0; i < nv; i++) {
        int n = 0;
        for (int w = 0; w < out_words; w++) n += snprintf(b + n, sizeof b - n, w ? " %llx" : "%llx", kout_word(h[i], w, out_words));
        b[n++] = ' ';
        s.append(b, n);
        if ((i + 1) % 8 == 0) s.push_back('\n');
    }
    s.push_back('\n');
    *n_vertex = nv;
}

template void EngineT<2>::build_edges(EdgeStats*, std::string*);
template void EngineT<4>::build_edges(EdgeStats*, std::string*);
template void EngineT<2>::vertices(std::string*, uint64_t*);
template void EngineT<4>::vertices(std::string*, uint64_t*);

}   // namespace pgb
