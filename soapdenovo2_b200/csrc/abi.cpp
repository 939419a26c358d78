// abi.cpp -- the extern "C" veneer of include/pregraph_b200.h over IEngine.  Errors never unwind across it: every entry point
// catches, keeps the message for pgb200_last_error() and returns its failure value.
#include "stage.h"
#include <cstring>
#include <memory>
#include <stdexcept>
#include <cuda_runtime_api.h>
using namespace pgb;
static thread_local std::string g_err;
struct pgb200_engine {
    std::unique_ptr<IEngine> e;
    PgParams prm;
};
// Runs f and returns its value; an exception becomes the calling thread's last error and `on_error` is returned.
template <class R, class F> static R guarded(R on_error, F&& f) {
    try { return f(); } catch (const std::exception& ex) { g_err = ex.what(); } catch (...) { g_err = "unknown error"; }
    return on_error;
}
// Engine entry points bind the calling thread to the engine's GPU first (one process may drive several engines), then run f(IEngine&):
// 0 on success, -1 on failure; with `on_error` given, f's value, or on_error on failure.
template <class F> static int abi_call(pgb200_engine* h, F&& f) { return guarded(-1, [&] { cudaSetDevice(h->prm.device); f(*h->e); return 0; }); }
template <class R, class F> static R abi_call(pgb200_engine* h, R on_error, F&& f) { return guarded(on_error, [&] { cudaSetDevice(h->prm.device); return f(*h->e); }); }

PgParams pgb::to_pg_params(const pgb200_params& p) {
    PgParams q;
    q.K = p.K; q.P = p.P; q.initG = p.initG; q.D = p.D; q.repsTie = p.repsTie; q.flavour127 = p.flavour127;
    q.device = p.device; q.max_rd_len = p.max_rd_len > 0 ? p.max_rd_len : 100; q.table_slots = p.table_slots;
    q.verbose = p.verbose; q.world = p.world > 0 ? p.world : 1; q.rank = p.rank;
    if (q.K < 13 || q.K % 2 == 0 || q.K > (q.flavour127 ? 127 : 63)) fail("pgb200: K must be odd, 13..63 (63-mer flavour) or 13..127 (127-mer flavour)");
    // first-occurrence rank = (read ordinal << 16) | k-mer position: positions must fit 16 bits
    if (q.max_rd_len - q.K + 1 > 65536) fail("pgb200: max_rd_len - K + 1 must not exceed 65536 (k-mer positions are 16-bit)");
    if (q.world > 16 || q.rank < 0 || q.rank >= q.world) fail("pgb200: world must be 1..16 and 0 <= rank < world");
    return q;
}
extern "C" const char* pgb200_last_error(void) { return g_err.c_str(); }
extern "C" void pgb200_default_params(pgb200_params* p) {
    memset(p, 0, sizeof *p);
    p->K = 23; p->P = 8; p->max_rd_len = 100; p->world = 1;
}
extern "C" pgb200_engine* pgb200_create(const pgb200_params* p) {
    return guarded<pgb200_engine*>(nullptr, [&] { const PgParams q = to_pg_params(*p); return new pgb200_engine{std::unique_ptr<IEngine>(make_engine(q)), q}; });
}
extern "C" void pgb200_destroy(pgb200_engine* e) { delete e; }
extern "C" void* pgb200_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { g_err = "cudaHostAlloc failed"; return nullptr; }
    return p;
}
extern "C" void pgb200_host_free(void* p) { if (p) cudaFreeHost(p); }
extern "C" int pgb200_feed_text(pgb200_engine* e, const char* text, size_t nbytes, int on_device, int fastq, uint64_t ord_base,
                                uint64_t ord_stride, int reverse_seq, int maxlen) {
    return abi_call(e, [&](IEngine& g) { g.feed_text(text, nbytes, on_device != 0, fastq, ord_base, ord_stride, reverse_seq, maxlen); });
}
extern "C" uint64_t pgb200_last_chunk_records(pgb200_engine* e) { return e->e->last_chunk_records(); }
extern "C" int pgb200_xchg_setup(pgb200_engine* e, uint64_t cap_records) { return abi_call(e, [&](IEngine& g) { g.xchg_setup(cap_records); }); }
extern "C" int pgb200_xchg_export(pgb200_engine* e, void* handle64) { return abi_call(e, [&](IEngine& g) { g.xchg_export(handle64); }); }
extern "C" int pgb200_xchg_import(pgb200_engine* e, int peer, const void* handle64) { return abi_call(e, [&](IEngine& g) { g.xchg_import(peer, handle64); }); }
extern "C" void* pgb200_xchg_base(pgb200_engine* e) { return abi_call<void*>(e, nullptr, [](IEngine& g) { return g.xchg_base(); }); }
extern "C" int pgb200_xchg_import_ptr(pgb200_engine* e, int peer, int peer_device, void* base) { return abi_call(e, [&](IEngine& g) { g.xchg_import_ptr(peer, peer_device, base); }); }
extern "C" int pgb200_xchg_fence(pgb200_engine* e) { return abi_call(e, [](IEngine& g) { g.xchg_fence(); }); }
extern "C" int pgb200_flush(pgb200_engine* e) { return abi_call(e, [](IEngine& g) { g.flush(); }); }
extern "C" int pgb200_xchg_room(pgb200_engine* e, uint64_t n_rec) { return abi_call(e, -1, [&](IEngine& g) { return g.xchg_room(n_rec) ? 1 : 0; }); }
extern "C" int pgb200_absorb(pgb200_engine* e, pgb200_engine* other) { return abi_call(e, [&](IEngine& g) { g.absorb(other->e.get()); }); }
extern "C" int pgb200_finish_pass1(pgb200_engine* e, pgb200_pass1_stats* st) {
    return abi_call(e, [&](IEngine& g) {
        Pass1Stats s;
        g.finish_pass1(&s);
        if (st) {
            st->records = s.records; st->reads_kept = s.reads_kept; st->instances = s.instances; st->distinct = s.distinct;
            st->table_slots = s.table_slots; st->launches = s.launches; st->ms_decode = s.ms_decode; st->ms_insert = s.ms_insert; st->ms_apply = s.ms_apply;
        }
    });
}
extern "C" int pgb200_reset_pass1(pgb200_engine* e) { return abi_call(e, [](IEngine& g) { g.reset_pass1(); }); }
extern "C" int pgb200_sweeps(pgb200_engine* e, long long hist[256], uint64_t* linear_marked, uint64_t* removed) {
    return abi_call(e, [&](IEngine& g) {
        SweepStats s;
        g.sweeps(&s);
        if (hist) memcpy(hist, s.hist, sizeof s.hist);
        if (linear_marked) *linear_marked = s.linear;
        if (removed) *removed = s.removed;
    });
}
extern "C" int pgb200_build_layout(pgb200_engine* e) { return abi_call(e, [](IEngine& g) { g.build_layout(); }); }
extern "C" uint64_t pgb200_node_count(pgb200_engine* e) { return e->e->node_count(); }
extern "C" int pgb200_dump_nodes(pgb200_engine* e, void* out) { return abi_call(e, [&](IEngine& g) { g.dump_nodes(out); }); }
extern "C" int pgb200_sample_table(pgb200_engine* e, uint64_t seed, uint32_t one_in, uint64_t* out, uint64_t cap, uint64_t* n_out) {
    return abi_call(e, [&](IEngine& g) { *n_out = g.sample_table(seed, one_in, out, cap); });
}

// ---- graph phases (stage.cpp)
extern "C" int pgb200_remove_tips(pgb200_engine* e, pgb200_graph_stats* st) { return abi_call(e, [&](IEngine& g) { phase_tips(g, e->prm, st); }); }
extern "C" int pgb200_kmer2edges(pgb200_engine* e, const char* prefix, pgb200_graph_stats* st) { return abi_call(e, [&](IEngine& g) { phase_edges(g, e->prm, prefix, st); }); }
extern "C" int pgb200_read2edge(pgb200_engine* e, const char* prefix, pgb200_graph_stats* st) { return abi_call(e, [&](IEngine& g) { phase_pass2(g, e->prm, prefix, st); }); }
extern "C" int pgb200_output_vertex(pgb200_engine* e, const char* prefix, pgb200_graph_stats* st) { return abi_call(e, [&](IEngine& g) { phase_vertex(g, e->prm, prefix, st); }); }

// ---- host logic only (stage_io.cpp)
extern "C" int pgb200_plan_files(const char* cfg, char* out, size_t cap) {   // "max_rd_len N", then "mate fastq reverse cut path" per file
    return guarded(-1, [&] {
        const ReadPlan plan = read_plan(cfg);
        std::string s = "max_rd_len " + std::to_string(plan.max_rd_len) + "\n";
        for (const PlanEntry& f : plan.files)
            s += std::to_string(f.mate) + " " + std::to_string((int)f.fastq) + " " + std::to_string(f.reverse) + " " + std::to_string(f.cut) + " " + f.path + "\n";
        if (s.size() + 1 > cap) fail("pgb200: the plan takes %zu bytes, more than the %zu given", s.size() + 1, cap);
        memcpy(out, s.c_str(), s.size() + 1);
        return 0;
    });
}
extern "C" size_t pgb200_cut_chunk(const char* buf, size_t n, int fastq) { return last_record_start(buf, n, fastq != 0); }
extern "C" int pgb200_edge_text_to_sidecar(const char* text, size_t nbytes, int K, int flavour127, uint64_t num_ed, const char* path) {
    return guarded(-1, [&] { edge_text_to_sidecar(text, nbytes, K, flavour127, num_ed, path); return 0; });
}
extern "C" int pgb200_sidecar_to_edge_gz(const char* prefix) { return guarded(-1, [&] { sidecar_to_edge_gz(prefix); return 0; }); }
