// stage.cpp -- the `pregraph -s cfg -K k -p P [-a G] [-d D] [-R] -o prefix` stage (CLI, call_pregraph) and the graph phases it shares
// with the C-ABI.  Mirrors, in new code, the host-side behaviour of (standardPregraph/):
//   call_pregraph / initenv        pregraph.c:62-220   (getopt string, K fix-ups, phase order, stderr lines)
//   phase files                    prlRead2path.c:426-476 (.preArc/.markOnEdge), output_pregraph.c:50-86 (.vertex, .preGraphBasic)
// All k-mer work happens on the GPU through IEngine; this file only moves bytes between files and the engines.
#include "stage.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <future>
#include <memory>
#include <stdexcept>
#include <getopt.h>
#include "cuda_owner.h"

namespace pgb {
void phase_tips(IEngine& e, const PgParams& p, pgb200_graph_stats* st) {
    TipStats t;
    e.remove_tips(&t);
    if ((signed char)p.D == 0) {
        fprintf(stderr, "Start to remove frequency-one-kmer tips shorter than %d.\n", 2 * p.K);
        fprintf(stderr, "Total %llu tip(s) removed.\n", (unsigned long long)t.single_tips);
        fprintf(stderr, "%llu linear node(s) marked.\n", (unsigned long long)t.single_relinear);
    }
    fprintf(stderr, "Start to remove tips with minority links.\n");
    for (size_t i = 0; i < t.minor_cycles.size(); i++) fprintf(stderr, "%llu tip(s) removed in cycle %zu.\n", (unsigned long long)t.minor_cycles[i], i + 1);
    fprintf(stderr, "Total %llu tip(s) removed.\n", (unsigned long long)t.minor_tips);
    fprintf(stderr, "%llu linear node(s) marked.\n", (unsigned long long)t.minor_relinear);
    if (st) { st->single_tips = t.single_tips; st->minor_tips = t.minor_tips; }
}
std::string phase_edges(IEngine& e, const PgParams& p, const char* prefix, pgb200_graph_stats* st) {
    EdgeStats es;
    std::string text;
    e.build_edges(&es, &text);
    if (prefix) write_edge_outputs(prefix, text, p, es.num_ed);
    fprintf(stderr, "%llu (%llu) edge(s) and %llu extra node(s) constructed.\n", (unsigned long long)es.num_ed, (unsigned long long)es.edges, (unsigned long long)es.extra_nodes);
    if (st) { st->num_ed = es.num_ed; st->edges = es.edges; st->extra_nodes = es.extra_nodes; }
    return text;
}
void phase_pass2(IEngine& e, const PgParams& p, const std::string& prefix, pgb200_graph_stats* st) {
    Pass2Stats ps;
    std::string arcs, path, mark;
    e.pass2(&ps, &arcs, &path, &mark);
    write_file(prefix + ".preArc", arcs.data(), arcs.size());
    if (p.repsTie) {
        write_file(prefix + ".path", path.data(), path.size());
        write_file(prefix + ".markOnEdge", mark.data(), mark.size());
        fprintf(stderr, "%llu marker(s) output.\n", (unsigned long long)ps.markers);
    }
    fprintf(stderr, "Reads alignment done, %llu read(s) deleted, %llu pre-arc(s) added.\n", (unsigned long long)ps.deleted_reads, (unsigned long long)ps.arcs);
    if (st) { st->deleted_reads = ps.deleted_reads; st->arcs = ps.arcs; }
}
void phase_vertex(IEngine& e, const PgParams& p, const std::string& prefix, pgb200_graph_stats* st) {
    std::string vt;
    uint64_t nv = 0;
    e.vertices(&vt, &nv);
    write_file(prefix + ".vertex", vt.data(), vt.size());
    fprintf(stderr, "%llu vertex(es) output.\n", (unsigned long long)nv);
    char buf[512];
    const uint64_t num_ed = e.num_ed();   // the engine's own count (st is an output here)
    int n = snprintf(buf, sizeof buf, "VERTEX %llu K %d\n\nEDGEs %llu\n\nMaxReadLen %d MinReadLen %d MaxNameLen %d\n", (unsigned long long)nv, p.K, (unsigned long long)num_ed, p.max_rd_len, 0, 256);
    write_file(prefix + ".preGraphBasic", buf, n);
    if (st) { st->vertices = nv; st->num_ed = num_ed; }
}

namespace {
// The stage's engines: engine g on GPU device0 + g.  IEngine's methods expect the calling thread to be bound to the engine's GPU
// (the C-ABI's entry points do that for their callers); at(g) does it here.
struct Engines {
    std::vector<std::unique_ptr<IEngine>> e;
    int device0 = 0;
    IEngine& at(size_t g) { cudaSetDevice(device0 + (int)g); return *e[g]; }
    Pass1Stats finish_pass1() {   // over every shard: the counts add up, the GPU times are the slowest shard's
        Pass1Stats sum;
        for (size_t g = 0; g < e.size(); g++) {
            Pass1Stats s;
            at(g).finish_pass1(&s);
            sum.distinct += s.distinct; sum.instances += s.instances; sum.table_slots += s.table_slots;
            sum.ms_decode = std::max(sum.ms_decode, s.ms_decode); sum.ms_insert = std::max(sum.ms_insert, s.ms_insert);
        }
        return sum;
    }
    SweepStats sweeps() {
        SweepStats sum{};
        for (size_t g = 0; g < e.size(); g++) {
            SweepStats s;
            at(g).sweeps(&s);
            for (int i = 0; i < 256; i++) sum.hist[i] += s.hist[i];
            sum.linear += s.linear; sum.removed += s.removed;
        }
        return sum;
    }
};
// One pinned staging buffer; chunk i goes to engine i % G.  feed_text returns when the chunk's H2D copy is done, its kernels keep
// running, so with several GPUs the copy of chunk i+1 (to the next GPU) overlaps the kernels of chunk i.
struct Feeder {
    static constexpr size_t kMaxChunksPerEpoch = 120;   // several GPUs: at most this many chunks (over all GPUs) between collective flushes
    Engines& engs;
    const size_t cap;         // chunk bytes
    size_t next = 0;          // engine of the next chunk
    Pinned<char> pin;
    size_t fed_in_epoch = 0;
    double ms_read = 0, ms_feed = 0;   // wall time reading the files, outside the chunks' feed / inside feed_text (PGB200_VERBOSE)
    void collective_flush() {
        in_step("pgb200: %s", [&] { for (size_t g = 0; g < engs.e.size(); g++) engs.at(g).xchg_fence(); for (size_t g = 0; g < engs.e.size(); g++) engs.at(g).flush(); });
        fed_in_epoch = 0;
    }
    // streams one file; returns number of records
    uint64_t run(const std::string& fn, bool fastq, uint64_t ord_base, uint64_t ord_stride, int reverse, int maxlen) {
        fprintf(stderr, "Import reads from file:\n %s\n", fn.c_str());
        if (!pin) in_step("pgb200: cudaHostAlloc failed", [&] { pin = make_pinned<char>(cap + 16); });
        uint64_t recs = 0;
        const double t_run = host_now();
        double ms_take = 0;
        read_chunks(fn, pin, cap, [&](const char* text, size_t n, bool at_eof) {
            const double t_take = host_now();
            const size_t cut = whole_records(text, n, fastq, at_eof);
            if (cut == 0) return cut;
            if (engs.e.size() > 1) {
                // several GPUs: room for this chunk's records in every arena region, and for its segment (128 per epoch over all GPUs)
                // reads in this chunk, estimated generously from the library's read length (a record is a header, the bases and,
                // for FASTQ, as many quality characters); an estimate that is too low is caught on the device (arena overflow error)
                const uint64_t L = (uint64_t)std::max(8, maxlen);
                const uint64_t upper = cut / (fastq ? L + 6 : L / 2 + 4) + 1;
                if (fed_in_epoch + engs.e.size() > kMaxChunksPerEpoch || !engs.e[next]->xchg_room(upper)) collective_flush();
            }
            const double t_f = host_now();
            IEngine& eng = engs.at(next);
            in_step("readseqInLib return error! please make sure input file is correct fastq/fasta file \n(%s)",
                    [&] { eng.feed_text(text, cut, false, fastq, ord_base + recs * ord_stride, ord_stride, reverse, maxlen); });
            ms_feed += host_now() - t_f;
            recs += eng.last_chunk_records();
            next = (next + 1) % engs.e.size();
            fed_in_epoch++;
            ms_take += host_now() - t_take;
            return cut;
        });
        ms_read += host_now() - t_run - ms_take;
        return recs;
    }
};
void usage(int flavour127) {
    fprintf(stderr, "\npregraph -s configFile -o outputGraph [-R] [-K kmer -p n_cpu -a initMemoryAssumption -d KmerFreqCutoff]\n");
    fprintf(stderr, "  -s <string>      configFile: the config file of solexa reads\n");
    fprintf(stderr, "  -o <string>      outputGraph: prefix of output graph file name\n");
    fprintf(stderr, "  -K <int>         kmer(min 13, max %d): kmer size, [23]\n", flavour127 ? 127 : 63);
    fprintf(stderr, "  -p <int>         n_cpu: number of reference hash sets (layout parameter of the GPU engine), [8]\n");
    fprintf(stderr, "  -a <int>         initMemoryAssumption: memory assumption initialized to avoid further reallocation, unit GB, [0]\n");
    fprintf(stderr, "  -R (optional)    output extra information for resolving repeats in contig step, [NO]\n");
    fprintf(stderr, "  -d <int>         KmerFreqCutoff: kmers with frequency no larger than KmerFreqCutoff will be deleted, [0]\n");
}
// PGB200_VERBOSE: where the stage's wall time went, in milliseconds (the reference's own "Time spent" lines are whole seconds)
struct Timeline {
    double t_prev;
    std::string text;
    void mark(const char* what) {
        const double t = host_now();
        char b[96];
        snprintf(b, sizeof b, "%s%s %.0f ms", text.empty() ? "" : ", ", what, t - t_prev);
        text += b;
        t_prev = t;
    }
};
int seconds_since(double t_ms) { return (int)((host_now() - t_ms) * 1e-3); }
// The stage; every failure throws with the text to print.
int pregraph(int argc, char** argv, int flavour127) {
    const double t_all = host_now();
    Timeline tl{t_all};
    fprintf(stderr, "\n********************\nPregraph\n********************\n\n");
    // ---- initenv (pregraph.c:142-220)
    pgb200_params prm;
    pgb200_default_params(&prm);
    prm.flavour127 = flavour127;
    std::string cfg, prefix;
    int inp = 0, outp = 0, c;
    optind = 1;
    fprintf(stderr, "Parameters: pregraph ");
    while ((c = getopt(argc, argv, "a:s:o:K:p:d:R")) != EOF) {
        switch (c) {
            case 's': fprintf(stderr, "-s %s ", optarg); inp = 1; cfg = optarg; break;
            case 'o': fprintf(stderr, "-o %s ", optarg); outp = 1; prefix = optarg; break;
            case 'K': fprintf(stderr, "-K %s ", optarg); prm.K = atoi(optarg); break;
            case 'p': fprintf(stderr, "-p %s ", optarg); prm.P = atoi(optarg); break;
            case 'R': prm.repsTie = 1; fprintf(stderr, "-R "); break;
            case 'd': fprintf(stderr, "-d %s ", optarg); prm.D = atoi(optarg) >= 0 ? atoi(optarg) : 0; break;
            case 'a': fprintf(stderr, "-a %s ", optarg); prm.initG = atoi(optarg); break;
            default:
                if (!inp || !outp) { usage(flavour127); exit(-1); }
        }
    }
    fprintf(stderr, "\n\n");
    if (!inp || !outp) { usage(flavour127); exit(-1); }
    // ---- K fix-ups (pregraph.c:71-97)
    if (prm.K % 2 == 0) { prm.K++; fprintf(stderr, "K should be an odd number.\n"); }
    if (prm.K < 13) { prm.K = 13; fprintf(stderr, "K should not be less than 13.\n"); }
    else if (prm.K > (flavour127 ? 127 : 63)) { prm.K = flavour127 ? 127 : 63; fprintf(stderr, "K should not be greater than %d.\n", prm.K); }
    const StageSettings env = stage_settings();
    prm.device = env.device;
    prm.verbose = env.verbose;
    if (const char* v = getenv("PGB200_TABLE_SLOTS")) prm.table_slots = strtoull(v, nullptr, 10);

    // ---- pass 1 (prlRead2HashTable)
    double t0 = host_now();
    const ReadPlan plan = read_plan(cfg.c_str());
    prm.max_rd_len = plan.max_rd_len;
    fprintf(stderr, "In %s, %d lib(s), maximum read length %d, maximum name length %d.\n\n", cfg.c_str(), plan.n_libs, prm.max_rd_len, 256);
    // ---- engines: one per GPU (PGB200_GPUS=n | all; default 1).  Pass 1 is sharded: GPU g owns bucket range g, every GPU decodes
    // and partitions the chunks dealt to it and stores the records straight into their owners' arenas (peer access).
    int n_gpus = 1;
    if (const char* v = getenv("PGB200_GPUS")) {
        int have = 0;
        cudaGetDeviceCount(&have);
        n_gpus = strcmp(v, "all") == 0 ? have : atoi(v);
        if (n_gpus < 1) n_gpus = 1;
        if (n_gpus > 16) n_gpus = 16;
        if (prm.device + n_gpus > have) fail("pgb200: PGB200_GPUS=%d but only %d GPU(s) visible", n_gpus, have);
    }
    prm.world = n_gpus;
    const PgParams p0 = in_step("pgb200: %s", [&] { return to_pg_params(prm); });   // engine 0's, the one that runs the graph phases
    {
        Engines engs{{}, p0.device};
        for (int g = 0; g < n_gpus; g++) {
            PgParams q = p0;
            q.device += g;
            q.rank = g;
            engs.e.emplace_back(in_step("pgb200: %s", [&] { return make_engine(q); }));
        }
        if (n_gpus > 1) {
            in_step("pgb200: exchange arena failed: %s", [&] { for (int g = 0; g < n_gpus; g++) engs.at(g).xchg_setup(0); });
            in_step("pgb200: peer access failed: %s", [&] {
                for (int g = 0; g < n_gpus; g++) for (int h = 0; h < n_gpus; h++) if (h != g) engs.at(g).xchg_import_ptr(h, p0.device + h, engs.e[h]->xchg_base());
            });
            fprintf(stderr, "[pgb200] pass 1 sharded over %d GPUs (minimizer-bucket ranges, records stored peer to peer)\n", n_gpus);
        }
        fprintf(stderr, "%d thread(s) initialized.\n", prm.P);
        tl.mark("engines");
        uint64_t ord_next = 0, n_reads = 0;
        {
            Feeder fd{engs, env.chunk_bytes};
            for (size_t i = 0; i < plan.files.size(); i++) {
                const PlanEntry& e = plan.files[i];
                if (e.mate == 0) {
                    // mates interleave r1,r2,r1,r2 (prlHashReads.c:480-583): ordinal = base + 2*pair + mate
                    uint64_t n1 = fd.run(e.path, e.fastq, ord_next, 2, e.reverse, e.cut);
                    const PlanEntry& m = plan.files[++i];
                    uint64_t n2 = fd.run(m.path, m.fastq, ord_next + 1, 2, m.reverse, m.cut);
                    if (n1 != n2) fail("pgb200: mate files hold different numbers of reads (%llu vs %llu): unsupported", (unsigned long long)n1, (unsigned long long)n2);
                    ord_next += 2 * n1; n_reads += 2 * n1;
                } else {
                    uint64_t n = fd.run(e.path, e.fastq, ord_next, 1, e.reverse, e.cut);
                    ord_next += n; n_reads += n;
                }
            }
            if (n_gpus > 1) fd.collective_flush();
            if (prm.verbose) fprintf(stderr, "[pgb200] reading the files: %.0f ms in fread, %.0f ms in feed_text (H2D copy + launches)\n", fd.ms_read, fd.ms_feed);
        }
        const Pass1Stats p1 = in_step("pgb200: pass 1 failed: %s", [&] { return engs.finish_pass1(); });
        const double t1 = host_now();
        tl.mark("reads -> k-mer table");
        fprintf(stderr, "Time spent on hashing reads: %ds, %lld read(s) processed.\n", (int)((t1 - t0) * 1e-3), (long long)n_reads);
        fprintf(stderr, "%lli node(s) allocated, %lli kmer(s) in reads, %lli kmer(s) processed.\n", (long long)p1.distinct, (long long)p1.instances, (long long)p1.instances);
        fprintf(stderr, "[pgb200] pass 1: %.3f s wall, decode %.1f ms + insert %.1f ms on the GPU%s, table %llu slots\n", (t1 - t0) * 1e-3, p1.ms_decode, p1.ms_insert,
                n_gpus > 1 ? " (slowest GPU)" : "", (unsigned long long)p1.table_slots);
        fprintf(stderr, "done hashing nodes\n");
        const SweepStats sw = in_step("pgb200: sweeps failed: %s", [&] { return engs.sweeps(); });
        tl.mark("sweeps");
        if ((signed char)prm.D) fprintf(stderr, "%llu kmer(s) removed.\n", (unsigned long long)sw.removed);
        fprintf(stderr, "%llu linear node(s) marked.\n", (unsigned long long)sw.linear);
        // The graph phases walk across buckets: the shards (tables with their swept flags, packed reads) are folded into GPU 0, which
        // runs layout, tips, edges and pass 2 exactly as in the single-GPU case.
        for (int g = 1; g < n_gpus; g++) {
            in_step("pgb200: gathering the table shards failed: %s", [&] { engs.at(0).absorb(engs.e[g].get()); });
            engs.e[g].reset();
        }
        if (n_gpus > 1) tl.mark("gather shards");
        write_kmer_freq(prefix, sw.hist);
        fprintf(stderr, "Time spent on pre-graph construction: %ds.\n\n", seconds_since(t0));
        if (getenv("PGB200_PASS1_ONLY")) return 0;

        // ---- layout + tips (removeSingleTips / removeMinorTips)
        t0 = host_now();
        in_step("pgb200: layout failed: %s", [&] { engs.at(0).build_layout(); });
        in_step("pgb200: tips failed: %s", [&] { phase_tips(engs.at(0), p0, nullptr); });
        tl.mark("layout + tips");
        fprintf(stderr, "Time spent on removing tips: %ds.\n\n", seconds_since(t0));
        // ---- edges (kmer2edges)
        t0 = host_now();
        const std::string edge_text = in_step("pgb200: edges failed: %s", [&] { return phase_edges(engs.at(0), p0, nullptr, nullptr); });
        const uint64_t num_ed = engs.e[0]->num_ed();
        // The deflate of the edge text is sequential host work (it has to be: the bytes must equal the reference's gz stream); it runs
        // on a host thread while the GPU does pass 2.  get() rethrows its failure; on every other way out the future's destructor waits.
        std::future<void> edge_files = std::async(std::launch::async, [&] { write_edge_outputs(prefix, edge_text, p0, num_ed); });
        tl.mark("edges");
        fprintf(stderr, "Time spent on constructing edges: %ds.\n\n", seconds_since(t0));
        // ---- pass 2 (prlRead2edge)
        t0 = host_now();
        in_step("pgb200: pass 2 failed: %s", [&] { phase_pass2(engs.at(0), p0, prefix, nullptr); });
        fprintf(stderr, "Time spent on aligning reads: %ds.\n\n", seconds_since(t0));
        tl.mark("pass 2 + its files");
        edge_files.get();
        tl.mark("waiting for the edge file");
        in_step("pgb200: vertex output failed: %s", [&] { phase_vertex(engs.at(0), p0, prefix, nullptr); });
    }   // the engine is released here, inside the "vertex + teardown" interval
    tl.mark("vertex + teardown");
    if (prm.verbose) fprintf(stderr, "[pgb200] stage wall %.2f s: %s\n", (host_now() - t_all) * 1e-3, tl.text.c_str());
    fprintf(stderr, "Overall time spent on constructing pre-graph: %dm.\n\n", seconds_since(t_all) / 60);
    return 0;
}
}   // namespace
}   // namespace pgb
// The reference ends the process on every error, and callers of call_pregraph rely on that: one handler prints the message and exits.
extern "C" int pgb200_pregraph_main(int argc, char** argv, int flavour127) {
    try { return pgb::pregraph(argc, argv, flavour127); } catch (const std::exception& ex) { fprintf(stderr, "%s\n", ex.what()); exit(-1); }
}
// The library's own call_pregraph has the 63-mer semantics (what dlopen / ctypes users get).  A SOAPdenovo-127mer build links
// pregraph_shim.c (-DPGB_FLAVOUR127=1) instead: the executable's definition takes precedence, so the flavour is fixed at link
// time exactly as the reference fixes it with -DMER63 / -DMER127 -- no environment variable is involved.
extern "C" int call_pregraph(int argc, char** argv) { return pgb200_pregraph_main(argc, argv, 0); }
