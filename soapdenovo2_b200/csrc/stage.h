// stage.h -- what abi.cpp (the C-ABI veneer), stage.cpp (the pregraph stage and its graph phases) and stage_io.cpp (config, chunk
// cutter, output files, edge sidecar; no GPU) share.  Internal to csrc/: not installed, and hidden from the library's exports.
#pragma once
#include "../../include/pregraph_b200.h"
#include "engine.h"

#pragma GCC visibility push(hidden)
namespace pgb {

[[noreturn]] void fail(const char* fmt, ...);     // throws std::runtime_error with the printf-formatted text the stage prints
PgParams to_pg_params(const pgb200_params& p);   // fills in defaults; checks K range, 16-bit k-mer positions, world / rank

// One implementation per graph phase: each prints the reference's stderr lines and fills its fields of *st (st may be null).
// phase_edges writes the edge files under `prefix` before its line, or leaves the returned text to the caller (prefix null).
void phase_tips(IEngine& e, const PgParams& p, pgb200_graph_stats* st);
std::string phase_edges(IEngine& e, const PgParams& p, const char* prefix, pgb200_graph_stats* st);
void phase_pass2(IEngine& e, const PgParams& p, const std::string& prefix, pgb200_graph_stats* st);
void phase_vertex(IEngine& e, const PgParams& p, const std::string& prefix, pgb200_graph_stats* st);

// The files of a library config in the order the reference opens them (openNextFile / nextValidIndex)
// mate: -1 single file; 0/1 = first/second file of an interleaved pair (ordinals base + 2*pair + mate)
struct PlanEntry { std::string path; bool fastq; int mate, reverse, cut; };
struct ReadPlan { int n_libs, max_rd_len; std::vector<PlanEntry> files; };
ReadPlan read_plan(const char* cfg);
// The map stage's plan: every library in config order after the sort by avg_ins, with the files map reads (paired ones, asm_flags 2|3)
// MapPlan::long_libs: the asm_flags=4 libraries (prlLongRead2Ctg), their p, f, q files in that order, each read cut to `cut` bases.
// long_len is getMaxLongReadLen (0: no long pass); the libraries' `cut` and the short pass's use max_len4all = max(max_rd_len,
// long_len).
struct MapLib { int avg_ins, reverse, map_len, rank, pair_num_cut; std::vector<PlanEntry> files; };
struct MapPlan { int max_rd_len, long_len = 0, max_len4all = 0; std::vector<MapLib> libs, long_libs; };
MapPlan map_plan(const char* cfg);   // refuses b= libraries and two-file pairs in asm_flags=4 libraries
size_t last_record_start(const char* buf, size_t n, bool fastq);   // the chunk cutter
void write_file(const std::string& name, const void* data, size_t n);
void write_kmer_freq(const std::string& prefix, const long long hist[256]);
void write_edge_outputs(const std::string& prefix, const std::string& text, const PgParams& p, uint64_t num_ed);
void edge_text_to_sidecar(const char* text, size_t nbytes, int K, int flavour127, uint64_t num_ed, const std::string& path);
void sidecar_to_edge_gz(const std::string& prefix);

}   // namespace pgb
#pragma GCC visibility pop
