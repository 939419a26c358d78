// stage.h -- what abi.cpp (the C-ABI veneer), stage.cpp (pregraph and its graph phases), map_stage.cpp (map) and stage_io.cpp (settings,
// config, chunked reads, output files, edge sidecar; no GPU) share.  Internal to csrc/: not installed, and hidden from the library's exports.
#pragma once
#include "../../include/pregraph_b200.h"
#include "engine.h"
#include <cstdio>
#include <exception>
#include <functional>

#pragma GCC visibility push(hidden)
namespace pgb {

[[noreturn]] void fail(const char* fmt, ...);     // throws std::runtime_error with the printf-formatted text the stage prints
// Runs f; a failure is rethrown as `fmt` with its message for the first %s, then a...: the text the stage prints for that step.
template <class F, class... A> auto in_step(const char* fmt, F&& f, A... a) -> decltype(f()) {
    try { return f(); } catch (const std::exception& ex) { fail(fmt, ex.what(), a...); }
}
PgParams to_pg_params(const pgb200_params& p);   // fills in defaults; checks K range, 16-bit k-mer positions, world / rank

// The environment settings both stages share, read once before any engine exists: PGB200_DEVICE (the stage's first GPU),
// PGB200_VERBOSE (where the time went) and PGB200_CHUNK_MB (the read files' chunk: a whole number of MB from 1 to 4095, so that a
// chunk stays under the engines' 4 GiB limit; default 256).
struct StageSettings { int device = 0, verbose = 0; size_t chunk_bytes = (size_t)256 << 20; };
StageSettings stage_settings();

FILE* ckopen(const std::string& name, const char* mode);   // fopen, or fail as the reference's ckopen (check.c:30-34)
std::string read_whole_file(FILE* f);                      // the rest of an open file
// Reads `path` through buf, cap bytes the caller owns.  take(text, n, at_eof) gets each chunk, which starts at a record start, and
// returns how many leading bytes it used; the rest starts the next chunk.  at_eof: the text ends at the end of the file (feof after
// the fread), and take uses all of it.  An empty file makes no call.  A full chunk of which take used nothing fails.
using ChunkTake = std::function<size_t(const char* text, size_t n, bool at_eof)>;
void read_chunks(const std::string& path, char* buf, size_t cap, const ChunkTake& take);
// Pass 1's record rule (single-line FASTA, 4-line FASTQ): the leading bytes of a chunk that hold whole records.  At the end of the
// file that is all of it but trailing blank lines; otherwise everything before the last record start.
size_t whole_records(const char* text, size_t n, bool fastq, bool at_eof);
// The contigs of <prefix>.contig that map hashes, read as prlContig2nodes reads them: readseqpar's pass over fgets pieces of 4949 bytes
// (its stats line goes to stderr), then readseq1by1's pieces of 4999 bytes, each record cut at readseqpar's maximum length, kept if
// it has at least K + 2 bases.  Bases are packed 2 bits each into one stream (LSB first); record r is [off[r], off[r + 1]).
struct Contigs {
    std::vector<unsigned long long> packed, off{0};
    std::vector<unsigned> id;   // atoi of a name that starts with a digit, else the record's ordinal (1-based, every record counted)
    unsigned long long n_kmers = 0;
};
Contigs read_contigs(const std::string& prefix, int K);

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
