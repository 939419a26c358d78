// engine.h -- C++ interface of the GPU pregraph engine (one instance == one GPU's share of the pregraph stage).
// The C-ABI in include/pregraph_b200.h is a thin veneer over this.  No torch types, no CUDA types in signatures.
#pragma once
#include <cstddef>
#include <cstdint>
#include <ctime>
#include <string>
#include <vector>

namespace pgb {

// monotonic host clock in milliseconds
inline double host_now() { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; }

struct PgParams {
    int K = 23;              // overlaplen after the reference's fix-ups (pregraph.c:71-97)
    int P = 8;               // -p: number of reference hash sets == LAYOUT parameter (SURVEY.md fact 1)
    int initG = 0;           // -a: GB assumed by the reference for its static tables (0 = dynamic growth)
    int D = 0;               // -d: deLowKmer
    int repsTie = 0;         // -R
    int flavour127 = 0;      // 0: SOAPdenovo-63mer semantics, 1: SOAPdenovo-127mer semantics (entry size 40, modular())
    int device = 0;
    int max_rd_len = 100;    // maxReadLen4all
    uint64_t table_slots = 0;   // capacity hint for the GPU table (rounded up to a power of two); 0 = derive
    int verbose = 0;
    // multi-GPU sharding of the k-mer space (rank r owns a contiguous range of minimizer buckets, skm.cuh)
    int world = 1, rank = 0;
};

struct Pass1Stats {
    uint64_t records = 0;        // reads seen ("read(s) processed")
    uint64_t reads_kept = 0;     // reads with len >= K+1
    uint64_t instances = 0;      // "kmer(s) in reads"
    uint64_t distinct = 0;       // "node(s) allocated"
    uint64_t table_slots = 0;
    double ms_decode = 0, ms_insert = 0;   // CUDA-event times accumulated over chunks (ms_insert includes ms_apply)
    uint64_t launches = 0;
    double ms_apply = 0;                   // the aggregation launches (k_skm_apply) alone
};

struct SweepStats {
    long long hist[256];
    uint64_t linear = 0, removed = 0;
};

struct TipStats {
    uint64_t single_tips = 0, single_relinear = 0;
    std::vector<uint64_t> minor_cycles;
    uint64_t minor_tips = 0, minor_relinear = 0;
    uint64_t rounds = 0;
};

struct EdgeStats {
    uint64_t num_ed = 0;      // edge_c incl. twins
    uint64_t edges = 0;       // emitted records
    uint64_t extra_nodes = 0; // length-1 edges
};

struct Pass2Stats {
    uint64_t deleted_reads = 0, arcs = 0, markers = 0;
};

class IEngine {
public:
    virtual ~IEngine() {}
    // ---- pass 1 (replaces prlRead2HashTable, prlHashReads.c:304-760)
    // Feed one chunk of FASTA/FASTQ text that starts at a record start and ends at a record end ('\n').
    // Record i of the chunk gets stream ordinal ord_base + i*ord_stride (defines first-occurrence order, SURVEY fact 2).
    virtual void feed_text(const char* text, size_t nbytes, bool on_device, int fastq, uint64_t ord_base, uint64_t ord_stride,
                           int reverse_seq, int maxlen) = 0;
    virtual uint64_t last_chunk_records() const = 0;
    // Aggregated pass 1 / multi-GPU exchange (skm.cu).  Every engine owns an arena that all engines of the job (itself included)
    // store super-k-mer records into; rank r aggregates the buckets it owns.  world == 1 needs none of these calls.
    //   xchg_setup -> [exchange handles / base pointers, xchg_import*] -> feed_text ... -> xchg_fence -> [barrier] -> flush
    virtual void xchg_setup(uint64_t cap_records) = 0;                 // arena capacity in records, summed over senders
    virtual void xchg_export(void* handle64) = 0;                      // CUDA IPC handle of the arena (other processes)
    virtual void xchg_import(int peer, const void* handle64) = 0;
    virtual void* xchg_base() = 0;                                      // arena base pointer (other GPUs of the same process)
    virtual void xchg_import_ptr(int peer, int peer_device, void* base) = 0;
    virtual void xchg_fence() = 0;    // every record this engine produced so far has reached its owner
    virtual void flush() = 0;         // aggregate the fenced records into the table (after every engine has fenced)
    virtual bool xchg_room(uint64_t n_rec) = 0;   // true: a chunk of n_rec reads surely fits this epoch (else: fence + flush all engines)
    // Fold another engine of the same job into this one (its table shard and its read store; peer access required): afterwards this
    // engine alone holds everything the graph phases need.  `other` must have finished pass 1 and its sweeps.
    virtual void absorb(IEngine* other) = 0;
    virtual void finish_pass1(Pass1Stats* st) = 0;
    virtual void reset_pass1() = 0;   // drop reads + table (bench: repeat the step)
    virtual void sweeps(SweepStats* st) = 0;            // delow + mark linear + kmerFreq histogram
    virtual void build_layout() = 0;                    // reference iteration order (needs -a for bit-exactness)
    virtual uint64_t node_count() const = 0;
    virtual void dump_nodes(void* host_out) = 0;        // node_count() records in reference iteration order
    // the entries whose key hashes (with seed) to 0 mod one_in, as {key[4] (zero-padded), payload, rank} u64 records; returns how many
    // there are (at most cap are written, in slot order: the caller sorts)
    virtual uint64_t sample_table(uint64_t seed, uint32_t one_in, uint64_t* host_out, uint64_t cap) = 0;
    // ---- graph phases
    virtual void remove_tips(TipStats* st) = 0;         // removeSingleTips (if D==0) + removeMinorTips
    virtual void build_edges(EdgeStats* st, std::string* edge_text) = 0;   // uncompressed .edge text, in edge order
    virtual void pass2(Pass2Stats* st, std::string* prearc_text, std::string* path_bin, std::string* mark_text) = 0;
    virtual void vertices(std::string* vertex_text, uint64_t* n_vertex) = 0;
    virtual uint64_t num_ed() const = 0;   // edge_c incl. twins, as of build_edges (the EDGEs line of .preGraphBasic)
};

IEngine* make_engine(const PgParams& p);   // picks 128- or 256-bit keys from K; throws std::runtime_error on CUDA errors

}   // namespace pgb
