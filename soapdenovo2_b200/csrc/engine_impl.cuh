// engine_impl.cuh -- EngineT<NW>: device state + phase methods; the methods are defined across decode.cu, pass1.cu, skm.cu,
// skm_apply.cu, table_build.cu, layout.cu, tips.cu, edges.cu, pass2.cu and explicitly instantiated for NW = 2 (K <= 63) and NW = 4
// (K <= 127).
#pragma once
#include "engine.h"
#include "cuda_owner.h"
#include "kmer.cuh"
#include "table.cuh"
#include "skm.cuh"
#include <cuda_runtime.h>
#include <cstdlib>
#include <ctime>
#include <string>
#include <vector>

namespace pgb {

inline u64 next_pow2(u64 x) { u64 p = 1; while (p < x) p <<= 1; return p; }

// One fed text chunk, decoded: 2-bit packed reads (LSB-first, W64 words per read) + lengths.  Stays resident in HBM so
// that pass 2 re-scans the reads without touching the text again (the reference re-parses every file, prlRead2path.c:786).
struct ReadChunk {
    u64* words = nullptr;
    u32* len = nullptr;
    u64 n_rec = 0;
    u64 ord_base = 0, ord_stride = 1;
};

enum Counter { C_DISTINCT = 0, C_INSTANCES, C_KEPT, C_LINEAR, C_REMOVED, C_MISC0, C_MISC1, C_MISC2, C_BADFMT, C_XERR, C_XUSED, C_RESERVED, C_DEFER, C_MAXU,
               C_XSEGS, C_XEPOCH, C_SPILLKEYS, C_REDO, C_SKM_STAGED, C_SKM_DRAINED, C_CARRY, C_BIN_OVF, C_COUNT };
               // C_SPILLKEYS: keys a region build stored WITHOUT the fused sweeps (its carries); C_REDO: records decoded by the general rules
               // (k_decode_fix); C_SKM_STAGED / C_SKM_DRAINED: records an aggregation read, distinct records it expanded (k_skm_apply);
               // C_CARRY: entries on the region build's remnant list (bin overflow + carries), C_BIN_OVF: the bin overflow among them

// What an aggregation launch reports: C_XERR .. C_MAXU, read with one copy
struct FlushOutcome { u64 xerr, xused, reserved, defer, maxu; };

// Counters moved with one copy or memset: C_XERR .. C_MAXU (FlushOutcome), C_LINEAR + C_REMOVED (reset by the sweeps),
// C_DISTINCT .. C_KEPT (absorb)
static_assert(C_XUSED == C_XERR + 1 && C_RESERVED == C_XERR + 2 && C_DEFER == C_XERR + 3 && C_MAXU == C_XERR + 4 &&
              sizeof(FlushOutcome) == (C_MAXU - C_XERR + 1) * sizeof(u64), "FlushOutcome mirrors C_XERR .. C_MAXU");
static_assert(C_REMOVED == C_LINEAR + 1, "C_LINEAR, C_REMOVED are reset together");
static_assert(C_INSTANCES == C_DISTINCT + 1 && C_KEPT == C_DISTINCT + 2, "absorb writes C_DISTINCT .. C_KEPT with one copy");

// Whether the end-of-pass sweeps (K4) already ran inside this pass's aggregation launch.  They can, when the launch is the pass so far (no
// key in the table, no launch and no per-instance insert before it): such a launch builds the table region by region (k_table_build,
// table_build.cu), every entry is final when its region is written, and one pass over the table is saved.  Without -d the sweeps only
// SET flags that k_sweep recomputes, so the build may do them speculatively; with -d the link counters are zeroed for good, so the
// launch must be known to be the last of the pass (finish_pass1 on one GPU).  Whatever touches the table afterwards -- another launch,
// a per-instance insert, a table growth, a bin overflow, more carries than the spill list holds -- makes the result Plain.
//   Untouched  no aggregation launch and no per-instance insert since reset_pass1
//   Fused      this pass's only launch was a region build that applied the sweeps, and they still hold: sweeps() sweeps the carries only
//   Plain      anything else: sweeps() runs k_sweep over the whole table
enum class PassSweeps { Untouched, Fused, Plain };

// The decode of one text chunk (decode.cu), shared by pass 1 (feed_text) and the map stage (map.cu).  decode_lines counts the
// records (one host sync of stream sd; h_cnt: pinned, C_COUNT + 1 words) and indexes their sequence lines in line_buf;
// decode_records packs them into words / lens (W64 words per read) and adds "kmer(s) in reads" / reads kept to d_cnt.
struct DecodeLines {
    u32* seq_start;
    u32* seq_end;
    u32* n_redo;   // records the fast decode could not handle (general rules: k_decode_fix) ...
    u32* redo;     // ... and their indices
    u32* flag;     // [n_rec] 1 once a record is on the redo list
    u64 n_rec;
};
void check_format(const u64* h_cnt);   // throws the malformed-input error when the line index flagged a bad record
DecodeLines decode_lines(const unsigned char* d_text, size_t nbytes, int fastq, int n_sm, DevBuf& scan_buf, DevBuf& line_buf, u64* d_cnt, u64* h_cnt,
                         cudaStream_t sd);
void decode_records(const unsigned char* d_text, size_t nbytes, const DecodeLines& L, int maxlen, int reverse, int K, int W64, int n_sm, u64* words,
                    u32* lens, u64* d_cnt, cudaStream_t sd);

// The aggregation launch whose outcome (deferred buckets, time) has not been read yet
struct PendingFlush {
    bool pending = false;
    bool region = false;  // the launch wrote its aggregates to the bins and k_table_build made the table from them
    bool sweep = false;   // ... and the build applied the end-of-pass sweeps
    int half = 0;         // the arena half it reads
};

struct BinArgs;   // table_build.cuh

template <int NW>
class EngineT : public IEngine {
public:
    explicit EngineT(const PgParams& p);
    ~EngineT() override;

    void feed_text(const char* text, size_t nbytes, bool on_device, int fastq, uint64_t ord_base, uint64_t ord_stride,
                   int reverse_seq, int maxlen) override;
    uint64_t last_chunk_records() const override { return last_records_; }
    void finish_pass1(Pass1Stats* st) override;
    void reset_pass1() override;
    void sweeps(SweepStats* st) override;
    void build_layout() override;
    uint64_t node_count() const override { return n_nodes_; }
    void dump_nodes(void* host_out) override;
    uint64_t sample_table(uint64_t seed, uint32_t one_in, uint64_t* host_out, uint64_t cap) override;
    void remove_tips(TipStats* st) override;
    void build_edges(EdgeStats* st, std::string* edge_text) override;
    void pass2(Pass2Stats* st, std::string* prearc_text, std::string* path_bin, std::string* mark_text) override;
    void vertices(std::string* vertex_text, uint64_t* n_vertex) override;
    uint64_t num_ed() const override { return num_ed_; }

    // ---- state
    PgParams prm_;
    KParams<NW> kp_;
    // Words per key in the output files (kout_word): the 127-mer build prints four at every K
    int out_words() const { return prm_.flavour127 ? 4 : 2; }
    // The 127-mer build's reverse complement of a (K+1) = 128-mer keeps its lowest word only (krc_ref)
    bool quirk128() const { return prm_.flavour127 && prm_.K + 1 == 128; }
    // Three streams make pass 1 a pipeline: st_copy_ (H2D of chunk c+1) | st_dec_ (line index + decode of chunk c: all a chunk's host
    // sync waits for) | st_ (partition, aggregation, every later phase).  With the per-instance insert (PGB200_SKM=0) decode runs on st_.
    Stream st_, st_dec_;
    static constexpr int EV_RING = 32;          // per-chunk event quads {decode begin, decode end, insert begin, insert end}
    Event ev_ring_[EV_RING][4];
    Event ev_dec_done_;
    unsigned ev_head_ = 0, ev_tail_ = 0;        // chunks [ev_tail_, ev_head_) have unsettled timings
    int W64_ = 0;   // packed words per read
    int n_sm_ = 0;  // SMs of the device: grid-stride kernels launch a fixed number of CTAs per SM
    std::vector<ReadChunk> chunks_;
    uint64_t last_records_ = 0, total_records_ = 0;
    Pass1Stats p1_;

    Table<NW> tab_{nullptr, 0};
    u64 cap_ = 0;
    DevBuf tab_buf_;
    DevBuf cnt_buf_;
    u64* d_cnt_ = nullptr;      // Counter[] (in cnt_buf_)
    Pinned<u64> h_cnt_;         // pinned mirror

    // decode scratch
    DevBuf text_bufs_[2], line_buf_, scan_buf_, hist_buf_;
    int text_flip_ = 0;
    Stream st_copy_;            // H2D of chunk i+1 overlaps the insert of chunk i
    Stream st_clear_;           // the table clear, queued before the first write that needs an empty table (clear_table_if_dirty)
    Event ev_clear_;
    bool clear_pending_ = false;
    bool table_dirty_ = false;  // the table memory holds no valid table (fresh allocation, or a previous pass): cleared lazily
    Event ev_copy_;
    void settle_timing();                        // waits for every fed chunk's kernels and books their times
    void settle_oldest();

    // layout
    u64 n_nodes_ = 0;           // distinct k-mers == entries in iteration order
    DevBuf order_buf_;          // u64 order[n_nodes_] : iteration index -> ktab slot
    // growth replay (no -a): per set, 1 if the set ends at its growth threshold and a later instance makes the reference grow it
    std::vector<uint32_t> late_growth(const std::vector<u64>& cnt, const std::vector<u64>& first, const u64* sort_keys);

    // edges / pass 2 state
    u64 num_ed_ = 0;
    DevBuf patch_buf_;          // (K+1)-mer patch table
    u64 patch_mask_ = 0;

    // pass 1, per-instance insert (pass1.cu): PGB200_SKM=0, single GPU only -- the second exact path the parity tests compare with
    void chop_insert_chunk(const ReadChunk& ch);
    void check_format_counter();
    // pass 1, aggregated: super-k-mer records scattered into the owners' arenas, one table update per DISTINCT k-mer
    // ... the exchange (skm.cu)
    int skm_mode_ = -1;          // -1: aggregated for device-resident text, per-instance inserts for host text; 0 / 1: forced (PGB200_SKM)
    int skm_flush_every_ = -1;   // single GPU: aggregate every n chunks (-1: host text whenever the insert stream is idle, device text only when the arena is full)
    SkmGeom skm_geom_;
    u32 skm_own_lo_ = 0, skm_own_hi_ = 0;
    int skm_own_shift_ = -1;
    int skm_part_threads_ = 128;
    DevBuf skm_cnt_, skm_segoff_, skm_cursor_, skm_scan_, skm_side_;
    DevBuf skm_scratch_;               // SkmScratch (skm.cu): the exchange's device-side cursors and scan total
    // the exchange arena: [SKM_ARENA_HALVES][nseg | ring | offsets | world x cap_pair records]; xa_peer_[o] = owner o's arena as mapped here
    SkmArenaGeom xa_geom_;
    DevBuf xa_buf_;
    std::vector<void*> xa_peer_;
    std::vector<IpcMapping> xa_ipc_opened_;
    u64 xa_send_epoch_ = 0, xa_flushed_epoch_ = 0;
    u32 xa_seg_idx_ = 0;
    std::vector<u64> xa_reads_cum_;   // reads fed in this epoch after 0, 1, 2, ... chunks (the fill known to the host lags behind)
    bool xa_dirty_ = false;
    void skm_init();
    void xchg_default_setup();
    u64 skm_room_estimate(u64 n_rec);
    void skm_make_room(u64 n_rec, bool host_text);
    void skm_feed_chunk(size_t ci);
    void skm_close_epoch(bool hard);
    void skm_fence();
    void skm_reset();
    void xchg_setup(uint64_t cap_records) override;
    void xchg_export(void* handle64) override;
    void xchg_import(int peer, const void* handle64) override;
    void* xchg_base() override;
    void xchg_import_ptr(int peer, int peer_device, void* base) override;
    void xchg_fence() override { skm_fence(); }
    bool xchg_room(uint64_t n_rec) override;
    // ... the bucket aggregation (skm_apply.cu)
    DevBuf skm_segs_;                  // SkmSegList (skm_apply.cu): the segments an aggregation launch reads
    DevBuf skm_deferred_[2];           // deferred buckets of an aggregation launch, read by the re-run that writes the other list
    PendingFlush flush_;
    PassSweeps pass_sweeps_ = PassSweeps::Untouched;
    Pinned<FlushOutcome> h_outcome_;   // as of the end of the last aggregation launch
    Event ev_flush_begin_, ev_flush_;
    void skm_launch_apply(const u32* list, u32 n_list, u32* deferred_out, bool region);
    void skm_flush(bool final_of_pass = false);
    void skm_flush_complete();
    void flush() override { skm_flush(); }
    // ... the region build (table_build.cu; PGB200_TABLE_BUILD=region, the default; merge: every launch merges into the global table
    // with the CAS protocol)
    bool table_build_region_ = true;
    int region_log2_ = 0;              // slots per region (and bin capacity) = 2^region_log2_
    DevBuf bin_cursor_;                // [regions] u32: entries the aggregation stored in each bin
    DevBuf carry_buf_;                 // remnant list: entries past their bin's capacity, then the build's carries (Slot<NW> format)
    u64 carry_cap_ = 0;
    DevBuf spill_list_;                // slots of the keys a Fused launch stored unswept (the region build's carries)
    static constexpr u64 SPILL_CAP = 1ull << 22;
    BinArgs bin_args() const;          // where a region-mode aggregation launch stores its aggregates (table_build.cuh)
    void table_build_prepare();
    void table_build_launch();
    bool table_build_redo();
    void absorb(IEngine* other) override;

    // helpers
    void ensure_table_bound(u64 have, u64 incoming);
    void create_table_if_needed(bool clean = true);   // clean = false: the caller overwrites every slot (region build)
    void clear_table_if_dirty();
    void alloc_first_table();
    std::vector<DevBuf> arena_;   // read-store blocks
    size_t arena_used_ = 0;
    void* arena_alloc(size_t bytes);
    void grow_table(u64 new_cap);
    bool grow_table_for(u64 need, double load, u64 headroom, bool partial);
    void alloc_table(u64 cap);
    void sync() {
        if (st_dec_) PG_CUDA(cudaStreamSynchronize(st_dec_));
        PG_CUDA(cudaStreamSynchronize(st_));
        if (clear_pending_) { PG_CUDA(cudaStreamSynchronize(st_clear_)); clear_pending_ = false; }
    }
    // The table clear runs on its own stream: decode and partition kernels (which do not touch the table) run beside the 17 GB memset
    // instead of behind it.  Whoever touches the table next orders the insert stream behind the clear.
    void join_table_clear() {
        if (!clear_pending_) return;
        PG_CUDA(cudaStreamWaitEvent(st_, ev_clear_, 0));
        clear_pending_ = false;
    }
    void read_counters() {   // everything queued so far has completed when this returns
        if (st_dec_) PG_CUDA(cudaStreamSynchronize(st_dec_));
        PG_CUDA(cudaMemcpyAsync(h_cnt_, d_cnt_, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, st_));
        PG_CUDA(cudaStreamSynchronize(st_));
    }
    void read_counters_on(cudaStream_t s) {   // per-chunk sync of the decode stream only: counters of st_ work may lag
        PG_CUDA(cudaMemcpyAsync(h_cnt_, d_cnt_, C_COUNT * sizeof(u64), cudaMemcpyDeviceToHost, s));
        PG_CUDA(cudaStreamSynchronize(s));
    }
};

// reference table geometry helpers (newhash.c:142-185, 200-233; prlHashReads.c:369-390)
inline bool ref_is_prime(u64 n) {
    if (n < 4) return true;
    if (n % 2 == 0) return false;
    u64 mx = (u64)__builtin_sqrtf((float)n);   // float sqrt, strict '<': squares of primes count as prime
    for (u64 i = 3; i < mx; i += 2)
        if (n % i == 0) return false;
    return true;
}
inline u64 ref_next_prime(u64 n) {
    if (n % 2 == 0) n++;
    while (!ref_is_prime(n)) n += 2;
    return n;
}
inline u64 ref_static_set_size(int initG, int P, bool flavour127) {
    u64 want = (u64)((double)initG * 1024.0f * 1024.0f * 1024.0f / (double)P / (flavour127 ? 40 : 24)), k = 0;
    do ++k; while (k * 0xFFFFFFULL < want);
    u64 init = k * 0xFFFFFFULL;
    return init < 3 ? 3 : ref_next_prime(init);
}

}   // namespace pgb
