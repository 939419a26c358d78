// engine_impl.cuh -- EngineT<NW>: device state + phase methods; the methods are defined across decode.cu, pass1.cu, skm.cu,
// layout.cu, tips.cu, edges.cu, pass2.cu and explicitly instantiated for NW = 2 (K <= 63) and NW = 4 (K <= 127).
#pragma once
#include "engine.h"
#include "kmer.cuh"
#include "table.cuh"
#include "skm.cuh"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <ctime>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

namespace pgb {

#define PG_CUDA(call)                                                                                         \
    do {                                                                                                      \
        cudaError_t e__ = (call);                                                                             \
        if (e__ != cudaSuccess) {                                                                             \
            char b__[512];                                                                                    \
            snprintf(b__, sizeof b__, "CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, \
                     cudaGetErrorString(e__));                                                                \
            throw std::runtime_error(b__);                                                                    \
        }                                                                                                     \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() {}
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(bytes, o.bytes); return *this; }
    ~DevBuf() { release(); }
    void alloc(size_t n) {
        release();
        if (n == 0) n = 16;
        PG_CUDA(cudaMalloc(&p, n));
        bytes = n;
    }
    void ensure(size_t n) { if (n > bytes) alloc(n + n / 4); }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Owner of a stream, an event or a pinned host block, in the style of DevBuf: released with its owner, moved but never copied.
template <class T, cudaError_t (*Release)(T)>
struct CudaOwned {
    T h = nullptr;
    CudaOwned() {}
    CudaOwned(CudaOwned&& o) noexcept : h(o.h) { o.h = nullptr; }
    CudaOwned& operator=(CudaOwned&& o) noexcept { std::swap(h, o.h); return *this; }
    ~CudaOwned() { if (h) Release(h); }
    operator T() const { return h; }
};
template <class T> cudaError_t free_pinned(T* p) { return cudaFreeHost(p); }
using Stream = CudaOwned<cudaStream_t, cudaStreamDestroy>;
using Event = CudaOwned<cudaEvent_t, cudaEventDestroy>;
template <class T> using Pinned = CudaOwned<T*, free_pinned<T>>;

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
               C_XSEGS, C_XEPOCH, C_SPILLKEYS, C_REDO, C_COUNT };   // C_SPILLKEYS: keys the aggregation stored WITHOUT the fused sweeps;
                                                                 // C_REDO: records decoded by the general rules (k_decode_fix)

// What an aggregation launch reports: C_XERR .. C_MAXU, read with one copy
struct FlushOutcome { u64 xerr, xused, reserved, defer, maxu; };

// Counters moved with one copy or memset: C_XERR .. C_MAXU (FlushOutcome), C_LINEAR + C_REMOVED (reset by the sweeps),
// C_DISTINCT .. C_KEPT (absorb)
static_assert(C_XUSED == C_XERR + 1 && C_RESERVED == C_XERR + 2 && C_DEFER == C_XERR + 3 && C_MAXU == C_XERR + 4 &&
              sizeof(FlushOutcome) == (C_MAXU - C_XERR + 1) * sizeof(u64), "FlushOutcome mirrors C_XERR .. C_MAXU");
static_assert(C_REMOVED == C_LINEAR + 1, "C_LINEAR, C_REMOVED are reset together");
static_assert(C_INSTANCES == C_DISTINCT + 1 && C_KEPT == C_DISTINCT + 2, "absorb writes C_DISTINCT .. C_KEPT with one copy");

// Whether the end-of-pass sweeps (K4) already ran inside this pass's aggregation launch.  The launch can apply them to every entry it
// stores only when it is the pass so far (empty table, no launch and no per-instance insert before it): each entry is then final, and
// one pass over the table is saved.  Without -d the sweeps only SET flags that k_sweep recomputes, so the launch may do them
// speculatively; with -d the link counters are zeroed for good, so the launch must be known to be the last of the pass (finish_pass1 on
// one GPU).  Whatever touches the table afterwards -- another launch, a per-instance insert, a table growth, more unswept keys than the
// spill list holds -- makes the result Plain.
//   Untouched  no aggregation launch and no per-instance insert since reset_pass1
//   Fused      this pass's only launch applied the sweeps and they still hold: sweeps() only sweeps the spill list
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
    bool sweep = false;   // the launch (and its deferred re-runs) applies the end-of-pass sweeps
    int half = 0;         // the arena half it reads
};

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
    Stream st_clear_;           // the table clear between two passes (reset_pass1)
    Event ev_clear_;
    bool clear_pending_ = false;
    Event ev_copy_;
    void settle_timing();                        // waits for every fed chunk's kernels and books their times
    void settle_oldest();

    // layout
    u64 n_nodes_ = 0;           // distinct k-mers == entries in iteration order
    DevBuf order_buf_;          // u64 order[n_nodes_] : iteration index -> ktab slot

    // edges / pass 2 state
    u64 num_ed_ = 0;
    DevBuf patch_buf_;          // (K+1)-mer patch table
    u64 patch_mask_ = 0;

    // pass 1, per-instance insert (pass1.cu): PGB200_SKM=0, single GPU only -- the second exact path the parity tests compare with
    void chop_insert_chunk(const ReadChunk& ch);
    void check_format_counter();
    // pass 1, aggregated (skm.cu): super-k-mer records scattered into the owners' arenas, one table update per DISTINCT k-mer
    int skm_mode_ = -1;          // -1: aggregated for device-resident text, per-instance inserts for host text; 0 / 1: forced (PGB200_SKM)
    int skm_flush_every_ = -1;   // single GPU: aggregate every n chunks (-1: host text whenever the insert stream is idle, device text only when the arena is full)
    SkmGeom skm_geom_;
    u32 skm_own_lo_ = 0, skm_own_hi_ = 0;
    int skm_own_shift_ = -1;
    int skm_part_threads_ = 128;
    DevBuf skm_cnt_, skm_segoff_, skm_cursor_, skm_scan_, skm_side_;
    DevBuf skm_scratch_;               // SkmScratch (skm.cu): the exchange's device-side cursors, scan total and segment list
    DevBuf skm_deferred_[2];           // deferred buckets of an aggregation launch, read by the re-run that writes the other list
    // the exchange arena: [SKM_ARENA_HALVES][nseg | ring | offsets | world x cap_pair records]; xa_peer_[o] = owner o's arena as mapped here
    SkmArenaGeom xa_geom_;
    DevBuf xa_buf_;
    std::vector<void*> xa_peer_, xa_ipc_opened_;
    u64 xa_send_epoch_ = 0, xa_flushed_epoch_ = 0;
    u32 xa_seg_idx_ = 0;
    PendingFlush flush_;
    PassSweeps pass_sweeps_ = PassSweeps::Untouched;
    DevBuf spill_list_;                // slots of the keys a Fused launch stored unswept (instances that did not fit a bucket's shared-memory table)
    static constexpr u64 SPILL_CAP = 1ull << 22;
    Pinned<FlushOutcome> h_outcome_;   // as of the end of the last aggregation launch
    Event ev_flush_begin_, ev_flush_;
    void skm_close_epoch(bool hard);
    void skm_flush_complete();
    void skm_launch_apply(const u32* list, u32 n_list, u32* deferred_out);
    std::vector<u64> xa_reads_cum_;   // reads fed in this epoch after 0, 1, 2, ... chunks (the fill known to the host lags behind)
    u64 skm_room_estimate(u64 n_rec);
    bool xa_dirty_ = false;
    void skm_init();
    void xchg_default_setup();
    void skm_send_args(void* out_args, int half);
    void skm_make_room(u64 n_rec, bool host_text);
    void skm_feed_chunk(size_t ci);
    void skm_fence();
    void skm_flush(bool final_of_pass = false);
    void skm_reset();
public:
    void xchg_setup(uint64_t cap_records) override;
    void xchg_export(void* handle64) override;
    void xchg_import(int peer, const void* handle64) override;
    void* xchg_base() override;
    void xchg_import_ptr(int peer, int peer_device, void* base) override;
    void xchg_fence() override { skm_fence(); }
    void flush() override { skm_flush(); }
    bool xchg_room(uint64_t n_rec) override;
    void absorb(IEngine* other) override;

    // helpers
    void ensure_table_bound(u64 have, u64 incoming);
    void create_table_if_needed();
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
    // reset_pass1 clears the table on its own stream: the next pass's decode and partition kernels (which do not touch the table) run
    // beside the 17 GB memset instead of behind it.  Whoever touches the table next orders the insert stream behind the clear.
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
