// skm_apply.cu -- aggregated pass 1, the bucket aggregation: one shared-memory aggregation per bucket of the records the exchange
// (skm.cu) delivered, ONE global table update per distinct k-mer.
//
//   flush (end of pass 1 / arena full):  k_skm_apply over the owned buckets; buckets whose worst case does not fit the global table
//                                     are deferred, the table grows, the deferred buckets run again.  When the table holds no key yet
//                                     (the pass's first launch: the normal case is one launch per pass) the launch stores its
//                                     aggregates into bins -- the table memory of their home region, no probe, no claim -- and
//                                     k_table_build makes each region in shared memory and writes it whole: no table clear, and the
//                                     end-of-pass sweeps -- delow, linear flag, coverage histogram (thread_delow / thread_mark /
//                                     freqStat, prlHashReads.c:953-1132) -- are applied to every entry as its region is written.
#include "engine_impl.cuh"
#include "table_build.cuh"
#include "chop.cuh"

namespace pgb {

constexpr int SKM_APPLY_THREADS = 256;
// Shared-memory table of a bucket: 1024 slots (32 KB at K <= 63) plus the record stage (2 x 128 records), the distinct-record buffer
// (SKM_BUF_RECS = 128 records, their reversed bases, counts and a 512-slot dedup table) put 4 CTAs = 32 warps on an H100 SM
// (4 x 54 KB of 228 KB) at 64 registers per thread; 256-bit keys (48 B slots, a 2 x 64-record stage, a 256-slot dedup table, 71 KB
// per CTA) run 3 CTAs at 74.  No stack frame and no spills at either width (skm_w).  5 or 6 CTAs spill at the register budget they
// allow.
#ifndef SKM_APPLY_MIN_BLOCKS_NW2
#define SKM_APPLY_MIN_BLOCKS_NW2 4
#endif
#ifndef SKM_APPLY_MIN_BLOCKS_NW4
#define SKM_APPLY_MIN_BLOCKS_NW4 3
#endif
#define SKM_APPLY_MIN_BLOCKS(NW) ((NW) == 2 ? SKM_APPLY_MIN_BLOCKS_NW2 : SKM_APPLY_MIN_BLOCKS_NW4)
constexpr int SKM_SOFT_LIMIT = SKM_SLOTS - SKM_APPLY_THREADS - 64;   // claims stop here: the table can never fill up completely

// ------------------------------------------------------------------------------------------------ aggregation
// Shared-memory table of one bucket, structure of arrays: key words [NW][S], payload [S], rank [S], claim list [S] (u16).
// Claim protocol: smem_find_or_claim.  Empty slots hold {PAYLOAD_FRESH, ~0} in their payload / rank words, so the claimer records its
// own instance together with the lanes that found the key (one update path).  The claimer also appends the slot to the claim list (the
// flush walks the list, not the table).  (Prefetching the k-mer's home slot of the GLOBAL table into L2 at claim time measured no
// difference and was dropped.)
// S slots (any size: the slot index is a multiply-shift range reduction of a 32-bit hash), claims stop at LIMIT so that the
// table can never fill up completely whatever the number of concurrent claimers; LT = type of the claim-list entries.
template <int NW, int S, int LIMIT, class LT>
struct SmemTable {
    u64* key;   // [NW * S]
    u64* pay;
    u64* rnk;
    LT* list;
    u32* count;
    // Two phases with a warp barrier between them (the caller's __syncwarp over the lanes that have an instance): first every lane
    // finds or claims its slot (lanes differ only in the number of probes), then the lanes that found an existing key apply their
    // instance TOGETHER (without the barrier the lanes that match on their first probe run the long update on their own while the
    // others keep probing: the update code then executes several times per step with a few active lanes each).
    // find(): 1 = key present at idx (found, or claimed by this lane just now), 3 = no room (caller spills)
    __device__ __forceinline__ int find(const Kmer<NW>& k, u32& idx) const {
        idx = (u32)(((u64)skm_slot_hash(k, 32) * (u64)S) >> 32);
        // an empty slot holds {PAYLOAD_FRESH, ~0}: the claimer records its instance with everybody else in apply()
        return smem_find_or_claim<NW, true>(key, 1, S, S, k, idx, [&] { return *(volatile u32*)count < (u32)LIMIT; }, [](u32) {},
                                            [&](u32 j, bool claimed) {
                                                if (claimed) list[atomicAdd(count, 1u)] = (LT)j;
                                            }) ? 1 : 3;
    }
    // c identical instances
    __device__ __forceinline__ void apply(u32 idx, unsigned left, unsigned right, u64 rank, unsigned c) const {
        payload_fold(&pay[idx], ((volatile u64*)pay)[idx], [=](u64 p) { return payload_apply_n(p, left, right, c); });
        rank_min(&rnk[idx], rank, rank < ((volatile u64*)rnk)[idx]);
    }
};

// the segments one aggregation launch reads, in device memory (built by k_skm_segs from what the senders published)
struct SkmSegList {
    const u64* recs[SKM_MAX_SEGS];
    const u32* segoff[SKM_MAX_SEGS];
    u32 n;
    u32 pad;
};
struct SkmFlushArgs {
    int world;
    u32 max_seg, bo_stride;
    u64 cap_pair;
    int rec_words;
    SkmArenaHalf half;   // the epoch half the launch reads
    SkmSegList* segs;
    u64* counters;
};
__global__ void __launch_bounds__(256) k_skm_segs(SkmFlushArgs a) {
    __shared__ u32 s_base[SKM_MAXW + 1];
    if (threadIdx.x == 0) {
        u32 acc = 0;
        for (int s = 0; s < a.world; s++) { s_base[s] = acc; acc += a.half.nseg[s] < a.max_seg ? a.half.nseg[s] : a.max_seg; }
        s_base[a.world] = acc;
        if (acc > (u32)SKM_MAX_SEGS) { atomicAdd(&a.counters[C_XERR], 1ull); acc = SKM_MAX_SEGS; }
        a.segs->n = acc;
        a.counters[C_RESERVED] = a.counters[C_DISTINCT];   // keys the table already holds; the launch that follows adds its reservations
        a.counters[C_DEFER] = 0;
        a.counters[C_MAXU] = 0;
    }
    __syncthreads();
    for (int s = 0; s < a.world; s++) {
        const u32 n = s_base[s + 1] - s_base[s];
        for (u32 i = threadIdx.x; i < n; i += blockDim.x) {
            const u32 j = s_base[s] + i;
            if (j >= (u32)SKM_MAX_SEGS) continue;
            const SkmSegDesc d = a.half.ring[(u64)s * a.max_seg + i];
            a.segs->recs[j] = a.half.recs + ((u64)s * a.cap_pair + d.rec_off) * a.rec_words;
            a.segs->segoff[j] = a.half.segoff + ((u64)s * a.max_seg + i) * a.bo_stride;
        }
    }
}

struct SkmApplyArgs {
    const SkmSegList* segs;
    const u32* bucket_list;   // nullptr: buckets 0 .. n_list-1; else the deferred buckets of the previous launch
    u32 n_list;
    u64* counters;            // C_RESERVED: keys the table is committed to hold; C_DEFER / C_MAXU: deferred buckets, their largest bound
    u64 limit;
    u32* deferred;
    BinArgs bins;             // k_skm_apply<NW, true>: where the aggregates go
    int collapse;             // SKM_COLLAPSE_OFF / _ON / _AUTO (PGB200_SKM_COLLAPSE): both ways of filling the buffer are exact.  256-bit
                              // keys only: at K <= 63 records repeat (0.553 of them distinct at 30x) and the kernel always collapses;
                              // its register budget at 4 CTAs per SM has no room for the copy path (DESIGN.md §5)
};
constexpr u64 SKM_CREDIT = 1ull << 16;   // table room a CTA reserves at a time (keys)
constexpr int SKM_COLLAPSE_OFF = 0, SKM_COLLAPSE_ON = 1, SKM_COLLAPSE_AUTO = 2;
// auto: a CTA measures its distinct / staged records over SKM_AUTO_PROBE collapsed buckets; above SKM_AUTO_NUM / SKM_AUTO_DEN the
// records hardly repeat and it copies the next SKM_AUTO_SKIP buckets' records straight into the buffer, then measures again
constexpr u32 SKM_AUTO_PROBE = 8, SKM_AUTO_SKIP = 56, SKM_AUTO_NUM = 9, SKM_AUTO_DEN = 10;

// -DSKM_PHASE_CLOCKS: k_skm_apply adds up clock64() per phase over all its threads (stage wait, instance build, find / claim, apply,
// spill to the global table, flush, record dedup), and thread 0 of every CTA splits the CTA's wall time between two of its
// barrier-delimited boundaries into SKM_WALL_PHASES phases that cover the whole kernel; the host prints both splits of every
// aggregation with PGB200_SKM_STATS.  Off: no code at all.
#ifdef SKM_PHASE_CLOCKS
constexpr int SKM_PHASES = 7;
__device__ unsigned long long g_skm_phase_clk[SKM_PHASES];
#define SKM_T0(v) const long long v = clock64()
#define SKM_ACC(i, v) clk[i] += (u64)(clock64() - (v))
// wall phases: top of bucket (scan + credit), stage wait, dedup or copy of a window incl. its barrier, drain pre-pass, drain steps
// incl. the barrier, flush incl. the barrier, other; then the kernel's end minus start and the number of CTAs (the check: the
// phases sum to it)
constexpr int SKM_WALL_PHASES = 7;
__device__ unsigned long long g_skm_wall_clk[SKM_WALL_PHASES + 2];
#define SKM_WALL(i)                                      \
    do {                                                 \
        if (tid == 0) {                                  \
            const long long t_ = clock64();              \
            s_wall[i] += (u64)(t_ - s_wall_last);        \
            s_wall_last = t_;                            \
        }                                                \
    } while (0)
#else
#define SKM_T0(v)
#define SKM_ACC(i, v)
#define SKM_WALL(i)
#endif

// Exclusive prefix sum over the CTA; *total = the sum.  The caller separates two calls with a __syncthreads (s_warp is reused).
__device__ __forceinline__ u32 cta_exclusive_scan(u32 v, u32* s_warp, u32& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    u32 inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 u = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += u;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    u32 off = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < SKM_APPLY_THREADS / 32; w++) {
        const u32 s = s_warp[w];
        off += w < wid ? s : 0u;
        tot += s;
    }
    total = tot;
    return off + inc - v;
}

// Records of one bucket staged per window: the window is W consecutive records of the bucket's concatenated segment ranges; every
// segment thread copies its part of the window with one bulk copy, completed on the half's mbarrier.  The stage is double-buffered:
// the next window (or the next bucket's first) is in flight while the current one is processed and synchronised.  A window is only
// collapsed into the distinct-record buffer (skm_dedup_insert), so the stage just has to keep the bulk copies ahead.
// Records per window: 128 at K <= 63 (2 x 4 KB of stage; a bucket's ~210 records at 30x take 2 windows instead of 4, so half the
// window barriers, and 128 threads collapse a window instead of 64), 64 at K > 63 (2 x 3 KB: what 3 CTAs per SM leave).
#ifndef SKM_STAGE_RECS_NW2
#define SKM_STAGE_RECS_NW2 128
#endif
#ifndef SKM_STAGE_RECS_NW4
#define SKM_STAGE_RECS_NW4 64
#endif
constexpr int SKM_BUF_RECS = 128;        // distinct records buffered before they are expanded into k-mer instances (a drain)
template <int NW>
__host__ __device__ constexpr int skm_w() { return NW == 2 ? SKM_STAGE_RECS_NW2 : SKM_STAGE_RECS_NW4; }
// the buffer's hash table (record -> buffer position): room for the buffered records and the FULL marks of one window, never full
template <int NW>
__host__ __device__ constexpr int skm_dd_slots() { return SKM_BUF_RECS + skm_w<NW>() < 256 ? 256 : 512; }
template <int NW>
__host__ __device__ constexpr bool skm_stage_ok() {
    return skm_w<NW>() <= SKM_BUF_RECS && SKM_BUF_RECS <= SKM_APPLY_THREADS && SKM_BUF_RECS % skm_w<NW>() == 0 &&
           SKM_BUF_RECS + skm_w<NW>() < skm_dd_slots<NW>();
}
static_assert(skm_stage_ok<2>() && skm_stage_ok<4>(), "one drain empties the buffer for a whole window, one thread per buffered record, "
                                                      "uncollapsed windows fill the buffer exactly, the dedup table never fills up");

constexpr u32 SKM_DD_EMPTY = 0xFFFFFFFFu, SKM_DD_BUSY = 0xFFFFFFFEu, SKM_DD_FULL = 0xFFFFFFFDu;
// One staged record r into the distinct-record buffer: find-or-claim its entry in the dedup table (claim: CAS EMPTY -> BUSY, take
// a buffer position, copy the record with count 1, fence, publish the position); a copy adds 1 to the count and lowers the buffered
// header to the smaller of the two (skm_rec_same).  Returns true when the record found no room (the claim came after the buffer's
// SKM_BUF_RECS positions were taken, or the probe met such a claim, marked FULL): the caller drains the buffer and calls again.
template <int NW>
__device__ __forceinline__ bool skm_dedup_insert(const u64* r, u64* buf, u32* cnt, u32* dd, u32* nbuf) {
    constexpr int RW = NW + 2;
    volatile u32* vdd = dd;
    constexpr int DS = skm_dd_slots<NW>();
    u32 idx = skm_rec_hash<NW>(r) >> (32 - __builtin_ctz(DS));
    for (;;) {
        u32 v = vdd[idx];
        if (v == SKM_DD_EMPTY) {
            v = atomicCAS(&dd[idx], SKM_DD_EMPTY, SKM_DD_BUSY);
            if (v == SKM_DD_EMPTY) {
                const u32 j = atomicAdd(nbuf, 1u);
                if (j >= (u32)SKM_BUF_RECS) {
                    vdd[idx] = SKM_DD_FULL;
                    return true;
                }
#pragma unroll
                for (int i = 0; i < RW; i++) buf[j * RW + i] = r[i];
                cnt[j] = 1;
                __threadfence_block();
                vdd[idx] = j;
                return false;
            }
        }
        while (v == SKM_DD_BUSY) v = vdd[idx];
        if (v == SKM_DD_FULL) return true;
        u64 b[RW];
        const volatile u64* vb = buf + v * RW;
#pragma unroll
        for (int i = 0; i < RW; i++) b[i] = vb[i];
        if (skm_rec_same<NW>(b, r)) {
            atomicAdd(&cnt[v], 1u);
            atomicMin((unsigned long long*)&buf[v * RW], (unsigned long long)r[0]);
            return false;
        }
        idx = (idx + 1) & (DS - 1);
    }
}

// A segment thread's part of one bucket: records lo .. lo+cnt-1 of its segment, at positions cum .. cum+cnt-1 of the bucket.
struct SkmSegRange {
    u32 lo, cnt, cum;
};
// Queue window w of a bucket of R records into a stage half.  Every thread calls it: thread 0 arrives with the window's byte count,
// the segment threads whose range meets the window copy their part.
template <int RW, int SKM_W>
__device__ __forceinline__ void skm_stage_window(u64* stage, u64* bar, const u64* my_recs, const SkmSegRange& sr, u32 R, u32 w) {
    const u32 a = w * (u32)SKM_W, e = min(R, a + (u32)SKM_W);
    if (threadIdx.x == 0) mbar_expect_tx(bar, (e - a) * (u32)(RW * sizeof(u64)));
    if (my_recs) {
        const u32 s0 = max(sr.cum, a), s1 = min(sr.cum + sr.cnt, e);
        if (s0 < s1) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic reads of this half come first
            tma_bulk_g2s(stage + (u64)(s0 - a) * RW, my_recs + (u64)(sr.lo + s0 - sr.cum) * RW, (s1 - s0) * (u32)(RW * sizeof(u64)), bar);
        }
    }
}

// One CTA per bucket (static round-robin over the list: buckets are hash-uniform), one shared-memory table per CTA.  REGION: the
// aggregates go to their bins (bin_store) and k_table_build makes the table; else they are merged into the table (table_merge).  A bucket is
// processed window by window (skm_stage_window); the table persists over the windows and is flushed once per bucket.  When a window
// has landed, one thread per record collapses it into the buffer of distinct records (skm_dedup_insert): at 30x most records of a
// bucket are copies of another one.  The buffer is drained into the table when it is full and at the end of the bucket: one thread
// per buffered record writes its k-mer count prefix P and its reversed bases (skm_rec_reverse), then the warps split the buffer's
// instances into contiguous slices and take 32 CONSECUTIVE instances per step -- all lanes busy whatever the run lengths: the
// records that start inside the step come from one lookahead load of P, and every lane builds its k-mer and reverse complement with
// two shifts of shared-memory words (skm_instance_staged) and applies it as many times as its record occurred.
template <int NW, bool REGION>
__global__ void __launch_bounds__(SKM_APPLY_THREADS, SKM_APPLY_MIN_BLOCKS(NW)) k_skm_apply(Table<NW> tab, KParams<NW> kp, SkmApplyArgs a) {
    constexpr int RW = NW + 2, WARPS = SKM_APPLY_THREADS / 32, C = SKM_BUF_RECS, SKM_W = skm_w<NW>(), SKM_DEDUP_SLOTS = skm_dd_slots<NW>();
    constexpr bool COPY_PATH = NW > 2;   // SKM_COLLAPSE_OFF / _AUTO exist for 256-bit keys only (see SkmApplyArgs::collapse)
    // key[NW][S], pay[S], rnk[S], stage[2][W][RW], buf[C][RW], rv[C][NW+1], list[S] (u16), P[C+1], cnt[C], dedup[DS]
    extern __shared__ __align__(16) u64 s_dyn[];
    u64* const s_stage = s_dyn + (NW + 2) * SKM_SLOTS;
    u64* const s_buf = s_stage + 2 * SKM_W * RW;
    u64* const s_rv = s_buf + C * RW;
    unsigned short* const s_list = reinterpret_cast<unsigned short*>(s_rv + C * (NW + 1));
    u32* const s_P = reinterpret_cast<u32*>(s_list + SKM_SLOTS);
    u32* const s_cnt = s_P + C + 1;
    u32* const s_dd = s_cnt + C;
    __shared__ __align__(8) u64 s_bar[2];
    __shared__ u32 s_warp[WARPS];
    __shared__ u32 s_count, s_defer, s_nbuf;
    __shared__ unsigned char s_pend[SKM_W];   // the window's records still to be collapsed into the buffer
    __shared__ unsigned s_new, s_tot_new;
    __shared__ u64 s_staged, s_drained;   // records staged, distinct records drained (PGB200_SKM_STATS)
    __shared__ u32 s_coll, s_ad_n;        // collapse the next bucket's records; buckets since the auto mode last decided
    __shared__ u64 s_ad_staged, s_ad_drained;   // s_staged, s_drained when it did
#ifdef SKM_PHASE_CLOCKS
    __shared__ u64 s_wall[SKM_WALL_PHASES];
    __shared__ long long s_wall_last;
    const long long t_kernel = clock64();
    if (threadIdx.x == 0) {
        for (int i = 0; i < SKM_WALL_PHASES; i++) s_wall[i] = 0;
        s_wall_last = t_kernel;
    }
#endif
    SmemTable<NW, SKM_SLOTS, SKM_SOFT_LIMIT, unsigned short> st{s_dyn, s_dyn + NW * SKM_SLOTS, s_dyn + (NW + 1) * SKM_SLOTS, s_list, &s_count};
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const unsigned lane_le = 0xffffffffu >> (31 - lane);
    for (int i = tid; i < SKM_SLOTS; i += SKM_APPLY_THREADS) {   // the flush re-empties what it merges
        st.key[i] = EMPTY64;
        st.pay[i] = PAYLOAD_FRESH;
        st.rnk[i] = ~0ull;
    }
    for (int i = tid; i < SKM_DEDUP_SLOTS; i += SKM_APPLY_THREADS) s_dd[i] = SKM_DD_EMPTY;   // each drain re-empties it
    if (tid == 0) {
        s_tot_new = 0;
        s_nbuf = 0;
        s_staged = 0;
        s_drained = 0;
        s_coll = a.collapse != SKM_COLLAPSE_OFF;
        s_ad_n = 0;
        s_ad_staged = 0;
        s_ad_drained = 0;
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
    }
    const int n_segs = (int)a.segs->n;
    const u32* my_so = tid < n_segs ? a.segs->segoff[tid] : nullptr;
    const u64* my_recs = tid < n_segs ? a.segs->recs[tid] : nullptr;
    __shared__ u64 s_credit;             // thread 0: table room this CTA holds (not in a register: the drain needs them all)
    u64& credit = s_credit;
    if (tid == 0) credit = 0;
#ifdef SKM_PHASE_CLOCKS
    u64 clk[SKM_PHASES] = {};
#endif
    auto seg_range = [&](u32 p, SkmSegRange& r) {   // this thread's range of the bucket at list position p (empty past the list)
        r.lo = r.cnt = 0;
        if (p < a.n_list && my_so) {
            const u32 b = a.bucket_list ? a.bucket_list[p] : p;
            r.lo = my_so[b];
            r.cnt = my_so[b + 1] - r.lo;
        }
    };
    u32 pos = blockIdx.x;
    SkmSegRange cur, nxt, nn;            // this thread's ranges of the current, the next and the one after
    seg_range(pos, cur);
    seg_range(pos + gridDim.x, nxt);
    u32 R_cur;
    cur.cum = cta_exclusive_scan(cur.cnt, s_warp, R_cur);
    unsigned half = 0, phase = 0;        // stage half of the current window; bit h: parity of half h's next completion
    __syncthreads();                     // the mbarriers are initialised
    if (pos < a.n_list) skm_stage_window<RW, SKM_W>(s_stage, &s_bar[0], my_recs, cur, R_cur, 0);
    for (; pos < a.n_list; pos += gridDim.x) {
        SKM_WALL(6);
        __syncthreads();   // previous bucket fully flushed (and the empty table visible on the first trip)
        u32 R_nxt;
        nxt.cum = cta_exclusive_scan(nxt.cnt, s_warp, R_nxt);
        seg_range(pos + 2 * gridDim.x, nn);
        if (tid == 0) { s_count = 0; s_new = 0; }
        const u32 R = R_cur;
        // ---- room in the global table: every k-mer instance could be a new key.  Credits are taken SKM_CREDIT keys at a time.
        if (tid == 0) {
            bool defer = false;
            const u64 bound = (u64)R * SKM_MAX_RUN;
            if (credit < bound) {
                unsigned long long* res = (unsigned long long*)&a.counters[C_RESERVED];
                const u64 want = bound - credit, ask = want > SKM_CREDIT ? want : SKM_CREDIT;
                u64 old = atomicAdd(res, (unsigned long long)ask);
                if (old + ask <= a.limit) credit += ask;
                else {
                    atomicAdd(res, (unsigned long long)(0ull - ask));
                    bool got = false;
                    if (ask != want) {
                        old = atomicAdd(res, (unsigned long long)want);
                        if (old + want <= a.limit) { credit += want; got = true; }
                        else atomicAdd(res, (unsigned long long)(0ull - want));
                    }
                    if (!got) {
                        defer = true;
                        const u32 b = a.bucket_list ? a.bucket_list[pos] : pos;
                        a.deferred[atomicAdd((unsigned long long*)&a.counters[C_DEFER], 1ull)] = b;
                        atomicMax((unsigned long long*)&a.counters[C_MAXU], (unsigned long long)bound);
                    }
                }
            }
            if (!defer) credit -= bound;
            s_defer = defer ? 1u : 0u;
        }
        __syncthreads();
        SKM_WALL(0);
        const bool run = !s_defer && R > 0;
        // ---- drain: the nb buffered records -> their k-mer instances -> the shared-memory table; the buffer is empty again
        auto drain = [&](u32 nb) {
            SKM_T0(t_pre);
            // per record: its k-mer count prefix and its reversed bases
            u32 n = 0;
            if ((u32)tid < nb) {
                const u64 hdr = s_buf[tid * RW];
                n = (u32)skm_rec_n(hdr);
                u64 rv[NW + 1];
                skm_rec_reverse<NW>(hdr, s_buf + tid * RW + 1, rv, kp.K);
#pragma unroll
                for (int i = 0; i < NW + 1; i++) s_rv[tid * (NW + 1) + i] = rv[i];
            }
            u32 I;
            const u32 p = cta_exclusive_scan(n, s_warp, I);
            if ((u32)tid < nb) s_P[tid] = p;
            if (tid == 0) s_P[nb] = I;
            __syncthreads();
            SKM_ACC(1, t_pre);
            SKM_WALL(3);
            // ---- the warps: contiguous slices of the buffer's instances, 32 consecutive instances per step
            const u32 steps = (I + 31) / 32, per = (steps + WARPS - 1) / WARPS;
            const u32 q_end = min(I, (wid + 1) * per * 32);
            u32 q0 = wid * per * 32;
            u32 r0 = 0;   // the record holding q0: the last record with P <= q0
            if (q0 < q_end) {
                u32 lo = 0, hi = nb;
                while (hi - lo > 1) {
                    const u32 mid = (lo + hi) >> 1;
                    if (s_P[mid] <= q0) lo = mid; else hi = mid;
                }
                r0 = lo;
            }
            for (; q0 < q_end; q0 += 32) {
                const u32 q = q0 + lane;
                const bool has = q < q_end;
                SKM_T0(t_inst);
                // the records that start at step positions 1 .. 31 (P is strictly increasing: every record holds a k-mer)
                const u32 pn = s_P[min(r0 + 1 + lane, nb)];
                const unsigned starts = __reduce_or_sync(0xffffffffu, pn - q0 - 1 < 31u ? 1u << (pn - q0) : 0u);
                const u32 rec = r0 + __popc(starts & lane_le);
                r0 += __popc(__ballot_sync(0xffffffffu, pn <= q0 + 32));
                const unsigned has_mask = __ballot_sync(0xffffffffu, has);
                if (has) {
                    const int t = (int)(q - s_P[rec]);
                    const u64 h = s_buf[rec * RW];
                    const unsigned c = s_cnt[rec];
                    const SkmInst<NW> in = skm_instance_staged<NW>(kp, h, s_buf + rec * RW + 1, s_rv + rec * (NW + 1), t);
                    const u64 rank = skm_rec_rank(h, t);
                    SKM_ACC(1, t_inst);
                    SKM_T0(t_find);
                    u32 slot;
                    const int state = st.find(in.canon, slot);
                    __syncwarp(has_mask);   // the lanes re-join before the counter update (see SmemTable)
                    SKM_ACC(2, t_find);
                    SKM_T0(t_upd);
                    if (state == 1) {
                        st.apply(slot, in.left, in.right, rank, c);
                        SKM_ACC(3, t_upd);
                    } else if (state == 3) {
                        // bucket holds more distinct k-mers than the shared-memory table: this k-mer goes to HBM directly (same result).
                        // Region mode: to its bin as a partial aggregate (counted as a new key: the bound the CTA's credit is settled
                        // with); else the CAS protocol, since lanes may spill the same new key at once.
                        if constexpr (REGION) {
                            bin_store(tab, a.bins, a.counters, in.canon, payload_apply_n(PAYLOAD_FRESH, in.left, in.right, c), rank);
                            atomicAdd(&s_new, 1u);
                        } else if (table_insert(tab, in.canon, in.left, in.right, rank, c)) {
                            atomicAdd(&s_new, 1u);
                        }
                        SKM_ACC(4, t_upd);
                    }
                }
                __syncwarp();
            }
            __syncthreads();   // the buffer, its counts, P and rv are free again
            if (!COPY_PATH || s_coll)
                for (int i = tid; i < SKM_DEDUP_SLOTS; i += SKM_APPLY_THREADS) s_dd[i] = SKM_DD_EMPTY;
            if (tid == 0) { s_nbuf = 0; s_drained += nb; }
            __syncthreads();
            SKM_WALL(4);
        };
        // ---- the windows of the bucket (a deferred or empty bucket still retires the window queued for it)
        for (u32 w = 0;; w++) {
            const bool more = run && (w + 1) * (u32)SKM_W < R;
            if (more) skm_stage_window<RW, SKM_W>(s_stage + (half ^ 1) * SKM_W * RW, &s_bar[half ^ 1], my_recs, cur, R, w + 1);
            else if (pos + gridDim.x < a.n_list) skm_stage_window<RW, SKM_W>(s_stage + (half ^ 1) * SKM_W * RW, &s_bar[half ^ 1], my_recs, nxt, R_nxt, 0);
            SKM_WALL(6);
            SKM_T0(t_wait);
            mbar_wait(&s_bar[half], (phase >> half) & 1u);
            SKM_ACC(0, t_wait);
            SKM_WALL(1);
            phase ^= 1u << half;
            if (run) {
                const u64* stg = s_stage + half * SKM_W * RW;
                const u32 nrec = min(R - w * (u32)SKM_W, (u32)SKM_W);
                if (tid == 0) s_staged += nrec;
                if (tid < SKM_W) s_pend[tid] = (u32)tid < nrec;   // (in shared memory: nothing of the window stays in registers over a drain)
                for (;;) {
                    SKM_T0(t_dd);
                    u32 nb;
                    if (!COPY_PATH || s_coll) {   // (read from shared memory, not held in a register over the drains; it only changes after a flush)
                        if (tid < SKM_W && s_pend[tid]) s_pend[tid] = skm_dedup_insert<NW>(stg + tid * RW, s_buf, s_cnt, s_dd, &s_nbuf);
                        __syncthreads();
                        nb = s_nbuf;
                    } else {
                        // Records that hardly repeat: the window is copied into the buffer with count 1, no dedup table.  Every window
                        // but a bucket's last is full, so window w goes to buffer position (w mod C/W) * W, and a full buffer is drained.
                        const u32 at = w % (u32)(C / SKM_W) * (u32)SKM_W;
                        if (tid < SKM_W && s_pend[tid]) {
#pragma unroll
                            for (int i = 0; i < RW; i++) s_buf[(at + tid) * RW + i] = stg[tid * RW + i];
                            s_cnt[at + tid] = 1;
                        }
                        __syncthreads();
                        nb = at + min(R - w * (u32)SKM_W, (u32)SKM_W);
                    }
                    SKM_ACC(6, t_dd);
                    SKM_WALL(2);
                    const bool full = nb > (u32)C;
                    if (!full && ((more && (!COPY_PATH || s_coll || nb < (u32)C)) || nb == 0)) break;
                    drain(min(nb, (u32)C));   // full (the records that found no room go into the emptied buffer), or the bucket's end
                    if (!full) break;
                }
            }
            __syncthreads();   // the window's stage half is free again
            half ^= 1;
            if (!more) break;
        }
        cur = nxt;
        nxt = nn;
        R_cur = R_nxt;
        if (!run) continue;
        // ---- flush: one global update per distinct k-mer of the bucket, walking the claim list (every thread busy)
        SKM_T0(t_flush);
        const u32 n_claimed = s_count;
        unsigned my_new = 0;
        for (u32 i = tid; i < n_claimed; i += SKM_APPLY_THREADS) {
            const u32 idx = st.list[i];
            Kmer<NW> k;
#pragma unroll
            for (int w = 0; w < NW; w++) k.w[w] = st.key[w * SKM_SLOTS + idx];
            if constexpr (REGION) {
                bin_store(tab, a.bins, a.counters, k, st.pay[idx], st.rnk[idx]);
                my_new++;   // an upper bound of the new keys: the CTA's credit is settled with it, C_DISTINCT comes from the build
            } else {
                bool claimed;
                table_merge<true>(tab, k, st.pay[idx], st.rnk[idx], &claimed);
                my_new += claimed;
            }
            st.key[idx] = EMPTY64;
            st.pay[idx] = PAYLOAD_FRESH;
            st.rnk[idx] = ~0ull;
        }
        if (my_new) atomicAdd(&s_new, my_new);
        __syncthreads();
        SKM_ACC(5, t_flush);
        SKM_WALL(5);
        if (tid == 0) {
            credit += (u64)R * SKM_MAX_RUN - (u64)s_new;   // what the bound over-reserved stays with the CTA
            s_tot_new += s_new;
            if (COPY_PATH && a.collapse == SKM_COLLAPSE_AUTO && ++s_ad_n == (s_coll ? SKM_AUTO_PROBE : SKM_AUTO_SKIP)) {
                // collapsing: go on while the distinct share of the records is at most the threshold; not collapsing: measure again
                s_coll = !s_coll || (s_drained - s_ad_drained) * SKM_AUTO_DEN <= (s_staged - s_ad_staged) * SKM_AUTO_NUM;
                s_ad_n = 0;
                s_ad_staged = s_staged;
                s_ad_drained = s_drained;
            }
        }
    }
    __syncthreads();
    if (tid == 0 && credit) atomicAdd((unsigned long long*)&a.counters[C_RESERVED], (unsigned long long)(0ull - credit));
    if (!REGION && tid == 0 && s_tot_new) atomicAdd(&a.counters[C_DISTINCT], (u64)s_tot_new);
    if (tid == 0 && s_staged) {
        atomicAdd(&a.counters[C_SKM_STAGED], s_staged);
        atomicAdd(&a.counters[C_SKM_DRAINED], s_drained);
    }
#ifdef SKM_PHASE_CLOCKS
    for (int i = 0; i < SKM_PHASES; i++) atomicAdd(&g_skm_phase_clk[i], (unsigned long long)clk[i]);
    SKM_WALL(6);
    if (tid == 0) {
        for (int i = 0; i < SKM_WALL_PHASES; i++) atomicAdd(&g_skm_wall_clk[i], (unsigned long long)s_wall[i]);
        atomicAdd(&g_skm_wall_clk[SKM_WALL_PHASES], (unsigned long long)(clock64() - t_kernel));
        atomicAdd(&g_skm_wall_clk[SKM_WALL_PHASES + 1], 1ull);
    }
#endif
}

// ------------------------------------------------------------------------------------------------ host side
template <int NW>
static constexpr size_t skm_apply_smem() {
    return ((size_t)(NW + 2) * SKM_SLOTS + 2 * skm_w<NW>() * (NW + 2) + SKM_BUF_RECS * (NW + 2) + SKM_BUF_RECS * (NW + 1)) * sizeof(u64) +
           (size_t)SKM_SLOTS * sizeof(unsigned short) + (2 * SKM_BUF_RECS + 1 + skm_dd_slots<NW>()) * sizeof(u32);
}
// An aggregation launch keeps the keys the table is committed to under this share of its capacity (buckets beyond it are deferred),
// and the growth before their re-run leaves this much HBM free
constexpr double SKM_TABLE_LOAD = 0.85;
constexpr u64 SKM_GROW_HEADROOM = 1ull << 28;

template <int NW>
void EngineT<NW>::skm_launch_apply(const u32* list, u32 n_list, u32* deferred_out, bool region) {
    SkmSegList* segs = skm_segs_.template as<SkmSegList>();
    SkmFlushArgs fa;
    fa.world = xa_geom_.world; fa.max_seg = xa_geom_.max_seg; fa.bo_stride = xa_geom_.bo_max + 1; fa.cap_pair = xa_geom_.cap_pair; fa.rec_words = NW + 2;
    fa.half = skm_arena_half(xa_geom_, xa_buf_.p, flush_.half);
    fa.segs = segs;
    fa.counters = d_cnt_;
    k_skm_segs<<<1, 256, 0, st_>>>(fa);   // segment list + C_RESERVED = keys in the table, C_DEFER = C_MAXU = 0
    PG_CUDA(cudaGetLastError());
    SkmApplyArgs aa;
    aa.segs = segs; aa.bucket_list = list; aa.n_list = n_list; aa.counters = d_cnt_;
    aa.limit = (u64)(SKM_TABLE_LOAD * (double)cap_);
    aa.deferred = deferred_out;
    aa.bins = bin_args();
    aa.collapse = SKM_COLLAPSE_AUTO;
    if (const char* e = getenv("PGB200_SKM_COLLAPSE")) {
        if (!strcmp(e, "off")) aa.collapse = SKM_COLLAPSE_OFF;
        else if (!strcmp(e, "on")) aa.collapse = SKM_COLLAPSE_ON;
        else if (strcmp(e, "auto")) throw std::runtime_error("pgb200: PGB200_SKM_COLLAPSE must be auto, on or off");
    }
    auto kern = region ? k_skm_apply<NW, true> : k_skm_apply<NW, false>;
    PG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)skm_apply_smem<NW>()));
    int per_sm = 0;
    PG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, SKM_APPLY_THREADS, skm_apply_smem<NW>()));
    if (per_sm < 1) per_sm = 1;
    const unsigned blocks = (unsigned)std::min<u64>((u64)n_list, (u64)n_sm_ * per_sm);   // persistent CTAs: as many as are resident
    if (blocks) kern<<<blocks, SKM_APPLY_THREADS, skm_apply_smem<NW>(), st_>>>(tab_, kp_, aa);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cudaMemcpyAsync(h_outcome_, d_cnt_ + C_XERR, sizeof(FlushOutcome), cudaMemcpyDeviceToHost, st_));
    p1_.launches += 2;
}

// Aggregate the closed epoch into the global table (several GPUs: only after every GPU has fenced -- the caller's barrier).
// Returns as soon as the work is queued; skm_flush_complete (next epoch close, pgb200_finish_pass1) reads the outcome.
template <int NW>
void EngineT<NW>::skm_flush(bool final_of_pass) {
    if (!xa_buf_.p || xa_flushed_epoch_ >= xa_send_epoch_) return;
    skm_flush_complete();
    if (xa_flushed_epoch_ + 1 != xa_send_epoch_) throw std::runtime_error("pgb200: internal: more than one unflushed exchange epoch");
    // The pass's first launch (no key in the table) builds the table region by region, and the end-of-pass sweeps ride on the build
    // (PassSweeps); the table memory is then the bins' storage and needs no clear.  Any other launch merges into the table.
    flush_.region = table_build_region_ && pass_sweeps_ == PassSweeps::Untouched;
    create_table_if_needed(!flush_.region);
    flush_.sweep = flush_.region && ((signed char)prm_.D <= 0 || final_of_pass);
    if (flush_.region) table_build_prepare();
    skm_segs_.ensure(sizeof(SkmSegList));
    pass_sweeps_ = flush_.sweep ? PassSweeps::Fused : PassSweeps::Plain;
    PG_CUDA(cudaMemsetAsync(d_cnt_ + C_SKM_STAGED, 0, 2 * sizeof(u64), st_));
    flush_.half = (int)(xa_flushed_epoch_ % SKM_ARENA_HALVES);
    PG_CUDA(cudaEventRecord(ev_flush_begin_, st_));
    skm_launch_apply(nullptr, skm_own_hi_ - skm_own_lo_, skm_deferred_[0].template as<u32>(), flush_.region);
    if (flush_.region) table_build_launch();
    PG_CUDA(cudaEventRecord(ev_flush_, st_));
    flush_.pending = true;
}

template <int NW>
void EngineT<NW>::skm_flush_complete() {
    if (!flush_.pending) return;
    flush_.pending = false;
    PG_CUDA(cudaEventSynchronize(ev_flush_));
    float ms;
    PG_CUDA(cudaEventElapsedTime(&ms, ev_flush_begin_, ev_flush_));
    int launches = 1, which = 0;
    // a merge-mode re-run of `list` (nullptr: every owned bucket), timed and waited for
    auto relaunch = [&](const u32* list, u32 n_list, u32* deferred_out) {
        PG_CUDA(cudaEventRecord(ev_flush_begin_, st_));
        skm_launch_apply(list, n_list, deferred_out, false);
        PG_CUDA(cudaEventRecord(ev_flush_, st_));
        PG_CUDA(cudaEventSynchronize(ev_flush_));
        float ms2;
        PG_CUDA(cudaEventElapsedTime(&ms2, ev_flush_begin_, ev_flush_));
        ms += ms2;
        launches++;
        return *h_outcome_;
    };
    FlushOutcome out = *h_outcome_;
    if (out.xerr) throw std::runtime_error("pgb200: too many segments in one exchange epoch (flush more often)");
    if (flush_.region && table_build_redo()) {
        // entries were dropped: the same records again, the classic way, into a cleared table (the launch found it empty)
        pass_sweeps_ = PassSweeps::Plain;
        PG_CUDA(cudaMemsetAsync(tab_buf_.p, 0xFF, cap_ * sizeof(Slot<NW>), st_));
        PG_CUDA(cudaMemsetAsync(d_cnt_ + C_DISTINCT, 0, sizeof(u64), st_));
        PG_CUDA(cudaMemsetAsync(d_cnt_ + C_SKM_STAGED, 0, 2 * sizeof(u64), st_));
        out = relaunch(nullptr, skm_own_hi_ - skm_own_lo_, skm_deferred_[0].template as<u32>());
    }
    while (out.defer) {
        // buckets whose worst case did not fit the table: grow so that (at least) the largest one fits, run them again
        read_counters();
        if (!grow_table_for(h_cnt_[C_DISTINCT] + out.maxu, SKM_TABLE_LOAD, SKM_GROW_HEADROOM, false))
            throw std::runtime_error("pgb200: k-mer table cannot grow further (out of HBM); use more GPUs");
        if (pass_sweeps_ == PassSweeps::Fused) pass_sweeps_ = PassSweeps::Plain;   // the spill list holds slots of the table just replaced
        out = relaunch(skm_deferred_[which].template as<u32>(), (u32)out.defer, skm_deferred_[which ^ 1].template as<u32>());
        which ^= 1;
    }
    // the epoch's half is free again: senders may use it from the epoch after next
    PG_CUDA(cudaMemsetAsync(skm_arena_half(xa_geom_, xa_buf_.p, flush_.half).nseg, 0, (size_t)xa_geom_.world * sizeof(u32), st_));
    p1_.ms_insert += ms;
    p1_.ms_apply += ms;
    xa_flushed_epoch_++;
    if (prm_.verbose >= 2 || getenv("PGB200_SKM_STATS")) {
        u64 rd[2];   // C_SKM_STAGED, C_SKM_DRAINED
        PG_CUDA(cudaMemcpy(rd, d_cnt_ + C_SKM_STAGED, sizeof(rd), cudaMemcpyDeviceToHost));
        fprintf(stderr, "[pgb200] aggregated epoch %llu: %u owned bucket(s), %d launch(es), %.2f ms, table %llu slots, %llu records staged, %llu distinct "
                        "drained (%.3f)\n", (unsigned long long)xa_flushed_epoch_, skm_own_hi_ - skm_own_lo_, launches, ms, (unsigned long long)cap_,
                (unsigned long long)rd[0], (unsigned long long)rd[1], rd[0] ? (double)rd[1] / (double)rd[0] : 0.0);
    }
#ifdef SKM_PHASE_CLOCKS
    if (getenv("PGB200_SKM_STATS")) {
        unsigned long long c[SKM_PHASES], zero[SKM_PHASES] = {}, tot = 0;
        PG_CUDA(cudaMemcpyFromSymbol(c, g_skm_phase_clk, sizeof(c)));
        PG_CUDA(cudaMemcpyToSymbol(g_skm_phase_clk, zero, sizeof(zero)));
        for (int i = 0; i < SKM_PHASES; i++) tot += c[i];
        fprintf(stderr, "[pgb200] aggregation phase clocks (thread-cycles, %% of %.3g): stage wait %.1f, instance build %.1f, find/claim %.1f, apply %.1f, "
                        "spill %.1f, flush %.1f, dedup %.1f\n", (double)tot, 100.0 * c[0] / tot, 100.0 * c[1] / tot, 100.0 * c[2] / tot, 100.0 * c[3] / tot,
                100.0 * c[4] / tot, 100.0 * c[5] / tot, 100.0 * c[6] / tot);
        unsigned long long wl[SKM_WALL_PHASES + 2], wzero[SKM_WALL_PHASES + 2] = {}, wsum = 0;
        PG_CUDA(cudaMemcpyFromSymbol(wl, g_skm_wall_clk, sizeof(wl)));
        PG_CUDA(cudaMemcpyToSymbol(g_skm_wall_clk, wzero, sizeof(wzero)));
        for (int i = 0; i < SKM_WALL_PHASES; i++) wsum += wl[i];
        const double ctas = wl[SKM_WALL_PHASES + 1] ? (double)wl[SKM_WALL_PHASES + 1] : 1.0, kern = wl[SKM_WALL_PHASES] ? (double)wl[SKM_WALL_PHASES] : 1.0;
        fprintf(stderr, "[pgb200] aggregation wall split (thread 0 of each of %.0f CTAs, %% of %.4g cycles per CTA): top of bucket %.1f, stage wait %.1f, "
                        "dedup/copy %.1f, drain pre-pass %.1f, drain steps %.1f, flush %.1f, other %.1f; phases sum to %.4f of kernel end - start\n",
                ctas, kern / ctas, 100.0 * wl[0] / kern, 100.0 * wl[1] / kern, 100.0 * wl[2] / kern, 100.0 * wl[3] / kern, 100.0 * wl[4] / kern,
                100.0 * wl[5] / kern, 100.0 * wl[6] / kern, (double)wsum / kern);
    }
#endif
}

#define PGB_INST(NW)                                                          \
    template void EngineT<NW>::skm_launch_apply(const u32*, u32, u32*, bool); \
    template void EngineT<NW>::skm_flush(bool);                               \
    template void EngineT<NW>::skm_flush_complete();
PGB_INST(2)
PGB_INST(4)

}   // namespace pgb
