// Host-side check of the record collapse of the aggregated pass 1 (skm_apply.cu: k_skm_apply, skm_dedup_insert), compiled with nvcc and
// run on the CPU by tests/test_skm_collapse_host.py.
//   * payload_apply_n(p, left, right, c) equals c calls of payload_apply for every left/right in 0..4 and c in 1..600, from the fresh
//     state, saturated links and coverage, `single`, and random payloads;
//   * a sequential restatement of the distinct-record buffer (capacity SKM_BUF_RECS, drained when full and at the end of the bucket,
//     the smallest header wins, skm_rec_same / skm_rec_hash as the key) gives, expanding every distinct record once with its count,
//     the same {payload, rank} per k-mer as applying every instance of every record -- on random reads and on heavily tiled ones,
//     K = 31, 63, 65, 127, with records of n = 1 and n = 32, has_prev = 0 and last = 1 all present.
#include "../soapdenovo2_b200/csrc/skm.cuh"
#include <cstdio>
#include <map>
#include <vector>
using namespace pgb;

static u64 rng_state = 0x2545F4914F6CDD1Dull;
static u64 rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

constexpr int C = 128;   // the kernel's SKM_BUF_RECS

static int check_apply_n() {
    std::vector<u64> starts = {PAYLOAD_FRESH, payload_apply(PAYLOAD_FRESH, 0, 3), payload_apply(PAYLOAD_FRESH, 4, 1), payload_apply(PAYLOAD_FRESH, 2, 4)};
    u64 sat = PAYLOAD_FRESH;   // every link and the coverage saturated
    for (int i = 0; i < 300; i++) for (unsigned l = 0; l < 4; l++) sat = payload_apply(sat, l, 3 - l);
    starts.push_back(sat);
    starts.push_back(sat | PL_SINGLE | PL_LINEAR);
    for (int i = 0; i < 40; i++) starts.push_back(rnd() & ~(3ull << 62));
    int bad = 0;
    for (u64 p0 : starts)
        for (unsigned l = 0; l <= 4; l++)
            for (unsigned r = 0; r <= 4; r++) {
                u64 p = p0;
                for (unsigned c = 1; c <= 600; c++) {
                    p = payload_apply(p, l, r);
                    if (payload_apply_n(p0, l, r, c) != p) bad++;
                }
            }
    printf("apply_n: starts=%zu errors=%d\n", starts.size(), bad);
    return bad;
}

template <int NW>
struct KeyLess { bool operator()(const Kmer<NW>& a, const Kmer<NW>& b) const { return kless(a, b); } };
struct Agg { u64 payload = PAYLOAD_FRESH; u64 rank = ~0ull; };
struct Run { u32 b; int start, n; bool last; };
struct EmitRuns {
    std::vector<Run>* v;
    void operator()(u32 b, int s, int n, bool last) { v->push_back(Run{b, s, n, last}); }
};

template <int NW>
static int run_case(int K, bool tiled, int n_reads, int L, u32 n_buckets) {
    constexpr int RW = NW + 2;
    const KParams<NW> kp = make_kparams<NW>(K);
    const SkmGeom g = make_skm_geom(K, n_buckets);
    const int W64 = (L + 31) / 32;
    std::vector<unsigned> genome(tiled ? 3 * L : 0);
    for (auto& b : genome) b = (unsigned)(rnd() & 3);
    std::vector<u32> ring(g.w);
    std::vector<std::vector<std::vector<u64>>> buckets(n_buckets);   // the records of each bucket, in stream order
    for (int r = 0; r < n_reads; r++) {
        std::vector<unsigned> seq(L);
        const int off = tiled ? (int)(rnd() % (2 * L)) : 0;
        const bool rc = tiled && (rnd() & 1);
        for (int i = 0; i < L; i++) seq[i] = !tiled ? (unsigned)(rnd() & 3) : rc ? genome[off + L - 1 - i] ^ 2u : genome[off + i];
        std::vector<u64> words(W64 + 1, 0);
        for (int i = 0; i < L; i++) words[i >> 5] |= (u64)seq[i] << (2 * (i & 31));
        std::vector<Run> runs;
        EmitRuns e{&runs};
        skm_scan_read(g, words.data(), L, ring.data(), 1, e);
        for (const Run& ru : runs) {
            const SkmRec<NW> rec = skm_make_rec<NW>(K, words.data(), W64, (u64)r, ru.start, ru.n, ru.last);
            buckets[ru.b].push_back(std::vector<u64>(rec.w, rec.w + RW));
        }
    }
    typedef std::map<Kmer<NW>, Agg, KeyLess<NW>> Map;
    Map direct, collapsed;
    long recs = 0, distinct = 0, drains = 0, n1 = 0, n32 = 0, noprev = 0, last = 0, maxc = 0;
    auto expand = [&](Map& m, const u64* rec, unsigned c) {
        u64 x[NW + 1];
        for (int i = 0; i <= NW; i++) x[i] = rec[1 + i];
        for (int t = 0; t < skm_rec_n(rec[0]); t++) {
            const SkmInst<NW> in = skm_instance_rec<NW>(kp, rec[0], x, t);
            Agg& a = m[in.canon];
            a.payload = payload_apply_n(a.payload, in.left, in.right, c);
            const u64 rk = skm_rec_rank(rec[0], t);
            if (rk < a.rank) a.rank = rk;
        }
    };
    int bad_hash = 0;
    for (auto& bk : buckets) {
        std::vector<std::vector<u64>> buf;   // distinct records, the smallest header of their copies
        std::vector<unsigned> cnt;
        auto drain = [&]() {
            for (size_t i = 0; i < buf.size(); i++) {
                expand(collapsed, buf[i].data(), cnt[i]);
                if ((long)cnt[i] > maxc) maxc = cnt[i];
            }
            distinct += (long)buf.size();
            drains += !buf.empty();
            buf.clear();
            cnt.clear();
        };
        for (const auto& rec : bk) {
            recs++;
            expand(direct, rec.data(), 1);
            const int n = skm_rec_n(rec[0]);
            n1 += n == 1; n32 += n == 32; noprev += !skm_rec_has_prev(rec[0]); last += skm_rec_last(rec[0]);
            size_t j = 0;
            while (j < buf.size() && !skm_rec_same<NW>(buf[j].data(), rec.data())) j++;
            if (j < buf.size()) {
                bad_hash += skm_rec_hash<NW>(buf[j].data()) != skm_rec_hash<NW>(rec.data());
                cnt[j]++;
                if (rec[0] < buf[j][0]) buf[j][0] = rec[0];
                continue;
            }
            if ((int)buf.size() == C) drain();
            buf.push_back(rec);
            cnt.push_back(1);
        }
        drain();
    }
    int bad = bad_hash + (direct.size() != collapsed.size());
    for (const auto& kv : direct) {
        auto it = collapsed.find(kv.first);
        if (it == collapsed.end() || it->second.payload != kv.second.payload || it->second.rank != kv.second.rank) bad++;
    }
    const bool shapes = n1 > 0 && noprev > 0 && last > 0;
    printf("K=%d %s reads=%d buckets=%u: records=%ld distinct=%ld drains=%ld max_count=%ld n1=%ld n32=%ld no_prev=%ld last=%ld kmers=%zu errors=%d\n", K,
           tiled ? "tiled" : "random", n_reads, n_buckets, recs, distinct, drains, maxc, n1, n32, noprev, last, direct.size(), bad + !shapes);
    return bad + !shapes;
}

int main() {
    int bad = check_apply_n();
    bad += run_case<2>(31, false, 3000, 100, 64);
    bad += run_case<2>(31, true, 6000, 100, 16);
    bad += run_case<2>(63, false, 3000, 150, 64);
    bad += run_case<2>(63, true, 8000, 150, 8);
    bad += run_case<4>(65, true, 6000, 150, 8);
    bad += run_case<4>(127, false, 2000, 200, 32);
    bad += run_case<4>(127, true, 6000, 200, 4);
    printf(bad ? "FAILED\n" : "ALL OK\n");
    return bad ? 1 : 0;
}
