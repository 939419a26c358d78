// Host check of k_map_long's parse1read (soapdenovo2_b200/csrc/map_group.cuh) against a literal sequential parse1read
// (prlRead2Ctg.c:260-361), compiled for the host by tests/test_map_long_host.py.  The CTA is simulated phase by phase: in the first
// round every hit is added in a random order (each add is one atomic step, so any order is an interleaving the kernel allows), in
// later rounds the threads run one after another in a random thread order, each over its own strided share of the span.  Table
// sizes from 1 slot up force the overflow rounds.  Spans: empty, no hits, one id across the whole span, ties between groups,
// groups exactly at `multi`, many distinct ids, K < 32 and K > 32.
#include "../soapdenovo2_b200/csrc/map_group.cuh"
#include <algorithm>
#include <cstdio>
#include <random>
#include <vector>
using namespace pgb;

struct Result {
    u32 counter, counter2, best_j;
    u64 best;
};

static Result parse1read_ref(std::vector<u64> h, int K, u32 multi) {   // the reference's loop, on a copy of the span
    Result r{0, 0, 0, 0};
    u32 max_occ = 0;
    for (size_t j = 0; j < h.size(); j++) {
        const u64 v = h[j];
        if (!v) continue;
        u32 flag = 1;
        for (size_t s = j + 1; s < h.size(); s++)
            if (h[s] && (u32)h[s] == (u32)v) { flag++; h[s] = 0; }
        if ((K < 32 && flag >= 2) || K > 32) r.counter2++;
        if (flag < multi) continue;
        r.counter++;
        if (flag > max_occ) { max_occ = flag; r.best_j = (u32)j; r.best = v; }
    }
    return r;
}

static Result parse1read_cta(std::vector<u64> h, int K, u32 multi, u32 n_groups, int nthr, std::mt19937_64& rng, int* rounds) {
    std::vector<u32> id(n_groups), cnt(n_groups), first(n_groups);
    const GroupTab t{id.data(), cnt.data(), first.data(), n_groups};
    GroupAcc acc{0, 0, 0};
    int pending = 0;
    const u32 nk = (u32)h.size();
    for (int tid = 0; tid < nthr; tid++) group_clear(t, tid, nthr);
    std::vector<u32> order;
    for (u32 j = 0; j < nk; j++) if (h[j]) order.push_back(j);
    std::shuffle(order.begin(), order.end(), rng);
    for (u32 j : order) group_add_hit(h.data(), j, t, &pending);
    std::vector<int> tids(nthr);
    for (int i = 0; i < nthr; i++) tids[i] = i;
    *rounds = 1;
    for (;;) {
        std::shuffle(tids.begin(), tids.end(), rng);
        for (int tid : tids) group_fold(t, K, multi, tid, nthr, &acc);
        if (!pending) break;
        for (int tid = 0; tid < nthr; tid++) group_clear(t, tid, nthr);
        pending = 0;
        std::shuffle(tids.begin(), tids.end(), rng);
        for (int tid : tids) group_round(h.data(), nk, t, tid, nthr, &pending);
        ++*rounds;
    }
    Result r{acc.counter, acc.counter2, 0, 0};
    if (acc.counter) { r.best_j = group_best_j(acc); r.best = h[r.best_j]; }
    return r;
}

static u64 hit(u32 id, std::mt19937_64& rng) {   // a hit's payload: contig id, a position, a twin, the read k-mer's isSmaller
    return HIT_VALID | (u64)id | ((rng() & 0xFFFFFFull) << 32) | ((rng() & 1ull) << 56) | ((rng() & 1ull) << HIT_SMALLER_SHIFT);
}

int main() {
    std::mt19937_64 rng(12345);
    long cases = 0, errors = 0, overflow_cases = 0;
    const u32 sizes[] = {1, 2, 3, 7, 64, MAP_GROUPS};
    const int threads[] = {1, 5, 128};
    auto check = [&](const std::vector<u64>& h, int K, u32 multi, const char* what) {
        const Result a = parse1read_ref(h, K, multi);
        std::vector<u32> ids;
        for (u64 v : h) if (v) ids.push_back((u32)v);
        std::sort(ids.begin(), ids.end());
        const size_t distinct = (size_t)(std::unique(ids.begin(), ids.end()) - ids.begin());
        for (u32 n : sizes)
            for (int nthr : threads) {
                if (distinct > 50 * (size_t)n) continue;   // one round per n ids: keeps the run short
                int rounds = 0;
                const Result b = parse1read_cta(h, K, multi, n, nthr, rng, &rounds);
                cases++;
                overflow_cases += rounds > 1;
                const bool same = a.counter == b.counter && (a.counter2 > 1) == (b.counter2 > 1) && a.counter2 == b.counter2 &&
                                  (!a.counter || (a.best_j == b.best_j && a.best == b.best));
                if (!same && errors++ < 10)
                    printf("MISMATCH %s nk=%zu K=%d multi=%u groups=%u threads=%d: counter %u/%u counter2 %u/%u j %u/%u\n", what, h.size(), K, multi, n,
                           nthr, a.counter, b.counter, a.counter2, b.counter2, a.best_j, b.best_j);
            }
    };
    for (int K : {25, 31, 63, 91}) {
        check({}, K, 2, "empty");
        check(std::vector<u64>(50, 0), K, 2, "no hits");
        std::vector<u64> one(300);
        for (auto& v : one) v = hit(77, rng);
        check(one, K, 2, "one id");
        check(one, K, 300, "one id at multi");
        check(one, K, 301, "one id below multi");
        // ties: two ids with equal counts, the later-starting one interleaved first-hit-last
        std::vector<u64> tie;
        for (int i = 0; i < 40; i++) { tie.push_back(hit(5, rng)); tie.push_back(0); tie.push_back(hit(9, rng)); }
        std::reverse(tie.begin(), tie.end());
        check(tie, K, 40, "tie at multi");
        check(tie, K, 2, "tie");
        for (int it = 0; it < 400; it++) {
            const size_t nk = (size_t)(rng() % 3000);
            const u32 pool = 1 + (u32)(rng() % (it % 4 == 0 ? 3 : it % 4 == 1 ? 40 : 2000));
            const double miss = (rng() % 100) / 100.0;
            std::vector<u64> h(nk);
            for (auto& v : h) v = (rng() % 1000) / 1000.0 < miss ? 0 : hit(1 + (u32)(rng() % pool), rng);
            const u32 multi = 2 + (u32)(rng() % (it % 3 == 0 ? 3 : 60));
            check(h, K, multi, "random");
        }
    }
    printf("cases=%ld overflow_cases=%ld errors=%ld\n", cases, overflow_cases, errors);
    if (errors == 0 && overflow_cases > 0) printf("ALL OK\n");
    return errors == 0 && overflow_cases > 0 ? 0 : 1;
}
