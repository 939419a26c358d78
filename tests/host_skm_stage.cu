// Host-side check of the staged instance construction of the aggregation kernel (soapdenovo2_b200/csrc/skm.cuh), compiled with nvcc
// and run on the CPU by tests/test_skm_stage.py.  For every odd K from 13 to 127 (128-bit keys up to K = 63, 256-bit keys for all K),
// every run length n from 1 to 32, every has_prev / last combination and random bases (including garbage past the record's bases),
// skm_instance_staged over the reversed base words of skm_rec_reverse must equal skm_instance_rec for every k-mer of the record.
#include "../soapdenovo2_b200/csrc/skm.cuh"
#include <cstdio>
using namespace pgb;

static u64 rng_state = 0x2545F4914F6CDD1Dull;
static u64 rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }

template <int NW>
static long check_k(int K, long& checked) {
    const KParams<NW> kp = make_kparams<NW>(K);
    long errors = 0;
    for (int n = 1; n <= SKM_MAX_RUN; n++)
        for (int flags = 0; flags < 4; flags++)
            for (int rep = 0; rep < 6; rep++) {
                const bool has_prev = flags & 1, last = (flags & 2) != 0;
                const u64 hdr = skm_rec_header(rnd() >> 30, has_prev ? 1 + (int)(rnd() % 1000) : 0, n, last);
                u64 x[NW + 1];
                for (int i = 0; i < NW + 1; i++) x[i] = rnd();
                if (rep & 1) {   // as skm_make_rec writes it: a dummy base 0 without a predecessor, nothing past the last base
                    if (!has_prev) x[0] &= ~3ull;
                    const int nb = n + K + (last ? 0 : 1);
                    for (int i = 0; i < NW + 1; i++) {
                        const int bits = 2 * nb - 64 * i;
                        if (bits <= 0) x[i] = 0;
                        else if (bits < 64) x[i] &= (1ull << bits) - 1ull;
                    }
                }
                u64 rv[NW + 1];
                skm_rec_reverse<NW>(hdr, x, rv, K);
                for (int t = 0; t < n; t++) {
                    const SkmInst<NW> a = skm_instance_staged<NW>(kp, hdr, x, rv, t);
                    const SkmInst<NW> b = skm_instance_rec<NW>(kp, hdr, x, t);
                    checked++;
                    if (!keq(a.canon, b.canon) || a.left != b.left || a.right != b.right) {
                        if (errors < 5) printf("MISMATCH NW=%d K=%d n=%d has_prev=%d last=%d t=%d\n", NW, K, n, (int)has_prev, (int)last, t);
                        errors++;
                    }
                }
            }
    return errors;
}

int main() {
    long errors = 0, checked = 0;
    for (int K = 13; K <= 127; K += 2) {
        long e = 0, c = 0;
        if (K <= 63) e += check_k<2>(K, c);
        e += check_k<4>(K, c);
        printf("K=%d instances=%ld errors=%ld\n", K, c, e);
        errors += e;
        checked += c;
    }
    printf("%s (%ld instances)\n", errors ? "FAILED" : "ALL OK", checked);
    return errors ? 1 : 0;
}
