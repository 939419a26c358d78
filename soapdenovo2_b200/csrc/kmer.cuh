// kmer.cuh -- 2-bit k-mer algebra for the GPU pregraph engine (host + device).
//
// Semantics follow the reference's MER63 / MER127 `Kmer` (standardPregraph/inc/def.h:46-56, kmer.c):
//   * base codes A0 C1 T2 G3, complement = code ^ 2                     (inc/def.h:39-42)
//   * k-mer right-aligned in NW 64-bit words, w[0] most significant; the LAST base sits in bits 1:0 of w[NW-1]
//   * nextKmer = shl 2, mask to 2K bits, or-in                          (kmer.c:696-702)
//   * prevKmer = shr 2, or-in at bit 2(K-1)                             (kmer.c:704-718)
//   * reverseComplement                                                 (kmer.c:819-845 / 507-581)
//   * KmerSmaller / KmerLarger = unsigned lexicographic compare on words (kmer.c:608-629)
// The code is new: the reference shifts word by word through tables; here everything is register arithmetic
// (funnel shifts, __brevll) so that one thread can roll a k-mer along a read with a handful of instructions.
#pragma once
#include <cstdint>
#include <cstddef>

#if defined(__CUDACC__)
#define PG_HD __host__ __device__ __forceinline__
#define PG_D __device__ __forceinline__
#else
#define PG_HD inline
#define PG_D inline
#endif

namespace pgb {

typedef unsigned long long u64;
typedef unsigned int u32;
typedef unsigned char u8;

template <int NW>
struct Kmer {
    u64 w[NW];
};

template <int NW>
PG_HD Kmer<NW> kzero() {
    Kmer<NW> k;
#pragma unroll
    for (int i = 0; i < NW; i++) k.w[i] = 0;
    return k;
}
template <int NW>
PG_HD bool keq(const Kmer<NW>& a, const Kmer<NW>& b) {
    bool e = true;
#pragma unroll
    for (int i = 0; i < NW; i++) e = e && (a.w[i] == b.w[i]);
    return e;
}
// a < b, unsigned, w[0] most significant (KmerSmaller, kmer.c:608-629)
template <int NW>
PG_HD bool kless(const Kmer<NW>& a, const Kmer<NW>& b) {
#pragma unroll
    for (int i = 0; i < NW; i++) {
        if (a.w[i] != b.w[i]) return a.w[i] < b.w[i];
    }
    return false;
}
template <int NW>
PG_HD Kmer<NW> kshl2(const Kmer<NW>& a) {
    Kmer<NW> r;
#pragma unroll
    for (int i = 0; i < NW; i++) r.w[i] = (a.w[i] << 2) | (i + 1 < NW ? (a.w[i + 1] >> 62) : 0ull);
    return r;
}
template <int NW>
PG_HD Kmer<NW> kshr2(const Kmer<NW>& a) {
    Kmer<NW> r;
#pragma unroll
    for (int i = NW - 1; i >= 0; i--) r.w[i] = (a.w[i] >> 2) | (i > 0 ? (a.w[i - 1] << 62) : 0ull);
    return r;
}
// generic right shift by `s` bits, 0 <= s < 64*NW.  The word offset is dispatched through a switch so that every w[] index is a
// compile-time constant: a dynamically indexed w[] lives in local memory on the GPU (LDL/STL in every reverse complement), and
// the shift amount is uniform (it depends on K only), so the switch is a uniform branch.
template <int NW, int WS>
PG_HD Kmer<NW> kshr_words(const Kmer<NW>& a, int bs) {
    Kmer<NW> r;
#pragma unroll
    for (int i = NW - 1; i >= 0; i--) {
        const u64 lo = i - WS >= 0 ? a.w[i - WS >= 0 ? i - WS : 0] : 0ull;
        const u64 hi = i - WS - 1 >= 0 ? a.w[i - WS - 1 >= 0 ? i - WS - 1 : 0] : 0ull;
        r.w[i] = bs ? ((lo >> bs) | (hi << (64 - bs))) : lo;
    }
    return r;
}
template <int NW>
PG_HD Kmer<NW> kshr(const Kmer<NW>& a, int s) {
    const int bs = s & 63;
    switch (s >> 6) {
        case 0: return kshr_words<NW, 0>(a, bs);
        case 1: return kshr_words<NW, 1>(a, bs);
        case 2: return kshr_words<NW, (NW > 2 ? 2 : 0)>(a, bs);
        default: return kshr_words<NW, (NW > 3 ? 3 : 0)>(a, bs);
    }
}

// Per-K constants (WORDFILTER = createFilter(K), kmer.c:738-758)
template <int NW>
struct KParams {
    Kmer<NW> mask;   // low 2K bits
    int K;
    int top_word;    // word holding bit 2(K-1)
    int top_shift;   // bit offset of the first base inside that word
};
template <int NW>
inline KParams<NW> make_kparams(int K) {
    KParams<NW> p;
    p.K = K;
    int bits = 2 * K;
    for (int i = NW - 1; i >= 0; i--) {
        p.mask.w[i] = bits >= 64 ? ~0ull : (bits > 0 ? ((1ull << bits) - 1) : 0ull);
        bits -= 64;
    }
    int b = 2 * (K - 1);
    p.top_word = NW - 1 - b / 64;
    p.top_shift = b % 64;
    return p;
}

template <int NW>
PG_HD Kmer<NW> knext(const Kmer<NW>& a, unsigned c, const KParams<NW>& p) {
    Kmer<NW> r = kshl2(a);
#pragma unroll
    for (int i = 0; i < NW; i++) r.w[i] &= p.mask.w[i];
    r.w[NW - 1] |= (u64)c;
    return r;
}
template <int NW>
PG_HD Kmer<NW> kprev(const Kmer<NW>& a, unsigned c, const KParams<NW>& p) {
    Kmer<NW> r = kshr2(a);
#pragma unroll
    for (int i = 0; i < NW; i++)
        if (i == p.top_word) r.w[i] |= (u64)c << p.top_shift;
    return r;
}
// the canonical k-mer, selected word by word so that both candidates stay in registers (a select of a whole Kmer by reference puts
// them in local memory)
template <int NW>
PG_D Kmer<NW> kcanon(const Kmer<NW>& f, const Kmer<NW>& rc, bool smaller) {
    Kmer<NW> c;
#pragma unroll
    for (int i = 0; i < NW; i++) c.w[i] = smaller ? f.w[i] : rc.w[i];
    return c;
}
// Word w of a key as the output files print it, out of out_words (EngineT::out_words): the 127-mer build prints four words at every
// K, so a key held in two words gets two leading zero words.  Selected like kfirst: a dynamically indexed w[] lives in local memory.
template <int NW>
PG_HD u64 kout_word(const Kmer<NW>& a, int w, int out_words) {
    const int src = w - (out_words - NW);
    u64 v = 0;
#pragma unroll
    for (int i = 0; i < NW; i++)
        if (i == src) v = a.w[i];
    return v;
}
template <int NW>
PG_HD unsigned klast(const Kmer<NW>& a) { return (unsigned)(a.w[NW - 1] & 3); }
template <int NW>
PG_HD unsigned kfirst(const Kmer<NW>& a, const KParams<NW>& p) {   // firstCharInKmer
    u64 v = 0;
#pragma unroll
    for (int i = 0; i < NW; i++)
        if (i == p.top_word) v = a.w[i];
    return (unsigned)((v >> p.top_shift) & 3);
}

PG_HD u64 rev2bit64(u64 x) {   // reverse the order of the 32 two-bit groups of x
#if defined(__CUDA_ARCH__)
    x = __brevll(x);
#else
    x = ((x >> 1) & 0x5555555555555555ull) | ((x & 0x5555555555555555ull) << 1);
    x = ((x >> 2) & 0x3333333333333333ull) | ((x & 0x3333333333333333ull) << 2);
    x = ((x >> 4) & 0x0F0F0F0F0F0F0F0Full) | ((x & 0x0F0F0F0F0F0F0F0Full) << 4);
    x = __builtin_bswap64(x);
#endif
    // bit-reversal also swapped the two bits inside each group: swap them back
    return ((x & 0xAAAAAAAAAAAAAAAAull) >> 1) | ((x & 0x5555555555555555ull) << 1);
}
// plain reverse complement of an n-mer (n bases right-aligned)
template <int NW>
PG_HD Kmer<NW> krc_n(const Kmer<NW>& a, int n) {
    Kmer<NW> t;
#pragma unroll
    for (int i = 0; i < NW; i++) t.w[i] = rev2bit64(a.w[NW - 1 - i] ^ 0xAAAAAAAAAAAAAAAAull);
    return kshr(t, 64 * NW - 2 * n);
}
// reverseComplement(seq, n) as the reference BINARY behaves: in the 127-mer build a (K+1)=128-mer hits a `char`
// overflow in fastReverseComp (kmer.c:532-542) and only the lowest word is complemented+reversed (SURVEY.md fact 11).
// quirk128 must be true only for (flavour127 && n == 128).
template <int NW>
PG_HD Kmer<NW> krc_ref(const Kmer<NW>& a, int n, bool quirk128) {
    if (NW == 4 && quirk128) {
        Kmer<NW> r = a;
        r.w[NW - 1] = rev2bit64(a.w[NW - 1] ^ 0xAAAAAAAAAAAAAAAAull);
        return r;
    }
    return krc_n(a, n);
}

// ---------------------------------------------------------------- CRC-32 set hash (hashFunction.c:28-82,123-131,155-158)
// Reflected CRC-32 (poly 0xEDB88320), register starts at 0, final XOR 0xFFFFFFFF, over the little-endian bytes of the
// words in struct order (w[0] first); returned as int sign-extended to 64 bits.  Only used to pick the reference "set"
// (crc % P) of each DISTINCT k-mer when the reference layout is reconstructed -- never on the per-instance hot path.
PG_HD u32 crc32_step_bitwise(u32 c, u32 byte) {
    c ^= byte;
#pragma unroll
    for (int j = 0; j < 8; j++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
    return c;
}
template <int NW>
PG_HD u64 crc_hash(const Kmer<NW>& k) {
    u32 c = 0;
#pragma unroll
    for (int i = 0; i < NW; i++) {
#pragma unroll
        for (int b = 0; b < 8; b++) c = crc32_step_bitwise(c, (u32)((k.w[i] >> (8 * b)) & 0xff));
    }
    c ^= 0xFFFFFFFFu;
    return (u64)(long long)(int)c;
}

// ---------------------------------------------------------------- home slot in the reference's prime-sized set
// 63-mer build: (u128)kmer % size (newhash.c:490-492).  127-mer build: chained 32-bit-limb modulo (newhash.c:36-47),
// which equals the true remainder while size < 2^32 and wraps (faithfully reproduced) beyond.
PG_HD u64 mod_u128(u64 hi, u64 lo, u64 m) {
#if defined(__CUDA_ARCH__)
    if (m < (1ull << 32)) {
        // Horner over 32-bit limbs: every partial value < m * 2^32 < 2^64
        u64 t = hi % m;
        t = ((t << 32) | (lo >> 32)) % m;
        t = ((t << 32) | (lo & 0xffffffffull)) % m;
        return t;
    }
    // general case: binary long division (only reached for > 4G-slot sets)
    u64 r = hi % m;
    for (int i = 63; i >= 0; i--) {
        u64 carry = r >> 63;
        r = (r << 1) | ((lo >> i) & 1);
        if (carry || r >= m) r -= m;
    }
    return r;
#else
    unsigned __int128 t = ((unsigned __int128)hi << 64) | lo;
    return (u64)(t % m);
#endif
}
template <int NW>
PG_HD u64 ref_home(const Kmer<NW>& k, u64 size, bool flavour127) {
    if (!flavour127) {
        // 63-mer build: Kmer = {high, low} = the two least-significant words (upper words are zero for K <= 63)
        return mod_u128(k.w[NW - 2], k.w[NW - 1], size);
    }
    u64 w0 = NW == 4 ? k.w[0] : 0ull, w1 = NW == 4 ? k.w[1] : 0ull, w2 = k.w[NW - 2], w3 = k.w[NW - 1];
    u64 t = (w0 % size) << 32 | (w1 >> 32 & 0xffffffffull);
    t = (t % size) << 32 | (w1 & 0xffffffffull);
    t = (t % size) << 32 | (w2 >> 32 & 0xffffffffull);
    t = (t % size) << 32 | (w2 & 0xffffffffull);
    t = (t % size) << 32 | (w3 >> 32 & 0xffffffffull);
    t = (t % size) << 32 | (w3 & 0xffffffffull);
    return t % size;
}

// ---------------------------------------------------------------- engine-private hash for the GPU k-mer table
// (not the reference's: slot position in the GPU table is an implementation detail; the reference layout is rebuilt later)
PG_HD u64 mix64(u64 x) {
    x ^= x >> 32;
    x *= 0xD6E8FEB86659FD93ull;
    x ^= x >> 32;
    x *= 0xD6E8FEB86659FD93ull;
    x ^= x >> 32;
    return x;
}
template <int NW>
PG_HD u64 table_hash(const Kmer<NW>& k) {
    u64 h = 0;
#pragma unroll
    for (int i = 0; i < NW; i++) h = (h ^ k.w[i]) * 0x9E3779B97F4A7C15ull + (h >> 29);
    return mix64(h);
}

}   // namespace pgb
