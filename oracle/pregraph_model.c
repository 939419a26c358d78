/*
 * oracle/pregraph_model.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by, or executed from the
 * product path (soapdenovo2_b200/, include/).  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may run it, and only as the checker.
 *
 * A single-threaded, deliberately plain C restatement of SOAPdenovo2's `pregraph` stage
 * (reference @ c7568cc; all file:line citations are relative to /root/reference/standardPregraph/).
 * It is NOT a copy of the reference: it re-derives every phase from the behaviour documented in
 * SURVEY.md Appendix A/C and is pinned by byte-comparing its seven output files against the
 * UNMODIFIED reference binary built by oracle/Makefile into oracle/_ref/ (tests/test_oracle_vs_ref.py).
 * The reference ships no tests / golden vectors of its own (SURVEY.md section 4), so that binary is the pin.
 *
 * Build:  gcc -O2 -DMODEL_W=128 (63-mer build, Kmer = 2 x u64)   |  -DMODEL_W=256 (127-mer build, 4 x u64)
 * Usage:  pregraph_model_63 -s cfg -o prefix [-K k] [-p P] [-a G] [-d D] [-R] [-T table_dump.bin] [-U tips_dump.bin] [-1]
 *         -T : dump {kmer words, l[4], r[4], cov, flags} of every node in reference iteration order
 *              right after pass 1 + mark-linear (before tips) -- the intermediate the CUDA kernels are checked on.
 *         -U : the same records right after tip removal (before the edges clear links and overlay edge ids).
 *         -1 : stop after pass 1 (.kmerFreq only); used by the cpu_baseline timing leg.
 *
 * Supported input domain (same as the engine's): single-line FASTA, 4-line FASTQ, files ending in '\n',
 * f1/f2, q1/q2, p, f, q keys; no BAM, no .gz (SURVEY.md A.9 lists the reference's reader quirks outside it).
 */
#define _GNU_SOURCE
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <math.h>
#include <time.h>
#include <unistd.h>
#include <zlib.h>

#ifndef MODEL_W
#define MODEL_W 128
#endif
#define NW (MODEL_W / 64)
typedef uint64_t u64;
typedef uint32_t u32;
typedef uint8_t u8;

/* ------------------------------------------------------------------ k-mer algebra (kmer.c:594-855 / 29-591) */
typedef struct { u64 w[NW]; } Kmer; /* w[0] most significant; memory order == reference struct order (def.h:46-56) */

static int K;              /* overlaplen */
static Kmer MASKK;         /* WORDFILTER, kmer.c:738-758 */

static Kmer kzero(void) { Kmer k; memset(&k, 0, sizeof k); return k; }
static int kcmp(Kmer a, Kmer b) { for (int i = 0; i < NW; i++) { if (a.w[i] < b.w[i]) return -1; if (a.w[i] > b.w[i]) return 1; } return 0; }
static int keq(Kmer a, Kmer b) { return kcmp(a, b) == 0; }
static Kmer kshl2(Kmer a) { Kmer r; for (int i = 0; i < NW; i++) r.w[i] = (a.w[i] << 2) | (i + 1 < NW ? a.w[i + 1] >> 62 : 0); return r; }
static Kmer kshr2(Kmer a) { Kmer r; for (int i = NW - 1; i >= 0; i--) r.w[i] = (a.w[i] >> 2) | (i > 0 ? a.w[i - 1] << 62 : 0); return r; }
static Kmer kand(Kmer a, Kmer b) { Kmer r; for (int i = 0; i < NW; i++) r.w[i] = a.w[i] & b.w[i]; return r; }
static Kmer kmask(int nbases) { /* low 2*nbases bits set */
    Kmer r = kzero(); int bits = 2 * nbases;
    for (int i = NW - 1; i >= 0 && bits > 0; i--) { r.w[i] = bits >= 64 ? ~0ULL : ((1ULL << bits) - 1); bits -= 64; }
    return r;
}
static Kmer kor_low(Kmer a, unsigned c) { a.w[NW - 1] |= c; return a; }
/* nextKmer: kmer.c:696-702 */
static Kmer knext(Kmer a, unsigned c) { return kor_low(kand(kshl2(a), MASKK), c); }
/* prevKmer: kmer.c:704-718 (shift right, new base enters at bit 2(K-1)) */
static Kmer kprev(Kmer a, unsigned c) {
    Kmer r = kshr2(a); int bit = 2 * (K - 1); int wi = NW - 1 - bit / 64;
    r.w[wi] |= (u64)c << (bit % 64); return r;
}
static unsigned klast(Kmer a) { return a.w[NW - 1] & 3; }
static unsigned kfirst(Kmer a) { int bit = 2 * (K - 1); return (a.w[NW - 1 - bit / 64] >> (bit % 64)) & 3; } /* firstCharInKmer */
/* plain reverse complement of an n-mer (complement = code ^ 2, def.h:39-42) */
static Kmer krc_n(Kmer a, int n) {
    Kmer r = kzero();
    for (int i = 0; i < n; i++) { r = kshl2(r); r.w[NW - 1] |= (a.w[NW - 1] & 3) ^ 2; a = kshr2(a); }
    return r;
}
/* reverseComplement(seq, n) as the reference binary actually behaves.  SURVEY.md fact 11: in the 127-mer build
 * fastReverseComp takes `char seq_size` (kmer.c:532); n == 128 overflows to -128 and only low2 is
 * complemented+reversed, the other three words are returned untouched.  Load-bearing for K=127 (K+1)-mers. */
static Kmer krc(Kmer a, int n) {
#if NW == 4
    if (n == 128) { Kmer r = a; u64 lo = a.w[3], o = 0; for (int i = 0; i < 32; i++) { o = (o << 2) | ((lo & 3) ^ 2); lo >>= 2; } r.w[3] = o; return r; }
#endif
    return krc_n(a, n);
}

/* ------------------------------------------------------------------ CRC hash (hashFunction.c:28-82,123-131,155-158) */
static u32 crc_tab[256];
static void crc_init(void) { /* standard reflected CRC-32 (poly 0xEDB88320) table -- same values as crc_table[] */
    for (u32 i = 0; i < 256; i++) { u32 c = i; for (int j = 0; j < 8; j++) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1; crc_tab[i] = c; }
}
static u64 hash_kmer(Kmer k) { /* register starts at 0, final xor 0xFFFFFFFF, returned as int -> sign-extended */
    u32 c = 0; const u8 *p = (const u8 *)k.w;
    for (size_t i = 0; i < sizeof(Kmer); i++) c = crc_tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
    c ^= 0xFFFFFFFFu; return (u64)(int64_t)(int32_t)c;
}

/* ------------------------------------------------------------------ node + KmerSet (newhash.h:77-113, newhash.c) */
typedef struct {
    Kmer seq; u8 l[4], r[4]; u8 cov; u8 single, linear, deleted, inEdge, twin; u32 eid;
} Node;
typedef struct {
    u32 *slot;      /* 0 = null, else node index + 1 (the reference stores kmer_t inline + 2-bit flags; layout-equivalent) */
    Node *pool; u64 npool, cpool;
    u64 size, count, max; float lf; int is_static;
} Set;

static int is_prime_kh(u64 n) { /* newhash.c:142-167: float sqrt, strict '<' => squares of primes pass */
    if (n < 4) return 1;
    if (n % 2 == 0) return 0;
    u64 mx = (u64)sqrt((float)n);
    for (u64 i = 3; i < mx; i += 2) if (n % i == 0) return 0;
    return 1;
}
static u64 next_prime_kh(u64 n) { if (n % 2 == 0) n++; while (!is_prime_kh(n)) n += 2; return n; } /* :169-185 */
static u64 home(const Set *s, Kmer k) {
#if NW == 2
    unsigned __int128 t = ((unsigned __int128)k.w[0] << 64) | k.w[1]; return (u64)(t % s->size);   /* newhash.c:490-492 */
#else
    u64 z = s->size, t;                                                                             /* newhash.c:36-47 */
    t = (k.w[0] % z) << 32 | (k.w[1] >> 32 & 0xffffffff);
    t = (t % z) << 32 | (k.w[1] & 0xffffffff);
    t = (t % z) << 32 | (k.w[2] >> 32 & 0xffffffff);
    t = (t % z) << 32 | (k.w[2] & 0xffffffff);
    t = (t % z) << 32 | (k.w[3] >> 32 & 0xffffffff);
    t = (t % z) << 32 | (k.w[3] & 0xffffffff);
    return t % z;
#endif
}
static Set *set_new(u64 init, float lf, int is_static) { /* init_kmerset newhash.c:200-233 */
    Set *s = calloc(1, sizeof *s);
    s->size = init < 3 ? 3 : next_prime_kh(init);
    s->max = (u64)(s->size * lf);          /* ubyte8 * float -> float32 product */
    s->lf = lf; s->is_static = is_static;
    s->slot = calloc(s->size, sizeof(u32));
    s->cpool = 1024; s->pool = malloc(s->cpool * sizeof(Node));
    return s;
}
static void set_encap(Set *s) { /* encap_kmerset newhash.c:340-455, num == 1 */
    if (s->count + 1 <= s->max) return;
    if (s->is_static) {
        /* :353-366.  NB `load_factor < 0.88` compares a float against a double; (double)0.88f < 0.88, so the
         * "exploded" abort is unreachable and the table simply keeps filling. */
        s->lf = 0.88f; s->max = (u64)(s->size * s->lf); return;
    }
    u64 n = s->size;
    do { if (n < 0xFFFFFFFU) n <<= 1; else n += 0xFFFFFFU; n = next_prime_kh(n); } while (n * s->lf < s->count + 1);
    u64 old = s->size;
    u32 *arr = realloc(s->slot, n * sizeof(u32));           /* array realloc'ed in place ... */
    u8 *oldocc = calloc(old, 1), *newocc = calloc(n, 1);    /* ... with a fresh flag array (all null) */
    for (u64 i = 0; i < old; i++) oldocc[i] = arr[i] != 0;
    memset(arr + old, 0, (n - old) * sizeof(u32));
    s->slot = arr; s->size = n; s->max = (u64)(n * s->lf);
    for (u64 i = 0; i < old; i++) {                          /* ascending old slot, displacement chains */
        if (!oldocc[i]) continue;
        u32 key = arr[i]; oldocc[i] = 0;
        for (;;) {
            u64 hc = home(s, s->pool[key - 1].seq);
            while (newocc[hc]) { if (++hc == n) hc = 0; }
            newocc[hc] = 1;
            if (hc < old && oldocc[hc]) { u32 t = key; key = arr[hc]; arr[hc] = t; oldocc[hc] = 0; }
            else { arr[hc] = key; break; }
        }
    }
    /* slots of the old range that were never re-occupied must read as null */
    for (u64 i = 0; i < old; i++) if (!newocc[i]) arr[i] = 0;
    free(oldocc); free(newocc);
}
/* put_kmerset newhash.c:473-528; returns node, *found = 1 if it existed */
static Node *set_put(Set *s, Kmer k, int *found) {
    if (s->count + 1 > s->max) set_encap(s);
    u64 hc = home(s, k);
    for (;;) {
        if (!s->slot[hc]) {
            if (s->npool == s->cpool) { s->cpool *= 2; s->pool = realloc(s->pool, s->cpool * sizeof(Node)); }
            Node *nd = &s->pool[s->npool++]; memset(nd, 0, sizeof *nd); nd->seq = k;
            s->slot[hc] = (u32)s->npool; s->count++; *found = 0; return nd;
        }
        Node *nd = &s->pool[s->slot[hc] - 1];
        if (keq(nd->seq, k)) { *found = 1; return nd; }
        if (++hc == s->size) hc = 0;
    }
}
static Node *set_find(Set *s, Kmer k) { /* search_kmerset newhash.c:277-318 */
    u64 hc = home(s, k);
    for (;;) {
        if (!s->slot[hc]) return NULL;
        Node *nd = &s->pool[s->slot[hc] - 1];
        if (keq(nd->seq, k)) return nd;
        if (++hc == s->size) hc = 0;
    }
}

/* ------------------------------------------------------------------ globals (inc/global.h defaults) */
static int P = 8, D = 0, repsTie = 0, initG = 0;
static Set **sets, **patch;
static Node **order; static u64 norder;      /* THE iteration order: set 0 slot 0.., set 1 ... (SURVEY A.5) */
static Node *lookup(Kmer c) { return set_find(sets[hash_kmer(c) % (u64)P], c); }
static int nb(const u8 *a) { return (a[0] > 0) + (a[1] > 0) + (a[2] > 0) + (a[3] > 0); }
static int first_nz(const u8 *a) { for (int i = 0; i < 4; i++) if (a[i]) return i; return 4; }

/* ------------------------------------------------------------------ config + read stream (lib.c, readseq1by1.c) */
typedef struct { int avg_ins, asm_flag, reverse, rd_len_cutoff; char **f[7]; int nf[7]; } Lib; /* f[1]=f1 f[2]=q1 f[3]=p f[5]=f f[6]=q; f2/q2 in f[0]/f[4] */
static Lib *libs; static int nlibs; static int max_rd_len = 0;
typedef struct { u8 *s; int len; } Read;
static Read *reads; static u64 nreads, creads; static long long n_records;

static int split_col(const char *line, char t0[1024], char t1[1024]) { /* splitColumn lib.c:70-108: runs of printable chars other than '=' */
    int n = 0, i = 0, len = (int)strlen(line); char *t[2] = { t0, t1 };
    while (i < len) {
        if (line[i] >= 32 && line[i] <= 126 && line[i] != '=') {
            int j = 0; while (i < len && line[i] >= 32 && line[i] <= 126 && line[i] != '=') t[n][j++] = line[i++];
            t[n][j] = 0; if (++n == 2) return 1;
        }
        i++;
    }
    return 0;
}
static void add_file(Lib *L, int slot, const char *name) { L->f[slot] = realloc(L->f[slot], (L->nf[slot] + 1) * sizeof(char *)); L->f[slot][L->nf[slot]++] = strdup(name); }
static int cmp_lib(const void *a, const void *b) { int x = ((const Lib *)a)->avg_ins, y = ((const Lib *)b)->avg_ins; return (x > y) - (x < y); }
static void scan_lib(const char *cfg) { /* scan_libInfo lib.c:130-506 */
    FILE *fp = fopen(cfg, "r"); if (!fp) { fprintf(stderr, "Cannot open %s. Now exit to system...\n", cfg); exit(-1); }
    char line[1024], t0[1024], t1[1024]; int i = -1;
    while (fgets(line, 1024, fp)) {
        if (strncmp(line, "[LIB]", 5) == 0) { i++; libs = realloc(libs, (i + 1) * sizeof(Lib)); memset(&libs[i], 0, sizeof(Lib)); libs[i].asm_flag = 3; continue; }
        if (!split_col(line, t0, t1)) continue;
        if (i < 0) { if (!strcmp(t0, "max_rd_len")) max_rd_len = atoi(t1); continue; }   /* only before the first [LIB] (lib.c:152-165) */
        Lib *L = &libs[i];
        if (!strcmp(t0, "f1")) add_file(L, 1, t1); else if (!strcmp(t0, "f2")) add_file(L, 0, t1);
        else if (!strcmp(t0, "q1")) add_file(L, 2, t1); else if (!strcmp(t0, "q2")) add_file(L, 4, t1);
        else if (!strcmp(t0, "p")) add_file(L, 3, t1); else if (!strcmp(t0, "f")) add_file(L, 5, t1);
        else if (!strcmp(t0, "q")) add_file(L, 6, t1);
        else if (!strcmp(t0, "avg_ins")) L->avg_ins = atoi(t1); else if (!strcmp(t0, "reverse_seq")) L->reverse = atoi(t1);
        else if (!strcmp(t0, "asm_flags")) L->asm_flag = atoi(t1); else if (!strcmp(t0, "rd_len_cutoff")) L->rd_len_cutoff = atoi(t1);
    }
    fclose(fp); nlibs = i + 1;
    if (!nlibs) { fprintf(stderr, "Config file error: no [LIB] in file\n"); exit(-1); }
    qsort(libs, nlibs, sizeof(Lib), cmp_lib);                                           /* lib.c:505 */
}
typedef struct { char *buf; size_t n, pos; int fastq; } Src;
static Src src_open(const char *fn, int fastq) {
    fprintf(stderr, "Import reads from file:\n %s\n", fn);
    FILE *f = fopen(fn, "rb"); if (!f) { fprintf(stderr, "Cannot open %s. Now exit to system...\n", fn); exit(-1); }
    Src s; fseek(f, 0, SEEK_END); s.n = ftell(f); fseek(f, 0, SEEK_SET); s.buf = malloc(s.n + 1);
    if (fread(s.buf, 1, s.n, f) != s.n) exit(-1);
    s.buf[s.n] = 0; fclose(f); s.pos = 0; s.fastq = fastq; return s;
}
static size_t line_end(const Src *s, size_t p) { while (p < s->n && s->buf[p] != '\n') p++; return p; }
/* one record -> base codes.  readseqInBuf readseq1by1.c:138-209 / readseqfq :279-360: first min(linelen, maxReadLen) chars of the
 * sequence line; letters map through (ch&6)>>1 (A0 C1 T2 G3, N->3), '.' -> 0, anything else is dropped. */
static int src_next(Src *s, u8 *out, int *len, int maxlen) {
    if (s->pos >= s->n) return 0;
    size_t e = line_end(s, s->pos);            /* header */
    size_t b = e + 1; if (b > s->n) return 0;
    e = line_end(s, b);
    int raw = (int)(e - b), use = raw > maxlen ? maxlen : raw, n = 0;
    for (int i = 0; i < use; i++) {
        unsigned char c = s->buf[b + i];
        if ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z')) out[n++] = (c & 6) >> 1; else if (c == '.') out[n++] = 0;
    }
    *len = n; s->pos = e + 1;
    if (s->fastq) { e = line_end(s, s->pos); s->pos = e + 1 + raw + 1; }   /* skip '+' line, then jump strlen(seq)+1 (:342-347) */
    return 1;
}
static void take_read(u8 *tmp, int len, int reverse) {
    n_records++;
    if (reverse) { for (int i = 0; i < len / 2; i++) { u8 t = tmp[i]; tmp[i] = tmp[len - 1 - i]; tmp[len - 1 - i] = t; } for (int i = 0; i < len; i++) tmp[i] ^= 2; } /* reverse2k :788-802 */
    if (len < K + 1) return;                                             /* prlHashReads.c:504,559,642 */
    if (nreads == creads) { creads = creads ? creads * 2 : 1024; reads = realloc(reads, creads * sizeof(Read)); }
    reads[nreads].s = malloc(len); memcpy(reads[nreads].s, tmp, len); reads[nreads].len = len; nreads++;
}
static void load_reads(void) { /* openNextFile prlHashReads.c:903-951 + nextValidIndex readseq1by1.c:595-674 */
    int mrl = max_rd_len ? max_rd_len : 100;                             /* prlHashReads.c:326-329 */
    u8 *tmp = malloc(mrl + 8);
    for (int li = 0; li < nlibs; li++) {
        Lib *L = &libs[li];
        if (L->asm_flag != 1 && L->asm_flag != 3) continue;
        int cut = (L->rd_len_cutoff > 0 && L->rd_len_cutoff < mrl) ? L->rd_len_cutoff : mrl;   /* :921-928 */
        for (int type = 1; type <= 6; type++) {
            if (type == 4) continue;                                     /* BAM: out of scope */
            for (int fi = 0; fi < L->nf[type]; fi++) {
                int fq = (type == 2 || type == 6), len;
                if (type <= 2) {                                         /* paired files: r1,r2,r1,r2,... until file 2 ends (:480-583) */
                    Src a = src_open(L->f[type][fi], fq), b = src_open(L->f[type == 1 ? 0 : 4][fi], fq);
                    for (;;) {
                        if (!src_next(&a, tmp, &len, cut)) break; take_read(tmp, len, L->reverse);
                        if (!src_next(&b, tmp, &len, cut)) break; take_read(tmp, len, L->reverse);
                        if (b.pos >= b.n) break;
                    }
                    free(a.buf); free(b.buf);
                } else {
                    Src a = src_open(L->f[type][fi], fq);
                    while (src_next(&a, tmp, &len, cut)) take_read(tmp, len, L->reverse);
                    free(a.buf);
                }
            }
        }
    }
    free(tmp);
}

/* ------------------------------------------------------------------ chop (prlHashReads.c:163-259, prlRead2path.c:271-345) */
typedef struct { Kmer c; u8 sm; } Chop;
static int chop(const Read *rd, Chop *out) {
    Kmer w = kzero(); int n = rd->len - K + 1;
    for (int i = 0; i < K; i++) w = kor_low(kshl2(w), rd->s[i]);
    for (int j = 0; j < n; j++) {
        if (j) w = knext(w, rd->s[j + K - 1]);
        Kmer r = krc(w, K);
        if (kcmp(w, r) < 0) { out[j].c = w; out[j].sm = 1; } else { out[j].c = r; out[j].sm = 0; }   /* KmerSmaller; tie -> rc branch */
    }
    return n;
}

/* ------------------------------------------------------------------ output helpers */
static char *prefix;
static FILE *open_out(const char *suffix) { char nm[4096]; snprintf(nm, sizeof nm, "%s%s", prefix, suffix); FILE *f = fopen(nm, "w"); if (!f) { perror(nm); exit(-1); } return f; }
static int hexwords(char *dst, Kmer k, char sep) { /* print_kmer: "%llx %llx" (63) / 4 words (127) */
    int n = 0; for (int i = 0; i < NW; i++) n += sprintf(dst + n, i ? " %llx" : "%llx", (unsigned long long)k.w[i]); dst[n++] = sep; dst[n] = 0; return n;
}

/* ------------------------------------------------------------------ pass 1 (prlHashReads.c:304-760) */
static long long kmer_instances;
static void pass1(void) {
    u64 init = 1024;
    if (initG) {                                                          /* prlHashReads.c:369-390 */
        u64 want = (u64)((double)initG * 1024.0f * 1024.0f * 1024.0f / (double)P / (NW == 2 ? 24 : 40)), k = 0;
        do ++k; while (k * 0xFFFFFFULL < want);
        init = k * 0xFFFFFFULL;
    }
    sets = malloc(P * sizeof(Set *));
    for (int i = 0; i < P; i++) sets[i] = set_new(init, 0.77f, initG != 0);
    Chop *ch = malloc(((max_rd_len ? max_rd_len : 100) + 8) * sizeof(Chop));
    for (u64 ri = 0; ri < nreads; ri++) {
        const Read *rd = &reads[ri]; int L = rd->len, n = chop(rd, ch);
        kmer_instances += n;
        for (int j = 0; j < n; j++) {
            int prev, nxt;                                                /* SURVEY A.2 */
            if (ch[j].sm) { prev = j > 0 ? rd->s[j - 1] : 4; nxt = j < L - K ? rd->s[j + K] : 4; }
            else { prev = j + K < L ? rd->s[j + K] ^ 2 : 4; nxt = j > 0 ? rd->s[j - 1] ^ 2 : 4; }   /* bal[i] = s[L-1-i]^2 */
            int found; Node *e = set_put(sets[hash_kmer(ch[j].c) % (u64)P], ch[j].c, &found);
            if (!found) {                                                 /* set_new_kmer newhash.c:123-140 */
                e->single = 1; e->cov = 1; if (prev < 4) e->l[prev] = 1; if (nxt < 4) e->r[nxt] = 1;
            } else {                                                      /* update_kmer newhash.c:74-106 */
                if (prev < 4 && e->l[prev] < 63) e->l[prev]++;
                if (nxt < 4 && e->r[nxt] < 63) e->r[nxt]++;
                if ((prev < 4 || nxt < 4) && e->cov < 255) e->cov++;
                e->single = 0;
            }
        }
    }
    free(ch);
    u64 alloc = 0; for (int i = 0; i < P; i++) alloc += sets[i]->count;
    fprintf(stderr, "%lli node(s) allocated, %lli kmer(s) in reads, %lli kmer(s) processed.\n", (long long)alloc, kmer_instances, kmer_instances);
    norder = alloc; order = malloc((norder + 1) * sizeof(Node *)); u64 o = 0;
    for (int i = 0; i < P; i++) for (u64 j = 0; j < sets[i]->size; j++) if (sets[i]->slot[j]) order[o++] = &sets[i]->pool[sets[i]->slot[j] - 1];
    if (D > 0) {                                                          /* thread_delow prlHashReads.c:953-996 */
        long long removed = 0;
        for (u64 i = 0; i < norder; i++) {
            Node *e = order[i];
            for (int c = 0; c < 4; c++) { if (e->l[c] > 0 && e->l[c] <= D) e->l[c] = 0; if (e->r[c] > 0 && e->r[c] <= D) e->r[c] = 0; }
            if (e->l[0] + e->l[1] + e->l[2] + e->l[3] == 0 && e->r[0] + e->r[1] + e->r[2] + e->r[3] == 0) { e->deleted = 1; removed++; }
        }
        fprintf(stderr, "%lld kmer(s) removed.\n", removed);
    }
    long long hist[257] = { 0 }, lin = 0;                                 /* thread_mark :1020-1077 (no deleted check) */
    for (u64 i = 0; i < norder; i++) { Node *e = order[i]; hist[e->cov]++; if (nb(e->l) == 1 && nb(e->r) == 1) { e->linear = 1; lin++; } }
    fprintf(stderr, "%lld linear node(s) marked.\n", lin);
    FILE *fo = open_out(".kmerFreq");                                     /* freqStat :1104-1132 */
    for (int i = 1; i < 256; i++) fprintf(fo, "%lld\n", hist[i]);
    fclose(fo);
}

static void dump_table(const char *fn) {
    FILE *f = fopen(fn, "wb"); if (!f) { perror(fn); exit(-1); }
    for (u64 i = 0; i < norder; i++) {
        Node *e = order[i]; u8 fl = e->single | e->linear << 1 | e->deleted << 2;
        fwrite(e->seq.w, 8, NW, f); fwrite(e->l, 1, 4, f); fwrite(e->r, 1, 4, f); fwrite(&e->cov, 1, 1, f); fwrite(&fl, 1, 1, f);
    }
    fclose(f);
}

/* ------------------------------------------------------------------ tips (cutTipPreGraph.c) */
typedef struct { Kmer word, bal; int sm; } Canon;
static Canon canon(Kmer w) { Canon c; Kmer b = krc(w, K); if (kcmp(w, b) > 0) { c.word = b; c.bal = w; c.sm = 0; } else { c.word = w; c.bal = b; c.sm = 1; } return c; } /* KmerLarger swap */
static void dislink_prev(Node *n, int ch, int sm) { if (sm) n->l[ch] = 0; else n->r[ch ^ 2] = 0; }   /* newhash.c:681-691 */
static void dislink_next(Node *n, int ch, int sm) { if (sm) n->r[ch] = 0; else n->l[ch ^ 2] = 0; }   /* newhash.c:707-717 */
static int tip_c;
static Node *must_lookup(Kmer w, Node *n1) {
    Node *o = lookup(w); if (!o) { char b[200]; hexwords(b, w, ' '); fprintf(stderr, "Kmer %s is not found (model)\n", b); (void)n1; exit(1); } return o;
}
static int clip(Node *n1, int cut, int THIN) { /* clipTipFromNode cutTipPreGraph.c:43-346 */
    int in = nb(n1->l), on = nb(n1->r); Kmer pre, word;
    if (in == 0 && on == 1) { pre = n1->seq; word = knext(pre, first_nz(n1->r)); }
    else if (in == 1 && on == 0) { pre = krc(n1->seq, K); word = knext(pre, first_nz(n1->l) ^ 2); }
    else return 0;
    int count = 1; Canon c = canon(word); Node *out = must_lookup(c.word, n1);
    while (out->linear) {
        count++;
        if (THIN && !out->single) break;
        if (count > cut) return 0;
        if (c.sm) { pre = c.word; word = knext(pre, first_nz(out->r)); }
        else { pre = c.bal; word = knext(pre, first_nz(out->l) ^ 2); }
        c = canon(word); out = must_lookup(c.word, n1);
    }
    if (nb(out->l) + nb(out->r) == 1) { tip_c++; n1->deleted = 1; out->deleted = 1; return 1; }
    int ch = kfirst(pre);
    if (THIN) { tip_c++; n1->deleted = 1; dislink_prev(out, ch, c.sm); out->linear = 0; return 1; }
    int mx = 0; for (int i = 0; i < 4; i++) { int v = c.sm ? out->l[i] : out->r[i]; if (v > mx) mx = v; }
    if ((c.sm && out->l[ch] < mx) || (!c.sm && out->r[ch ^ 2] < mx)) {
        tip_c++; n1->deleted = 1; dislink_prev(out, ch, c.sm);
        if (nb(out->l) == 1 && nb(out->r) == 1) out->linear = 1;
        return 1;
    }
    return 0;
}
static void remark(void) { /* cutTipPreGraph.c:532-564 */
    long long c = 0;
    for (u64 i = 0; i < norder; i++) { Node *e = order[i]; if (!e->deleted && !e->linear && nb(e->l) == 1 && nb(e->r) == 1) { e->linear = 1; c++; } }
    fprintf(stderr, "%lld linear node(s) marked.\n", c);
}
static void tips(void) {
    int cut = 2 * K;
    if (D == 0) {                                                         /* pregraph.c:106-113, removeSingleTips :363-399 */
        fprintf(stderr, "Start to remove frequency-one-kmer tips shorter than %d.\n", cut);
        tip_c = 0;
        for (u64 i = 0; i < norder; i++) { Node *e = order[i]; if (!e->linear && !e->deleted && e->single) clip(e, cut, 1); }
        fprintf(stderr, "Total %d tip(s) removed.\n", tip_c);
        remark();
    }
    fprintf(stderr, "Start to remove tips with minority links.\n");       /* removeMinorTips :414-488 */
    tip_c = 0; int flag = 1, round = 1;
    while (flag) {
        flag = 0;
        for (u64 i = 0; i < norder; i++) { Node *e = order[i]; if (!e->linear && !e->deleted) flag += clip(e, cut, 0); }
        fprintf(stderr, "%d tip(s) removed in cycle %d.\n", flag, round++);
    }
    fprintf(stderr, "Total %d tip(s) removed.\n", tip_c);
    remark();
}

/* ------------------------------------------------------------------ edges (node2edge.c, output_pregraph.c:88-110) */
typedef struct { Node *nd; int sm; Kmer ori; } Bead;
static Bead *st; static int nst, cst;
static void st_push(Node *nd, int sm, Kmer ori) { if (nst == cst) { cst = cst ? cst * 2 : 1024; st = realloc(st, cst * sizeof(Bead)); } st[nst].nd = nd; st[nst].sm = sm; st[nst].ori = ori; nst++; }
static u32 edge_c; static long long extra_nodes, edge_counter;
static gzFile egz;
static void string_beads(int nextch) { /* stringBeads node2edge.c:86-218 */
    Canon c = canon(knext(st[0].ori, nextch)); Node *out = lookup(c.word);
    while (out && out->linear) {
        Kmer ori = c.sm ? c.word : c.bal; st_push(out, c.sm, ori);
        c = canon(knext(ori, c.sm ? first_nz(out->r) : (first_nz(out->l) ^ 2))); out = lookup(c.word);
    }
    if (!out) { fprintf(stderr, "model: edge walk fell off the table\n"); exit(1); }
    st_push(out, c.sm, c.sm ? c.word : c.bal);
}
static void merge_linear(int bal_edge) { /* merge_linearV2 node2edge.c:430-609 */
    int length = nst - 1; Bead *first = &st[0], *second = &st[1], *second_last = &st[nst - 2], *last = &st[nst - 1];
    dislink_prev(last->nd, kfirst(second_last->ori), last->sm);
    dislink_next(first->nd, klast(second->ori), first->sm);
    Kmer frm = first->ori, to = last->ori;
    edge_c++; edge_counter++;
    if (length == 1) {                                                    /* (K+1)-mer patch entry :481-541 */
        extra_nodes++;
        Kmer wp = kor_low(kshl2(frm), klast(to)), bwp = krc(wp, K + 1); int found; Node *n;
        if (kcmp(wp, bwp) < 0) { n = set_put(patch[hash_kmer(wp) % (u64)P], wp, &found); n->eid = edge_c; n->twin = (bal_edge + 1) & 3; }
        else { n = set_put(patch[hash_kmer(bwp) % (u64)P], bwp, &found); n->eid = edge_c + bal_edge; n->twin = (1 - bal_edge) & 3; }
    }
    long long symbol = 0;
    for (int i = nst - 2; i >= 1; i--) { st[i].nd->inEdge = 1; symbol += st[i].nd->l[0] + st[i].nd->l[1] + st[i].nd->l[2] + st[i].nd->l[3]; }
    for (int i = nst - 2; i >= 1; i--) {                                  /* edgeId overlays l_links+cov (union, newhash.h:83-88) */
        Node *nd = st[i].nd;
        if (st[i].sm) { nd->eid = edge_c; nd->twin = (bal_edge + 1) & 3; } else { nd->eid = edge_c + bal_edge; nd->twin = (1 - bal_edge) & 3; }
        nd->l[0] = nd->l[1] = nd->l[2] = nd->l[3] = 0xEE; /* poison: the reference's l_links are garbage from here on; nobody may read them */
    }
    int cvg = 0;
    if (length > 1) { long long v = symbol / (length - 1) * 10; cvg = v > 16000 ? 16000 : (int)v; }
    char hb[256]; int n = sprintf(hb, ">length %d,", length); n += hexwords(hb + n, frm, ','); n += hexwords(hb + n, to, ','); n += sprintf(hb + n, "cvg %d, %d\n", cvg, bal_edge);
    gzwrite(egz, hb, n);
    char *seq = malloc(length + length / 100 + 2); int m = 0;
    for (int i = 0; i < length; i++) { seq[m++] = "ACTG"[klast(st[i + 1].ori)]; if ((i + 1) % 100 == 0) seq[m++] = '\n'; }
    if (length % 100 != 0) seq[m++] = '\n';
    gzwrite(egz, seq, m); free(seq);
    edge_c += bal_edge;
}
static void edges(void) {
    char nm[4096]; snprintf(nm, sizeof nm, "%s.edge.gz", prefix); egz = gzopen(nm, "w");
    patch = malloc(P * sizeof(Set *)); for (int i = 0; i < P; i++) patch[i] = set_new(1000, 0.75f, 0);  /* node2edge.c:371-376; dynamic (pregraph.c:122) */
    edge_c = 0;
    for (u64 i = 0; i < norder; i++) {                                    /* make_edge :366-411, startEdgeFromNode :237-352 */
        Node *e = order[i]; if (e->linear || e->deleted) continue;
        Kmer w1 = e->seq, b1 = krc(w1, K);
        for (int side = 0; side < 2; side++) for (int ch = 0; ch < 4; ch++) {
            if (!(side == 0 ? e->r[ch] : e->l[ch])) continue;             /* read at this moment: merge clears links */
            nst = 0; st_push(e, side == 0, side == 0 ? w1 : b1);
            string_beads(side == 0 ? ch : ch ^ 2);
            int pal = 1; for (int q = 0; q < nst; q++) if (!keq(st[nst - 1 - q].ori, krc(st[q].ori, K))) { pal = 0; break; }
            merge_linear(pal ? 0 : 1);
        }
    }
    gzclose(egz);
    fprintf(stderr, "%d (%lld) edge(s) and %lld extra node(s) constructed.\n", edge_c, edge_counter, extra_nodes);
}

/* ------------------------------------------------------------------ pass 2 (prlRead2path.c) */
typedef struct Arc { u32 to, mult; struct Arc *next; } Arc;
static void pass2(void) {
    u32 num_ed = edge_c; Arc **arcs = calloc(num_ed + 1, sizeof(Arc *)); u8 *marker = calloc(num_ed + 1, 1);
    FILE *pf = repsTie ? open_out(".path") : NULL;
    int mrl = max_rd_len ? max_rd_len : 100; long long deleted_reads = 0, arc_c = 0;
    u32 *pathbuf = malloc((mrl + 8) * sizeof(u32));
    Chop *ks = malloc((mrl + 8) * sizeof(Chop)); Kmer *mix = malloc((mrl + 8) * sizeof(Kmer)); u8 *flag = malloc(mrl + 8), *smb = malloc(mrl + 8);
    for (u64 ri = 0; ri < nreads; ri++) {
        int n = chop(&reads[ri], ks); int retain = 0, pos = 0, IsPrev = 0; Kmer prevK = kzero();
        for (int j = 0; j < n; j++) smb[j] = ks[j].sm;
        for (int j = 0; j < n; j++) {                                     /* parse1read :598-745 */
            Node *nd = lookup(ks[j].c);
            if (!nd) { fprintf(stderr, "model: pass-2 lookup miss\n"); exit(1); }
            if (nd->deleted || (nd->linear && !nd->inEdge)) { if (retain < 2) { retain = 0; pos = 0; continue; } break; }   /* IsPrev/prevK NOT reset */
            int sm = smb[j];
            if (nd->linear) {
                u32 ei = sm ? nd->eid : nd->eid + nd->twin - 1;
                if (retain == 0 || IsPrev) { retain++; mix[pos] = kzero(); mix[pos].w[NW - 1] = ei; flag[pos++] = 0; IsPrev = 0; }
                else if (ei != (u32)mix[pos - 1].w[NW - 1]) { retain++; mix[pos] = kzero(); mix[pos].w[NW - 1] = ei; flag[pos++] = 0; }
            } else {
                Kmer cur = sm ? nd->seq : krc(nd->seq, K);
                if (IsPrev) {
                    retain++; Kmer wp = kor_low(kshl2(prevK), klast(cur)), bwp = krc(wp, K + 1);
                    if (kcmp(wp, bwp) < 0) { smb[pos] = 1; mix[pos] = wp; } else { smb[pos] = 0; mix[pos] = bwp; }
                    flag[pos++] = 1;
                }
                IsPrev = 1; prevK = cur;
            }
        }
        if (retain < 1) deleted_reads++;
        if (retain < 2) continue;
        u32 *path = pathbuf; int np = pos;
        for (int j = 0; j < pos; j++) {                                   /* search1kmerPlus :558-596 */
            if (flag[j]) { Node *ln = set_find(patch[hash_kmer(mix[j]) % (u64)P], mix[j]); path[j] = !ln ? 0 : (smb[j] ? ln->eid : ln->eid + ln->twin - 1); }
            else path[j] = (u32)mix[j].w[NW - 1];
        }
        for (int j = 0; j + 1 < np; j++) {                                /* thread_add1preArc :388-403 (head insert) */
            if (path[j] == 0 || path[j + 1] == 0) break;
            Arc *a = arcs[path[j]]; while (a && a->to != path[j + 1]) a = a->next;
            if (a) a->mult++; else { a = malloc(sizeof *a); a->to = path[j + 1]; a->mult = 1; a->next = arcs[path[j]]; arcs[path[j]] = a; arc_c++; }
        }
        if (repsTie && n >= 3 && np >= 3 && path[0] && path[1] && path[2]) {   /* recordPathBin :478-543 */
            u8 cnt = 0; u32 seg[256];
            for (int j = 0; j < np && path[j]; j++) { seg[cnt++] = path[j]; if (marker[path[j]] < 255) marker[path[j]]++; }
            fwrite(&cnt, 1, 1, pf); fwrite(seg, 4, cnt, pf);
        }
    }
    fprintf(stderr, "%lld pre-arcs built, %lld read(s) deleted (model)\n", arc_c, deleted_reads);
    FILE *fa = open_out(".preArc"), *fm = repsTie ? open_out(".markOnEdge") : NULL;   /* output_arcs :426-476 */
    for (u32 i = 1; i <= num_ed; i++) {
        if (fm) fprintf(fm, "%d\n", marker[i]);
        if (!arcs[i]) continue;
        fprintf(fa, "%u", i); for (Arc *a = arcs[i]; a; a = a->next) fprintf(fa, " %u %u", a->to, a->mult); fprintf(fa, "\n");
    }
    fclose(fa); if (fm) fclose(fm); if (pf) fclose(pf);
}

static void vertices(void) { /* output_vertex output_pregraph.c:50-86 */
    FILE *fv = open_out(".vertex"); int c = 0; char hb[200];
    for (u64 i = 0; i < norder; i++) { Node *e = order[i]; if (!e->linear && !e->deleted) { c++; int n = hexwords(hb, e->seq, ' '); fwrite(hb, 1, n, fv); if (c % 8 == 0) fputc('\n', fv); } }
    fputc('\n', fv); fclose(fv);
    fprintf(stderr, "%d vertex(es) output.\n", c);
    FILE *fb = open_out(".preGraphBasic");
    fprintf(fb, "VERTEX %d K %d\n\nEDGEs %d\n\nMaxReadLen %d MinReadLen %d MaxNameLen %d\n", c, K, edge_c, max_rd_len ? max_rd_len : 100, 0, 256);
    fclose(fb);
}

/* -V : print known-answer vectors of the restated primitives (compared with tests/golden/kats.json by tests/test_kats.py) */
static void self_kats(void) {
    const char *s = "ACGTTGCATGCAAGCTTAGCTAGGATCCATCGATCGGGCTATATCGCGATTAGCCATGCAGGT";
    K = 63; crc_init(); MASKK = kmask(K);
    Kmer f = kzero(), r;
    for (const char *p = s; *p; p++) f = knext(f, (*p & 6) >> 1);
    r = krc(f, K);
    printf("hash_zero 0x%llx\n", (unsigned long long)hash_kmer(kzero()));
    printf("kmer63_fwd 0x%llx 0x%llx\n", (unsigned long long)f.w[NW - 2], (unsigned long long)f.w[NW - 1]);
    printf("kmer63_rc 0x%llx 0x%llx\n", (unsigned long long)r.w[NW - 2], (unsigned long long)r.w[NW - 1]);
    printf("kmer63_smaller_fwd_rc %d\n", kcmp(f, r) < 0);
    printf("kmer63_hash_fwd 0x%llx\n", (unsigned long long)(hash_kmer(f) & 0xffffffffULL));
    printf("kmer63_hash_rc 0x%llx\n", (unsigned long long)(hash_kmer(r) & 0xffffffffULL));
    Set *a = set_new(1024, 0.77f, 0), *b = set_new(3 * 0xFFFFFFULL, 0.77f, 1);
    printf("init_kmerset_0 %llu %llu\n", (unsigned long long)a->size, (unsigned long long)a->max);
    printf("init_kmerset_1 %llu %llu\n", (unsigned long long)b->size, (unsigned long long)b->max);
}

int main(int argc, char **argv) {
    const char *cfg = NULL, *tdump = NULL, *udump = NULL; int only1 = 0, c; K = 23;
    if (argc > 1 && !strcmp(argv[1], "-V")) { self_kats(); return 0; }
    if (argc > 1 && !strcmp(argv[1], "pregraph")) { argv++; argc--; }
    while ((c = getopt(argc, argv, "a:s:o:K:p:d:RT:U:1")) != -1) switch (c) {
        case 's': cfg = optarg; break; case 'o': prefix = optarg; break; case 'K': K = atoi(optarg); break;
        case 'p': P = atoi(optarg); break; case 'R': repsTie = 1; break; case 'd': D = atoi(optarg) >= 0 ? atoi(optarg) : 0; break;
        case 'a': initG = atoi(optarg); break; case 'T': tdump = optarg; break; case 'U': udump = optarg; break; case '1': only1 = 1; break;
    }
    if (!cfg || !prefix) { fprintf(stderr, "usage: pregraph_model -s cfg -o prefix [-K k -p P -a G -d D -R]\n"); return -1; }
    /* pregraph.c:71-97 */
    if (K % 2 == 0) K++;
    if (K < 13) K = 13;
    if (K > MODEL_W / 2 - 1) K = MODEL_W / 2 - 1;
    D = (signed char)D;                                                   /* deLowKmer is a char (global.h:67) */
    crc_init(); MASKK = kmask(K);
    scan_lib(cfg);
    struct timespec t0, t1; clock_gettime(CLOCK_MONOTONIC, &t0);
    load_reads();
    clock_gettime(CLOCK_MONOTONIC, &t1);
    fprintf(stderr, "model: %lld record(s), %llu read(s) kept, load %.3fs\n", n_records, (unsigned long long)nreads, (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec));
    pass1();
    clock_gettime(CLOCK_MONOTONIC, &t0);
    fprintf(stderr, "model: pass1 %.3fs\n", (t0.tv_sec - t1.tv_sec) + 1e-9 * (t0.tv_nsec - t1.tv_nsec));
    if (tdump) dump_table(tdump);
    if (only1) return 0;
    tips();
    if (udump) dump_table(udump);
    edges(); pass2(); vertices();
    return 0;
}
