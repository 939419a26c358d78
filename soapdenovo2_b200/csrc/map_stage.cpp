// map_stage.cpp -- the `map -s cfg -g prefix [-f] [-p n] [-k k] [-h len]` stage (call_align).  Mirrors, in new code, the host-side
// behaviour of (standardPregraph/):
//   call_align / initenv / getMinOverlap   map.c:48-240           (getopt string, K from .preGraphBasic, -k, stderr lines)
//   prlContig2nodes (host part)            prlHashCtg.c:325-467   (the stats lines; .contig itself is read by read_contigs, stage_io.cpp)
//   basicContigInfo                        prlRead2Ctg.c:727-763  (.ContigIndex -> lengths, bal_edge)
//   prlRead2Ctg / recordAlldgn / getReadIngap / output1read_gz / getPEreadOnContig   prlRead2Ctg.c:427-712, 779-1053
//   prlLongRead2Ctg / recordLongRead / output1read         prlRead2Ctg.c:456-492, 612-625, 1080-1298
// The k-mer work (contig table, read scan, parse1read) runs on the GPU (map.cu); the .contig text is parsed on the host: it is a
// few hundred MB at most, multi-line, and is read once.
//
// Long-read libraries (asm_flags=4) are mapped first, when getMaxLongReadLen >= 1, and write .longReadInGap (.RlongReadInGap with
// -f); configs without them give the same output and stderr as a stage without the long pass.  Both passes' reads are decoded
// before any output file is opened, so every refusal -- BAM, two-file pairs in a long library, a read that would overflow the
// reference's read buffers -- comes before the first output.  locate1read
// (prlRead2Ctg.c:389-425) is not restated: recordAlldgn calls it only for a read with footprint set whose contig id is < 1, but
// parse1read sets footprint only after it chose a contig, and a chosen contig id is either atoi(name) > 0, an ordinal >= 1, or its
// twin id, which is >= 1 as well.
//
// `.readInGap.gz` depends on -p.  Its records are packed into rcSeq[1] (writeChar2tightString, seq.c:81), which masks only the
// 2-bit fields it writes, so the last byte of a record carries bits of whatever the buffer held.  The reference's thread 0 also uses
// rcSeq[1] as the reverse-complement scratch of the reads it chops, reads i == 0 (mod P) of each batch with len >= K+1, before the
// batch is recorded.  `RcSeqModel` keeps a byte-exact copy of that buffer: one base code per byte after a chop, then every tight-
// string write in order.  It starts as zeros (ckalloc is calloc).
#include "stage.h"
#include "map.h"
#include "deflate.h"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <future>
#include <memory>
#include <stdexcept>
#include <getopt.h>
#include <zlib.h>

namespace pgb {
namespace {

void map_usage(int flavour127) {   // display_map_usage, map.c:227-240
    fprintf(stderr, "\nmap -s configFile -g inputGraph [-f] [-p n_cpu -k kmer_R2C] [-h contig_total_length]\n");
    fprintf(stderr, "  -s <string>        configFile: the config file of solexa reads\n");
    fprintf(stderr, "  -g <string>        inputGraph: prefix of input graph file names\n");
    fprintf(stderr, "  -h (optional)      total length of contigs for init hash table. [1024]\n");
    fprintf(stderr, "  -f (optional)      output gap related reads in map step for using SRkgf to fill gap, [NO]\n");
    fprintf(stderr, "  -p <int>           n_cpu: number of cpu for use, [8]\n");
    fprintf(stderr, "  -k <int>           kmer_R2C(min 13, max %d): kmer size used for mapping read to contig, [K]\n", flavour127 ? 127 : 63);
}

int min_overlap(const std::string& prefix) {   // getMinOverlap, map.c:48-76
    int K = 23, n;
    char ch, line[1024];
    FILE* fp = fopen((prefix + ".preGraphBasic").c_str(), "r");
    if (!fp) return K;
    while (fgets(line, sizeof line, fp))
        if (line[0] == 'V') sscanf(line + 6, "%d %c %d", &n, &ch, &K);
    fclose(fp);
    return K;
}

// basicContigInfo: contig_array[1..num_all].{length, bal_edge}
struct ContigInfo { std::vector<u32> length; std::vector<int> bal_edge; int num_all = 0; };
ContigInfo contig_info(const std::string& prefix) {
    FILE* fp = ckopen(prefix + ".ContigIndex", "r");
    char line[1024];
    ContigInfo ci;
    int num_long = 0, index, length, bal;
    if (fgets(line, sizeof line, fp) && strlen(line) > 8) sscanf(line + 8, "%d %d", &ci.num_all, &num_long);
    ci.length.assign((size_t)std::max(ci.num_all, 0) + 1, 0);
    ci.bal_edge.assign(ci.length.size(), 0);
    if (!fgets(line, sizeof line, fp)) line[0] = 0;
    num_long = 0;
    while (fgets(line, sizeof line, fp)) {
        if (sscanf(line, "%d %d %d", &index, &length, &bal) != 3) continue;
        if (num_long + 2 >= (int)ci.length.size()) { ci.length.resize(num_long + 3, 0); ci.bal_edge.resize(num_long + 3, 0); }
        ci.length[++num_long] = (u32)length;
        ci.bal_edge[num_long] = bal + 1;
        if (index != num_long) fprintf(stderr, "BasicContigInfo: %d vs %d.\n", index, num_long);
        if (bal == 0) continue;
        ci.length[++num_long] = (u32)length;
        ci.bal_edge[num_long] = -bal + 1;
    }
    fclose(fp);
    return ci;
}

// The reads of one pass, in the order read1seqInLib returns them (short pass: mates interleaved), each packed 2 bits per base (LSB
// first) at its own length, ceil(len / 32) words at wofs[r]; wofs[n] is the word total
struct Reads {
    std::vector<u64> words, wofs;
    std::vector<u32> lens;
    std::vector<int> lib;   // index into MapPlan::libs / long_libs
};

// The stage's reader of read files, with one chunk buffer for the whole stage.  read() appends one file's reads to *words / *lens,
// each cut to maxlen bases.  fgets_gstr < 0: pass 1's reader (decode_text: single-line FASTA, 4-line FASTQ) with pass 1's record rule.
// Otherwise the fgets reader (read_text, reader.cu), which reads wrapped records as readseq1by1 / read1seqfq do, in fgets pieces (see
// load_reads), and finds the cut.
struct FileReader {
    IMapEngine& eng;
    const size_t cap;
    std::unique_ptr<char[]> buf{new char[cap]};
    void read(const PlanEntry& f, int maxlen, int fgets_gstr, std::vector<u64>* words, std::vector<u32>* lens) {
        const int piece = fgets_gstr < 0 ? 0 : fgets_gstr ? f.cut : 4999;
        read_chunks(f.path, buf.get(), cap, [&](const char* text, size_t n, bool at_eof) {
            if (piece)
                return in_step("%s (%s)", [&] { return eng.read_text(text, n, f.fastq, piece, maxlen, f.reverse, at_eof, words, lens); }, f.path.c_str());
            const size_t cut = whole_records(text, n, f.fastq, at_eof);
            in_step("readseqInLib return error! please make sure input file is correct fastq/fasta file \n(%s)",
                    [&] { eng.decode_text(text, cut, f.fastq, f.reverse, maxlen, words, lens); });
            return cut;
        });
    }
};

// One pass's reads, decoded before anything is written: every refusal comes before the first output file.  The stderr lines the
// reference prints while it reads go to *log, to be printed where the pass prints them.  A read longer than `room` would run past
// the reference's seqBuffer (allocated for `room` bases): no output is defined for it, so it is refused.  Each file is read with a
// cut one base past `room` so that such a read shows.  fgets_gstr < 0: pass 1's reader (single-line FASTA, 4-line FASTQ);
// otherwise the fgets reader, whose pieces are the cutoff long when the pass allocated gStr (fgets_gstr = 1) and gLineLen - 1 = 4999
// bytes long when it did not (readseq1by1.c:54-66, prlRead2Ctg.c:826, 1133).
Reads load_reads(FileReader& files, const std::vector<MapLib>& libs, bool long_pass, int room, int fgets_gstr, std::string* log) {
    Reads rd;
    char line[256];
    auto say = [&](const char* fmt, auto... a) { snprintf(line, sizeof line, fmt, a...); *log += line; };
    for (size_t li = 0; li < libs.size(); li++) {
        const MapLib& L = libs[li];
        const size_t lib_begin = rd.lens.size();
        for (size_t fi = 0; fi < L.files.size(); fi++) {
            const PlanEntry& e = L.files[fi];
            const int maxlen = std::min(e.cut, room + 1);
            const size_t before = rd.lens.size();
            if (e.mate == 0) {
                // openFileInLib names both mates before the first read; mates then alternate r1, r2, r1, r2
                const PlanEntry& m = L.files[++fi];
                say("Import reads from file:\n %s\n", e.path.c_str());
                say("Import reads from file:\n %s\n", m.path.c_str());
                std::vector<u64> w1, w2;
                std::vector<u32> l1, l2;
                files.read(e, maxlen, fgets_gstr, &w1, &l1);
                files.read(m, maxlen, fgets_gstr, &w2, &l2);
                if (l1.size() != l2.size())
                    fail("pgb200: mate files hold different numbers of reads (%zu vs %zu): unsupported", l1.size(), l2.size());
                const size_t w0 = rd.words.size();
                rd.words.resize(w0 + w1.size() + w2.size());
                u64* dst = rd.words.data() + w0;
                const u64 *s1 = w1.data(), *s2 = w2.data();
                auto copy_read = [&](const u64*& src, u32 len) {
                    const size_t nw = (len + 31) / 32;
                    memcpy(dst, src, nw * sizeof(u64));
                    dst += nw;
                    src += nw;
                    rd.lens.push_back(len);
                };
                for (size_t r = 0; r < l1.size(); r++) {
                    copy_read(s1, l1[r]);
                    copy_read(s2, l2[r]);
                }
            } else {
                say("Import reads from file:\n %s\n", e.path.c_str());
                files.read(e, maxlen, fgets_gstr, &rd.words, &rd.lens);
            }
            for (size_t r = before; r < rd.lens.size(); r++)
                if ((int)rd.lens[r] > room)
                    fail("pgb200: %s holds a read longer than %d bases (%s); the reference would write past its read buffer", e.path.c_str(), room,
                         long_pass ? "the long-read length, getMaxLongReadLen"
                                   : "max_rd_len: the long-read libraries raise the short reads' length cutoff to maxReadLen4all");
            rd.lib.resize(rd.lens.size(), (int)li);
            if (rd.lens.size() > before && lib_begin == before) {
                if (long_pass) say("Map_len %d.\n", std::max(L.map_len, 35));   // prlRead2Ctg.c:1198-1204
                else say("Current insert size is %d, map_len is %d.\n", L.avg_ins, L.avg_ins > 1000 ? std::max(L.map_len, 35) : std::max(L.map_len, 32));   // :903-919
            }
            for (size_t r = before; r < rd.lens.size(); r++)
                if ((r + 1) % 100000000 == 0) say("--- %lldth reads.\n", (long long)(r + 1));
        }
    }
    rd.wofs.resize(rd.lens.size() + 1);
    u64 o = 0;
    for (size_t r = 0; r < rd.lens.size(); r++) { rd.wofs[r] = o; o += (rd.lens[r] + 31) / 32; }
    rd.wofs.back() = o;
    return rd;
}

template <class T> void put(std::string& s, const T& v) { s.append(reinterpret_cast<const char*>(&v), sizeof v); }

struct RcSeqModel {
    std::vector<unsigned char> b;
    // writeChar2tightString of every base of w (seq.c:81-107), then the len / 4 + 1 bytes the record takes from the buffer
    void append_tight(std::string& s, const u64* w, int len) {
        for (int i = 0; i < len; i++) {
            const unsigned c = (unsigned)(w[i >> 5] >> (2 * (i & 31))) & 3u;
            unsigned char& x = b[i / 4];
            const int sh = 6 - 2 * (i % 4);
            x = (unsigned char)((x & ~(3u << sh)) | (c << sh));
        }
        s.append(reinterpret_cast<const char*>(b.data()), (size_t)(len / 4 + 1));
    }
    // thread 0's chops of a batch of n reads leave their reverse complements here (chopKmer4read, prlRead2Ctg.c:153-187): reads
    // t = 0 (mod P) with len >= K+1, the later ones over the earlier ones
    void chops(u64 n, int P, int K, const u32* lens, const u64* W, const u64* wofs) {
        size_t covered = 0;
        for (long long t = ((long long)n - 1) / P * P; t >= 0 && covered < b.size(); t -= P) {
            const int len = (int)lens[t];
            if (len < K + 1 || (size_t)len <= covered) continue;
            const u64* w = W + wofs[t];
            for (size_t i = covered; i < (size_t)len; i++) {
                const int src = len - 1 - (int)i;
                b[i] = (unsigned char)((((w[src >> 5] >> (2 * (src & 31))) & 3u)) ^ 2u);
            }
            covered = (size_t)len;
        }
    }
};

// parse1read's output arrays for one batch: the contig lengths and twins applied to the GPU's placements
struct Placement {
    std::vector<u32> ctg;
    std::vector<int> pos;
    std::vector<char> orien, footprint;
    explicit Placement(size_t n) : ctg(n), pos(n), orien(n, 0), footprint(n) {}
    void set(const MapHit* hit, u64 n, const ContigInfo& ci, int K, const std::string& prefix) {
        for (u64 t = 0; t < n; t++) {
            const MapHit& h = hit[t];
            footprint[t] = (h.flags & MAP_FOOTPRINT) ? 1 : 0;
            if (!(h.flags & MAP_PLACED)) { ctg[t] = 0; continue; }
            if (h.ctg >= ci.length.size()) fail("pgb200: contig %u is not in %s.ContigIndex", h.ctg, prefix.c_str());
            const u32 len = ci.length[h.ctg];
            if (h.flags & MAP_MINUS) {
                orien[t] = '-';
                ctg[t] = h.ctg + (u32)ci.bal_edge[h.ctg] - 1u;   // getTwinCtg, attachPEinfo.c:666-669
                pos[t] = (int)(len - (u32)h.node_pos - (u32)K - (u32)h.i + 1u);
            } else {
                orien[t] = '+';
                ctg[t] = h.ctg;
                pos[t] = (int)((u32)h.node_pos - (u32)h.i + 1u);
            }
        }
    }
};

long long batch_reads(const char* what, int read_len, int K) {   // maxReadNum, prlRead2Ctg.c:814-815 and 1115-1116
    if (read_len - K + 1 <= 0) fail("pgb200: %s %d is shorter than K %d", what, read_len, K);
    long long m = 100000000 / (read_len - K + 1);
    if (m % 2) m--;
    if (m < 2) fail("pgb200: %s %d leaves no room for a read pair in a batch", what, read_len);
    return m;
}

void print_libs(const MapPlan& plan) {   // free_libs, lib.c:516-520
    fprintf(stderr, "LIB(s) information:\n");
    for (size_t i = 0; i < plan.libs.size(); i++) fprintf(stderr, " [LIB] %zu, avg_ins %d, reverse %d.\n", i, plan.libs[i].avg_ins, plan.libs[i].reverse);
}

// The batch work both passes share: reads [b0, b0 + n) of rd, their word offsets rebased to the batch, through parse1read on the
// GPU (k_map_long, one CTA per read, when per_read_cta; else k_map_reads), then thread 0's chops into rc (a zeroed buffer of the
// pass's read length: ckalloc is calloc) and the placements into pl.  read(t) is the batch's read t.
struct BatchMapper {
    IMapEngine& eng;
    const Reads& rd;
    const ContigInfo& ci;
    const int K, P;
    const std::string& prefix;
    std::vector<MapHit> hit;
    Placement pl;
    RcSeqModel rc;
    std::vector<u64> wofs;
    const u64* W = nullptr;
    const u32* lens = nullptr;
    BatchMapper(IMapEngine& eng, const Reads& rd, long long max_read_num, int read_len, const ContigInfo& ci, int K, int P, const std::string& prefix)
        : eng(eng), rd(rd), ci(ci), K(K), P(P), prefix(prefix), hit((size_t)std::min<long long>(max_read_num, (long long)std::max<size_t>(rd.lens.size(), 1))),
          pl(hit.size()), rc{std::vector<unsigned char>((size_t)read_len, 0)} {}
    const u64* read(u64 t) const { return W + wofs[t]; }
    // returns the host time at which the GPU's placements were in
    double map(u64 b0, u64 n, int alignlen, bool per_read_cta, const char* fail_fmt) {
        const u64 w0 = rd.wofs[b0];
        wofs.resize(n);
        for (u64 t = 0; t < n; t++) wofs[t] = rd.wofs[b0 + t] - w0;
        W = rd.words.data() + w0;
        lens = rd.lens.data() + b0;
        in_step(fail_fmt, [&] { eng.map_batch(W, rd.wofs[b0 + n] - w0, wofs.data(), lens, n, alignlen, per_read_cta, hit.data()); });
        const double t_mapped = host_now();
        rc.chops(n, P, K, lens, W, wofs.data());
        pl.set(hit.data(), n, ci, K, prefix);
        return t_mapped;
    }
};

// The gap record of output1read / output1read_gz: len, contig, pos, then the read packed from rcSeq[1]
void put_gap(std::string& s, RcSeqModel& rc, const u64* w, int len, int ctg, int pos) {
    put(s, len); put(s, ctg); put(s, pos);
    rc.append_tight(s, w, len);
}
// The -f text record: ">len\tctg\tpos\torien\tins\tdh\n", then the bases
void put_text(std::string& s, const u64* w, int len, int ctg, int pos, char o, int ins, int dh) {
    char line[128];
    s.append(line, (size_t)snprintf(line, sizeof line, ">%d\t%d\t%d\t%c\t%d\t%d\n", len, ctg, pos, o, ins, dh));
    for (int i = 0; i < len; i++) s.push_back("ACTG"[(w[i >> 5] >> (2 * (i & 31))) & 3]);
    s.push_back('\n');
}

// prlLongRead2Ctg once its reads are in: batches of maxReadNum reads (from longReadLen) and recordLongRead / output1read.  Every
// long read has insert size 18; a read whose footprint is set goes to .longReadInGap (with this pass's own rcSeq[1], of longReadLen
// bytes) and, with -f, as text to .RlongReadInGap.  Both are plain files.
void map_long_reads(IMapEngine& eng, const MapPlan& plan, const Reads& rd, long long max_read_num, const ContigInfo& ci, int K, int P, int fill,
                    const std::string& prefix) {
    const u64 n_reads = rd.lens.size();
    BatchMapper bm(eng, rd, max_read_num, plan.long_len, ci, K, P, prefix);
    const Placement& pl = bm.pl;
    std::unique_ptr<FILE, int (*)(FILE*)> f_gap(ckopen(prefix + ".longReadInGap", "wb"), fclose);
    std::unique_ptr<FILE, int (*)(FILE*)> f_txt(fill ? ckopen(prefix + ".RlongReadInGap", "w") : nullptr, fclose);
    auto put_file = [&](FILE* f, const std::string& s, const char* suffix) {
        if (!s.empty() && fwrite(s.data(), 1, s.size(), f) != s.size()) fail("short write on %s%s", prefix.c_str(), suffix);
    };
    long long read_counter = 0, in_gap = 0, last_batch = 0;
    std::string s_gap, s_txt;
    for (u64 b0 = 0; b0 < n_reads; b0 += (u64)max_read_num) {
        const u64 n = std::min<u64>((u64)max_read_num, n_reads - b0);
        last_batch = (long long)n;
        const int alignlen = std::max(plan.long_libs[rd.lib[b0 + n - 1]].map_len, 35);   // ALIGNLEN after the batch's last read (:1198-1204)
        bm.map(b0, n, alignlen, true, "pgb200: long-read scan failed: %s");
        s_gap.clear(); s_txt.clear();
        for (u64 t = 0; t < n; t++) {   // recordLongRead, output1read (prlRead2Ctg.c:456-492, 612-625)
            read_counter++;
            if (!pl.footprint[t]) continue;
            const int len = (int)bm.lens[t];
            in_gap++;
            put_gap(s_gap, bm.rc, bm.read(t), len, (int)pl.ctg[t], pl.pos[t]);
            if (fill && len > 0) put_text(s_txt, bm.read(t), len, (int)pl.ctg[t], pl.pos[t], pl.orien[t], 18, 0);
        }
        put_file(f_gap.get(), s_gap, ".longReadInGap");
        if (fill) put_file(f_txt.get(), s_txt, ".RlongReadInGap");
    }
    if (n_reads && last_batch != max_read_num)   // a batch that ends exactly at the last read is recorded inside the reference's loop
        fprintf(stderr, "Output %lld out of %lld (%.1f)%% reads in gaps.\n", in_gap, read_counter, (float)in_gap / read_counter * 100);
}

// The map .gz outputs: gzopen + gzwrite bytes, deflated on the GPU of the stage (deflate.cu; PGB200_GZ=host: zlib)
struct GzOut {
    std::unique_ptr<GzFile> f;
    std::string name;
    void open(const std::string& n, int device) {
        name = n;
        try { f.reset(gz_open(n, device)); } catch (const std::exception&) { fail("Cannot open %s. Now exit to system...", n.c_str()); }
    }
    void write(const std::string& s) { f->write(s.data(), s.size(), false); }
    void close() { if (f) f->close(); f.reset(); }
};

// prlRead2Ctg once its reads are in: the output files, batches of maxReadNum reads (from max_rd_len), recordAlldgn with its mates
// (getReadIngap, getPEreadOnContig) and output1read_gz, the closing counts and .peGrads.  long_all: the batches through k_map_long.
void map_short_reads(IMapEngine& eng, const MapPlan& plan, const Reads& rd, const std::string& log, long long max_read_num, const ContigInfo& ci, int K,
                     int P, int fill, bool long_all, const std::string& prefix, int device, double* ms_record, double* ms_deflate) {
    GzOut f_gap, f_short, f_on, f_pe;
    f_gap.open(prefix + ".readInGap.gz", device);
    if (fill) f_short.open(prefix + ".shortreadInGap.gz", device);
    f_on.open(prefix + ".readOnContig.gz", device);
    if (fill) f_pe.open(prefix + ".PEreadOnContig.gz", device);
    f_on.write("read\tcontig\tpos\n");
    fputs(log.c_str(), stderr);
    struct Grad { int ins; long long bound; int rank, cut; };
    std::vector<Grad> grads;   // a library's boundary is the count of reads up to its last one (readseq1by1.c:1092-1102)
    for (size_t r = 0; r < rd.lens.size(); r++)
        if (r + 1 == rd.lens.size() || rd.lib[r + 1] != rd.lib[r]) {
            const MapLib& L = plan.libs[rd.lib[r]];
            grads.push_back({L.avg_ins, (long long)r + 1, L.rank, L.pair_num_cut});
        }
    const u64 n_reads = rd.lens.size();

    BatchMapper bm(eng, rd, max_read_num, plan.max_rd_len, ci, K, P, prefix);
    std::vector<u32>& ctg_arr = bm.pl.ctg;
    std::vector<int>& pos_arr = bm.pl.pos;
    const std::vector<char>&orien = bm.pl.orien, &footprint = bm.pl.footprint;
    long long read_counter = 0, map_counter = 0, in_gap = 0;
    int alignlen = 0, prev_lib = -1;
    // everything the writer thread touches is declared before the writer, whose destructor waits for the thread on every way out
    std::string s_gap, s_short, s_on, s_pe;
    std::future<void> writer;
    auto join = [&] {
        const double t_join = host_now();
        if (writer.valid()) writer.get();   // rethrows the writer's failure
        *ms_deflate += host_now() - t_join;
    };
    long long last_batch = 0;
    for (u64 b0 = 0; b0 < n_reads; b0 += (u64)max_read_num) {
        const u64 n = std::min<u64>((u64)max_read_num, n_reads - b0);
        last_batch = (long long)n;
        for (u64 r = b0; r < b0 + n; r++) {   // ALIGNLEN as it stands after the batch's last read (prlRead2Ctg.c:903-926)
            const MapLib& L = plan.libs[rd.lib[r]];
            if (rd.lib[r] != prev_lib) { prev_lib = rd.lib[r]; alignlen = L.avg_ins > 1000 ? std::max(L.map_len, 35) : std::max(L.map_len, 32); }
            if (L.avg_ins > 1000) alignlen = std::max(alignlen, (int)(rd.lens[r] / 2 + 1));
        }
        const double t_rec = bm.map(b0, n, alignlen, long_all, "pgb200: read scan failed: %s");
        // recordAlldgn (prlRead2Ctg.c:627-712) into this batch's byte strings
        join();
        s_gap.clear(); s_short.clear(); s_on.clear(); s_pe.clear();
        auto ins_of = [&](u64 t) { return plan.libs[rd.lib[b0 + t]].avg_ins; };
        auto output1read = [&](u64 t, char o, int dh) {   // output1read_gz
            const int len = (int)bm.lens[t];
            in_gap++;
            put_gap(s_gap, bm.rc, bm.read(t), len, (int)ctg_arr[t], pos_arr[t]);
            if (fill && ins_of(t) < 2000 && len > 0) put_text(s_short, bm.read(t), len, (int)ctg_arr[t], pos_arr[t], o, ins_of(t), dh);
        };
        auto read_in_gap = [&](u64 t, bool read_one) {   // getReadIngap
            const u64 r1 = read_one ? t : t - 1, r2 = read_one ? t + 1 : t;
            const u64 placed = read_one ? r2 : r1, gap = read_one ? r1 : r2;
            const char o = orien[placed] == '+' ? '-' : '+';
            ctg_arr[gap] = ctg_arr[placed];
            pos_arr[gap] = pos_arr[placed] + ins_of(gap) - (int)bm.lens[gap];
            output1read(gap, o, read_one ? 1 : 2);
        };
        auto pe_on_contig = [&](u64 t) {   // getPEreadOnContig
            if (!(ins_of(t) < 2000 && ins_of(t) == ins_of(t - 1))) return;
            for (u64 r = t - 1; r <= t; r++) {
                const int len = (int)bm.lens[r];
                put(s_pe, len); put(s_pe, (int)ctg_arr[r]); put(s_pe, pos_arr[r]); put(s_pe, orien[r]); put(s_pe, ins_of(r));
                bm.rc.append_tight(s_pe, bm.read(r), len);
            }
        };
        char line[96];
        for (u64 t = 0; t < n; t++) {
            read_counter++;
            bool rd1gap = false, rd2gap = false;
            const int ctg_id = (int)ctg_arr[t];
            if (t % 2 == 1) {
                if (ctg_arr[t] < 1 && ctg_arr[t - 1] > 0) { read_in_gap(t, false); rd2gap = true; }
                else if (ctg_arr[t] > 0 && ctg_arr[t - 1] < 1) { read_in_gap(t - 1, true); rd1gap = true; }
                else if (ctg_arr[t] > 0 && ctg_arr[t - 1] > 0 && fill) pe_on_contig(t);
            }
            if (ctg_id < 1) continue;
            map_counter++;
            s_on.append(line, (size_t)snprintf(line, sizeof line, "%lld\t%u\t%d\t%c\n", read_counter, ctg_arr[t], pos_arr[t], orien[t]));
            if (t % 2 == 0) continue;
            if (footprint[t - 1] && !rd1gap) output1read(t - 1, orien[t] == '+' ? '-' : '+', 1);
            if (footprint[t] && !rd2gap) output1read(t, orien[t - 1] == '+' ? '-' : '+', 2);
        }
        *ms_record += host_now() - t_rec;
        // the deflate runs beside the next batch's GPU work, on the writers' own streams
        writer = std::async(std::launch::async, [&] { f_gap.write(s_gap); if (fill) f_short.write(s_short); f_on.write(s_on); if (fill) f_pe.write(s_pe); });
    }
    join();
    if (n_reads && last_batch != max_read_num) {   // a batch that ends exactly at the last read is recorded inside the reference's loop
        fprintf(stderr, "\nTotal reads         %lld\n", read_counter);
        fprintf(stderr, "Reads in gaps       %lld\n", in_gap);
        fprintf(stderr, "Ratio               %.1f%%\n", (float)in_gap / read_counter * 100);
    }
    fprintf(stderr, "Reads on contigs    %lld\n", map_counter);
    fprintf(stderr, "Ratio               %.1f%%\n", (float)map_counter / read_counter * 100);
    f_on.close();
    {
        FILE* fo = ckopen(prefix + ".peGrads", "w");
        fprintf(fo, "grads&num: %d\t%lld\t%d\n", (int)grads.size(), (long long)n_reads, plan.max_len4all);
        if (!grads.empty()) fprintf(stderr, "%d pe insert size, the largest boundary is %lld.\n\n", (int)grads.size(), grads.back().bound);
        else fprintf(stderr, "No paired reads found.\n");
        for (const Grad& g : grads) fprintf(fo, "%d\t%lld\t%d\t%d\n", g.ins, g.bound, g.rank, g.cut);
        fclose(fo);
    }
    f_gap.close(); f_short.close(); f_pe.close();
}

int map_stage(int argc, char** argv, int flavour127) {
    const double t_all = host_now();
    fprintf(stderr, "\n********************\nMap\n********************\n\n");
    std::string cfg, prefix;
    int inp = 0, outp = 0, c, P = 8, small_k = 0, fill = 0;
    optind = 1;
    fprintf(stderr, "Parameters: map ");
    while ((c = getopt(argc, argv, "s:g:K:p:k:h:f")) != EOF) {
        switch (c) {
            case 's': fprintf(stderr, "-s %s ", optarg); inp = 1; cfg = optarg; break;
            case 'g': fprintf(stderr, "-g %s ", optarg); outp = 1; prefix = optarg; break;
            case 'K': fprintf(stderr, "-K %s ", optarg); break;   // parsed, then replaced by the K of .preGraphBasic (map.c:104)
            case 'p': fprintf(stderr, "-p %s ", optarg); P = atoi(optarg); break;
            case 'k': fprintf(stderr, "-k %s ", optarg); small_k = atoi(optarg); break;
            case 'h': fprintf(stderr, "-h %s ", optarg); break;   // sizes the reference's initial hash only
            case 'f': fill = 1; fprintf(stderr, "-f "); break;
            default:
                if (!inp || !outp) { map_usage(flavour127); exit(1); }
        }
    }
    fprintf(stderr, "\n\n");
    if (!inp || !outp) { map_usage(flavour127); exit(1); }
    int K = min_overlap(prefix);
    const int kmax = flavour127 ? 127 : 63;
    if (small_k > 12 && small_k <= kmax && small_k % 2 == 1) K = small_k;
    fprintf(stderr, "Kmer size: %d.\n", K);
    if (K < 13 || K > kmax || K % 2 == 0) fail("pgb200: K %d is outside 13..%d or even", K, kmax);
    if (P < 1) fail("pgb200: -p must be at least 1");
    fprintf(stderr, "Contig length cutoff: %d.\n", K + 2);
    const StageSettings env = stage_settings();

    // ---- prlContig2nodes
    double t0 = host_now();
    const Contigs ctg = read_contigs(prefix, K);
    const double ms_parse = host_now() - t0;
    fprintf(stderr, "Time spent on parsing contigs file: %ds.\n", (int)(ms_parse * 1e-3));
    fprintf(stderr, "%d thread(s) initialized.\n", P);
    // the plan is read before the engine so that a refused library stops the stage before any output
    const MapPlan plan = map_plan(cfg.c_str());
    if (plan.max_rd_len - K + 1 <= 0) fail("pgb200: max_rd_len %d is shorter than K %d", plan.max_rd_len, K);
    const bool long_pass = plan.long_len >= 1;   // prlRead2Ctg.c:1099-1104
    std::unique_ptr<IMapEngine> eng(in_step("pgb200: %s", [&] { return make_map_engine(K, env.device); }));
    const double t_hash = host_now();
    u64 distinct = 0;
    in_step("pgb200: contig hash failed: %s", [&] { eng->hash_contigs(ctg.packed.data(), ctg.off.back(), ctg.off.data(), ctg.id.data(), ctg.id.size(), &distinct); });
    fprintf(stderr, "Time spent on hashing contigs: %ds.\n", (int)((host_now() - t_hash) * 1e-3));
    fprintf(stderr, "%lli node(s) allocated, %lli kmer(s) in contigs, %lli kmer(s) processed.\n", (long long)distinct, (long long)ctg.n_kmers, (long long)ctg.n_kmers);
    fprintf(stderr, "Time spent on graph construction: %ds.\n\n", (int)((host_now() - t0) * 1e-3));

    // ---- the reads of both passes, before any output file
    t0 = host_now();
    std::string long_log, short_log;
    // The long pass reads with the fgets reader: long reads are commonly wrapped.  PGB200_MAP_READER=fgets sends the short pass
    // through it as well, a second exact implementation of the reads the parity tests can run over every short-read scenario.  gStr:
    // the long pass allocates it for longReadLen > gLineLen (prlRead2Ctg.c:1133), the short pass for max_rd_len > gLineLen (:826).
    const char* reader_env = getenv("PGB200_MAP_READER");
    const bool fgets_short = reader_env && !strcmp(reader_env, "fgets");
    FileReader files{*eng, env.chunk_bytes};
    const Reads lrd = long_pass ? load_reads(files, plan.long_libs, true, plan.long_len, plan.long_len > 5000 ? 1 : 0, &long_log) : Reads{};
    MapTimes t_lrd;
    eng->times(&t_lrd);
    const double ms_read_long = host_now() - t0;
    const Reads rd = load_reads(files, plan.libs, false, plan.max_rd_len, fgets_short ? (plan.max_rd_len > 5000 ? 1 : 0) : -1, &short_log);
    const double ms_read = host_now() - t0;
    const long long max_read_num = batch_reads("max_rd_len", plan.max_rd_len, K);
    const long long max_long_num = long_pass ? batch_reads("long read length", plan.long_len, K) : 0;
    const char* long_env = getenv("PGB200_MAP_LONG");
    const bool long_all = long_env && !strcmp(long_env, "all");   // the short pass through k_map_long too: a second exact implementation

    // ---- prlLongRead2Ctg
    ContigInfo ci;
    t0 = host_now();
    if (long_pass) {
        fprintf(stderr, "In file: %s, long read len %d, max name len %d.\n", cfg.c_str(), plan.long_len, 256);
        fprintf(stderr, "%d thread(s) initialized.\n", P);
        ci = contig_info(prefix);   // basicContigInfo runs once: here, not in the short pass
        fprintf(stderr, "%d edge(s) in the graph.\n", ci.num_all);
        fputs(long_log.c_str(), stderr);
        map_long_reads(*eng, plan, lrd, max_long_num, ci, K, P, fill, prefix);
        print_libs(plan);
        fprintf(stderr, "0 reads deleted.\n");
        if (env.verbose) {
            MapTimes tm;
            eng->times(&tm);
            fprintf(stderr, "[pgb200] map long pass: %zu reads, %.0f ms (host), long-read scan %.1f ms (GPU events), %llu lookups; reading %.0f ms (host), "
                            "reader %.1f ms (GPU events)\n",
                    lrd.lens.size(), host_now() - t0, tm.ms_long, (unsigned long long)tm.lookups_long, ms_read_long, t_lrd.ms_decode);
        }
    }
    fprintf(stderr, "Time spent on aligning long reads: %ds.\n\n", (int)((host_now() - t0) * 1e-3));

    // ---- prlRead2Ctg
    t0 = host_now();
    fprintf(stderr, "In file: %s, max seq len %d, max name len %d\n", cfg.c_str(), plan.max_rd_len, 256);
    fprintf(stderr, "%d thread(s) initialized.\n", P);
    if (!long_pass) {
        ci = contig_info(prefix);
        fprintf(stderr, "%d edge(s) in the graph.\n", ci.num_all);
    }
    double ms_record = 0, ms_deflate = 0;
    map_short_reads(*eng, plan, rd, short_log, max_read_num, ci, K, P, fill, long_all, prefix, env.device, &ms_record, &ms_deflate);
    print_libs(plan);
    fprintf(stderr, "Time spent on aligning reads: %ds.\n\n", (int)((host_now() - t0) * 1e-3));
    if (env.verbose) {
        MapTimes tm;
        eng->times(&tm);
        fprintf(stderr, "[pgb200] map: parse .contig %.0f ms (host), contig hash %.1f ms, read decode %.1f ms, read scan %.1f ms (GPU events); reading %.0f ms, "
                        "record pass %.0f ms, waiting for the deflate %.0f ms (host)\n",
                ms_parse, tm.ms_hash, tm.ms_decode, long_all ? tm.ms_long : tm.ms_scan, ms_read, ms_record, ms_deflate);
    }
    eng.reset();
    fprintf(stderr, "Overall time spent on alignment: %dm.\n\n", (int)((host_now() - t_all) * 1e-3) / 60);
    return 0;
}

}   // namespace
}   // namespace pgb

extern "C" int pgb200_map_main(int argc, char** argv, int flavour127) {
    try { return pgb::map_stage(argc, argv, flavour127); } catch (const std::exception& ex) { fprintf(stderr, "%s\n", ex.what()); exit(-1); }
}
