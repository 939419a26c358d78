// stage_io.cpp -- the stage's host-only work: config, read-stream plan, chunk cutter, output files, edge-sidecar codec.  Mirrors, in
// new code, the host-side behaviour of (standardPregraph/):
//   scan_libInfo / splitColumn     lib.c:70-506        (key=value config, [LIB] sections, sort by avg_ins)
//   openNextFile / nextValidIndex  prlHashReads.c:903-951, readseq1by1.c:595-674 (library + file-type iteration order)
//   file writers                   prlHashReads.c:1104-1132 (.kmerFreq), node2edge.c:61-70 (.edge.gz via zlib)
#include "stage.h"
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <zlib.h>

namespace pgb {
void fail(const char* fmt, ...) {
    va_list ap, ap2;
    va_start(ap, fmt); va_copy(ap2, ap);
    std::string s((size_t)vsnprintf(nullptr, 0, fmt, ap), '\0');
    vsnprintf(&s[0], s.size() + 1, fmt, ap2);   // writes s's own terminator too
    va_end(ap); va_end(ap2);
    throw std::runtime_error(s);
}

namespace {   // the library config (lib.c)
struct Lib {
    int avg_ins = 0, asm_flag = 3, reverse = 0, rd_len_cutoff = 0, map_len = 0, rank = 0, pair_num_cut = 0;
    std::vector<std::string> f[7];   // [1]=f1 [0]=f2 [2]=q1 [4]=q2 [3]=p [5]=f [6]=q
};
}   // namespace
static bool split_column(const char* line, std::string& a, std::string& b) {   // splitColumn lib.c:70-108
    int len = (int)strlen(line), i = 0, n = 0;
    std::string* t[2] = {&a, &b};
    a.clear(); b.clear();
    while (i < len) {
        if (line[i] >= 32 && line[i] <= 126 && line[i] != '=') {
            while (i < len && line[i] >= 32 && line[i] <= 126 && line[i] != '=') t[n]->push_back(line[i++]);
            if (++n == 2) return true;
        }
        i++;
    }
    return false;
}
static std::vector<Lib> scan_lib(const char* cfg, int* max_rd_len) {
    FILE* fp = fopen(cfg, "r");
    if (!fp) fail("Cannot open %s. Now exit to system...", cfg);
    std::vector<Lib> libs;
    char line[1024];
    std::string a, b;
    bool bam = false;
    *max_rd_len = 0;
    while (!bam && fgets(line, sizeof line, fp)) {
        if (strncmp(line, "[LIB]", 5) == 0) { libs.emplace_back(); continue; }
        if (!split_column(line, a, b)) continue;
        if (libs.empty()) { if (a == "max_rd_len") *max_rd_len = atoi(b.c_str()); continue; }   // only before the first [LIB] (lib.c:152-165)
        Lib& L = libs.back();
        if (a == "f1") L.f[1].push_back(b); else if (a == "f2") L.f[0].push_back(b);
        else if (a == "q1") L.f[2].push_back(b); else if (a == "q2") L.f[4].push_back(b);
        else if (a == "p") L.f[3].push_back(b); else if (a == "f") L.f[5].push_back(b); else if (a == "q") L.f[6].push_back(b);
        else if (a == "b") bam = true;
        else if (a == "avg_ins") L.avg_ins = atoi(b.c_str()); else if (a == "reverse_seq") L.reverse = atoi(b.c_str());
        else if (a == "asm_flags") L.asm_flag = atoi(b.c_str()); else if (a == "rd_len_cutoff") L.rd_len_cutoff = atoi(b.c_str());
        else if (a == "map_len") L.map_len = atoi(b.c_str()); else if (a == "rank") L.rank = atoi(b.c_str());
        else if (a == "pair_num_cutoff") L.pair_num_cut = atoi(b.c_str());
    }
    fclose(fp);
    if (bam) fail("pgb200: BAM input (b=) is not supported by the GPU engine");
    if (libs.empty()) fail("Config file error: no [LIB] in file");
    for (size_t i = 0; i < libs.size(); i++) {
        if (libs[i].f[1].size() != libs[i].f[0].size()) fail("Config file error: the number of mark \"f1\" is not the same as \"f2\"!");
        if (libs[i].f[2].size() != libs[i].f[4].size()) fail("Config file error: the number of mark \"q1\" is not the same as \"q2\"!");
        bool pe = !libs[i].f[1].empty() || !libs[i].f[2].empty() || !libs[i].f[3].empty();
        if (pe && libs[i].avg_ins == 0) fail("Config file error: PE reads need avg_ins in [LIB] %zu", i + 1);
    }
    std::stable_sort(libs.begin(), libs.end(), [](const Lib& x, const Lib& y) { return x.avg_ins < y.avg_ins; });   // qsort by avg_ins, lib.c:505
    if (!*max_rd_len) *max_rd_len = 100;   // prlHashReads.c:326-329
    return libs;
}

// Libraries sorted by avg_ins, only asm_flags 1|3; inside a library f1/f2 pairs, q1/q2 pairs, p, (b: unsupported), f, q.
ReadPlan read_plan(const char* cfg) {
    ReadPlan plan;
    const std::vector<Lib> libs = scan_lib(cfg, &plan.max_rd_len);
    plan.n_libs = (int)libs.size();
    for (const Lib& L : libs) {
        if (L.asm_flag != 1 && L.asm_flag != 3) continue;                           // nextValidIndex, readseq1by1.c:601
        int cut = (L.rd_len_cutoff > 0 && L.rd_len_cutoff < plan.max_rd_len) ? L.rd_len_cutoff : plan.max_rd_len;   // prlHashReads.c:921-928
        for (int type = 1; type <= 6; type++) {
            if (type == 4) continue;
            bool fq = (type == 2 || type == 6);
            for (size_t fi = 0; fi < L.f[type].size(); fi++) {
                if (type <= 2) {
                    plan.files.push_back({L.f[type][fi], fq, 0, L.reverse, cut});
                    plan.files.push_back({L.f[type == 1 ? 0 : 4][fi], fq, 1, L.reverse, cut});
                } else plan.files.push_back({L.f[type][fi], fq, -1, L.reverse, cut});
            }
        }
    }
    return plan;
}

// The map stage reads twice.  The long pass (prlLongRead2Ctg) reads with pair = 0 and asm_ctg = 4: the asm_flags=4 libraries, and
// inside each the p, f and q files (two-file pairs are refused: read unpaired they would be mates taken as single reads).  The short
// pass reads with pair = 1 and asm_ctg = 0 (prlRead2Ctg.c:887, readseq1by1.c:595-674): libraries with asm_flags 2|3, and inside each
// only the f1/f2 pairs, q1/q2 pairs and p files.  Every library is kept for the "LIB(s) information" lines.  Each read is cut to
// min(rd_len_cutoff, maxReadLen4all), or maxReadLen4all without a cutoff (readseq1by1.c:1083-1090); maxReadLen4all is max_rd_len
// raised to longReadLen by the long pass (prlRead2Ctg.c:1106).
MapPlan map_plan(const char* cfg) {
    MapPlan plan;
    const std::vector<Lib> libs = scan_lib(cfg, &plan.max_rd_len);
    bool has_long = false;
    for (const Lib& L : libs) {   // getMaxLongReadLen, lib.c:43-68
        if (L.asm_flag != 4) continue;
        has_long = true;
        plan.long_len = std::max(plan.long_len, L.rd_len_cutoff);
        if (!L.f[1].empty() || !L.f[2].empty())
            fail("pgb200: long-read libraries (asm_flags=4) are not supported with two-file pairs (f1/f2, q1/q2); list long reads as f=, q= or p=");
    }
    if (has_long && plan.long_len <= 0) plan.long_len = plan.max_rd_len;
    plan.max_len4all = std::max(plan.max_rd_len, plan.long_len);
    for (const Lib& L : libs) {
        MapLib m{L.avg_ins, L.reverse, L.map_len, L.rank, L.pair_num_cut, {}};
        const int cut = L.rd_len_cutoff > 0 ? std::min(L.rd_len_cutoff, plan.max_len4all) : plan.max_len4all;   // readseq1by1.c:1083-1090
        if (L.asm_flag == 4) {
            for (int type : {3, 5, 6})
                for (const std::string& path : L.f[type]) m.files.push_back({path, type == 6, -1, L.reverse, cut});
            plan.long_libs.push_back(m);
            m.files.clear();
        }
        if (L.asm_flag == 2 || L.asm_flag == 3)
            for (int type = 1; type <= 3; type++)
                for (size_t fi = 0; fi < L.f[type].size(); fi++) {
                    const bool fq = type == 2;
                    if (type <= 2) {
                        m.files.push_back({L.f[type][fi], fq, 0, L.reverse, cut});
                        m.files.push_back({L.f[type == 1 ? 0 : 4][fi], fq, 1, L.reverse, cut});
                    } else m.files.push_back({L.f[type][fi], fq, -1, L.reverse, cut});
                }
        plan.libs.push_back(std::move(m));
    }
    return plan;
}

// Chunks are cut at record boundaries on the host (only the tail of each chunk is inspected); the GPU does the parsing.
size_t last_record_start(const char* buf, size_t n, bool fastq) {
    // returns the offset of the last position that starts a record, such that buf[0..off) holds whole records
    if (n == 0) return 0;
    size_t p = n;
    for (;;) {
        if (p == 0) return 0;
        size_t q = p - 1;
        while (q > 0 && buf[q - 1] != '\n') q--;
        if (!fastq) { if (buf[q] == '>') return q; }
        else if (buf[q] == '@') {
            // a FASTQ header is followed two lines later by a '+' line; a quality line starting with '@' is followed
            // two lines later by a sequence line, which never starts with '+'
            const char* e1 = (const char*)memchr(buf + q, '\n', n - q);
            if (e1) {
                const char* e2 = (const char*)memchr(e1 + 1, '\n', n - (e1 + 1 - buf));
                if (e2 && (size_t)(e2 + 1 - buf) < n && e2[1] == '+') return q;
            }
        }
        p = q;
    }
}

void write_file(const std::string& name, const void* data, size_t n) {
    FILE* f = fopen(name.c_str(), "wb");
    if (!f) fail("Cannot open %s. Now exit to system...", name.c_str());   // ckopen, check.c:30-34
    if (n && fwrite(data, 1, n, f) != n) { fclose(f); fail("short write on %s", name.c_str()); }
    fclose(f);
}
void write_kmer_freq(const std::string& prefix, const long long hist[256]) {   // freqStat, prlHashReads.c:1104-1132
    std::string s;
    char b[32];
    for (int i = 1; i < 256; i++) { snprintf(b, sizeof b, "%lld\n", hist[i]); s += b; }
    write_file(prefix + ".kmerFreq", s.data(), s.size());
}
// gzopen(name,"w") + gzwrite: same zlib, same default level => the same byte stream as the reference's gzprintf calls
static void write_edge_gz(const std::string& name, const std::string& text) {
    gzFile gz = gzopen(name.c_str(), "w");
    if (!gz) fail("Cannot open %s", name.c_str());
    size_t off = 0;
    while (off < text.size()) {
        size_t n = std::min<size_t>(text.size() - off, 1u << 30);
        if (gzwrite(gz, text.data() + off, (unsigned)n) != (int)n) { gzclose(gz); fail("gzwrite failed on %s", name.c_str()); }
        off += n;
    }
    gzclose(gz);
}
// PGB200_EDGE_SIDECAR unset: <prefix>.edge.gz only (the reference's output).  Set: the sidecar first (a fraction of a second, so a
// contig that links contig_sidecar.c never waits for the deflate), then the .edge.gz.  "only": the sidecar alone -- the deflate of
// the edge text is sequential host work (its bytes must equal the reference's gz stream) and is the longest single item of a
// full-size stage run, so a pipeline whose contig reads the sidecar can leave it out.
void write_edge_outputs(const std::string& prefix, const std::string& text, const PgParams& p, uint64_t num_ed) {
    const char* sc = getenv("PGB200_EDGE_SIDECAR");
    if (sc) edge_text_to_sidecar(text.data(), text.size(), p.K, p.flavour127, num_ed, prefix + ".edge.b200");
    if (!(sc && !strcmp(sc, "only"))) write_edge_gz(prefix + ".edge.gz", text);
}

// f2: the edges as a binary sidecar for a `contig` that links csrc/contig_sidecar.c (format: pgb200_edge_sidecar_header).  Converts
// the edge TEXT the GPU emitted (">length L,<from>,<to>,cvg C, B" + bases, output_pregraph.c:88-110).
static bool parse_hex_words(const char*& p, const char* end, uint64_t* w, int n) {
    for (int i = 0; i < n; i++) {
        uint64_t v = 0;
        int digits = 0;
        while (p < end) {
            char c = *p;
            int d = c >= '0' && c <= '9' ? c - '0' : (c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1);
            if (d < 0) break;
            v = (v << 4) | (uint64_t)d;
            p++; digits++;
        }
        if (!digits) return false;
        w[i] = v;
        if (i + 1 < n) { if (p >= end || *p != ' ') return false; p++; }
    }
    return true;
}
static bool parse_int(const char*& p, const char* end, long long* out) {
    long long v = 0;
    int digits = 0;
    while (p < end && *p >= '0' && *p <= '9') { v = v * 10 + (*p - '0'); p++; digits++; }
    *out = v;
    return digits > 0;
}
static bool expect(const char*& p, const char* end, const char* lit) {
    size_t n = strlen(lit);
    if ((size_t)(end - p) < n || memcmp(p, lit, n) != 0) return false;
    p += n;
    return true;
}
void edge_text_to_sidecar(const char* text, size_t nbytes, int K, int flavour127, uint64_t num_ed, const std::string& path) {
    const int kw = flavour127 ? 4 : 2;
    pgb200_edge_sidecar_header h = {{0}, PGB200_SIDECAR_VERSION, (uint32_t)K, (uint32_t)kw, 0, 0, num_ed, 0};
    memcpy(h.magic, PGB200_SIDECAR_MAGIC, sizeof h.magic);
    std::string out;
    out.reserve(nbytes / 3 + 4096);
    out.append(sizeof h, '\0');   // the header goes in last, once n_records is known
    const char* p = text;
    const char* end = text + nbytes;
    while (p < end) {
        long long length, cvg, bal;
        uint64_t from[4], to[4];
        if (!expect(p, end, ">length ") || !parse_int(p, end, &length) || !expect(p, end, ",") || !parse_hex_words(p, end, from, kw) || !expect(p, end, ",") ||
            !parse_hex_words(p, end, to, kw) || !expect(p, end, ",cvg ") || !parse_int(p, end, &cvg) || !expect(p, end, ", ") || !parse_int(p, end, &bal) ||
            !expect(p, end, "\n"))
            fail("pgb200: edge text does not parse (record %llu)", (unsigned long long)h.n_records);
        int32_t rec[4] = {(int32_t)length, (int32_t)cvg, (int32_t)bal, (int32_t)(length / 4 + 1)};
        out.append(reinterpret_cast<const char*>(rec), sizeof rec);
        out.append(reinterpret_cast<const char*>(from), kw * 8);
        out.append(reinterpret_cast<const char*>(to), kw * 8);
        const size_t seq0 = out.size();
        out.append((size_t)rec[3], '\0');
        long long pos = 0;
        while (pos < length) {
            if (p >= end) fail("pgb200: edge text ends inside a sequence");
            const char c = *p++;
            if (c == '\n') continue;
            const unsigned code = ((unsigned)c & 6u) >> 1;                       // base2int, inc/def.h:39
            out[seq0 + (size_t)(pos >> 2)] |= (char)(code << (6 - 2 * (pos & 3)));   // writeChar2tightString, seq.c:81-107
            pos++;
        }
        if (p < end && *p == '\n') p++;
        h.n_records++;
    }
    memcpy(&out[0], &h, sizeof h);
    write_file(path, out.data(), out.size());
}
// The way back: <prefix>.edge.b200 -> the byte-identical <prefix>.edge.gz (the sidecar holds every field of the text; the record
// layout is output_pregraph.c:88-110: header line, then the bases 100 per line).  A pipeline that ran the stage with
// PGB200_EDGE_SIDECAR=only can produce the .edge.gz later, or beside `contig`, with `pregraph-b200-<flavour> edgegz -g prefix`.
void sidecar_to_edge_gz(const std::string& prefix) {
    const std::string in = prefix + ".edge.b200";
    FILE* f = fopen(in.c_str(), "rb");
    if (!f) fail("pgb200: cannot open %s", in.c_str());
    std::string raw;
    char buf[1 << 16];
    size_t got;
    while ((got = fread(buf, 1, sizeof buf, f)) > 0) raw.append(buf, got);
    fclose(f);
    pgb200_edge_sidecar_header h;
    if (raw.size() < sizeof h) fail("pgb200: %s is truncated", in.c_str());
    memcpy(&h, raw.data(), sizeof h);
    if (memcmp(h.magic, PGB200_SIDECAR_MAGIC, sizeof h.magic) != 0 || h.version != PGB200_SIDECAR_VERSION || (h.kmer_words != 2 && h.kmer_words != 4))
        fail("pgb200: %s is not an edge sidecar", in.c_str());
    const int kw = (int)h.kmer_words;
    std::string text;
    text.reserve(raw.size() * 4 + (1 << 20));
    size_t off = sizeof h;
    for (uint64_t r = 0; r < h.n_records; r++) {
        int32_t rec[4];
        uint64_t km[8];
        if (off + sizeof rec + (size_t)kw * 16 > raw.size()) fail("pgb200: %s is truncated", in.c_str());
        memcpy(rec, raw.data() + off, sizeof rec); off += sizeof rec;
        memcpy(km, raw.data() + off, (size_t)kw * 16); off += (size_t)kw * 16;
        if (rec[0] < 0 || rec[3] != rec[0] / 4 + 1 || off + (size_t)rec[3] > raw.size()) fail("pgb200: %s is corrupt", in.c_str());
        int n = snprintf(buf, sizeof buf, ">length %d,", rec[0]);
        for (int side = 0; side < 2; side++) {
            for (int w = 0; w < kw; w++) n += snprintf(buf + n, sizeof buf - n, w ? " %llx" : "%llx", (unsigned long long)km[side * kw + w]);
            buf[n++] = ',';
        }
        n += snprintf(buf + n, sizeof buf - n, "cvg %d, %d\n", rec[1], rec[2]);
        text.append(buf, (size_t)n);
        const unsigned char* seq = reinterpret_cast<const unsigned char*>(raw.data() + off);
        for (int i = 0; i < rec[0]; i++) {
            text.push_back("ACTG"[(seq[i >> 2] >> (6 - 2 * (i & 3))) & 3]);
            if ((i + 1) % 100 == 0) text.push_back('\n');
        }
        if (rec[0] % 100 != 0) text.push_back('\n');
        off += (size_t)rec[3];
    }
    write_edge_gz(prefix + ".edge.gz", text);
}
}   // namespace pgb
