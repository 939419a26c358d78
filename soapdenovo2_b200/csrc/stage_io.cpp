// stage_io.cpp -- the stages' host-only work: settings, config, read-stream plan, chunked reads, output files, edge-sidecar codec.
// Mirrors, in new code, the host-side behaviour of (standardPregraph/):
//   scan_libInfo / splitColumn     lib.c:70-506        (key=value config, [LIB] sections, sort by avg_ins)
//   openNextFile / nextValidIndex  prlHashReads.c:903-951, readseq1by1.c:595-674 (library + file-type iteration order)
//   file writers                   prlHashReads.c:1104-1132 (.kmerFreq), node2edge.c:61-70 (.edge.gz via zlib)
//   map's .contig reader           prlHashCtg.c:297-425, readseq1by1.c:50-136, 225-277 (getID, prlContig2nodes, readseq1by1, readseqpar)
#include "stage.h"
#include "deflate.h"
#include <algorithm>
#include <cctype>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
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

StageSettings stage_settings() {
    StageSettings s;
    if (const char* v = getenv("PGB200_DEVICE")) s.device = atoi(v);
    if (const char* v = getenv("PGB200_VERBOSE")) s.verbose = atoi(v);
    if (const char* v = getenv("PGB200_CHUNK_MB")) {
        char* end;
        const long mb = strtol(v, &end, 10);
        if (end == v || *end || mb < 1 || mb > 4095) fail("pgb200: PGB200_CHUNK_MB must be a whole number of MB from 1 to 4095, not \"%s\"", v);
        s.chunk_bytes = (size_t)mb << 20;
    }
    return s;
}

FILE* ckopen(const std::string& name, const char* mode) {
    FILE* fp = fopen(name.c_str(), mode);
    if (!fp) fail("Cannot open %s. Now exit to system...", name.c_str());
    return fp;
}
std::string read_whole_file(FILE* f) {
    std::string s;
    char buf[1 << 16];
    size_t got;
    while ((got = fread(buf, 1, sizeof buf, f)) > 0) s.append(buf, got);
    return s;
}

void read_chunks(const std::string& path, char* buf, size_t cap, const ChunkTake& take) {
    std::unique_ptr<FILE, int (*)(FILE*)> f(ckopen(path, "rb"), fclose);
    size_t have = 0;
    for (;;) {
        have += fread(buf + have, 1, cap - have, f.get());
        if (ferror(f.get())) fail("pgb200: read error on %s", path.c_str());   // on Linux also a directory, which fopen accepts
        if (have == 0) return;   // the fread found the end, and nothing was carried
        const bool at_eof = feof(f.get()) != 0;
        const size_t used = take(buf, have, at_eof);
        if (at_eof) return;
        if (used == 0 && have == cap) fail("pgb200: a single record exceeds the %zu MB chunk", cap >> 20);
        memmove(buf, buf + used, have - used);
        have -= used;
    }
}
size_t whole_records(const char* text, size_t n, bool fastq, bool at_eof) {
    if (!at_eof) return last_record_start(text, n, fastq);
    while (n > 1 && text[n - 1] == '\n' && text[n - 2] == '\n') n--;   // trailing blank lines are harmless
    return n == 1 && text[0] == '\n' ? 0 : n;
}

namespace {
// fgets(str, size, fp) over a file's text: each piece is at most size - 1 bytes and ends after the first '\n'.  eof is feof after
// the call: a piece that ran into the end of the text before its '\n' or its size limit sets it, as does a call at the end.
struct Fgets {
    const std::string& t;
    size_t at = 0;
    bool eof = false;
    bool next(size_t size, const char** s, size_t* n) {
        if (at == t.size()) { eof = true; return false; }
        const size_t lim = std::min(t.size(), at + size - 1);
        const char* nl = (const char*)memchr(t.data() + at, '\n', lim - at);
        const size_t end = nl ? (size_t)(nl - t.data()) + 1 : lim;
        eof = !nl && end - at < size - 1;
        *s = t.data() + at;
        *n = strnlen(*s, end - at);   // strlen(str): the piece up to a NUL byte
        at = end;
        return true;
    }
};
// sscanf(&str[1], "%s", name) on a '>' piece: leading whitespace skipped; a piece with no token leaves name as it was
void scan_name(const char* s, size_t n, std::string* name) {
    size_t i = 1;
    while (i < n && isspace((unsigned char)s[i])) i++;
    size_t j = i;
    while (j < n && !isspace((unsigned char)s[j])) j++;
    if (j > i) name->assign(s + i, j - i);
}
}   // namespace

Contigs read_contigs(const std::string& prefix, int K) {
    FILE* fp = ckopen(prefix + ".contig", "r");
    const std::string text = read_whole_file(fp);
    fclose(fp);
    const char* s;
    size_t n;
    std::string name;
    // readseqpar (readseq1by1.c:225-277): pieces of fgets(str, 4950); each piece but a '>' one adds strlen - 1 to the record's length
    long long num = -1;
    int max_len = 10, min_len = 1000, name_len = 10, len = 0;
    for (Fgets f{text}; f.next(4950, &s, &n);) {
        if (s[0] != '>') { len += (int)n - 1; continue; }
        if (num >= 0) { max_len = std::max(max_len, len); min_len = std::min(min_len, len); }
        len = 0;
        num++;
        scan_name(s, n, &name);
        name_len = std::max(name_len, (int)name.size());
    }
    max_len = std::max(max_len, len); min_len = std::min(min_len, len);
    fprintf(stderr, "\n%lld contig(s), maximum sequence length %d, minimum sequence length %d, maximum name length %d.\n", num + 1, max_len, min_len, name_len);
    // prlContig2nodes' loop (prlHashCtg.c:393-425) over readseq1by1 (readseq1by1.c:50-136) with gStr NULL: pieces of
    // fgets(str, gLineLen = 5000), '#' pieces skipped, each record cut where strlen + bases > maxReadLen = max_len
    Fgets f{text};
    std::vector<unsigned char> codes;
    auto record = [&] {   // one record's bases, up to the next '>' piece (whose name is the next record's) or the end
        codes.clear();
        while (f.next(5000, &s, &n)) {
            if (s[0] == '#') continue;
            if (s[0] == '>') { scan_name(s, n, &name); return; }
            const size_t room = (size_t)max_len - codes.size(), m = std::min(n, room);
            for (size_t i = 0; i < m; i++) {
                const unsigned ch = (unsigned char)s[i];
                if ((ch >= 'a' && ch <= 'z') || (ch >= 'A' && ch <= 'Z')) codes.push_back((unsigned char)((ch & 6u) >> 1));   // base2int
                else if (ch == '.') codes.push_back(0);
            }
        }
    };
    Contigs c;
    name.clear();   // next_name starts empty (ckalloc is calloc)
    record();       // the bytes before the first '>' are read and dropped
    unsigned long long n_bases = 0;
    for (unsigned ordinal = 1; !f.eof; ordinal++) {
        const unsigned cid = name[0] >= '0' && name[0] <= '9' ? (unsigned)atoi(name.c_str()) : 0u;   // getID, prlHashCtg.c:297-307
        record();
        const int clen = (int)codes.size();
        if (clen < K + 1 || clen < K + 2) continue;   // len_cut = ctg_short = K + 2
        c.id.push_back(cid > 0 ? cid : ordinal);
        for (unsigned char b : codes) {
            if ((n_bases & 31) == 0) c.packed.push_back(0);
            c.packed.back() |= (unsigned long long)b << (2 * (n_bases & 31));
            n_bases++;
        }
        c.off.push_back(n_bases);
        c.n_kmers += (unsigned long long)(clen - K + 1);
    }
    return c;
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
    FILE* fp = ckopen(cfg, "r");
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
    FILE* f = ckopen(name, "wb");
    if (n && fwrite(data, 1, n, f) != n) { fclose(f); fail("short write on %s", name.c_str()); }
    fclose(f);
}
void write_kmer_freq(const std::string& prefix, const long long hist[256]) {   // freqStat, prlHashReads.c:1104-1132
    std::string s;
    char b[32];
    for (int i = 1; i < 256; i++) { snprintf(b, sizeof b, "%lld\n", hist[i]); s += b; }
    write_file(prefix + ".kmerFreq", s.data(), s.size());
}
// gzopen(name,"w") + gzwrite: the reference's gzprintf calls write the same byte stream.  The deflate runs on the GPU (deflate.cu;
// PGB200_GZ=host: zlib), with the same bytes.
static void write_edge_gz(const std::string& name, const std::string& text, int device) {
    std::unique_ptr<GzFile> gz(gz_open(name, device));
    gz->write(text.data(), text.size(), false);
    gz->close();
}
// PGB200_EDGE_SIDECAR unset: <prefix>.edge.gz only (the reference's output).  Set: the sidecar first (a fraction of a second, so a
// contig that links contig_sidecar.c never waits for the deflate), then the .edge.gz.  "only": the sidecar alone -- the deflate of
// the edge text is sequential host work (its bytes must equal the reference's gz stream) and is the longest single item of a
// full-size stage run, so a pipeline whose contig reads the sidecar can leave it out.
void write_edge_outputs(const std::string& prefix, const std::string& text, const PgParams& p, uint64_t num_ed) {
    const char* sc = getenv("PGB200_EDGE_SIDECAR");
    if (sc) edge_text_to_sidecar(text.data(), text.size(), p.K, p.flavour127, num_ed, prefix + ".edge.b200");
    if (!(sc && !strcmp(sc, "only"))) write_edge_gz(prefix + ".edge.gz", text, p.device);
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
    const std::string raw = read_whole_file(f);
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
    char buf[512];
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
    write_edge_gz(prefix + ".edge.gz", text, stage_settings().device);
}
}   // namespace pgb
