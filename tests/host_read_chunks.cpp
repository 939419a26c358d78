// host_read_chunks.cpp -- runs the stages' chunked reader (read_chunks, soapdenovo2_b200/csrc/stage_io.cpp) over one file with pass
// 1's record rule (whole_records) and a chunk of `cap` bytes, as the pregraph feed and map's default short-pass reader do.  Prints one
// line per call, "call <n> <at_eof> <taken>", and writes the bytes taken, in order, to <out>.  A failure prints its message; exit 1.
//   host_read_chunks <path> fasta|fastq <cap> <out>
#include "../soapdenovo2_b200/csrc/stage.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>

int main(int argc, char** argv) {
    if (argc != 5) { fprintf(stderr, "usage: %s path fasta|fastq cap out\n", argv[0]); return 2; }
    const bool fastq = strcmp(argv[2], "fastq") == 0;
    const size_t cap = strtoull(argv[3], nullptr, 10);
    std::unique_ptr<char[]> buf(new char[cap]);
    std::unique_ptr<FILE, int (*)(FILE*)> out(fopen(argv[4], "wb"), fclose);
    try {
        pgb::read_chunks(argv[1], buf.get(), cap, [&](const char* text, size_t n, bool at_eof) {
            const size_t cut = pgb::whole_records(text, n, fastq, at_eof);
            printf("call %zu %d %zu\n", n, at_eof ? 1 : 0, cut);
            fwrite(text, 1, cut, out.get());
            return cut;
        });
    } catch (const std::exception& ex) {
        fprintf(stderr, "%s\n", ex.what());
        return 1;
    }
    return 0;
}
