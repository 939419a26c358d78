// host_read_contigs.cpp -- runs the map stage's .contig reader (read_contigs, soapdenovo2_b200/csrc/stage_io.cpp) on <prefix>.contig
// with K.  The reader prints its stats line to stderr; this prints "kmers <n>" and then one line per kept contig, "<id> <length>
// <hash>", the hash being the 64-bit FNV-1a of its base codes (one byte each, 0..3).  A failure prints its message; exit 1.
//   host_read_contigs <prefix> <K>
#include "../soapdenovo2_b200/csrc/stage.h"
#include <cstdio>
#include <cstdlib>
#include <stdexcept>

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s prefix K\n", argv[0]); return 2; }
    try {
        const pgb::Contigs c = pgb::read_contigs(argv[1], atoi(argv[2]));
        printf("kmers %llu\n", c.n_kmers);
        for (size_t r = 0; r < c.id.size(); r++) {
            unsigned long long h = 1469598103934665603ull;
            for (unsigned long long i = c.off[r]; i < c.off[r + 1]; i++) {
                h ^= (c.packed[i >> 5] >> (2 * (i & 31))) & 3;
                h *= 1099511628211ull;
            }
            printf("%u %llu %llu\n", c.id[r], c.off[r + 1] - c.off[r], h);
        }
    } catch (const std::exception& ex) {
        fprintf(stderr, "%s\n", ex.what());
        return 1;
    }
    return 0;
}
