// map.h -- what the map stage's host side (map_stage.cpp) and its GPU side (map.cu) share.  Internal to csrc/, like stage.h.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#pragma GCC visibility push(hidden)
namespace pgb {

typedef unsigned long long u64;   // as in kmer.cuh
typedef unsigned int u32;
typedef unsigned char u8;

enum : u32 { MAP_PLACED = 1, MAP_MINUS = 2, MAP_FOOTPRINT = 4 };
// One read's placement as parse1read (prlRead2Ctg.c:260-361) leaves it, before the contig lengths are applied: the winning group's
// contig id, the position its first hit has on that contig, i = (that hit's index in the read) + 1, and MAP_* flags.  MAP_MINUS:
// the hit's twin equals the read k-mer's isSmaller, i.e. the read lies on the reverse strand.
struct MapHit {
    u32 ctg;
    int32_t node_pos;
    int32_t i;
    u32 flags;
};

// CUDA-event milliseconds so far, and the long scan's k-mer lookups
struct MapTimes {
    double ms_hash, ms_decode, ms_scan, ms_long;
    u64 lookups_long;
};

class IMapEngine {
public:
    virtual ~IMapEngine() {}
    virtual int words_per_read() const = 0;   // W64: 2-bit packed words per read (LSB first), from max_rd_len
    // the contig k-mer table: bases packed 2 bits each (LSB first) into one stream, contig c = bases [ctg_off[c], ctg_off[c+1])
    virtual void hash_contigs(const u64* packed, u64 n_bases, const u64* ctg_off, const u32* ctg_id, u64 n_ctg,
                              u64* distinct) = 0;
    // one chunk of whole FASTA/FASTQ records, each cut to maxlen bases -> its reads appended to *words and *lens: `stride` words per
    // read (>= (maxlen + 31) / 32), or with stride 0 each read packed at its own length, ceil(len / 32) words, one after another
    virtual void decode_text(const char* text, size_t nbytes, int fastq, int reverse, int maxlen, int stride, std::vector<u64>* words,
                             std::vector<u32>* lens) = 0;
    // one batch of reads (parse1read reads ALIGNLEN once per batch: alignlen is its value after the batch's last read)
    virtual void map_batch(const u64* words, const u32* lens, u64 n, int alignlen, MapHit* out) = 0;
    // the same for reads located by word offsets into words[0, n_words) -- long reads, one CTA per read (k_map_long)
    virtual void map_long_batch(const u64* words, u64 n_words, const u64* wofs, const u32* lens, u64 n, int alignlen, MapHit* out) = 0;
    virtual void times(MapTimes* t) const = 0;
};
IMapEngine* make_map_engine(int K, int device, int max_rd_len);   // 128-bit keys for K <= 63, else 256-bit

}   // namespace pgb
#pragma GCC visibility pop
