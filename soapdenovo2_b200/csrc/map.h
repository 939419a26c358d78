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

class IMapEngine {
public:
    virtual ~IMapEngine() {}
    virtual int words_per_read() const = 0;   // W64: 2-bit packed words per read (LSB first), from max_rd_len
    // the contig k-mer table: bases packed 2 bits each (LSB first) into one stream, contig c = bases [ctg_off[c], ctg_off[c+1])
    virtual void hash_contigs(const u64* packed, u64 n_bases, const u64* ctg_off, const u32* ctg_id, u64 n_ctg,
                              u64* distinct) = 0;
    // one chunk of whole FASTA/FASTQ records -> its reads appended to *words (W64 per read) and *lens
    virtual void decode_text(const char* text, size_t nbytes, int fastq, int reverse, int maxlen, std::vector<u64>* words,
                             std::vector<u32>* lens) = 0;
    // one batch of reads (parse1read reads ALIGNLEN once per batch: alignlen is its value after the batch's last read)
    virtual void map_batch(const u64* words, const u32* lens, u64 n, int alignlen, MapHit* out) = 0;
    // CUDA-event milliseconds so far: contig hash, read decode, read scan
    virtual void times(double* ms_hash, double* ms_decode, double* ms_scan) const = 0;
};
IMapEngine* make_map_engine(int K, int device, int max_rd_len);   // 128-bit keys for K <= 63, else 256-bit

}   // namespace pgb
#pragma GCC visibility pop
