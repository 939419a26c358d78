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
    // the contig k-mer table: bases packed 2 bits each (LSB first) into one stream, contig c = bases [ctg_off[c], ctg_off[c+1])
    virtual void hash_contigs(const u64* packed, u64 n_bases, const u64* ctg_off, const u32* ctg_id, u64 n_ctg,
                              u64* distinct) = 0;
    // Reads come back, and go into map_batch, packed 2 bits per base (LSB first) at their own lengths: ceil(len / 32) words each, one
    // after another.
    // one chunk of whole FASTA/FASTQ records (pass 1's reader: single-line FASTA, 4-line FASTQ), each cut to maxlen bases -> its reads
    // appended to *words and *lens
    virtual void decode_text(const char* text, size_t nbytes, int fastq, int reverse, int maxlen, std::vector<u64>* words, std::vector<u32>* lens) = 0;
    // one chunk of a FASTA/FASTQ file read as the reference's map stage reads it (readseq1by1 / read1seqfq: fgets pieces of piece_len
    // bytes, wrapped records, the raw-length cut at `cutoff`; reader.cu) -> its reads appended to *words and *lens.  at_eof: the chunk
    // ends the file.  Returns the byte offset where the chunk's unfinished record starts (nbytes at the end of the file): the caller
    // prepends text[result, nbytes) to its next chunk.
    virtual size_t read_text(const char* text, size_t nbytes, int fastq, int piece_len, int cutoff, int reverse, bool at_eof, std::vector<u64>* words,
                             std::vector<u32>* lens) = 0;
    // one batch of reads, read r at words[wofs[r] ...) within words[0, n_words) (parse1read reads ALIGNLEN once per batch: alignlen
    // is its value after the batch's last read).  per_read_cta: one CTA per read (k_map_long, for long reads), else one thread per
    // read (k_map_reads); their GPU times are kept apart, as ms_long and ms_scan.
    virtual void map_batch(const u64* words, u64 n_words, const u64* wofs, const u32* lens, u64 n, int alignlen, bool per_read_cta, MapHit* out) = 0;
    virtual void times(MapTimes* t) const = 0;
};
IMapEngine* make_map_engine(int K, int device);   // 128-bit keys for K <= 63, else 256-bit

}   // namespace pgb
#pragma GCC visibility pop
