// reader.cuh -- the map stage's fgets reader (reader.cu): the reference's line-by-line FASTA / FASTQ readers on the GPU.
#pragma once
#include "engine_impl.cuh"
#include <vector>

namespace pgb {

constexpr int FG_NAME_MAX = 256;   // the reference's read_name holds maxNameLen = 256 bytes plus the terminating NUL

// One chunk of one file, read as readseq1by1 (FASTA) / read1seqfq (FASTQ) read it with fgets(str, piece_len + 1, fp): each read cut
// with the raw-length rule at `cutoff`, reverse-complemented when `reverse`.  The reads are appended to *lens and, packed 2 bits per
// base (LSB first) at their own lengths, ceil(len / 32) words each, to *words.  at_eof: the chunk ends the file.  Otherwise only the
// records a later header completes are returned, and the result is the byte offset where the rest starts (the caller prepends
// text[result, nbytes) to the next chunk); at the end of the file the result is nbytes.  d_text: 16-byte aligned, 16 bytes of slack.
// Throws on a NUL byte and on a header name longer than FG_NAME_MAX, before anything is appended.
class FgetsReader {
public:
    size_t read(const unsigned char* d_text, size_t nbytes, int fastq, int piece_len, int cutoff, int reverse, bool at_eof, int n_sm, cudaStream_t st,
                std::vector<u64>* words, std::vector<u32>* lens);

private:
    Pinned<u64> h_;
    DevBuf slots_, scan_, tiles_, nl_, lpb_, pstart_, role_, hdr_, val_, pfx_, lens_, fix_, redo_, wofs_, words_;
};

}   // namespace pgb
