/*
 * pregraph_b200.h -- C-ABI of libpregraph_b200.so, the H100-native (sm_90a) replacement for SOAPdenovo2's `pregraph` stage.
 *
 * Plain C: pointers, sizes, ints.  No CUDA / torch / C++ types cross this boundary; errors never unwind across it
 * (every int-returning entry point returns 0 on success, non-zero on failure, message via pgb200_last_error()).
 *
 * What each entry point replaces in the reference (file:line relative to /root/reference/standardPregraph/):
 *
 *   call_pregraph                 int call_pregraph(int argc, char **argv)            pregraph.c:62  (declared main.c:29,
 *                                 called main.c:74 and main.c:341).  Same argv contract ("pregraph -s cfg -o prefix
 *                                 [-K k -p P -a G -d D -R]"), same files written, same stderr counters, returns 0.
 *                                 The library's own call_pregraph has the 63-mer semantics; a SOAPdenovo-127mer build links
 *                                 csrc/pregraph_shim.c (-DPGB_FLAVOUR127=1), which fixes the flavour at BUILD time like the
 *                                 reference's -DMER63 / -DMER127 (Makefile:51-66) and keeps the `all` pipeline's globals.
 *   pgb200_pregraph_main          the stage with the flavour as an argument (what the shim and the CLI front ends call).
 *                                 PGB200_GPUS=n shards pass 1 over n GPUs of the box (see pgb200_xchg_* below).
 *   pgb200_map_main               int call_align(int argc, char **argv)                map.c:96.  The `map` stage: same argv contract
 *                                 ("map -s cfg -g prefix [-f] [-p n -k k -h len]"), same .readOnContig.gz / .readInGap.gz / .peGrads
 *                                 (and with -f .shortreadInGap.gz / .PEreadOnContig.gz), same stderr counters; -p is a layout
 *                                 parameter of .readInGap.gz, as in the reference.  One GPU (PGB200_DEVICE).  Long-read
 *                                 libraries (asm_flags=4) and BAM are refused.  Returns 0; a failure ends the process, as there.
 *                                 The drop-in's call_align (csrc/pregraph_shim.c) calls it.
 *   pgb200_feed_text + pgb200_finish_pass1 + pgb200_sweeps
 *                                 boolean prlRead2HashTable(char *libfile, char *outfile)   prlHashReads.c:304
 *                                 (readers readseq1by1.c:138-360, chopKmer4read :163-259, put_kmerset newhash.c:473-528,
 *                                  thread_delow/thread_mark/freqStat :953-1132)
 *   pgb200_build_layout           the iteration order implied by KmerSets[] (newhash.c:200-233, 473-528; SURVEY A.4/A.5)
 *   pgb200_remove_tips            void removeSingleTips(), void removeMinorTips()     cutTipPreGraph.c:363, 414
 *   pgb200_kmer2edges             void kmer2edges(char *outfile)                      node2edge.c:61
 *   pgb200_read2edge              void prlRead2edge(char *libfile, char *outfile)     prlRead2path.c:786
 *   pgb200_output_vertex          void output_vertex(char *outfile)                   output_pregraph.c:50
 *   pgb200_destroy                void free_Sets(KmerSet **, int)                     newhash.c:601
 *
 * Threading: call from one host thread per engine (every entry point binds the calling thread to its engine's GPU); an engine
 * owns its CUDA streams.  pgb200_feed_text returns when the chunk's text has been consumed (host buffers may be reused) while its
 * kernels may still run; pgb200_finish_pass1 and every later phase call return with the device work completed.  Not re-entrant
 * per engine (the reference is not re-entrant at all).
 */
#ifndef PREGRAPH_B200_H
#define PREGRAPH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pgb200_engine pgb200_engine;

typedef struct pgb200_params {
    int K;            /* k-mer size after the reference's fix-ups (odd, 13..63 or 13..127)                     */
    int P;            /* -p: number of reference hash sets; a LAYOUT parameter, not a thread count              */
    int initG;        /* -a: reference memory assumption in GB (static tables); 0 = dynamic                     */
    int D;            /* -d: k-mers with frequency <= D are deleted                                             */
    int repsTie;      /* -R                                                                                      */
    int flavour127;   /* 0 = SOAPdenovo-63mer semantics, 1 = SOAPdenovo-127mer semantics                        */
    int device;       /* CUDA device ordinal                                                                     */
    int max_rd_len;   /* maxReadLen4all (config max_rd_len, default 100)                                         */
    uint64_t table_slots; /* GPU k-mer table capacity hint (0 = derive from -a / grow on demand)                */
    int verbose;
    int world, rank;  /* k-mer space sharding across GPUs: this engine owns bucket range `rank` of `world` (see pgb200_xchg_*) */
} pgb200_params;

typedef struct pgb200_pass1_stats {
    uint64_t records, reads_kept, instances, distinct, table_slots, launches;
    double ms_decode, ms_insert;   /* CUDA-event times; ms_insert = partition + aggregation */
    double ms_apply;               /* the aggregation launches alone */
} pgb200_pass1_stats;

const char *pgb200_last_error(void);
void pgb200_default_params(pgb200_params *p);
pgb200_engine *pgb200_create(const pgb200_params *p);
void pgb200_destroy(pgb200_engine *e);

/* pinned host staging buffers for pgb200_feed_text(on_device = 0) */
void *pgb200_host_alloc(size_t bytes);
void pgb200_host_free(void *p);

/* Pass 1.  `text` holds whole FASTA (single-line) or FASTQ (4-line) records, starts at a record start, ends with '\n'.
 * on_device != 0: `text` is a device pointer (any alignment; 16-byte aligned pointers avoid one device-to-device copy).  Record i gets stream ordinal ord_base + i*ord_stride
 * (stride 2 + mate offset for f1/f2, q1/q2 files: the reference interleaves mates, prlHashReads.c:480-583).       */
int pgb200_feed_text(pgb200_engine *e, const char *text, size_t nbytes, int on_device, int fastq, uint64_t ord_base,
                     uint64_t ord_stride, int reverse_seq, int maxlen);
uint64_t pgb200_last_chunk_records(pgb200_engine *e);

/* Multi-GPU (params.world > 1).  Pass 1 is aggregated per minimizer bucket (super-k-mer records, csrc/skm.cuh); engine `rank` owns a
 * contiguous range of the buckets.  Every engine has an ARENA that all engines of the job store records into: pgb200_feed_text
 * decodes the chunk, partitions it and stores every record STRAIGHT INTO ITS OWNER'S ARENA (peer stores over NVLink from the
 * partition kernel; senders have private regions, so no negotiation and no library collective on the data path).
 * This replaces the reference's "every thread scans the whole batch and keeps hash % thrd_num == id" (prlHashReads.c:79-90).
 *   setup, once:   pgb200_xchg_setup(cap)  ->  exchange arenas: other processes  pgb200_xchg_export / pgb200_xchg_import (64-byte
 *                  cudaIpcMemHandle_t), same process  pgb200_xchg_base / pgb200_xchg_import_ptr (peer access)
 *   per epoch:     pgb200_feed_text ... (any number of chunks, each engine its own)  ->  pgb200_xchg_fence  ->  [caller: barrier over
 *                  all engines]  ->  pgb200_flush  (aggregates what this engine received into its table)
 * Arenas are double-buffered by epoch: an engine may start feeding the next epoch while others still aggregate.
 * world == 1 needs none of this (the engine sets up a private arena and flushes by itself).
 * cap_records = arena capacity in records (32 B for K <= 63, 48 B for K <= 127), summed over the `world` senders.            */
int pgb200_xchg_setup(pgb200_engine *e, uint64_t cap_records);
int pgb200_xchg_export(pgb200_engine *e, void *handle64);
int pgb200_xchg_import(pgb200_engine *e, int peer, const void *handle64);
void *pgb200_xchg_base(pgb200_engine *e);
int pgb200_xchg_import_ptr(pgb200_engine *e, int peer, int peer_device, void *base);
int pgb200_xchg_fence(pgb200_engine *e);
int pgb200_flush(pgb200_engine *e);
/* 1: a chunk of up to n_rec reads surely fits this engine's arena regions and segment ring in the current epoch; 0: fence + flush all
 * engines first (what the multi-GPU CLI does between chunks); -1: error.                                                          */
int pgb200_xchg_room(pgb200_engine *e, uint64_t n_rec);
/* Same process, after pass 1 + sweeps of both: fold `other`'s table shard and packed reads into `e` (peer access).  The graph phases
 * (layout, tips, edges, pass 2) walk across buckets and run on ONE GPU: the multi-GPU CLI (PGB200_GPUS=n) absorbs every shard
 * into GPU 0 and continues there.                                                                                                */
int pgb200_absorb(pgb200_engine *e, pgb200_engine *other);
int pgb200_finish_pass1(pgb200_engine *e, pgb200_pass1_stats *st);
int pgb200_reset_pass1(pgb200_engine *e);
/* delow (-d) + mark linear + coverage histogram (thread_delow / thread_mark / freqStat, prlHashReads.c:953-1132): hist[c] = number of
 * k-mers with coverage c (the .kmerFreq lines are hist[1..255]).  When the pass was one aggregation launch the sweeps were already
 * applied to every entry as it was stored and this call only returns the numbers; otherwise it runs the pass over the table.  May be
 * called again: same numbers.                                                                                                      */
int pgb200_sweeps(pgb200_engine *e, long long hist[256], uint64_t *linear_marked, uint64_t *removed);

int pgb200_build_layout(pgb200_engine *e);
uint64_t pgb200_node_count(pgb200_engine *e);
/* parity/debug: node_count() records {kmer words (2 or 4 x u64), l[4], r[4], cov, flags(1 single, 2 linear, 4 deleted)}
 * in reference iteration order; record size = 8*words + 10 bytes                                                    */
int pgb200_dump_nodes(pgb200_engine *e, void *out);
/* a seeded sample of the k-mer table: the entries whose key hashes (with `seed`) to 0 mod `one_in`, as 6 x u64 records {key words
 * (zero-padded to 4), payload (kmer_t bit layout), first-occurrence rank}; *n_out = how many there are, at most `cap` are written
 * (in table order: sort them).  The choice depends on the keys only, so runs over the same reads sample the same k-mers.        */
int pgb200_sample_table(pgb200_engine *e, uint64_t seed, uint32_t one_in, uint64_t *out, uint64_t cap, uint64_t *n_out);

typedef struct pgb200_graph_stats {
    uint64_t single_tips, minor_tips, num_ed, edges, extra_nodes, deleted_reads, arcs, vertices;
} pgb200_graph_stats;
int pgb200_remove_tips(pgb200_engine *e, pgb200_graph_stats *st);
int pgb200_kmer2edges(pgb200_engine *e, const char *outfile_prefix, pgb200_graph_stats *st);
int pgb200_read2edge(pgb200_engine *e, const char *outfile_prefix, pgb200_graph_stats *st);
int pgb200_output_vertex(pgb200_engine *e, const char *outfile_prefix, pgb200_graph_stats *st);

/* Host logic only (no GPU): the read-stream plan of a library config -- one "mate fastq reverse_seq cut path" line per file in
 * the order the reference opens them (scan_libInfo lib.c:130-506, nextValidIndex readseq1by1.c:595-674); first line "max_rd_len N". */
int pgb200_plan_files(const char *cfg, char *out, size_t cap);
/* Host logic only: where the stage cuts a text buffer that ends in the middle of a record -- the offset of the last record start such
 * that buf[0..off) holds whole records and the record at `off` is known to be a record start (FASTA: a line starting with '>';
 * FASTQ: a line starting with '@' whose line after next starts with '+', which a quality line starting with '@' never has).
 * 0: no such position in the buffer (the caller reads more).  The reference reads line by line (readseq1by1.c:138-209, 279-360). */
size_t pgb200_cut_chunk(const char *buf, size_t n, int fastq);

/* f2 (SURVEY 8f): binary edge sidecar `<prefix>.edge.b200` for a `contig` that links csrc/contig_sidecar.c -- the edges without
 * the gzip'ed text (the reference's loader: loadPreGraph.c:448-544).  Written by the stage when PGB200_EDGE_SIDECAR is set (the
 * byte-identical .edge.gz is still written, unless the value is "only").  The file is this header, then n_records records
 *   { i32 length, cvg, bal_ed, seq_bytes = length / 4 + 1; u64 from[kmer_words], to[kmer_words]; u8 seq[seq_bytes] }
 *   (seq: 4 bases per byte, first base in bits 7:6, codes A0 C1 T2 G3 -- writeChar2tightString, seq.c:81)                         */
#define PGB200_SIDECAR_MAGIC "PGB2EDGE"   /* the 8 bytes of magic[], no terminating NUL */
#define PGB200_SIDECAR_VERSION 1
typedef struct pgb200_edge_sidecar_header {
    char magic[8];
    uint32_t version, K, kmer_words, reserved0;   /* kmer_words: 2 (63-mer flavour) or 4 (127-mer flavour); reserved0 = 0 */
    uint64_t n_records, num_ed, reserved1;        /* num_ed: edges including twins (the EDGEs line of .preGraphBasic)     */
} pgb200_edge_sidecar_header;
#ifdef __cplusplus
static_assert(sizeof(pgb200_edge_sidecar_header) == 48, "the sidecar header is 48 bytes");
#else
_Static_assert(sizeof(pgb200_edge_sidecar_header) == 48, "the sidecar header is 48 bytes");
#endif
/* Converts edge TEXT (the uncompressed content of an .edge.gz) into a sidecar, on the host. */
int pgb200_edge_text_to_sidecar(const char *text, size_t nbytes, int K, int flavour127, uint64_t num_ed, const char *path);
/* The way back, host only: `<prefix>.edge.b200` -> the byte-identical `<prefix>.edge.gz` (record text of output_pregraph.c:88-110, deflated
 * like the stage does).  For pipelines that ran the stage with PGB200_EDGE_SIDECAR=only and want the .edge.gz later / in the background. */
int pgb200_sidecar_to_edge_gz(const char *prefix);

/* gzip files byte-identical to zlib's gzopen(path, "w") + gzwrite + gzclose (default level 6), deflated on the GPU (csrc/deflate.cu).
 * PGB200_GZ=host writes with zlib itself; the GPU writer is also left for zlib when the runtime zlib's level-6 bytes differ from
 * the ones it reproduces (pgb200_gz_gpu_exact).  The stages write their .gz outputs through these.                              */
typedef struct pgb200_gz pgb200_gz;
/* gzopen(path, "w"): NULL on error (pgb200_last_error says why). */
pgb200_gz *pgb200_gz_open(const char *path, int device);
/* gzwrite(file, buf, n): buf is host memory, or device memory on the writer's device when on_device.  0 on success. */
int pgb200_gz_write(pgb200_gz *h, const void *buf, size_t n, int on_device);
/* gzclose(file): writes the last block and the trailer and frees the handle (also after an error).  0 on success. */
int pgb200_gz_close(pgb200_gz *h);
/* 1: the GPU writer's bytes equal the runtime zlib's deflateInit2(6, Z_DEFLATED, 31, 8, Z_DEFAULT_STRATEGY) on the probe text. */
int pgb200_gz_gpu_exact(int device);

/* The drop-in stage entry points. */
int pgb200_pregraph_main(int argc, char **argv, int flavour127);
int pgb200_map_main(int argc, char **argv, int flavour127);
int call_pregraph(int argc, char **argv);

#ifdef __cplusplus
}
#endif
#endif
