/*
 * spades_b200.h -- C ABI of libspades_b200.so: the GPU-native (H100, sm_90a) k-mer counting / de Bruijn construction path.
 *
 * Plain pointers and sizes only; every function returns 0 on success or a positive error code (never exits,
 * never throws); sgpu_last_error() gives the message. One sgpu_ctx per process per GPU, used from one host
 * thread at a time (the reference calls this path from a single thread too, SURVEY 8b).
 *
 * Each entry point replaces one piece of the reference (paths relative to the SPAdes source tree):
 *
 *   sgpu_reads_*            io/reads binary read records: Sequence::BinRead (common/sequence/sequence.hpp:808-830),
 *                           SingleReadSeq (common/io/reads/single_read.hpp:307-323) -- 2-bit packed reads
 *   sgpu_count              kmers::KMerDiskCounter<RtSeq>::Count over a DeBruijnReadKMerSplitter<..., StoringTypeFilter<
 *                           InvertableStoring>> (SGPU_CANONICAL; common/kmer_index/kmer_mph/kmer_index_builder.hpp:306-332,
 *                           kmer_splitters.hpp:112-136) or over spades-kmercount's ParallelSortingSplitter (SGPU_ALL_WINDOWS;
 *                           projects/spades_tools/kmercount.cpp:48-122,219-220)
 *   sgpu_kmers_from_kpomers KMerDiskCounter::Count over DeBruijnKMerKMerSplitter (kmer_splitters.hpp:138-207), as called by
 *                           DeBruijnExtensionIndexBuilder::BuildExtensionIndexFromKPOMers (extension_index/
 *                           kmer_extension_index_builder.hpp:83-96)
 *   sgpu_kset_*             kmers::KMerDiskStorage<RtSeq> (kmer_index_builder.hpp:47-256): bucket_size, bucket files, merge()
 *   sgpu_mphf_build         kmers::KMerIndexBuilder<Index>::BuildIndex(index, storage) (kmer_index_builder.hpp:448-498)
 *   sgpu_mphf_serialize     kmers::KMerIndex::serialize (kmer_mph/kmer_index.hpp:102-108), byte compatible
 *   sgpu_mphf_lookup        kmers::KMerIndex::seq_idx (kmer_index.hpp:88-93)
 *   sgpu_graph_build        FillExtensionsFromIndex (kmer_extension_index_builder.hpp:45-60,102-105) +
 *                           UnbranchingPathExtractor::ExtractUnbranchingPathsAndLoops (assembly_graph/construction/
 *                           debruijn_graph_constructor.hpp:399-406) + CoverageHashMapBuilder::BuildIndex
 *                           (ph_map/coverage_hash_map_builder.hpp:42-56) + FillCoverageAndFlankingFromPHM (raw coverage part,
 *                           assembly_graph/graph_support/coverage_filling.hpp:90-96)
 *   sgpu_graph_build_ex     the same preceded by EarlyTipClipperProcessor::ClipTips (assembly_graph/construction/
 *                           early_simplification.hpp:38-162; stages/construction.cpp:289-302)
 *   sgpu_graph_build_opts   the same preceded, optionally, by EarlyLowComplexityClipperProcessor::RemoveATEdges / RemoveATTips
 *                           (early_simplification.hpp:164-347; EarlyATClipper of the RNA pipeline, stages/construction.cpp:317-340)
 *   sgpu_graph_masks        DeBruijnExtensionIndex::raw_data() (extension_index/kmer_extension_index.hpp:83-84)
 *   sgpu_graph_coverage     PerfectHashMap<RtSeq,uint32_t>::values() of the coverage map (stages/construction.cpp:371-395)
 *   sgpu_graph_histogram    the multiplicity histogram of PHMCoverageFiller (stages/construction.cpp:404-418)
 *   sgpu_graph_unitig*      std::vector<Sequence> returned by ExtractUnbranchingPathsAndLoops
 *   sgpu_edge_index_*       EdgeIndex<Graph>::Refill (alignment/edge_index.hpp:88-110; assembly_graph/index/edge_index_builders.hpp:154-307,
 *                           edge_info_updater.hpp:38-101)
 *   sgpu_graph_gfa          FastGraphFromSequencesConstructor::ConstructGraph (debruijn_graph_constructor.hpp:506-567) +
 *                           gfa::GFAWriter::WriteSegmentsAndLinks (io/graph/gfa_writer.cpp:36-116)
 */
#ifndef SPADES_B200_H_
#define SPADES_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sgpu_ctx sgpu_ctx;
typedef struct sgpu_kset sgpu_kset;     /* a counted k-mer set resident in HBM, or in host memory (== KMerDiskStorage contents) */
typedef struct sgpu_mphf sgpu_mphf;     /* a boomphf-compatible KMerIndex resident in HBM */
typedef struct sgpu_graph sgpu_graph;   /* masks + coverage + unitigs + link records */

typedef struct sgpu_config {
    int device;                 /* CUDA device ordinal */
    uint64_t hbm_budget_bytes;  /* 0 = whatever is free on the device */
    int verbose;
    uint64_t stream;            /* a cudaStream_t to run on (e.g. the caller's timing stream); 0 = create a private stream */
} sgpu_config;

enum { SGPU_CANONICAL = 0, SGPU_ALL_WINDOWS = 1 };
/* OR-ed into the mode of sgpu_count / sgpu_dist_begin: the k-mer set is returned in pinned host memory instead of HBM, so a set
 * larger than the device can be counted. Each pass's result is copied to the host while the next pass runs; only the pass in
 * flight keeps its result on the device. */
#define SGPU_RESULT_ON_HOST 0x100

enum {
    SGPU_OK = 0, SGPU_EINVAL = 2, SGPU_ENODEV = 3, SGPU_ENOMEM = 4, SGPU_ECUDA = 5, SGPU_EINTERNAL = 6, SGPU_EUNSUPPORTED = 7,
    SGPU_EIO = 8
};

/* device-side milliseconds of the last sgpu_count / sgpu_kmers_from_kpomers / sgpu_mphf_build, measured with CUDA events
 * on the context's stream, plus the number of kernels launched since the context was created */
typedef struct sgpu_times {
    float extract_count_ms, extract_scatter_ms, refine_ms, local_sort_ms, compact_ms, mphf_ms, exchange_ms;
    uint64_t instances;   /* records the partition kernel wrote */
    uint64_t passes;      /* bucket-group passes */
    uint64_t launches;    /* kernels launched by this context so far */
    uint64_t peak_bytes;  /* peak device memory held by this context */
    uint64_t cached_bytes;/* freed device blocks kept by the context's caching allocator (reusable) */
    /* which paths of the count ran (last sgpu_count / sgpu_kmers_from_kpomers / sgpu_dist_begin .. sgpu_dist_end) */
    uint64_t level_a_key_bits;      /* rA: key bits folded into a level-A partition id */
    uint64_t level_a_scatters;      /* level-A scatter launches (one per source, pass and partition sub-range) */
    uint64_t refine_rounds_max;     /* most refinement rounds any pass ran, the gather round included */
    uint64_t refine_splits_round0;  /* segments the first refinement round (the gather) added beyond the partitions */
    uint64_t refine_splits_later;   /* segments the later refinement rounds added */
    uint64_t sort_lsd_fallbacks;    /* local-sort segments that took the exact LSD fallback */
    uint64_t sort_oversize_equal;   /* segments longer than the local-sort capacity whose records are all equal */
    /* a count with SGPU_RESULT_ON_HOST (last sgpu_count / sgpu_dist_begin .. sgpu_dist_end) */
    uint64_t result_d2h_bytes;      /* bytes of records and multiplicities copied to host memory */
    float result_d2h_wait_ms;       /* host time the count spent waiting for those copies */
    /* bytes of host-set chunks uploaded to the device since the last sgpu_kmers_from_kpomers_ex, sgpu_mphf_build or graph build
     * began (0 when its sets live in HBM) */
    uint64_t stage_h2d_bytes;
    uint64_t graph_junction_batches; /* junction batches of the last graph build (0 when it had no junctions, e.g. no k-mers or
                                      * only perfect loops); a batch never spans the junctions of two chunks of the k-mer set */
    /* the last sgpu_reads_cov_filter / sgpu_reads_cov_filter_ex */
    uint64_t cov_filter_passes;      /* key-range passes of the counting table (1 = one table) */
    uint64_t cov_filter_table_bytes; /* device bytes of one pass's table */
} sgpu_times;

int sgpu_create(const sgpu_config *cfg, sgpu_ctx **out);
/* k-mer sets, indexes, graphs and distributed counts created from a context keep device memory of that context. Destroying the
 * context while some are alive is safe in any order: the context is torn down when the last of them has been freed. */
void sgpu_destroy(sgpu_ctx *ctx);
const char *sgpu_last_error(const sgpu_ctx *ctx);
int sgpu_get_times(const sgpu_ctx *ctx, sgpu_times *out);

/* reads: read r occupies words[offs[r] .. offs[r]+ceil(lens[r]/32)), nucleotide i at bits 2(i%32) of word i/32, A=0 C=1 G=2 T=3
 * (N-free: apply LongestValid first, io/reads/longest_valid_wrapper.hpp:16-53). offs are relative to `words`. */
int sgpu_reads_clear(sgpu_ctx *ctx);
int sgpu_reads_append_packed(sgpu_ctx *ctx, const uint64_t *words, uint64_t nwords, const uint64_t *offs, const uint32_t *lens, int64_t nreads);
/* replace the read set with these HOST buffers, copied straight to the device (pinned buffers copy at full PCIe rate). The copies
 * are enqueued on the context's stream and the call returns: the buffers must stay valid and unmodified until the next
 * sgpu_count / sgpu_dist_begin on this context has returned (both synchronise the stream). */
int sgpu_reads_upload(sgpu_ctx *ctx, const uint64_t *words, uint64_t nwords, const uint64_t *offs, const uint32_t *lens, int64_t nreads);
/* GPU-side packing (SURVEY 8f-2): the host only locates the sequence of every read inside a text buffer (FASTA/FASTQ file contents:
 * byte offset + length of each single-line sequence; sgpu_text_index_fastx does it for 2-line FASTA / 4-line FASTQ); the device applies
 * io::LongestValid (io/reads/longest_valid_wrapper.hpp:16-53; longest_valid = 0: a read with any non-ACGT symbol contributes nothing)
 * and packs 2 bits per base (Sequence::BinWrite payload). Replaces the context's read set; reads without a valid base keep a slot of
 * length 0. */
int sgpu_reads_pack_text(sgpu_ctx *ctx, const char *text, uint64_t text_bytes, const uint64_t *seq_off, const uint32_t *seq_len, int64_t nreads,
                         int longest_valid);
/* the context's current (packed) read set: sizes, and a copy to host arrays of those sizes (any pointer may be NULL) */
int sgpu_reads_info(sgpu_ctx *ctx, int64_t *nreads, uint64_t *nwords);
int sgpu_reads_download(sgpu_ctx *ctx, uint64_t *words, uint64_t *offs, uint32_t *lens);
/* Coverage pre-filter of the construction stage (SURVEY 8f-3; the pipeline's CoverageFilter phase, stages/construction.cpp:167-198, active
 * when read_cov_threshold > 0): K = k + 1. (1) HyperLogLog upper bound of the distinct K-mers (EstimateCardinalityUpperBound,
 * kmer_index/kmer_counting.hpp:215-249; adt/hll.hpp) with rolling_hash::SymmetricCyclicHash (adt/cyclichash.hpp:187-259); (2) the counting
 * quotient filter sized from it (qf::cqf, adt/cqf.hpp:28-37) filled up to `threshold` per key (FillCoverageHistogram, kmer_counting.hpp:251-282);
 * (3) io::CovFilteringWrap (io/reads/coverage_filtering_read_wrapper.hpp): a read survives iff the median multiplicity of its K-mers is >=
 * threshold. keep_out (may be NULL): one byte per read of the CURRENT read set, 1 = survives. apply != 0: the survivors (order kept) become
 * the context's read set, as the wrapper does to the pipeline's streams. stats (may be NULL): [0] cardinality upper bound, [1] key bits of
 * the filter (qbits + 8), [2] distinct keys counted, [3] reads kept.
 * The counting table takes 12 bytes per key of the bound in one piece (1.5 x the bound, 8-byte entries). When it does not fit the
 * device memory left (the context's hbm_budget_bytes minus what it holds, or 90 % of the arena's free bytes), the key space is split
 * into P ranges and the reads, which stay on the device, are rolled twice per range (fill, then lookup) against a table of about
 * 1/P of the size: the smallest P that fits, at most 256, else SGPU_ENOMEM. The outputs are the same for every P. */
int sgpu_reads_cov_filter(sgpu_ctx *ctx, int K, unsigned threshold, int apply, uint8_t *keep_out, uint64_t *stats);
/* the same with the passes chosen by the caller: 0 = planned as above, 1 = one table whatever the memory left, 2 .. 256 = that many
 * key ranges */
int sgpu_reads_cov_filter_ex(sgpu_ctx *ctx, int K, unsigned threshold, int apply, int passes, uint8_t *keep_out, uint64_t *stats);
/* the pass plan alone (pure host arithmetic, no GPU): for a cardinality bound, n reads and the device bytes left after the bound,
 * the key-range passes and the entries of one pass's table. budget_bytes also covers the filter's four per-read arrays (n + 1
 * entries, 13 bytes per entry in all, each array in 512-byte blocks) and two 512-byte blocks. SGPU_ENOMEM (passes = 0) when 256
 * passes do not fit. */
int sgpu_cov_pass_plan_host(uint64_t cardinality_bound, int64_t nreads, uint64_t budget_bytes, int *passes, uint64_t *pass_capacity);
/* use a read set that already lives in device memory (not copied, must stay valid while the context uses it) */
int sgpu_reads_adopt_device(sgpu_ctx *ctx, const uint64_t *d_words, uint64_t nwords, const uint64_t *d_offs, const uint32_t *d_lens, int64_t nreads);

/* ---- read ingest (pure host code: no GPU, no context needed). Replaces the front end of the tools: io::FastaFastqGzParser
 * over kseq + zlib (io/reads/fasta_fastq_gz_parser.hpp:25-150), io::LongestValid (io/reads/longest_valid_wrapper.hpp:16-53, applied
 * by io_helper.cpp:30-31 and read_converter.cpp:115,121) and the binary read streams <prefix>.seq / <prefix>.off that
 * io::BinaryWriter::ToBinary writes and io::BinaryFileStream<SingleReadSeq> reads (io/reads/binary_converter.cpp:84-145,
 * binary_streams.hpp:54-102; record = Sequence::BinWrite + SingleReadSeq::BinWrite, sequence.hpp:817-830, single_read.hpp:325-338).
 * A batch holds 2-bit packed reads in the layout sgpu_reads_append_packed / sgpu_reads_upload take. Reads without any valid
 * base are dropped (they contribute no k-mer). On failure *out is still a batch whose sgpu_read_batch_error() says why. */
typedef struct sgpu_read_batch sgpu_read_batch;
int sgpu_fastx_parse(const char *path, int longest_valid, sgpu_read_batch **out);      /* FASTA / FASTQ, plain or gzip */
/* nthreads > 1: an uncompressed file is parsed in parallel pieces, accepted only where the sequential parser provably stands at
 * the same place (otherwise, and for gzip, the sequential parse runs); 0 = hardware threads (SGPU_INGEST_THREADS overrides), 1 = sequential */
int sgpu_fastx_parse_threads(const char *path, int longest_valid, int nthreads, sgpu_read_batch **out);
int sgpu_seqfile_parse(const char *prefix, sgpu_read_batch **out);                     /* <prefix>.seq of the reference */
int sgpu_read_batch_write_seqfile(const sgpu_read_batch *b, const char *prefix);       /* <prefix>.seq + <prefix>.off */
int64_t sgpu_read_batch_num_reads(const sgpu_read_batch *b);
uint64_t sgpu_read_batch_num_words(const sgpu_read_batch *b);
const uint64_t *sgpu_read_batch_words(const sgpu_read_batch *b);
const uint64_t *sgpu_read_batch_offs(const sgpu_read_batch *b);
const uint32_t *sgpu_read_batch_lens(const sgpu_read_batch *b);
int sgpu_read_batch_stats(const sgpu_read_batch *b, uint64_t *out3);   /* records in the file, reads trimmed by LongestValid, reads dropped */
const char *sgpu_read_batch_error(const sgpu_read_batch *b);
void sgpu_read_batch_free(sgpu_read_batch *b);
/* host side of sgpu_reads_pack_text: sequence ranges of a strictly 2-line FASTA ('>') / 4-line FASTQ ('@', '+', quality as long as the
 * sequence) text; a trailing '\r' is excluded. out arrays must hold max_reads entries; returns the number of reads, -1 if the text is
 * not in that strict layout (then use sgpu_fastx_parse, which implements kseq's general record semantics), -2 if max_reads is too small */
int64_t sgpu_text_index_fastx(const char *text, uint64_t text_bytes, uint64_t *seq_off, uint32_t *seq_len, int64_t max_reads);
/* sgpu_reads_append_packed of a whole batch */
int sgpu_reads_append_batch(sgpu_ctx *ctx, const sgpu_read_batch *b);

/* mode: SGPU_CANONICAL or SGPU_ALL_WINDOWS, optionally | SGPU_RESULT_ON_HOST. A host set answers every sgpu_kset_* call and
 * sgpu_mphf_build exactly as a device set does (the index is built chunk by chunk, uploading each chunk while the one before is
 * placed), and sgpu_kmers_from_kpomers_ex and sgpu_graph_build_streamed take it. sgpu_kmers_from_kpomers and the older
 * sgpu_graph_build* calls need their sets in HBM and return SGPU_EUNSUPPORTED for a host set. */
int sgpu_count(sgpu_ctx *ctx, int K, int num_buckets, int mode, sgpu_kset **out);
int sgpu_kmers_from_kpomers(sgpu_ctx *ctx, const sgpu_kset *kpomers, int num_buckets, sgpu_kset **out);
/* the k-mers of a (k+1)-mer set in HBM or in host memory; mode = 0 (result in HBM) or SGPU_RESULT_ON_HOST. A host (k+1)-mer
 * set is uploaded chunk by chunk, once per histogram super-range and once per pass, the next chunk while the current one is read. */
int sgpu_kmers_from_kpomers_ex(sgpu_ctx *ctx, const sgpu_kset *kpomers, int num_buckets, int mode, sgpu_kset **out);

int64_t sgpu_kset_size(const sgpu_kset *s);
int sgpu_kset_k(const sgpu_kset *s);
int sgpu_kset_num_buckets(const sgpu_kset *s);
int sgpu_kset_record_bytes(const sgpu_kset *s);                       /* KMerCounter::kmer_size(): 8*ceil(K/32) */
int sgpu_kset_on_host(const sgpu_kset *s);                            /* 1: the set lives in host memory, 0: in HBM, -1: NULL */
int sgpu_kset_bucket_sizes(const sgpu_kset *s, int64_t *out);         /* num_buckets entries */
/* records [first, first+n) of final_kmers order (KMerDiskStorage::merge, kmer_index_builder.hpp:190-203) to host memory */
/* order-independent checksums computed on the device: out4 = { number of records, weighted sum of all record words, xor of
 * the rotated record words, sum of the multiplicities } (mod 2^64). Disjoint bucket sets add / xor up, so the per-rank sets of a
 * multi-GPU count can be checked against a single-GPU count of the union without moving records. */
int sgpu_kset_checksum(const sgpu_kset *s, uint64_t *out4);
int sgpu_kset_download_keys(const sgpu_kset *s, int64_t first, int64_t n, uint64_t *out);
int sgpu_kset_download_counts(const sgpu_kset *s, int64_t first, int64_t n, uint32_t *out);   /* SGPU_CANONICAL sets only */
/* writes <prefix>.<b> for every bucket in the reference's bucket file format (raw W-byte records) */
int sgpu_kset_write_buckets(const sgpu_kset *s, const char *prefix);
/* the buckets a set holds (flags: num_buckets bytes, 1 = owned): every bucket for a single-GPU set, this rank's share of every pass
 * for a set from sgpu_dist_end. sgpu_kset_write_owned_buckets writes <prefix>.<b> for the owned buckets only, so the ranks of a
 * distributed count writing into one directory leave each bucket file once: together the complete set of bucket files. */
int sgpu_kset_owned_buckets(const sgpu_kset *s, uint8_t *flags);
int sgpu_kset_write_owned_buckets(const sgpu_kset *s, const char *prefix);
int sgpu_kset_write_final(const sgpu_kset *s, const char *path);      /* final_kmers */
void sgpu_kset_free(sgpu_kset *s);

int sgpu_mphf_build(sgpu_ctx *ctx, const sgpu_kset *s, sgpu_mphf **out);
int64_t sgpu_mphf_serialized_size(const sgpu_mphf *m);
int sgpu_mphf_serialize(const sgpu_mphf *m, uint8_t *out, int64_t cap);
/* the serialized buckets [b_lo, b_hi) alone: the bytes sgpu_mphf_serialize writes for them between num_segments and segment_starts.
 * A bucket's bytes depend on its own keys only, so the index of a distributed k-mer set is assembled from its owners' buckets.
 * The size is -1 for a bad range. */
int64_t sgpu_mphf_serialized_size_buckets(const sgpu_mphf *m, int b_lo, int b_hi);
int sgpu_mphf_serialize_buckets(const sgpu_mphf *m, int b_lo, int b_hi, uint8_t *out, int64_t cap);
int sgpu_mphf_lookup(const sgpu_mphf *m, const uint64_t *keys, int64_t n, uint64_t *out_idx);   /* host keys, stored (minimal) form */
void sgpu_mphf_free(sgpu_mphf *m);

/* kpomers must come from sgpu_count(k+1, B, SGPU_CANONICAL); kmers/kmer_index from sgpu_kmers_from_kpomers / sgpu_mphf_build.
 * kpomer_index may be NULL (then no coverage: DP/KC are 0 and sgpu_graph_coverage fails). The graph borrows its inputs. */
int sgpu_graph_build(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index,
                     const sgpu_mphf *kpomer_index, int keep_perfect_loops, sgpu_graph **out);
/* sgpu_graph_build plus the pipeline's early tip clipper between the mask fill and the unitig extraction:
 * EarlyTipClipperProcessor::ClipTips (assembly_graph/construction/early_simplification.hpp:38-162) as run by the Construction
 * stage (stages/construction.cpp:289-302, modules/graph_construction.hpp:32-36) with length_bound = read length - k.
 * early_tip_length_bound = 0 switches it off (== sgpu_graph_build, what spades-gbuilder does). sgpu_graph_masks then returns
 * the clipped array. stats: removed k-mers (ClipTips' return value), tipped junctions, clipped links (its INFO counters). */
int sgpu_graph_build_ex(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index,
                        const sgpu_mphf *kpomer_index, int keep_perfect_loops, uint64_t early_tip_length_bound, sgpu_graph **out);
int sgpu_graph_tip_clipper_stats(const sgpu_graph *g, uint64_t *out3);
/* all options of the Construction stage's graph phases in one call. early_at_clipper: EarlyLowComplexityClipperProcessor::
 * RemoveATEdges + RemoveATTips (assembly_graph/construction/early_simplification.hpp:164-347), the EarlyATClipper phase the RNA
 * pipeline runs before the tip clipper (stages/construction.cpp:317-340,447-448 with at_ratio 0.8, min_length 10, max_length 200;
 * min_length must not exceed k). sgpu_graph_masks then returns the array after both clippers. */
typedef struct sgpu_graph_options {
    int keep_perfect_loops;
    uint64_t early_tip_length_bound;   /* 0 = off */
    int early_at_clipper;              /* 0 = off */
    double at_ratio;
    uint64_t at_min_length, at_max_length;
} sgpu_graph_options;
int sgpu_graph_build_opts(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index,
                          const sgpu_mphf *kpomer_index, const sgpu_graph_options *opts, sgpu_graph **out);
/* sgpu_graph_build_opts over sets in HBM or host memory, in any combination; the sets are read chunk by chunk (a host set's chunks
 * are uploaded while the one before is used). The device keeps both indexes, the masks, the coverage and the clippers' flags; the
 * unbranching paths are extracted in batches of junctions sized from the memory left. Same results as sgpu_graph_build_opts. */
int sgpu_graph_build_streamed(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index,
                              const sgpu_mphf *kpomer_index, const sgpu_graph_options *opts, sgpu_graph **out);
/* stats: edges collected (RemoveATEdges' return value), links removed, k-mers removed (RemoveATTips' return value), clipped tips */
int sgpu_graph_at_clipper_stats(const sgpu_graph *g, uint64_t *out4);
int sgpu_graph_masks(const sgpu_graph *g, uint8_t *out, int64_t n);           /* n = number of k-mers */
int sgpu_graph_coverage(const sgpu_graph *g, uint32_t *out, int64_t n);       /* n = number of (k+1)-mers */
int64_t sgpu_graph_histogram(const sgpu_graph *g, uint64_t *out, int64_t cap);/* returns the histogram length (max coverage) */
int64_t sgpu_graph_num_unitigs(const sgpu_graph *g);
int64_t sgpu_graph_unitig_bases(const sgpu_graph *g);
/* ASCII unitigs concatenated into out (sgpu_graph_unitig_bases() bytes) and their lengths */
int sgpu_graph_unitigs(const sgpu_graph *g, char *out, uint32_t *lens);
int64_t sgpu_graph_gfa(const sgpu_graph *g, const char *version, char *out, int64_t cap);   /* returns the text size */
int sgpu_graph_write_gfa(const sgpu_graph *g, const char *version, const char *path);
void sgpu_graph_free(sgpu_graph *g);

/* ---- EdgeIndex refill (the next consumer of the graph in the pipeline): debruijn_graph::EdgeIndex<Graph>::Refill
 * (alignment/edge_index.hpp:88-110, modules/graph_construction.hpp:74-82) = GraphPositionFillingIndexBuilder::BuildIndexFromGraph
 * (assembly_graph/index/edge_index_builders.hpp:154-307) + EdgeInfoUpdater::UpdateAll (edge_info_updater.hpp:38-101) over the
 * graph's own unitigs. num_buckets = 10 x the reference's threads in both cases: K = 0 means k+1 -- the reference then walks the
 * edges in that many vertex chunks and builds ONE index segment (num_buckets only decides a serialization detail, see
 * edge_index.cu); any other K counts through DeBruijnGraphKMerSplitter + KMerDiskCounter into num_buckets buckets. The index holds every K-mer of every edge
 * and of its conjugate (KmerFreeEdgeIndex, DefaultStoring); a slot's value is (EdgeId::int_id(), offset) -- edge i of
 * sgpu_graph_unitigs has id 3 + 2i, its conjugate 3 + 2i + 1 -- or (~1, 0x7ffffffe) when the K-mer occurs more than once in the
 * graph (EdgeInfo TOMBSTONE, edge_position_index.hpp:29-30,152-167). The graph may be freed afterwards. */
typedef struct sgpu_edge_index sgpu_edge_index;
int sgpu_edge_index_build(sgpu_ctx *ctx, const sgpu_graph *g, int K, int num_buckets, sgpu_edge_index **out);
int sgpu_edge_index_k(const sgpu_edge_index *e);
int64_t sgpu_edge_index_size(const sgpu_edge_index *e);                              /* number of K-mers = number of slots */
int64_t sgpu_edge_index_serialized_size(const sgpu_edge_index *e);
int sgpu_edge_index_serialize(const sgpu_edge_index *e, uint8_t *out, int64_t cap);   /* KMerIndex::serialize bytes */
int sgpu_edge_index_values(const sgpu_edge_index *e, uint64_t *edge_ids, uint32_t *offsets, int64_t n);   /* slot order */
int sgpu_edge_index_lookup(const sgpu_edge_index *e, const uint64_t *keys, int64_t n, uint64_t *out_idx);  /* host keys -> slots */
void sgpu_edge_index_free(sgpu_edge_index *e);

/* ---- multi-GPU count (one process per GPU; SURVEY 8e). Replaces hpcspades' shared-filesystem + MPI pattern
 * (projects/hpcspades/mpi/stages/construction_mpi.cpp:222-300, mpi/kmer_index/kmer_extension_index_builder_mpi.hpp:87,190):
 * buckets are owned by ranks; every rank partitions its own reads into a staging buffer (same kernels as sgpu_count), then
 * sgpu_dist_exchange is ONE kernel on the owner that pulls its pieces from all peers' staging buffers over NVLink peer memory
 * (cudaIpc mappings of the peers' memory arenas, opened once per process) and merges them partition by partition. The host
 * language only moves small tables between ranks (torch.distributed / MPI all_gather) and provides the barriers:
 *   begin -> local_counts -> [all_gather counts] -> plan ->
 *   repeat: free_bytes -> [all_reduce MIN] -> next_pass (-1 = done) -> ipc_handle -> [all_gather descriptors] -> open_peers ->
 *           scatter [barrier] exchange [barrier] sort
 *   -> end (k-mer set holding this rank's buckets)
 * Passes are planned one at a time against the memory every rank has free at that moment (like sgpu_count's bucket-group passes). */
typedef struct sgpu_dist sgpu_dist;
int sgpu_dist_begin(sgpu_ctx *ctx, int K, int num_buckets, int mode, int world, int rank, sgpu_dist **out);
/* the same sequence over this rank's (k+1)-mer set instead of its reads: sgpu_kmers_from_kpomers_ex distributed. mode = 0 or
 * SGPU_RESULT_ON_HOST; the source may live in HBM or in host memory (its chunks are uploaded for the histogram and every scatter).
 * Every rank passes the same num_buckets and a set of the same k + 1 >= 2; the sets may be any (k+1)-mer sets, and may overlap:
 * the ranks end with the k-mers of the union of the sets, each bucket on its owner, without multiplicities. The source must not
 * change while the count runs; sgpu_kset_free of it is deferred until sgpu_dist_free. */
int sgpu_dist_begin_kpomers(sgpu_ctx *ctx, const sgpu_kset *kpomers, int num_buckets, int mode, int world, int rank, sgpu_dist **out);
int64_t sgpu_dist_num_partitions(const sgpu_dist *d);
int sgpu_dist_local_counts(sgpu_dist *d, uint64_t *out);                 /* num_partitions host entries */
int sgpu_dist_plan(sgpu_dist *d, const uint64_t *all_counts /* world x num_partitions, rank-major, host */, uint64_t *total_records);
int sgpu_dist_free_bytes(sgpu_dist *d, uint64_t *out);                  /* device bytes this rank can allocate for the next pass */
/* budget_bytes: the MINIMUM of sgpu_dist_free_bytes over the ranks (identical inputs give identical decisions on every rank).
 * *pass = index of the pass that was planned and whose buffers were allocated, or -1 when all buckets are done */
int sgpu_dist_next_pass(sgpu_dist *d, uint64_t budget_bytes, int *pass);
#define SGPU_IPC_BYTES 96
/* this rank's descriptor for the current pass: cudaIpcMemHandle_t of its memory arena + the offsets of its staging buffer and
 * piece tables inside it */
int sgpu_dist_ipc_handle(sgpu_dist *d, uint8_t *out /* SGPU_IPC_BYTES */);
int sgpu_dist_open_peers(sgpu_dist *d, const uint8_t *descriptors /* world x SGPU_IPC_BYTES, rank-major */);
int sgpu_dist_scatter(sgpu_dist *d, int pass);                          /* partition this rank's shard into its staging buffer */
int sgpu_dist_exchange(sgpu_dist *d, int pass);                         /* fused NVLink exchange + merge: pulls the owned pieces from every peer */
int sgpu_dist_sort(sgpu_dist *d, int pass);                             /* refinement + local sort + compaction of what arrived */
int sgpu_dist_end(sgpu_dist *d, sgpu_kset **out);
void sgpu_dist_free(sgpu_dist *d);
/* the planning step alone (pure host arithmetic, no GPU): returns npass and fills pass_bounds[0..npass] */
int sgpu_dist_plan_host(int world, int num_buckets, int key_bits_in_partition, const uint64_t *all_counts, uint64_t budget_bytes,
                        int record_bytes, int *pass_bounds, uint64_t *max_recv);

/* ---- multi-GPU coverage pre-filter (one process per GPU). sgpu_reads_cov_filter over a read set sharded across ranks: the result
 * is what one GPU computes over the union of the shards (concatenated in rank order): the same cardinality bound and key width on
 * every rank, the same verdict for every read, the distinct keys summed over the ranks. The HLL registers of the union are the
 * element-wise maximum of the ranks' registers; the counting table is split into one slice per rank, and a key lives in the slice of
 * its owner (a hash of the key, independent of the slot inside the slice). Ranks insert into and look up in the owners' slices
 * through cudaIpc mappings of the peers' memory arenas (the same mappings as sgpu_dist_*). The host language moves the two
 * descriptors and provides the barriers:
 *   begin -> ipc_handle -> [all_gather descriptors] -> open_peers -> bound -> ipc_handle -> [all_gather descriptors] -> open_peers ->
 *   fill [barrier] filter [barrier] free
 * begin: HLL registers of this rank's shard (K = k + 1). bound: the union's bound and key width, and this rank's empty slice.
 * fill: every window of this rank's reads into its owner's slice, counts stopping at the threshold. filter: the verdicts of this
 * rank's reads; keep_out, apply and stats as sgpu_reads_cov_filter, except stats[2] = distinct keys in THIS rank's slice (the
 * union's number is the sum over the ranks) and stats[3] = reads kept on this rank. A slice that fills up fails the filter on
 * every rank (SGPU error 6). */
typedef struct sgpu_dist_cov sgpu_dist_cov;
int sgpu_dist_cov_begin(sgpu_ctx *ctx, int K, unsigned threshold, int world, int rank, sgpu_dist_cov **out);
int sgpu_dist_cov_ipc_handle(sgpu_dist_cov *d, uint8_t *out /* SGPU_IPC_BYTES */);
int sgpu_dist_cov_open_peers(sgpu_dist_cov *d, const uint8_t *descriptors /* world x SGPU_IPC_BYTES, rank-major */);
int sgpu_dist_cov_bound(sgpu_dist_cov *d);
int sgpu_dist_cov_fill(sgpu_dist_cov *d);
int sgpu_dist_cov_filter(sgpu_dist_cov *d, int apply, uint8_t *keep_out, uint64_t *stats);
void sgpu_dist_cov_free(sgpu_dist_cov *d);
/* the layout alone (pure host arithmetic, no GPU): the owner rank of each masked key, and the capacity of a rank's slice (entries)
 * for a cardinality bound */
int sgpu_dist_cov_layout_host(int world, uint64_t cardinality_bound, const uint64_t *keys, int64_t n, uint32_t *owners, uint64_t *slice_capacity);

/* ---- multi-GPU extension masks and coverage (one process per GPU). Every rank brings its bucket-owned (k+1)-mer set (with
 * multiplicities, from a distributed canonical count) and its index, and its bucket-owned k-mer set (from sgpu_dist_begin_kpomers)
 * and its index; owners[b] is the rank whose k-mer set holds bucket b (every rank passes the same table). Each rank ends with its
 * slices of what sgpu_graph_masks / _coverage / _histogram give on one GPU over the union (early clippers off): the masks of its
 * k-mers and the coverage of its (k+1)-mers, both in the slot order of its own indexes (a key's slot in the union's index is the
 * same rank inside its bucket, after the union's earlier buckets), and the histogram of its coverage slice (the union's histogram
 * is the element-wise sum over the ranks). A (k+1)-mer's two mask bits usually belong to k-mers other ranks own: per pass, a range
 * of destination buckets, every rank writes its contributions into a staging buffer grouped by owner, and every owner streams its
 * pieces out of the peers' staging buffers (cudaIpc mappings of their arenas, as sgpu_dist_*) into its slice. The coverage needs
 * no exchange and is filled by begin. kpomer_index = NULL: masks only; the (k+1)-mer sets may then overlap (the coverage needs
 * every (k+1)-mer bucket on exactly one rank). The sets and indexes must stay alive until sgpu_dist_ext_free.
 *   begin -> local_counts -> [all_gather counts] -> plan ->
 *   repeat: free_bytes -> [all_reduce MIN] -> next_pass (-1 = done) -> ipc_handle -> [all_gather descriptors] -> open_peers ->
 *           scatter [barrier] apply [barrier]
 *   -> masks / coverage / histogram -> free */
typedef struct sgpu_dist_ext sgpu_dist_ext;
int sgpu_dist_ext_begin(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_mphf *kpomer_index /* NULL: masks only */, const sgpu_kset *kmers,
                        const sgpu_mphf *kmer_index, const int32_t *owners /* num_buckets */, int world, int rank, sgpu_dist_ext **out);
int sgpu_dist_ext_local_counts(const sgpu_dist_ext *d, uint64_t *out);     /* num_buckets: this rank's contributions per destination bucket */
int sgpu_dist_ext_plan(sgpu_dist_ext *d, const uint64_t *all_counts /* world x num_buckets, rank-major */, uint64_t *total_records);
int sgpu_dist_ext_free_bytes(sgpu_dist_ext *d, uint64_t *out);
int sgpu_dist_ext_next_pass(sgpu_dist_ext *d, uint64_t budget_bytes, int *pass);     /* budget: the MINIMUM of free_bytes over the ranks */
int sgpu_dist_ext_ipc_handle(sgpu_dist_ext *d, uint8_t *out /* SGPU_IPC_BYTES */);
int sgpu_dist_ext_open_peers(sgpu_dist_ext *d, const uint8_t *descriptors /* world x SGPU_IPC_BYTES, rank-major */);
int sgpu_dist_ext_scatter(sgpu_dist_ext *d, int pass);
int sgpu_dist_ext_apply(sgpu_dist_ext *d, int pass);
int sgpu_dist_ext_masks(const sgpu_dist_ext *d, uint8_t *out, int64_t n);          /* n = this rank's k-mers */
int sgpu_dist_ext_coverage(const sgpu_dist_ext *d, uint32_t *out, int64_t n);      /* n = this rank's (k+1)-mers */
int64_t sgpu_dist_ext_histogram(const sgpu_dist_ext *d, uint64_t *out, int64_t cap);/* returns this rank's histogram length */
/* milliseconds spent so far in: the contribution histogram, the scatters, the applies, the coverage fill, the coverage histogram */
int sgpu_dist_ext_times(const sgpu_dist_ext *d, float *out5);
void sgpu_dist_ext_free(sgpu_dist_ext *d);
/* the pass plan alone (pure host arithmetic, no GPU), for a fixed budget and records of record_bytes: returns npass and fills
 * pass_bounds[0..npass] and the most records any rank sends or any owner receives in one pass */
int sgpu_dist_ext_plan_host(int world, int num_buckets, const int32_t *owners, const uint64_t *all_counts, uint64_t budget_bytes, int record_bytes,
                            int *pass_bounds, uint64_t *max_records);

/* ---- multi-GPU unitigs and perfect loops (one process per GPU), from a rank's sgpu_dist_ext after its passes: the edges one GPU's
 * sgpu_graph_build gives over the union (sgpu_dist_graph_begin_opts: the early clippers first, as sgpu_graph_build_opts). Every rank walks from the junctions and the loop leaders among the
 * k-mers it owns; a walk reads the index, masks, visited flags and coverage of whichever rank owns each k-mer it meets, in place,
 * through cudaIpc mappings of the peers' arenas (the owners' per-bucket index rows are copied to every rank once). Link records
 * carry union slots. kmer_owners[b] / kpomer_owners[b]: the rank whose k-mer / (k+1)-mer set holds bucket b (kpomer_owners may be
 * NULL without coverage); kmer_bucket_sizes[b]: the union's k-mers in bucket b. budget_bytes sizes the junction batches (0: the
 * memory left). The extension index, its sets and indexes must stay alive until sgpu_dist_graph_free.
 *   begin (working copy of the masks, junction list) -> ipc_handle -> [all_gather descriptors] -> open_peers -> unitigs [barrier]
 *   -> clear_visited [barrier] -> ipc_handle -> [all_gather] -> open_peers -> loops [barrier] -> edges / bucket_counts -> free
 * (without perfect loops, stop after unitigs). A rank's edges are its unitigs in its final_kmers x out-edge order, then its loops
 * in its leaders' order; bucket_counts gives per bucket the unitig edges that start at a junction of that bucket and the loop
 * edges whose leader lies in it, so that the ranks' edges interleave into the single-GPU order: the unitig edges bucket by bucket,
 * then the loop edges bucket by bucket. */
#define SGPU_DIST_GRAPH_IPC_BYTES 256
typedef struct sgpu_dist_graph sgpu_dist_graph;
int sgpu_dist_graph_begin(sgpu_ctx *ctx, const sgpu_dist_ext *ext, const int32_t *kmer_owners, const int32_t *kpomer_owners,
                          const uint64_t *kmer_bucket_sizes, uint64_t budget_bytes, sgpu_dist_graph **out);
/* sgpu_dist_graph_begin with the Construction stage's early clippers (sgpu_graph_build_opts; keep_perfect_loops is the caller's
 * choice of running clear_visited and loops). The options are refused with SGPU_EINVAL as sgpu_graph_build_opts refuses them,
 * before anything is allocated; min_length > k is refused on every rank, whether it owns k-mers or not. Every rank passes the
 * same options. With a clipper on, the phases between the first open_peers and the unitigs are, each followed by a barrier:
 *   A/T clipper:  at_edges_probe, at_edges_apply, at_tips_probe, isolate, unlink
 *   tip clipper:  tip_probe, isolate, unlink
 *   then junctions (the junction list over the clipped masks)
 * A phase called out of order, or for a clipper that is off, is refused with SGPU_EINVAL and changes nothing. Every probe reads
 * the owners' masks as they were when the phase began: its flags are final on every rank before any rank's isolate or apply
 * changes a mask. The probes set the IsolateVertex and root flags in the owners' slices; at_edges_apply clears the deleted links'
 * bits in both k-mers' owners' masks (32-bit atomics: with the A/T clipper on, open_peers refuses a peer on another device
 * without native peer atomics); isolate and unlink change only this rank's slice. A rank allocates 1 B per owned k-mer for the
 * marks, 2 B for the tip clipper's flags and 4 B for the A/T clipper's, released by junctions. */
int sgpu_dist_graph_begin_opts(sgpu_ctx *ctx, const sgpu_dist_ext *ext, const int32_t *kmer_owners, const int32_t *kpomer_owners,
                               const uint64_t *kmer_bucket_sizes, uint64_t budget_bytes, const sgpu_graph_options *opts, sgpu_dist_graph **out);
int sgpu_dist_graph_at_edges_probe(sgpu_dist_graph *d);
int sgpu_dist_graph_at_edges_apply(sgpu_dist_graph *d);
int sgpu_dist_graph_at_tips_probe(sgpu_dist_graph *d);
int sgpu_dist_graph_tip_probe(sgpu_dist_graph *d);
int sgpu_dist_graph_isolate(sgpu_dist_graph *d);
int sgpu_dist_graph_unlink(sgpu_dist_graph *d);
int sgpu_dist_graph_junctions(sgpu_dist_graph *d);
/* after junctions: this rank's slice of what sgpu_graph_masks gives on one GPU over the union (the clipped masks, or the extension
 * index's when no clipper is on), n = this rank's k-mers */
int sgpu_dist_graph_masks(const sgpu_dist_graph *d, uint8_t *out, int64_t n);
/* this rank's counters: at4 and tc3 as sgpu_graph_at_clipper_stats / _tip_clipper_stats (the union's are the sums over the ranks),
 * remote3: the mark stores, root stores and bit clears that landed in another rank's slice */
int sgpu_dist_graph_clipper_stats(const sgpu_dist_graph *d, uint64_t *at4, uint64_t *tc3, uint64_t *remote3);
/* milliseconds spent so far in: A/T edges probe, A/T edges apply, A/T tips probe, tip probe, isolate (both clippers), unlink (both) */
int sgpu_dist_graph_clipper_times(const sgpu_dist_graph *d, float *out6);
int sgpu_dist_graph_ipc_handle(sgpu_dist_graph *d, uint8_t *out /* SGPU_DIST_GRAPH_IPC_BYTES */);
int sgpu_dist_graph_open_peers(sgpu_dist_graph *d, const uint8_t *descriptors /* world x SGPU_DIST_GRAPH_IPC_BYTES, rank-major */);
int sgpu_dist_graph_unitigs(sgpu_dist_graph *d);
int sgpu_dist_graph_clear_visited(sgpu_dist_graph *d);
int sgpu_dist_graph_loops(sgpu_dist_graph *d);
/* out4: this rank's edges, its unitig edges (the first ones), the bases of their text, its junction batches */
int sgpu_dist_graph_stats(const sgpu_dist_graph *d, uint64_t *out4);
/* this rank's edges: text (stats[2] bytes), lengths, link records (LinkRecord hash_and_mask, ~0 = self-conjugate end), raw coverage */
int sgpu_dist_graph_edges(const sgpu_dist_graph *d, char *seq, uint32_t *lens, uint64_t *link_start, uint64_t *link_end, uint32_t *raw_cov);
int sgpu_dist_graph_bucket_counts(const sgpu_dist_graph *d, uint64_t *unitig_counts /* num_buckets */, uint64_t *loop_counts /* num_buckets */);
/* milliseconds spent so far in: begin (mask copy + junction list), unitigs, clear_visited, loops */
int sgpu_dist_graph_times(const sgpu_dist_graph *d, float *out4);
void sgpu_dist_graph_free(sgpu_dist_graph *d);
/* a host-only graph from n assembled edges (text = the edges' bases concatenated, nbases = the sum of lens; every length >= k + 1):
 * sgpu_graph_num_unitigs / _unitig_bases / _unitigs / _gfa / _write_gfa / _free work on it, the device accessors (masks, coverage,
 * histogram, clipper statistics, sgpu_edge_index_build) return SGPU_EINVAL */
int sgpu_graph_from_edges(int k, const char *seq, int64_t nbases, const uint32_t *lens, const uint64_t *link_start, const uint64_t *link_end,
                          const uint32_t *raw_cov, int64_t n, sgpu_graph **out);

/* ---- multi-GPU EdgeIndex refill (one process per GPU): sgpu_edge_index_build over the union of the ranks' edges, from each rank's
 * sgpu_dist_graph after its walks. Every rank ends with the union's index (serialize, lookup and size give one GPU's bytes and slots)
 * and the values of its slot range [n r / W, n (r+1) / W) (values: as sgpu_edge_index_values gives them, with the union's edge ids).
 * K and num_buckets as sgpu_edge_index_build; every rank passes the same ones. unitig_counts_all / loop_counts_all: world x B
 * (rank-major; B = the graph's k-mer buckets) of every rank's sgpu_dist_graph_bucket_counts, from which each rank numbers its edges
 * in the order assemble_graph lays them out (more than 2^31 - 2 union edges: SGPU_EUNSUPPORTED).
 *   begin -> count_begin (an ordinary distributed count, sgpu_dist_*, over this rank's edges; free it before the index) ->
 *   keys -> ipc_handle -> [all_gather descriptors] -> open_peers ->
 *   repeat: [barrier] merge [barrier] advance -> [all_reduce SUM live] -> level_done (more = 0: placed) ->
 *   ranks [barrier] fill [barrier] -> values / serialize / lookup / size / slot_range / times -> free
 * count_begin: K = k + 1 counts into the graph's k-mer buckets (they only decide which rank owns a key; the index has one segment),
 * any other K into num_buckets (at most 8192). keys: this rank's set from that count (in HBM), the union's size of each of its
 * buckets (the sums of every rank's sgpu_kset_bucket_sizes), and, for K = k + 1, whether the index is serialized as the reference's
 * single-index branch (num_buckets > 1 and at least num_buckets / 2 distinct edge ends in the union; sgpu_edge_index_vertex_prefix_host
 * gives each rank's part of that decision). keys lays out the union's index on every rank, allocates this rank's slot slice and
 * inserts its keys into level 0 of its copy. merge: every rank's copy of the current level and of its collision words, read through
 * the peer mappings, merged into scratch; advance: the merge becomes the level, this rank's keys whose bit was cleared go into the
 * next level (live: this rank's keys still unplaced); level_done: the union's live keys (SGPU_EUNSUPPORTED when keys remain after
 * the last level). fill: every window of this rank's edges is put into its slot's owner's slice with a 64-bit system-scope CAS
 * (open_peers refuses a peer on another device without native peer atomics). Steps out of order are refused with SGPU_EINVAL.
 * Every rank holds the union's index (about 0.65 B per union key) and, until ranks, collision and merge words of the largest level
 * (about 1 B per union key). */
#define SGPU_DIST_EDGE_INDEX_IPC_BYTES 128
typedef struct sgpu_dist_edge_index sgpu_dist_edge_index;
int sgpu_dist_edge_index_begin(sgpu_ctx *ctx, const sgpu_dist_graph *dg, int K, int num_buckets, const uint64_t *unitig_counts_all,
                               const uint64_t *loop_counts_all, sgpu_dist_edge_index **out);
int sgpu_dist_edge_index_count_begin(sgpu_dist_edge_index *d, int world, int rank, sgpu_dist **out);
int sgpu_dist_edge_index_keys(sgpu_dist_edge_index *d, const sgpu_kset *keys, const uint64_t *union_bucket_sizes, int single);
int sgpu_dist_edge_index_ipc_handle(sgpu_dist_edge_index *d, uint8_t *out /* SGPU_DIST_EDGE_INDEX_IPC_BYTES */);
int sgpu_dist_edge_index_open_peers(sgpu_dist_edge_index *d, const uint8_t *descriptors /* world x SGPU_DIST_EDGE_INDEX_IPC_BYTES */);
int sgpu_dist_edge_index_merge(sgpu_dist_edge_index *d);
int sgpu_dist_edge_index_advance(sgpu_dist_edge_index *d, uint64_t *live);
int sgpu_dist_edge_index_level_done(sgpu_dist_edge_index *d, uint64_t union_live, int *more);
int sgpu_dist_edge_index_ranks(sgpu_dist_edge_index *d);
int sgpu_dist_edge_index_fill(sgpu_dist_edge_index *d);
int sgpu_dist_edge_index_values(const sgpu_dist_edge_index *d, uint64_t *edge_ids, uint32_t *offsets, int64_t n);   /* n = this rank's slots */
int sgpu_dist_edge_index_k(const sgpu_dist_edge_index *d);
int64_t sgpu_dist_edge_index_size(const sgpu_dist_edge_index *d);                     /* the union's K-mers (after ranks) */
int sgpu_dist_edge_index_slot_range(const sgpu_dist_edge_index *d, int64_t *lo, int64_t *hi);
int64_t sgpu_dist_edge_index_serialized_size(const sgpu_dist_edge_index *d);
int sgpu_dist_edge_index_serialize(const sgpu_dist_edge_index *d, uint8_t *out, int64_t cap);
int sgpu_dist_edge_index_lookup(const sgpu_dist_edge_index *d, const uint64_t *keys, int64_t n, uint64_t *out_idx);
/* host milliseconds spent so far in: begin (edge numbers and packing), keys, the levels (merges and advances), ranks, fill, values */
int sgpu_dist_edge_index_times(const sgpu_dist_edge_index *d, float *out6);
void sgpu_dist_edge_index_free(sgpu_dist_edge_index *d);
/* pure host arithmetic (no GPU): the union number of each of a rank's edges (unitig edges first, then loops, as its sgpu_dist_graph
 * lists them), as above; the sorted distinct vertex slots (LinkRecord >> 2; an end of ~0 is none) of n edges, the first
 * ceil(num_buckets / 2) of them into out (returns how many, -1 for bad arguments); a rank's slot range of n slots */
int sgpu_dist_edge_numbers_host(int world, int rank, int num_buckets, const int32_t *owners, const uint64_t *unitig_counts_all,
                                const uint64_t *loop_counts_all, uint64_t unitig_edges, uint64_t edges, uint64_t *out);
int64_t sgpu_edge_index_vertex_prefix_host(const uint64_t *link_start, const uint64_t *link_end, int64_t n, int num_buckets, uint64_t *out);
int sgpu_dist_slot_range_host(uint64_t n, int world, int rank, uint64_t *lo, uint64_t *hi);

/* self tests of the shared host/device arithmetic (tests only): op 0 = xxh3_64, 1 = xxh3_128 lo, 2 = xxh3_128 hi, 3 = bucket(arg),
 * 4 = is_minimal, 5.. = rc word j. keys: n records of ceil(K/32) words. on_device != 0 runs the same code in a kernel. */
int sgpu_selftest(sgpu_ctx *ctx, int on_device, int op, int K, uint64_t arg, const uint64_t *keys, int64_t n, uint64_t *out);

#ifdef __cplusplus
}
#endif
#endif
