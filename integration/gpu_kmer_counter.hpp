// integration/gpu_kmer_counter.hpp -- the reference-side adapters of INTEGRATION.md as compilable code.
//
// Header-only C++ that a SPAdes maintainer drops into src/common/kmer_index/kmer_mph/: it implements the reference's OWN
// interfaces on top of the C ABI of libspades_b200.so (include/spades_b200.h), so everything downstream in SPAdes
// (KMerDiskStorage::merge, KMerIndexBuilder, DeBruijnExtensionIndexBuilder::BuildExtensionIndexFromKPOMers,
// CoverageHashMapBuilder, the hammer / ionhammer / mts clients) consumes the result unchanged.
//
//   kmers::GpuKMerDiskCounter      kmers::KMerCounter<RtSeq>  (kmer_index/kmer_mph/kmer_index_builder.hpp:259-282)
//                                  replacing KMerDiskCounter<RtSeq> + its splitter (:284-431, kmer_splitters.hpp:28-136,
//                                  projects/spades_tools/kmercount.cpp:48-122)
//   kmers::BuildIndexOnGpu         KMerIndexBuilder<Index>::BuildIndex(index, storage) (:448-498) through
//                                  KMerIndex::deserialize (kmer_index.hpp:110-124)
//
// It is compiled against the UNMODIFIED reference headers by integration/Makefile (where the reference sources are, like oracle/_ref).
#pragma once
#include <sstream>
#include <string>

#include "sequence/rtseq.hpp"
#include "sequence/sequence.hpp"
#include "kmer_index/kmer_mph/kmer_index_traits.hpp"
#include "kmer_index/kmer_mph/kmer_index.hpp"
#include "kmer_index/kmer_mph/kmer_index_builder.hpp"
#include "spades_b200.h"

namespace kmers {

// Seq = RtSeq for the assembler's own clients (spades-kmercount, Construction, EdgeIndex, MTS' KmerMultiplicityCounter,
// projects/mts/kmer_multiplicity_counter.cpp:156-161) or a fixed-length Seq<K> such as BayesHammer's hammer::KMer = Seq<21>
// (projects/hammer/kmer_stat.hpp:32-33, kmer_data.cpp:40-47,333-344): both pack 2 bits per nucleotide from bit 0 of word 0 and hash
// their words with XXH3 (rtseq.hpp:690-696, seq.hpp:465-471), so records and buckets are the same bytes.
template<class Seq>
class GpuKMerDiskCounterT : public KMerCounter<Seq> {
  public:
    // mode: SGPU_ALL_WINDOWS = every window and its reverse complement (spades-kmercount's splitter, kmercount.cpp:48-122; BayesHammer's
    //                          BufferFiller pushes seq and !seq, hammer/kmer_data.cpp:75-82),
    //       SGPU_CANONICAL   = DeBruijnReadKMerSplitter with the IsMinimal filter (kmer_splitters.hpp:112-136, storing_traits.hpp:92-101)
    // result_on_host: the counted set is kept in pinned host memory (SGPU_RESULT_ON_HOST), so it may be larger than the device; the
    // bucket files and the GPU index are made from it as from a device set, the graph phases need a device set
    GpuKMerDiskCounterT(fs::TmpDir work_dir, unsigned K, sgpu_ctx *ctx, int mode, bool result_on_host = false)
            : KMerCounter<Seq>(K), work_dir_(work_dir), ctx_(ctx), mode_(result_on_host ? (mode | SGPU_RESULT_ON_HOST) : mode) {
        check(sgpu_reads_clear(ctx_));
    }
    ~GpuKMerDiskCounterT() override { if (last_) sgpu_kset_free(last_); }

    // the payload of the reference's binary read records: Sequence::data(), ceil(size/32) words (sequence.hpp:808-830). Reads are
    // collected in a host batch and cross the C ABI kBatchReads at a time (one call per read would be 100 M calls for config 3).
    void AddRead(const Sequence &s) {
        if (s.size() == 0) return;
        const size_t nw = (s.size() + 31) / 32, w0 = words_.size();
        words_.resize(w0 + nw, 0);
        uint64_t *w = words_.data() + w0;
        for (size_t i = 0; i < s.size(); ++i) w[i >> 5] |= (uint64_t)s[i] << ((i & 31) << 1);          // rtseq.hpp:379-382 packing
        offs_.push_back((uint64_t)w0);
        lens_.push_back((uint32_t)s.size());
        if (lens_.size() >= kBatchReads) Flush();
    }
    // a stretch of nucleotides given as text (BayesHammer: the valid stretches ValidKMerGenerator walks, hammer/valid_kmer_generator.hpp)
    void AddString(const char *acgt, size_t n) {
        if (n == 0) return;
        const size_t nw = (n + 31) / 32, w0 = words_.size();
        words_.resize(w0 + nw, 0);
        uint64_t *w = words_.data() + w0;
        for (size_t i = 0; i < n; ++i) w[i >> 5] |= (uint64_t)dignucl(acgt[i]) << ((i & 31) << 1);
        offs_.push_back((uint64_t)w0);
        lens_.push_back((uint32_t)n);
        if (lens_.size() >= kBatchReads) Flush();
    }
    // one K-mer as a read of exactly K bases (MTS: DeBruijnKMerKMerSplitter over a k-mer file with K_source == K_target)
    void AddKMer(const Seq &kmer) {
        const size_t nw = Seq::GetDataSize(this->k()), w0 = words_.size();
        words_.insert(words_.end(), kmer.data(), kmer.data() + nw);
        offs_.push_back((uint64_t)w0);
        lens_.push_back((uint32_t)this->k());
        if (lens_.size() >= kBatchReads) Flush();
    }
    // every read of a stream (io::ReadStream<io::SingleReadSeq> and friends: `stream >> read` until eof(), read.sequence())
    template<class Stream>
    size_t AddStream(Stream &stream) {
        typename Stream::ReadT r;
        size_t n = 0;
        while (!stream.eof()) { stream >> r; AddRead(r.sequence()); ++n; }
        return n;
    }
    void Flush() {
        if (lens_.empty()) return;
        check(sgpu_reads_append_packed(ctx_, words_.data(), words_.size(), offs_.data(), lens_.data(), (int64_t)lens_.size()));
        words_.clear(); offs_.clear(); lens_.clear();
    }

    // a whole FASTA / FASTQ (plain or gzip) file through the library's ingest (kseq semantics + LongestValid, like io::EasyStream,
    // io_helper.cpp:21-35); returns the number of reads taken
    size_t AddFile(const std::string &path) {
        sgpu_read_batch *b = nullptr;
        if (sgpu_fastx_parse(path.c_str(), /* longest_valid */ 1, &b)) {
            std::string why = sgpu_read_batch_error(b);
            sgpu_read_batch_free(b);
            FATAL_ERROR("spades_b200: " << why);
        }
        Flush();                                                     // keep the order of reads added one by one before the file
        const size_t n = (size_t)sgpu_read_batch_num_reads(b);
        const int rc = sgpu_reads_append_batch(ctx_, b);
        sgpu_read_batch_free(b);
        check(rc);
        return n;
    }

    size_t kmer_size() const override { return Seq::GetDataSize(this->k()) * sizeof(typename Seq::DataType); }

    KMerDiskStorage<Seq> Count(unsigned num_buckets, unsigned /* num_threads */) override {
        Flush();
        if (last_) { sgpu_kset_free(last_); last_ = nullptr; }
        check(sgpu_count(ctx_, (int)this->k(), (int)num_buckets, mode_, &last_));
        INFO("K-mer counting done on the GPU. There are " << sgpu_kset_size(last_) << " kmers in total. ");
        KMerDiskStorage<Seq> res(work_dir_, this->k(), kmer::KMerSegmentPolicy<Seq>(num_buckets));
        // the storage creates (and keeps owning) the bucket files <prefix>.<i>; the library fills them
        std::string prefix;
        for (unsigned i = 0; i < num_buckets; ++i) {
            auto f = res.create(i);
            if (i == 0) { prefix = f->file().native(); prefix.resize(prefix.rfind('.')); }
        }
        check(sgpu_kset_write_buckets(last_, prefix.c_str()));
        return res;
    }

    KMerDiskStorage<Seq> CountAll(unsigned num_buckets, unsigned num_threads, bool merge = true) override {
        auto storage = Count(num_buckets, num_threads);
        if (merge) storage.merge();
        return storage;
    }

    const sgpu_kset *device_set() const { return last_; }      // the same set, still resident (HBM or host memory), for the GPU index / graph phases

  private:
    void check(int rc) const { if (rc) FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx_)); }          // logger.hpp:185-261 convention
    fs::TmpDir work_dir_;
    sgpu_ctx *ctx_;
    int mode_;
    sgpu_kset *last_ = nullptr;
    static constexpr size_t kBatchReads = 1u << 20;
    std::vector<uint64_t> words_, offs_;
    std::vector<uint32_t> lens_;
};
using GpuKMerDiskCounter = GpuKMerDiskCounterT<RtSeq>;

// The splitter-level seam: kmers::KMerSplitter<RtSeq> (kmer_splitter.hpp:25-53). Split() leaves, per bucket, ONE sorted-unique run
// of W-byte records in <tmp>/kmers_raw.<i> plus <file>.idx holding its length (what KMerSortingSplitter::DumpBuffers appends per
// dump, kmer_splitter.hpp:123-170), so the reference's own KMerDiskCounter<RtSeq>(work_dir, GpuKMerSplitter(...)) merges them
// (one run each: a copy) and everything downstream is untouched:
//     kmers::KMerDiskCounter<RtSeq> counter(workdir, kmers::GpuKMerSplitter(workdir, K, ctx, SGPU_CANONICAL));
//     auto storage = counter.Count(num_buckets, nthreads);
// Reads are added to the context beforehand (GpuKMerDiskCounter::AddRead / AddFile or sgpu_reads_* directly).
class GpuKMerSplitter : public KMerSplitter<RtSeq> {
  public:
    using typename KMerSplitter<RtSeq>::RawKMers;
    GpuKMerSplitter(fs::TmpDir work_dir, unsigned K, sgpu_ctx *ctx, int mode) : KMerSplitter<RtSeq>(work_dir, K), ctx_(ctx), mode_(mode) {}
    GpuKMerSplitter(const std::filesystem::path &work_dir, unsigned K, sgpu_ctx *ctx, int mode)
            : KMerSplitter<RtSeq>(work_dir, K), ctx_(ctx), mode_(mode) {}

    RawKMers Split(size_t num_files, unsigned /* nthreads */) override {
        this->bucket_.reset(num_files);
        sgpu_kset *ks = nullptr;
        if (sgpu_count(ctx_, (int)this->K_, (int)num_files, mode_, &ks)) FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx_));
        RawKMers out;
        auto tmp_prefix = this->work_dir_->tmp_file("kmers_raw");
        for (unsigned i = 0; i < num_files; ++i) out.emplace_back(tmp_prefix->CreateDep(std::to_string(i)));
        std::string prefix = out[0]->file().native();
        prefix.resize(prefix.rfind('.'));
        if (sgpu_kset_write_buckets(ks, prefix.c_str())) { sgpu_kset_free(ks); FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx_)); }
        std::vector<int64_t> bsz(num_files);
        sgpu_kset_bucket_sizes(ks, bsz.data());
        for (unsigned i = 0; i < num_files; ++i) {                   // run lengths: one run per bucket
            const std::string idx = out[i]->file().native() + ".idx";
            FILE *f = fopen(idx.c_str(), "wb");
            if (!f) FATAL_ERROR("spades_b200: cannot write " << idx);
            const size_t n = (size_t)bsz[i];
            if (n) fwrite(&n, sizeof n, 1, f);
            fclose(f);
        }
        sgpu_kset_free(ks);
        return out;
    }

  private:
    sgpu_ctx *ctx_;
    int mode_;
};

// index: kmers::KMerIndex<traits>. KMerIndex befriends only KMerIndexBuilder (kmer_index.hpp:149-150) but deserialize is public
// and sgpu_mphf_serialize emits exactly the bytes KMerIndex::serialize writes.
template<class Index>
void BuildIndexOnGpu(Index &index, sgpu_ctx *ctx, const sgpu_kset *ks) {
    sgpu_mphf *m = nullptr;
    if (sgpu_mphf_build(ctx, ks, &m)) FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx));
    std::string bytes((size_t)sgpu_mphf_serialized_size(m), '\0');
    if (sgpu_mphf_serialize(m, (uint8_t *)&bytes[0], (int64_t)bytes.size())) FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx));
    sgpu_mphf_free(m);
    std::istringstream is(bytes);
    index.deserialize(is);
}

}  // namespace kmers
