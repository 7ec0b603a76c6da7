// integration/spades_kmercount_gpu.cpp -- spades-kmercount (projects/spades_tools/kmercount.cpp:191-230) with the counter
// swapped for the GPU adapter: REFERENCE host code (KMerDiskStorage, KMerIndexBuilder, KMerIndex, RtSeq, Sequence, fs::TmpDir,
// logger -- all unmodified, compiled where they lie) calling hand-written sm_90a CUDA through the C ABI.
//
//   spades_kmercount_gpu <reads.txt> <k> <workdir> [num_buckets=16] [--host-result]
//
// --host-result: the count's result stays in host memory (SGPU_RESULT_ON_HOST) instead of HBM; the tool needs only final_kmers,
// so its result may be larger than the device.
//
// reads: FASTA / FASTQ, plain or gzip (parsed by the library's ingest with the original tool's semantics: kseq records +
// LongestValid), or one ACGT read per line (ref_probe's format). Output: <workdir>/final_kmers, byte-identical to the original
// tool's. It then proves the GPU-written storage is a drop-in for the rest of SPAdes:
//   1. the reference's OWN KMerIndexBuilder::BuildIndex runs over the GPU-written bucket files,
//   2. the GPU-built MPHF goes through the reference's OWN KMerIndex::deserialize,
//   3. both indices map every k-mer of final_kmers to the same slot (and that map is a bijection onto [0, n)).
// Exit code 0 only if all of that holds.
#include "gpu_kmer_counter.hpp"
#include <iterator>

#include "kmer_index/kmer_mph/kmer_index_traits.hpp"
#include "kmer_index/kmer_mph/kmer_splitter.hpp"
#include "kmer_index/kmer_mph/kmer_splitters.hpp"
#include "kmer_index/ph_map/storing_traits.hpp"
#include "sequence/seq.hpp"
#include "utils/logger/log_writers.hpp"
#include "utils/filesystem/temporary.hpp"

#include <fstream>
#include <iostream>
#include <vector>

static void create_console_logger() {
    using namespace logging;
    logger *lg = create_logger("");
    lg->add_writer(std::make_shared<console_writer>());
    attach_logger(lg);
}

// ---- a second client of the counter API: BayesHammer's k-mer value type (hammer::KMer = Seq<21>, projects/hammer/kmer_stat.hpp:32-33).
// Reference side: a KMerSortingSplitter<Seq<21>> that pushes every window and its reverse complement, exactly what hammer's BufferFiller
// does with the k-mers ValidKMerGenerator yields (projects/hammer/kmer_data.cpp:61-85), driven by the reference's own KMerDiskCounter.
typedef Seq<21> HKMer;
class RefHammerLikeSplitter : public kmers::KMerSortingSplitter<HKMer> {
  public:
    using typename kmers::KMerSortingSplitter<HKMer>::RawKMers;
    RefHammerLikeSplitter(const std::filesystem::path &work_dir, const std::vector<std::string> &reads)
            : kmers::KMerSortingSplitter<HKMer>(work_dir, 21), reads_(reads) {}
    RawKMers Split(size_t num_files, unsigned) override {
        auto out = this->PrepareBuffers(num_files, 1, 0);
        for (const std::string &r : reads_) {
            if (r.size() < 21) continue;
            HKMer kmer(r, 0, 21);                               // the (string, offset, count) constructor; Seq(const char*) wants strlen == 21
            bool stop = false;
            for (size_t i = 21;; ++i) {
                stop |= this->push_back_internal(kmer, 0);
                stop |= this->push_back_internal(!kmer, 0);
                if (i >= r.size()) break;
                kmer = kmer << r[i];
            }
            if (stop) this->DumpBuffers(out);
        }
        this->DumpBuffers(out);
        this->ClearBuffers();
        return out;
    }
  private:
    const std::vector<std::string> &reads_;
};

static std::string slurp(const std::filesystem::path &p) {
    std::ifstream f(p, std::ios::binary);
    return std::string((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

// returns the number of problems found
static int hammer_client_check(sgpu_ctx *ctx, const std::vector<std::string> &reads, const std::filesystem::path &workdir, unsigned B) {
    int bad = 0;
    kmers::KMerDiskCounter<HKMer> ref(workdir, RefHammerLikeSplitter(workdir, reads));
    // unmerged storages first: bucket by bucket (KMerDiskStorage::merge drops the bucket list, kmer_index_builder.hpp:190-201)
    auto ref_storage = ref.CountAll(B, 1, /* merge */ false);
    kmers::GpuKMerDiskCounterT<HKMer> gpu(fs::tmp::make_temp_dir(workdir, "hammer_gpu"), 21, ctx, SGPU_ALL_WINDOWS);
    for (const std::string &r : reads) gpu.AddString(r.data(), r.size());
    auto gpu_storage = gpu.CountAll(B, 1, /* merge */ false);
    if (gpu_storage.total_kmers() != ref_storage.total_kmers()) { ERROR("hammer client: k-mer counts differ"); ++bad; }
    for (unsigned b = 0; b < B; ++b)
        if (gpu_storage.bucket_size(b) != ref_storage.bucket_size(b)) { ERROR("hammer client: bucket " << b << " differs in size"); ++bad; break; }
    typedef kmers::KMerIndex<kmers::kmer_index_traits<HKMer>> HIndex;                // HammerKMerIndex, projects/hammer/kmer_data.hpp:21
    HIndex index;
    kmers::KMerIndexBuilder<HIndex>(1).BuildIndex(index, gpu_storage);
    if (index.size() != gpu_storage.total_kmers()) { ERROR("hammer client: index size"); ++bad; }
    gpu_storage.merge();
    ref_storage.merge();
    if (slurp(gpu_storage.final_kmers()->file()) != slurp(ref_storage.final_kmers()->file())) { ERROR("hammer client: final_kmers differ"); ++bad; }
    if (!bad) INFO("hammer::KMer client (Seq<21>): GPU counter == reference KMerDiskCounter<Seq<21>> (" << gpu_storage.total_kmers() << " k-mers), index built");
    return bad;
}

int main(int argc, char **argv) {
    const bool host_result = argc > 4 && std::string(argv[argc - 1]) == "--host-result";
    if (host_result) --argc;
    if (argc < 4) { fprintf(stderr, "usage: %s reads.txt k workdir [num_buckets] [--host-result]\n", argv[0]); return 2; }
    const std::string reads_path = argv[1];
    const unsigned K = (unsigned)atoi(argv[2]);
    const std::filesystem::path workdir = argv[3];
    const unsigned B = argc > 4 ? (unsigned)atoi(argv[4]) : 16;      // kmercount.cpp:220
    create_console_logger();
    std::filesystem::create_directories(workdir);

    sgpu_config cfg = {0, 0, 0, 0};
    sgpu_ctx *ctx = nullptr;
    if (int rc = sgpu_create(&cfg, &ctx)) {
        fprintf(stderr, "spades_kmercount_gpu: cannot create a GPU context (error %d): there is no CPU fallback\n", rc);
        return 3;
    }
    INFO("K-mer length set to " << K);
    typedef kmers::KMerIndex<kmers::kmer_index_traits<RtSeq>> Index;
    int bad = 0;
    {
        kmers::GpuKMerDiskCounter counter(fs::tmp::make_temp_dir(workdir, "kmer_counter"), K, ctx, SGPU_ALL_WINDOWS, host_result);
        std::vector<std::string> plain_reads;                                  // kept for the Seq<21> client check below (K == 21 only)
        {
            std::ifstream is(reads_path, std::ios::binary);
            const int c0 = is.get(), c1 = is.get();
            is.seekg(0);
            if (c0 == '>' || c0 == '@' || (c0 == 0x1f && c1 == 0x8b)) {       // FASTA / FASTQ / gzip: what the original tool takes
                is.close();
                INFO("Parsed " << counter.AddFile(reads_path) << " reads from " << reads_path);
            } else {                                                            // one ACGT read per line (ref_probe's format)
                std::string line;
                while (std::getline(is, line))
                    if (!line.empty()) { counter.AddRead(Sequence(line)); if (K == 21) plain_reads.push_back(line); }
            }
        }
        auto storage = counter.Count(B, 1);                         // KMerDiskStorage<RtSeq>, buckets written from HBM (or host memory)
        const size_t total = storage.total_kmers();
        if (!storage.is_unique_and_sorted()) { ERROR("GPU-written buckets are not sorted/unique"); ++bad; }

        Index ref_index, gpu_index;
        kmers::KMerIndexBuilder<Index>(1).BuildIndex(ref_index, storage);         // 1. reference builder over GPU-written files
        kmers::BuildIndexOnGpu(gpu_index, ctx, counter.device_set());             // 2. GPU MPHF through the reference's deserialize
        if (ref_index.size() != total || gpu_index.size() != total) { ERROR("index sizes differ from the storage"); ++bad; }

        // 3. same slot for every k-mer, bijection
        std::vector<char> seen(total, 0);
        size_t checked = 0;
        for (unsigned b = 0; b < B && !bad; ++b) {
            for (auto it = storage.bucket_begin(b), e = storage.bucket_end(b); it != e; ++it) {
                const RtSeq kmer(K, (*it).first);
                const size_t a = ref_index.seq_idx(kmer), g = gpu_index.seq_idx(kmer);
                if (a != g || a >= total || seen[a]) { ERROR("index mismatch at k-mer " << kmer.str() << ": " << a << " vs " << g); ++bad; break; }
                seen[a] = 1; ++checked;
            }
        }
        if (checked != total) ++bad;
        INFO("Checked " << checked << " k-mers: reference-built and GPU-built KMerIndex agree");

        storage.merge();                                             // the reference's own merge (kmer_index_builder.hpp:190-203)
        auto final_kmers = storage.final_kmers();
        const std::filesystem::path out = workdir / "final_kmers";
        std::rename(final_kmers->file().c_str(), out.c_str());       // kmercount.cpp:222-223
        INFO("K-mer counting done, kmers saved to " << out);

        // 4. the splitter-level seam: the reference's OWN KMerDiskCounter over kmers::GpuKMerSplitter (one sorted-unique run + .idx per
        //    bucket) must arrive at the same final_kmers
        {
            kmers::KMerDiskCounter<RtSeq> ref_counter(workdir, kmers::GpuKMerSplitter(workdir, K, ctx, SGPU_ALL_WINDOWS));
            auto st2 = ref_counter.CountAll(B, 1, /* merge */ true);
            std::ifstream a(out, std::ios::binary), b2(st2.final_kmers()->file(), std::ios::binary);
            const std::string sa((std::istreambuf_iterator<char>(a)), std::istreambuf_iterator<char>());
            const std::string sb((std::istreambuf_iterator<char>(b2)), std::istreambuf_iterator<char>());
            if (st2.total_kmers() != total || sa != sb) { ERROR("KMerDiskCounter over GpuKMerSplitter differs from GpuKMerDiskCounter"); ++bad; }
            else INFO("reference KMerDiskCounter over GpuKMerSplitter: identical final_kmers (" << st2.total_kmers() << " k-mers)");
        }
        // 5. another client of the same API with its own k-mer value type (SURVEY 8f-4)
        if (K == 21 && !plain_reads.empty()) bad += hammer_client_check(ctx, plain_reads, workdir, B);
        // 6. MTS' KmerMultiplicityCounter::BuildKmerIndex (projects/mts/kmer_multiplicity_counter.cpp:149-163): a k-mer FILE goes through
        //    DeBruijnKMerKMerSplitter(K -> K, add_rc) + KMerDiskCounter with 16 buckets = canonicalise + dedup. GPU: every k-mer is a read
        //    of exactly K bases, canonical count.
        {
            using KMerStorage = kmers::KMerDiskStorage<RtSeq>;
            kmers::DeBruijnKMerKMerSplitter<kmers::StoringTypeFilter<kmers::InvertableStoring>, KMerStorage::kmer_iterator>
                    splitter(fs::tmp::make_temp_dir(workdir, "mts_ref"), K, K, true, 0);
            splitter.AddKMers(adt::make_range(KMerStorage::kmer_iterator(out, K), KMerStorage::kmer_iterator()));
            kmers::KMerDiskCounter<RtSeq> mts_ref_counter(workdir, std::move(splitter));
            auto ref_st = mts_ref_counter.CountAll(16, 1, true);
            kmers::GpuKMerDiskCounter gpu_counter(fs::tmp::make_temp_dir(workdir, "mts_gpu"), K, ctx, SGPU_CANONICAL);
            for (auto it = KMerStorage::kmer_iterator(out, K), e = KMerStorage::kmer_iterator(); it != e; ++it) gpu_counter.AddKMer(RtSeq(K, (*it).first));
            auto gpu_st = gpu_counter.CountAll(16, 1, true);
            if (gpu_st.total_kmers() != ref_st.total_kmers() || slurp(gpu_st.final_kmers()->file()) != slurp(ref_st.final_kmers()->file())) {
                ERROR("MTS client: canonical k-mer sets differ"); ++bad;
            } else INFO("MTS client (k-mer file -> canonical set, 16 buckets): GPU counter == reference (" << gpu_st.total_kmers() << " k-mers)");
        }
    }
    sgpu_destroy(ctx);
    return bad ? 1 : 0;
}

namespace llvm {      // see oracle/ref_probe.cpp: the profiler hooks are no-ops unless the profiler was initialised
TimeTraceProfiler *getTimeTraceProfilerInstance() { return nullptr; }
void timeTraceProfilerBegin(StringRef, StringRef) {}
void timeTraceProfilerEnd() {}
}
