// integration/spades_gbuilder_gpu.cpp -- the condensed-graph half of the drop-in: spades-gbuilder's flow
// (projects/spades_tools/gbuilder.cpp:157-225) with the hot path on the GPU and EVERYTHING DOWNSTREAM done by the unmodified
// reference on the GPU's output:
//
//   GPU (C ABI)                                                     reference (compiled where it lies)
//   -----------------------------------------------------------     -------------------------------------------------------------
//   (k+1)-mers of reads, canonical      sgpu_count                  KMerDiskStorage owning the GPU-written bucket files
//   k-mers of the (k+1)-mers            sgpu_kmers_from_kpomers     kmers::BuildIndex(ext_index, counter, ...)  -- its own KMerIndexBuilder
//                                                                   over the GPU-written k-mer buckets, final_kmers, index.kmers_
//   extension masks                     sgpu_graph_build/_masks --> DeBruijnExtensionIndex<>::raw_data()       (kmer_extension_index.hpp:83-84)
//   (k+1)-mer multiplicities            sgpu_graph_coverage     --> PerfectHashMap<RtSeq,uint32_t>::values()   (stages/construction.cpp:371-395)
//                                                                   UnbranchingPathExtractor::ExtractUnbranchingPathsAndLoops
//                                                                   FastGraphFromSequencesConstructor::ConstructGraph
//                                                                   FillCoverageAndFlankingFromPHM, gfa::GFAWriter
//   unitigs, GFA                        sgpu_graph_unitigs/_gfa     compared with the reference's, byte for byte
//
// This only works because the GPU's MPHF is bit-identical to the one the reference builds: the mask / coverage arrays are indexed
// by it. Exit code 0 iff the reference, fed with the GPU's arrays, extracts the GPU's unitigs and writes the GPU's GFA.
//
//   spades_gbuilder_gpu <reads (FASTA/FASTQ[.gz] or one read per line)> <k> <workdir> [num_buckets=16] [early_tip_length_bound=0]
//                       [--host-result] [--fastg]
//
// --host-result: both counts keep their sets in host memory (SGPU_RESULT_ON_HOST), so they may be larger than the device, and the
// graph comes from sgpu_graph_build_streamed, which reads the sets chunk by chunk. The checks against the reference are the same.
// --fastg: also gbuilder's other two outputs. The GPU writes graph.fastg (sgpu_graph_write_fastg) and unitigs.fasta
// (sgpu_graph_write_unitigs_fasta); the reference writes graph_ref.fastg with io::FastgWriter over its own graph, graph_nocov_ref.fastg
// with it before FillCoverageAndFlankingFromPHM (what gbuilder without -c writes), and unitigs_ref.fasta with gbuilder's unitig loop
// (gbuilder.cpp:191-200) over its own unitigs. graph.fastg and unitigs.fasta must equal the reference's byte for byte.
#include "gpu_kmer_counter.hpp"

#include "kmer_index/ph_map/kmer_maps.hpp"
#include "kmer_index/ph_map/perfect_hash_map_builder.hpp"
#include "kmer_index/extension_index/kmer_extension_index.hpp"
#include "assembly_graph/core/graph.hpp"
#include "assembly_graph/construction/debruijn_graph_constructor.hpp"
#include "assembly_graph/construction/early_simplification.hpp"
#include "assembly_graph/graph_support/coverage_filling.hpp"
#include "io/graph/gfa_writer.hpp"
#include "io/graph/fastg_writer.hpp"
#include "io/reads/header_naming.hpp"
#include "io/reads/osequencestream.hpp"
#include "utils/logger/log_writers.hpp"
#include "utils/filesystem/temporary.hpp"
#include "version.hpp"

#include <fstream>
#include <iostream>
#include <sstream>
#include <vector>

using namespace debruijn_graph;

static void create_console_logger() {
    using namespace logging;
    logger *lg = create_logger("");
    lg->add_writer(std::make_shared<console_writer>());
    attach_logger(lg);
}

// kmers::KMerCounter<RtSeq> over the k-mers of an already counted (k+1)-mer set: replaces KMerDiskCounter over
// DeBruijnKMerKMerSplitter (kmer_extension_index_builder.hpp:83-96, kmer_splitters.hpp:138-207)
class GpuKmersFromKpomersCounter : public kmers::KMerCounter<RtSeq> {
  public:
    // mode: 0, or SGPU_RESULT_ON_HOST to keep the k-mer set in host memory
    GpuKmersFromKpomersCounter(fs::TmpDir work_dir, unsigned k, sgpu_ctx *ctx, const sgpu_kset *kpomers, int mode = 0)
            : kmers::KMerCounter<RtSeq>(k), work_dir_(work_dir), ctx_(ctx), kpomers_(kpomers), mode_(mode) {}
    ~GpuKmersFromKpomersCounter() override { if (last_) sgpu_kset_free(last_); }
    size_t kmer_size() const override { return RtSeq::GetDataSize(this->k()) * sizeof(RtSeq::DataType); }
    kmers::KMerDiskStorage<RtSeq> Count(unsigned num_buckets, unsigned) override {
        if (sgpu_kmers_from_kpomers_ex(ctx_, kpomers_, (int)num_buckets, mode_, &last_)) FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx_));
        kmers::KMerDiskStorage<RtSeq> res(work_dir_, this->k(), kmer::KMerSegmentPolicy<RtSeq>(num_buckets));
        std::string prefix;
        for (unsigned i = 0; i < num_buckets; ++i) {
            auto f = res.create(i);
            if (i == 0) { prefix = f->file().native(); prefix.resize(prefix.rfind('.')); }
        }
        if (sgpu_kset_write_buckets(last_, prefix.c_str())) FATAL_ERROR("spades_b200: " << sgpu_last_error(ctx_));
        return res;
    }
    kmers::KMerDiskStorage<RtSeq> CountAll(unsigned num_buckets, unsigned num_threads, bool merge = true) override {
        auto storage = Count(num_buckets, num_threads);
        if (merge) storage.merge();
        return storage;
    }
    const sgpu_kset *device_set() const { return last_; }

  private:
    fs::TmpDir work_dir_;
    sgpu_ctx *ctx_;
    const sgpu_kset *kpomers_;
    int mode_;
    sgpu_kset *last_ = nullptr;
};

#define CK(call) do { if (int rc_ = (call)) { fprintf(stderr, "spades_b200 error %d: %s\n", rc_, sgpu_last_error(ctx)); return 4; } } while (0)

static std::string file_text(const std::filesystem::path &p) {
    std::ifstream f(p, std::ios::binary);
    std::ostringstream s;
    s << f.rdbuf();
    return s.str();
}

int main(int argc, char **argv) {
    bool host_result = false, fastg = false;
    while (argc > 4) {                                   // trailing flags, in any order
        const std::string a = argv[argc - 1];
        if (a == "--host-result") host_result = true;
        else if (a == "--fastg") fastg = true;
        else break;
        --argc;
    }
    if (argc < 4) { fprintf(stderr, "usage: %s reads k workdir [num_buckets] [early_tip_length_bound] [--host-result] [--fastg]\n", argv[0]); return 2; }
    const std::string reads_path = argv[1];
    const unsigned k = (unsigned)atoi(argv[2]);
    const std::filesystem::path workdir = argv[3];
    const unsigned B = argc > 4 ? (unsigned)atoi(argv[4]) : 16;
    const uint64_t early_tc = argc > 5 ? (uint64_t)atoll(argv[5]) : 0;
    create_console_logger();
    std::filesystem::create_directories(workdir);
    if (k % 2 == 0) { fprintf(stderr, "k must be odd\n"); return 2; }          // gbuilder.cpp:125

    sgpu_config cfg = {0, 0, 0, 0};
    sgpu_ctx *ctx = nullptr;
    if (int rc = sgpu_create(&cfg, &ctx)) {
        fprintf(stderr, "spades_gbuilder_gpu: cannot create a GPU context (error %d): there is no CPU fallback\n", rc);
        return 3;
    }
    int bad = 0;
    {
        auto tmp = fs::tmp::make_temp_dir(workdir, "construction");
        // ---- (k+1)-mers on the GPU
        kmers::GpuKMerDiskCounter kpomer_counter(tmp, k + 1, ctx, SGPU_CANONICAL, host_result);
        {
            std::ifstream is(reads_path, std::ios::binary);
            const int c0 = is.get(), c1 = is.get();
            is.seekg(0);
            if (c0 == '>' || c0 == '@' || (c0 == 0x1f && c1 == 0x8b)) { is.close(); kpomer_counter.AddFile(reads_path); }
            else { std::string line; while (std::getline(is, line)) if (!line.empty()) kpomer_counter.AddRead(Sequence(line)); }
        }
        auto kpomers = kpomer_counter.Count(B, 1);
        // ---- k-mers on the GPU, the extension index's MPHF by the reference's own builder over the GPU-written buckets
        kmers::DeBruijnExtensionIndex<> ext(k);
        GpuKmersFromKpomersCounter kmer_counter(tmp, k, ctx, kpomer_counter.device_set(), host_result ? SGPU_RESULT_ON_HOST : 0);
        kmers::BuildIndex(ext, kmer_counter, B, 1);                  // KeyIteratingIndexBuilder: index + data_ size + kmers_ = final_kmers
        // ---- masks / coverage / unitigs / GFA on the GPU
        sgpu_mphf *mk = nullptr, *mkp = nullptr;
        sgpu_graph *gg = nullptr;
        CK(sgpu_mphf_build(ctx, kmer_counter.device_set(), &mk));
        CK(sgpu_mphf_build(ctx, kpomer_counter.device_set(), &mkp));
        if (host_result) {
            const sgpu_graph_options o = {/* keep_perfect_loops */ 1, early_tc, 0, 0.8, 10, 200};
            CK(sgpu_graph_build_streamed(ctx, kpomer_counter.device_set(), kmer_counter.device_set(), mk, mkp, &o, &gg));
        } else {
            CK(sgpu_graph_build_ex(ctx, kpomer_counter.device_set(), kmer_counter.device_set(), mk, mkp, /* keep_perfect_loops */ 1, early_tc, &gg));
        }
        if ((size_t)sgpu_kset_size(kmer_counter.device_set()) != ext.size()) { ERROR("k-mer count differs from the reference index size"); ++bad; }
        // the GPU's mask array straight into the reference's extension index (after the early tip clipper, if requested)
        CK(sgpu_graph_masks(gg, (uint8_t *)ext.raw_data(), (int64_t)ext.raw_size()));
        // ---- the reference takes over: unitigs
        std::vector<Sequence> edges = UnbranchingPathExtractor(ext, k).ExtractUnbranchingPathsAndLoops(16);
        {
            const int64_t ne = sgpu_graph_num_unitigs(gg), nb = sgpu_graph_unitig_bases(gg);
            std::string buf((size_t)nb, '\0');
            std::vector<uint32_t> lens((size_t)ne);
            CK(sgpu_graph_unitigs(gg, &buf[0], lens.data()));
            bool same = (size_t)ne == edges.size();
            size_t off = 0;
            for (size_t i = 0; same && i < edges.size(); ++i) { same = edges[i].str() == buf.substr(off, lens[i]); off += lens[i]; }
            if (!same) { ERROR("the reference's unitigs over the GPU's masks differ from the GPU's unitigs"); ++bad; }
            else INFO("Unitigs agree: " << edges.size());
        }
        // ---- the reference's graph, coverage from the GPU, the reference's GFA writer
        DeBruijnGraph g(k);
        FastGraphFromSequencesConstructor<DeBruijnGraph>(k, ext).ConstructGraph(g, edges);
        using CoverageMap = kmers::PerfectHashMap<RtSeq, uint32_t, kmers::slim_kmer_index_traits<RtSeq>, kmers::DefaultStoring>;
        CoverageMap coverage_map(k + 1);
        kmers::BuildIndex(coverage_map, kpomers, 1);                  // the reference's MPHF over the GPU-written (k+1)-mer buckets
        if (coverage_map.values().size() != (size_t)sgpu_kset_size(kpomer_counter.device_set())) { ERROR("(k+1)-mer count differs"); ++bad; }
        else CK(sgpu_graph_coverage(gg, coverage_map.values().data(), (int64_t)coverage_map.values().size()));
        if (fastg) io::FastgWriter(g, workdir / "graph_nocov_ref.fastg").WriteSegmentsAndLinks();
        omnigraph::FlankingCoverage<DeBruijnGraph> flanking_cov(g, 50);
        FillCoverageAndFlankingFromPHM(coverage_map, g, flanking_cov);
        if (fastg) {
            io::FastgWriter(g, workdir / "graph_ref.fastg").WriteSegmentsAndLinks();
            {
                size_t idx = 1;
                std::ofstream f(workdir / "unitigs_ref.fasta");
                for (const auto &edge : edges) {
                    f << std::string(">") << io::MakeContigId(idx++, edge.size(), "EDGE") << std::endl;
                    io::WriteWrapped(edge.str(), f);
                }
            }
            CK(sgpu_graph_write_fastg(ctx, gg, (workdir / "graph.fastg").c_str()));
            CK(sgpu_graph_write_unitigs_fasta(ctx, gg, (workdir / "unitigs.fasta").c_str()));
            const std::string gf = file_text(workdir / "graph.fastg"), uf = file_text(workdir / "unitigs.fasta");
            if (gf != file_text(workdir / "graph_ref.fastg")) { ERROR("the GPU's FASTG differs from the reference's FastgWriter output"); ++bad; }
            else INFO("FASTG agrees: " << gf.size() << " bytes");
            if (uf != file_text(workdir / "unitigs_ref.fasta")) { ERROR("the GPU's unitig FASTA differs from the reference's"); ++bad; }
            else INFO("Unitig FASTA agrees: " << uf.size() << " bytes");
        }
        std::ostringstream ref_gfa;
        { gfa::GFAWriter w(g, ref_gfa); w.WriteSegmentsAndLinks(); }
        const std::string version = std::string(version::flavour()) + "-" + version::package();      // what GFAWriter prints (gfa_writer.cpp:115)
        const int64_t n = sgpu_graph_gfa(gg, version.c_str(), nullptr, 0);
        std::string gpu_gfa((size_t)(n > 0 ? n : 0), '\0');
        if (n > 0) sgpu_graph_gfa(gg, version.c_str(), &gpu_gfa[0], n);
        if (ref_gfa.str() != gpu_gfa) { ERROR("the reference's GFA over the GPU's arrays differs from the GPU's GFA"); ++bad; }
        else INFO("GFA agrees: " << gpu_gfa.size() << " bytes");
        { std::ofstream f(workdir / "graph.gfa"); f << ref_gfa.str(); }
        { std::ofstream f(workdir / "graph_gpu.gfa"); f << gpu_gfa; }
        sgpu_graph_free(gg); sgpu_mphf_free(mk); sgpu_mphf_free(mkp);
    }
    sgpu_destroy(ctx);
    return bad ? 1 : 0;
}

namespace llvm {      // see oracle/ref_probe.cpp
TimeTraceProfiler *getTimeTraceProfilerInstance() { return nullptr; }
void timeTraceProfilerBegin(StringRef, StringRef) {}
void timeTraceProfilerEnd() {}
}
