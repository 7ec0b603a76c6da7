// graph.h -- condensed de Bruijn graph artefacts (device masks/coverage + host unitigs and link records)
#pragma once
#include <string>
#include <vector>

#include "sgpu_internal.h"

namespace sg {

struct Graph {
    Ctx *ctx = nullptr;
    int k = 0;
    const KSet *kp = nullptr, *km = nullptr;
    const Mphf *mk = nullptr, *mkp = nullptr;
    DArr<uint8_t> masks;         // working copy (mutated by RemoveSequences semantics), k-mer MPHF order
    DArr<uint8_t> masks_final;   // extension masks as the reference's DeBruijnExtensionIndex holds them
    DArr<uint32_t> cov;          // (k+1)-mer multiplicities, (k+1)-mer MPHF order (the reference's coverage_map)
    // edges in the reference's order: unbranching paths in final_kmers x out-edge order, then perfect loops
    std::string seq;             // ASCII, concatenated
    std::vector<uint64_t> edge_off;
    std::vector<uint32_t> edge_len;
    std::vector<uint64_t> link_start, link_end;   // LinkRecord::hash_and_mask_ (debruijn_graph_constructor.hpp:422-452)
    std::vector<uint32_t> raw_cov;                // CoverageIndex raw coverage per edge
    uint64_t tc_stats[3] = {0, 0, 0};             // early tip clipper: removed k-mers, tipped junctions, clipped links
    uint64_t at_stats[4] = {0, 0, 0, 0};          // early A/T clipper: edges collected, links removed, k-mers removed, clipped tips
};

struct GraphOptions {
    bool keep_perfect_loops = true;
    uint64_t early_tip_length_bound = 0;          // 0 = no early tip clipper
    bool early_at = false;                        // early low-complexity (poly A/T) clipper of the RNA pipeline, before the tip clipper
    double at_ratio = 0.8;
    uint64_t at_min_len = 10, at_max_len = 200;
};

Graph *graph_build(Ctx *ctx, const KSet *kp, const KSet *km, const Mphf *mk, const Mphf *mkp, const GraphOptions &opt);
std::vector<uint64_t> graph_histogram(Ctx *ctx, const Graph *g);
// the same two steps outside a graph build: cov[mphf(kpomer)] = multiplicity over a sweep of the (k+1)-mers (cov zeroed by the
// caller, one entry per key of the index), and the histogram of n coverage values (hist[c - 1] += 2, as long as the largest c)
void coverage_fill(Ctx *ctx, ChunkStager &kpomers, const Mphf *mkp, uint32_t *cov);
std::vector<uint64_t> coverage_histogram(Ctx *ctx, const uint32_t *cov, int64_t n);

// dist_graph.cu : the early clippers, unitigs and perfect loops of one rank's share of a distributed graph
// (DistributedGraphConstructor), from its extension index slices (dist_ext.cu). Phases, with a barrier between them: begin (a
// working copy of the masks; the junction list when no clipper is on), ipc_handle / open_peers, the clippers' phases and the
// junction list (dgraph_clip_phase), unitigs, clear_visited, ipc_handle / open_peers again (the remaining slots' positions), loops.
struct DistGraph;
struct ExtDist;
DistGraph *dgraph_begin(Ctx *ctx, const ExtDist *ext, const int *kmer_owner, const int *kpomer_owner, const uint64_t *kmer_bucket_sizes, uint64_t budget,
                        const GraphOptions &opt);
void dgraph_ipc_handle(DistGraph *d, uint8_t *out256);
void dgraph_open_peers(DistGraph *d, const uint8_t *descs);
// the phases between begin and the unitigs, in the order they run (a clipper's phases only when it is on)
enum { kAtEdgesProbe, kAtEdgesApply, kAtTipsProbe, kAtIsolate, kAtUnlink, kTipProbe, kTipIsolate, kTipUnlink, kJunctions };
// the next of them, when it is phase a or b; refuses any other
void dgraph_clip_phase(DistGraph *d, int a, int b);
void dgraph_unitigs(DistGraph *d);
void dgraph_clear_visited(DistGraph *d);
void dgraph_loops(DistGraph *d);
const Graph &dgraph_edges(const DistGraph *d);                   // its unitigs in its final_kmers order, then its loops
void dgraph_stats(const DistGraph *d, uint64_t *out4);           // edges, unitig edges, bases, junction batches
void dgraph_bucket_counts(const DistGraph *d, uint64_t *unitigs, uint64_t *loops);
void dgraph_times(const DistGraph *d, float *out4);
void dgraph_clip_times(const DistGraph *d, float *out6);         // A/T edges probe, A/T edges apply, A/T tips probe, tip probe, isolate, unlink
void dgraph_clip_stats(const DistGraph *d, uint64_t *at4, uint64_t *tc3, uint64_t *remote3);
void dgraph_masks(const DistGraph *d, uint8_t *out, int64_t n);  // the clipped slice (the extension index's when no clipper ran)
void dgraph_free(DistGraph *d);

// edge_index.cu : KmerFreeEdgeIndex refill over the graph's own unitigs (alignment/edge_index.hpp, assembly_graph/index/edge_index_builders.hpp)
struct EdgeIndex {
    Ctx *ctx = nullptr;
    int K = 0;
    bool single_segment = false;   // K == k+1: built like KMerIndexBuilder's single-index branch (its segment_starts_[1] stays 0)
    KSet *ks = nullptr;            // the minimal form of every K-mer of every edge (owned)
    Mphf *m = nullptr;             // its KMerIndex (owned)
    DArr<uint64_t> edge_id;        // per MPHF slot: EdgeId::int_id(), ~1 = removed (the K-mer occurs more than once), ~0 = cleared
    DArr<uint32_t> offset;         // per MPHF slot: offset on that edge (EdgeInfo::TOMBSTONE / CLEARED otherwise)
    ~EdgeIndex();
};
EdgeIndex *edge_index_build(Ctx *ctx, const Graph *g, int K, int num_buckets);

// host_graph.cpp : FastGraphFromSequencesConstructor::ConstructGraph + GFAWriter
std::string graph_gfa(const Graph *g, const char *version);
std::vector<std::string> graph_gfa_chunks(const Graph *g, const char *version);   // the same text in consecutive pieces (built on the host threads)

}  // namespace sg
