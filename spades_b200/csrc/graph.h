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
// what the distributed EdgeIndex refill reads of a rank's share of the graph
struct DistGraphInfo {
    Ctx *ctx;
    int world, rank, B, k;
    const std::vector<int> *owner;                    // B: the rank owning each k-mer bucket
    const std::vector<uint64_t> *ucnt, *lcnt;         // B: this rank's unitig edges by start junction's bucket, loop edges by leader's
    uint64_t unitig_edges;
    const Graph *edges;
};
DistGraphInfo dgraph_info(const DistGraph *d);
void dgraph_free(DistGraph *d);
// the visible device with this UUID, -1 if none
int device_of(const cudaUUID_t &u);

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
// the sorted distinct vertex slots (LinkRecord >> 2) of g's edge ends, the first `cap` of them
std::vector<uint64_t> edge_vertex_slots(const Graph *g, uint64_t cap);

// dist_edge_index.cu : the EdgeIndex refill across GPUs (DistributedEdgeIndex), from each rank's share of a distributed graph. Every
// rank ends with the union's index and the values of its slot range.
struct DistEdgeIndex;
DistEdgeIndex *dei_begin(Ctx *ctx, const DistGraph *dg, int K, int num_buckets, const uint64_t *ucnt_all, const uint64_t *lcnt_all);
DistState *dei_count_begin(DistEdgeIndex *d, int world, int rank);
void dei_keys(DistEdgeIndex *d, const KSet *ks, const uint64_t *union_bucket_sizes, int single);
void dei_ipc_handle(DistEdgeIndex *d, uint8_t *out128);
void dei_open_peers(DistEdgeIndex *d, const uint8_t *descs);
void dei_merge(DistEdgeIndex *d);
uint64_t dei_advance(DistEdgeIndex *d);
int dei_level_done(DistEdgeIndex *d, uint64_t union_live);     // 1: another level follows
void dei_ranks(DistEdgeIndex *d);
void dei_fill(DistEdgeIndex *d);
void dei_values(const DistEdgeIndex *d, uint64_t *ids, uint32_t *offs, int64_t n);
const Mphf *dei_index(const DistEdgeIndex *d);
bool dei_single(const DistEdgeIndex *d);
int dei_k(const DistEdgeIndex *d);
void dei_slot_range(const DistEdgeIndex *d, uint64_t *lo, uint64_t *hi);
void dei_times(const DistEdgeIndex *d, float *out6);
void dei_free(DistEdgeIndex *d);
// pure host arithmetic (exported for CPU tests): the union number of each of a rank's edges, in assemble_graph's order (the unitig
// edges bucket by bucket, each bucket's from its owner, then the loop edges bucket by bucket); and a rank's slot range
void dist_edge_numbers(int world, int rank, int B, const int *owner, const uint64_t *ucnt_all, const uint64_t *lcnt_all, uint64_t unitig_edges,
                       uint64_t edges, uint64_t *out);
__host__ __device__ inline uint64_t dist_slot_lo(uint64_t n, int world, int r) { return n * (uint64_t)r / (uint64_t)world; }

// host_graph.cpp : FastGraphFromSequencesConstructor::ConstructGraph + GFAWriter
std::string graph_gfa(const Graph *g, const char *version);
std::vector<std::string> graph_gfa_chunks(const Graph *g, const char *version);   // the same text in consecutive pieces (built on the host threads)

}  // namespace sg
