// edge_index.cu -- the EdgeIndex refill (SURVEY 8f-1): the very next consumer of the condensed graph in the pipeline
// (modules/graph_construction.hpp:74-82 -> alignment/edge_index.hpp Refill -> GraphPositionFillingIndexBuilder::BuildIndexFromGraph,
// assembly_graph/index/edge_index_builders.hpp:154-307, and EdgeInfoUpdater::UpdateAll, edge_info_updater.hpp:38-101). Reuses the
// whole counting / MPHF machinery with the GPU's own unitigs as the record source:
//   1. keys   : the MINIMAL form of every K-mer of every edge (KmerFreeEdgeIndex is an InvertableStoring map -- `typedef InvertableStoring
//               DefaultStoring`, ph_map/storing_traits.hpp:74 -- so its storages filter with IsMinimal, :92-101). For K == k+1 the
//               reference iterates the edges (KMerFullGraphStorage, one MPHF segment); for any other K it counts through
//               DeBruijnGraphKMerSplitter + KMerDiskCounter with 10 x threads buckets (:274-307). Both are the canonical count
//               (SGPU_CANONICAL) over the primary strand of the unitigs: conjugate edges add no new canonical K-mer.
//   2. index  : boomphf over the distinct K-mers (mphf.cu; byte-identical KMerIndex::serialize).
//   3. values : EdgeInfoUpdater::UpdateKMers puts (EdgeId, offset) for every window of every edge -- conjugate edges included -- that
//               is minimal as it stands (edge_info_updater.hpp:41-47); a K-mer that is put twice ends as a TOMBSTONE (PutInIndex,
//               edge_position_index.hpp:152-167) -- order independent: one put -> its position, more -> removed (a self-reverse-
//               complementary K-mer is minimal on both strands: on an ordinary edge it is put from the edge and its conjugate and
//               removed; at the centre of a self-conjugate edge, visited once, it is put once and keeps its position -- with K = k+1
//               every self-conjugate edge has one). Edge ids as FastGraphFromSequencesConstructor hands them out: edge i -> 3 + 2i,
//               conjugate +1, a self-conjugate edge has one id and is visited once (graph_core.hpp:233,514-531).
#include <algorithm>
#include <thread>
#include <vector>

#include "edge_dev.cuh"
#include "host_par.h"

namespace sg {

template <int NW>
__global__ void edge_occ_k(UnitigTable u, int K, uint64_t nwork, MphfDev m, uint32_t *__restrict__ occ) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    uint32_t e, off; int s; Kmer<NW> k;
    if (!edge_window<NW>(u, K, w, &e, &s, &off, &k)) return;
    const uint64_t idx = mphf_lookup_dev<NW>(m, k);
    atomicAdd(&occ[idx], 1u);
}
template <int NW>
__global__ void edge_fill_k(UnitigTable u, int K, uint64_t nwork, MphfDev m, const uint32_t *__restrict__ occ, uint64_t *__restrict__ edge_id,
                            uint32_t *__restrict__ offset) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    uint32_t e, off; int s; Kmer<NW> k;
    if (!edge_window<NW>(u, K, w, &e, &s, &off, &k)) return;
    const uint64_t idx = mphf_lookup_dev<NW>(m, k);
    if (occ[idx] == 1u) { edge_id[idx] = 3ull + 2ull * e + (uint64_t)s; offset[idx] = off; }
    else { edge_id[idx] = ~1ull; offset[idx] = kEdgeInfoTombstone; }     // put more than once: removed (same value from every writer)
}

template <int NW>
static void edge_index_fill_nw(Ctx *ctx, EdgeIndex *ei, const UnitigTable &u, uint64_t nwork) {
    cudaStream_t st = ctx->stream;
    const uint64_t n = (uint64_t)ei->ks->n;
    MphfDev m = mphf_dev(ei->m);
    DArr<uint32_t> occ(ctx, n + 1);
    SG_CUDA(cudaMemsetAsync(occ.p, 0, occ.bytes(), st));
    SG_CUDA(cudaMemsetAsync(ei->edge_id.p, 0xff, ei->edge_id.bytes(), st));                 // CLEARED: no edge (never read back for a key of the set)
    if (nwork) {
        const int grid = div_up((int64_t)nwork, 256);
        edge_occ_k<NW><<<grid, 256, 0, st>>>(u, ei->K, nwork, m, occ.p);
        edge_fill_k<NW><<<grid, 256, 0, st>>>(u, ei->K, nwork, m, occ.p, ei->edge_id.p, ei->offset.p);
        ctx->launches += 2;
        SG_CUDA(cudaGetLastError());
    }
    SG_CUDA(cudaStreamSynchronize(st));
}

EdgeIndex::~EdgeIndex() { delete m; delete ks; }

__global__ void fill_u32_k(uint32_t *__restrict__ p, uint64_t n, uint32_t v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}

std::vector<uint64_t> edge_vertex_slots(const Graph *g, uint64_t cap) {
    std::vector<uint64_t> vk;
    vk.reserve(2 * g->edge_len.size());
    for (size_t i = 0; i < g->edge_len.size(); ++i) {
        vk.push_back(g->link_start[i] >> 2);
        if (g->link_end[i] != ~0ull) vk.push_back(g->link_end[i] >> 2);
    }
    par_sort(vk, [](uint64_t a, uint64_t b) { return a < b; });
    vk.erase(std::unique(vk.begin(), vk.end()), vk.end());
    if (vk.size() > cap) vk.resize(cap);
    return vk;
}

void edge_pack(Ctx *ctx, const Graph *g, int K, EdgePack *out) {
    cudaStream_t st = ctx->stream;
    const size_t E = g->edge_len.size();
    // ---- unitigs -> 2-bit packed "reads" (primary strand), self-conjugate flags, window prefix
    std::vector<uint64_t> woff(E + 1, 0), wstart(E + 1, 0);
    std::vector<uint32_t> lens(E + 1, 0);
    std::vector<uint8_t> selfc(E + 1, 0);
    for (size_t i = 0; i < E; ++i) {
        const uint32_t L = g->edge_len[i];
        lens[i] = L;
        woff[i + 1] = woff[i] + (L + 31) / 32;
        selfc[i] = g->link_end[i] == ~0ull ? 1 : 0;              // LinkRecord() of a self-conjugate edge (graph.cu / host_graph.cpp)
        const uint64_t nwin = L >= (uint32_t)K ? (uint64_t)(L - K + 1) : 0;
        wstart[i + 1] = wstart[i] + nwin * (selfc[i] ? 1 : 2);
    }
    std::vector<uint64_t> words(woff[E] + 4, 0);
    {
        // 2-bit packing of the unitig text on the host threads (10^9..10^10 bases for config 3)
        unsigned hw = std::thread::hardware_concurrency();
        const int T = E < 4096 ? 1 : (int)std::min<unsigned>(hw ? hw : 1, 64u);
        auto pack_range = [&](size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) {
                const uint32_t L = g->edge_len[i];
                const char *s = g->seq.data() + g->edge_off[i];
                uint64_t *w = words.data() + woff[i];
                for (uint32_t p = 0; p < L; ++p) {
                    const char c = s[p];
                    const uint64_t code = c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : 3;
                    w[p >> 5] |= code << ((p & 31) << 1);
                }
            }
        };
        if (T <= 1) pack_range(0, E);
        else {
            // chunks of equal word counts
            std::vector<std::thread> th;
            size_t lo = 0;
            for (int t = 0; t < T; ++t) {
                const uint64_t target = woff[E] * (uint64_t)(t + 1) / (uint64_t)T;
                size_t hi = (size_t)(std::upper_bound(woff.begin(), woff.end(), target) - woff.begin());
                hi = t == T - 1 ? E : std::min(E, std::max(hi ? hi - 1 : 0, lo));
                th.emplace_back(pack_range, lo, hi);
                lo = hi;
            }
            for (auto &x : th) x.join();
        }
    }
    out->words.alloc(ctx, words.size()); out->woff.alloc(ctx, E + 1); out->wstart.alloc(ctx, E + 1);
    out->lens.alloc(ctx, E + 1);
    out->selfc.alloc(ctx, E + 8);
    SG_CUDA(cudaMemcpyAsync(out->words.p, words.data(), words.size() * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(out->woff.p, woff.data(), (E + 1) * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(out->wstart.p, wstart.data(), (E + 1) * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(out->lens.p, lens.data(), (E + 1) * 4, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(out->selfc.p, selfc.data(), E + 1, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaStreamSynchronize(st));
    out->nwords = words.size(); out->nwork = wstart[E]; out->E = (int64_t)E;
}

EdgeIndex *edge_index_build(Ctx *ctx, const Graph *g, int K, int B) {
    if (K == 0) K = g->k + 1;
    SG_CHECK(K >= 1 && K <= g->k + 1 && K <= 128, 2, "edge index: K must be in [1, k+1]");
    SG_CHECK(B >= 1, 2, "edge index: num_buckets must be >= 1");
    // K == k+1: the reference takes the K-mers straight from the edges (KMerFullGraphStorage: the edges of `num_buckets` = 10 x threads
    // vertex chunks, ONE index segment). With more than one chunk KMerIndexBuilder takes its "single index parallel over buckets" branch
    // (kmer_index_builder.hpp:481-493), which never fills segment_starts_[1] -> it serializes as 0; a graph with fewer vertices than
    // chunks yields one chunk (graph_iterators.hpp:471-498) and the segmented branch, which stores n there.
    bool single = false;
    if (K == g->k + 1) {
        const uint64_t vertices = 2 * (uint64_t)edge_vertex_slots(g, ~0ull).size();      // every vertex and its conjugate (k is odd)
        single = B > 1 && vertices / (uint64_t)B > 0;
        B = 1;
    }
    cudaStream_t st = ctx->stream;
    EdgePack pk;
    edge_pack(ctx, g, K, &pk);
    const size_t E = (size_t)pk.E;
    EdgeIndex *ei = new EdgeIndex();
    ei->ctx = ctx; ei->K = K; ei->single_segment = single;
    try {
        // ---- keys: the canonical count over the unitigs (the context's read set is swapped for the duration of the call)
        const uint64_t *sv_w = ctx->d_words, *sv_o = ctx->d_offs; const uint32_t *sv_l = ctx->d_lens;
        const int64_t sv_n = ctx->n_reads; const uint64_t sv_nw = ctx->n_words; const bool sv_dirty = ctx->staged_dirty;
        ctx->d_words = pk.words.p; ctx->d_offs = pk.woff.p; ctx->d_lens = pk.lens.p; ctx->n_reads = (int64_t)E; ctx->n_words = pk.nwords; ctx->staged_dirty = false;
        try { ei->ks = count_from_reads(ctx, K, B, kCanonical); } catch (...) {
            ctx->d_words = sv_w; ctx->d_offs = sv_o; ctx->d_lens = sv_l; ctx->n_reads = sv_n; ctx->n_words = sv_nw; ctx->staged_dirty = sv_dirty;
            throw;
        }
        ctx->d_words = sv_w; ctx->d_offs = sv_o; ctx->d_lens = sv_l; ctx->n_reads = sv_n; ctx->n_words = sv_nw; ctx->staged_dirty = sv_dirty;
        ei->m = mphf_build(ctx, ei->ks);
        // ---- values
        const uint64_t n = (uint64_t)ei->ks->n;
        ei->edge_id.alloc(ctx, n + 1, true);
        ei->offset.alloc(ctx, n + 1, true);
        fill_u32_k<<<ctx->num_sms * 4, 256, 0, st>>>(ei->offset.p, n + 1, kEdgeInfoCleared);
        ctx->launches++;
        const UnitigTable u = pk.table();
        if (E) {
            switch (nwords_of(K)) {
                case 1: edge_index_fill_nw<1>(ctx, ei, u, pk.nwork); break;
                case 2: edge_index_fill_nw<2>(ctx, ei, u, pk.nwork); break;
                case 3: edge_index_fill_nw<3>(ctx, ei, u, pk.nwork); break;
                default: edge_index_fill_nw<4>(ctx, ei, u, pk.nwork); break;
            }
        }
    } catch (...) { delete ei; throw; }
    return ei;
}

}  // namespace sg
