// graph.cu -- extension masks, coverage, unitigs (unbranching paths + perfect loops), link records. Replaces
//   DeBruijnExtensionIndexBuilder::FillExtensionsFromIndex (src/common/kmer_index/extension_index/kmer_extension_index_builder.hpp:45-60)
//   InOutMask (…/extension_index/inout_mask.hpp:55-221)
//   CoverageHashMapBuilder (src/common/kmer_index/ph_map/coverage_hash_map_builder.hpp:16-57) -- counts come from the sort's run lengths
//   UnbranchingPathExtractor (src/common/assembly_graph/construction/debruijn_graph_constructor.hpp:184-410)
//   FastGraphFromSequencesConstructor::CollectLinkRecords (…:473-487) and GraphCoverageFiller (graph_support/coverage_filling.hpp:52-70)
#include <algorithm>
#include <array>
#include <optional>

#include "graph_dev.cuh"
#include "masks_dev.cuh"

namespace sg {

// ---- masks -------------------------------------------------------------------------------------------------------
template <int NW, int NWS>
__global__ void masks_k(const uint64_t *__restrict__ kp, int64_t n, int K, MphfDev mk, unsigned *__restrict__ masks32) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Kmer<NWS> x;
#pragma unroll
    for (int q = 0; q < NWS; ++q) x.w[q] = kp[i * NWS + q];
    const int pnucl = kpomer_side_nucl<1, NWS>(x, K), nnucl = kpomer_side_nucl<0, NWS>(x, K);
    auto slot = [&](const Kmer<NW> &key) { return mphf_lookup_dev<NW>(mk, key); };
    {
        const auto c = kpomer_side<0, NW, NWS>(x, K, slot);                       // AddOutgoing(prefix, nnucl)
        mask_or(masks32, c.value, mask_bit<0>(c.is_min, nnucl));
    }
    {
        const auto c = kpomer_side<1, NW, NWS>(x, K, slot);                       // AddIncoming(suffix, pnucl)
        mask_or(masks32, c.value, mask_bit<1>(c.is_min, pnucl));
    }
}

// coverage array in the reference's layout: cov[mphf(kpomer)] = multiplicity
template <int NWS>
__global__ void cov_perm_k(const uint64_t *__restrict__ kp, const uint32_t *__restrict__ counts, int64_t n, MphfDev mkp, uint32_t *__restrict__ cov) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Kmer<NWS> x;
#pragma unroll
    for (int q = 0; q < NWS; ++q) x.w[q] = kp[i * NWS + q];
    cov[mphf_lookup_dev<NWS>(mkp, x)] = counts[i];
}

// stages/construction.cpp:404-418 : hist[cov-1] += 2
__global__ void hist_max_k(const uint32_t *__restrict__ cov, int64_t n, unsigned *__restrict__ mx) {
    unsigned m = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) m = max(m, cov[i]);
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(mx, m);
}
__global__ void hist_fill_k(const uint32_t *__restrict__ cov, int64_t n, unsigned long long *__restrict__ hist) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t c = cov[i];
        if (c) atomicAdd(&hist[c - 1], 2ull);
    }
}

// ---- unbranching paths ---------------------------------------------------------------------------------------------
// The kernels below that walk the k-mer set run once per chunk: `keys` holds the chunk's n records, and `base` is the position
// of its first record in final_kmers order, so every thread keeps its global k-mer position.
template <int NW>
__global__ void junction_flags_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, uint32_t *__restrict__ flag) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    Kmer<NW> k = key_at<NW>(keys, j);
    const uint8_t m = masks[mphf_lookup_dev<NW>(mk, k)];
    // IsJunction (:194-200). An isolated k-mer (mask 0, e.g. a clipped tip's) is one too, but starts no path: it is left out of
    // the list, which then costs nothing for the clipped k-mers
    flag[j] = (m && (uniq4(m & 15) < 0 || uniq4(m >> 4) < 0)) ? 1u : 0u;
}
// kept slots -> dense (offset, length) table of the path edges (eidx = rank among the kept slots, eoff = first base)
__global__ void edge_table_k(const uint32_t *__restrict__ len, const uint64_t *__restrict__ eidx, const uint64_t *__restrict__ eoff, int64_t nslots,
                             uint64_t *__restrict__ out_off, uint32_t *__restrict__ out_len) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nslots || !len[i]) return;
    out_off[eidx[i]] = eoff[i];
    out_len[eidx[i]] = len[i];
}

// the flagged keys of a chunk, in chunk order
template <int NW>
__global__ void compact_keys_k(const uint32_t *__restrict__ flag, const uint64_t *__restrict__ pos, const uint64_t *__restrict__ keys, int64_t n,
                               uint64_t *__restrict__ list) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n || !flag[j]) return;
#pragma unroll
    for (int q = 0; q < NW; ++q) list[pos[j] * NW + q] = keys[j * NW + q];
}

// the walks (graph_dev.cuh) over this GPU's index and arrays
template <int NW>
__global__ void unitig_probe_k(const uint64_t *__restrict__ jkeys, int64_t njunc, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                               uint64_t nk, uint32_t *__restrict__ len /*[njunc*8] 0 = none*/, uint8_t *__restrict__ selfc) {
    unitig_probe<NW>(LocalView{mk, masks}, jkeys, njunc, K, nk, len, selfc);
}

template <int NW, int NWS>
__global__ void unitig_write_k(const uint64_t *__restrict__ jkeys, int64_t njunc, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                               uint64_t nk, const uint32_t *__restrict__ len, const uint8_t *__restrict__ selfc, const uint64_t *__restrict__ eidx,
                               const uint64_t *__restrict__ eoff, MphfDev mkp, const uint32_t *__restrict__ cov, EdgeOut o) {
    unitig_write<NW, NWS>(LocalView{mk, masks, mkp, cov, o.visited}, jkeys, njunc, K, nk, len, selfc, eidx, eoff, o);
}

// also marks the remaining slots (unvisited, neither junction nor dead end: the vertices of perfect loops) in rem_bits, one bit per
// slot: warp w writes word w (the grid covers whole warps)
__global__ void masks_clear_visited_k(uint8_t *__restrict__ masks, const uint8_t *__restrict__ visited, uint64_t n, unsigned long long *__restrict__ remaining,
                                      uint32_t *__restrict__ rem_bits) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool rem = false;
    if (i < n) {
        if (visited[i]) masks[i] = 0;                      // RemoveSequences, kmer_extension_index.hpp:141-147
        const uint8_t m = masks[i];
        rem = m && uniq4(m & 15) >= 0 && uniq4(m >> 4) >= 0;
    }
    const unsigned b = __ballot_sync(0xffffffffu, rem);
    if ((threadIdx.x & 31) == 0 && i < n) rem_bits[i >> 5] = b;
    if (b && (threadIdx.x & 31) == 0) atomicAdd(remaining, (unsigned long long)__popc(b));
}

// ---- early clippers (graph_dev.cuh) over this GPU's index and masks ---------------------------------------------------------
template <int NW>
__global__ void tc_probe_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, uint32_t bound,
                           uint8_t *__restrict__ mark, uint8_t *__restrict__ tipped /*[2 * all k-mers]*/, unsigned long long *__restrict__ stats) {
    LocalView v{mk, masks};
    v.marks = mark;
    tc_probe<NW>(v, keys, base, n, K, bound, tipped, stats);
}
__global__ void tc_apply_k(uint8_t *__restrict__ masks, const uint8_t *__restrict__ mark, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && mark[i]) masks[i] = 0;
}
template <int NW>
__global__ void tc_links_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, int K, MphfDev mk, uint8_t *__restrict__ masks,
                           const uint8_t *__restrict__ tipped, unsigned long long *__restrict__ stat_clipped, int flags_by_slot) {
    LocalView v{mk, masks};
    v.roots = const_cast<uint8_t *>(tipped);
    tc_links<NW>(v, keys, base, n, K, tipped, stat_clipped, flags_by_slot);
}
template <int NW>
__global__ void at_edges_probe_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, AtParams ap,
                                 uint8_t *__restrict__ eflag /*[2 * all k-mers]*/, unsigned long long *__restrict__ stats) {
    LocalView v{mk, masks};
    v.eflags = eflag;
    at_edges_probe<NW>(v, keys, n, K, ap, stats);
}
template <int NW>
__global__ void at_edges_apply_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, uint8_t *__restrict__ masks, const uint8_t *__restrict__ eflag,
                                 unsigned long long *__restrict__ stats) {
    LocalView v{mk, masks};
    v.eflags = const_cast<uint8_t *>(eflag);
    at_edges_apply<NW>(v, keys, n, K, stats);
}
template <int NW>
__global__ void at_tips_probe_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, AtParams ap,
                                uint8_t *__restrict__ mark, uint8_t *__restrict__ rooted /*[2 * all k-mers]*/, unsigned long long *__restrict__ stats) {
    LocalView v{mk, masks};
    v.marks = mark; v.roots = rooted;
    at_tips_probe<NW>(v, keys, n, K, ap, stats);
}

// ---- perfect loops (CollectLoops :359-397) --------------------------------------------------------------------------
__global__ void popc_words_k(const uint32_t *__restrict__ bits, uint64_t nw, uint32_t *__restrict__ cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nw) cnt[i] = (uint32_t)__popc(bits[i]);
}
template <int NW>
__global__ void loop_pos_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, MphfDev mk, RemSlots rs, uint64_t *__restrict__ pos) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint64_t r = rs.rank(mphf_lookup_dev<NW>(mk, key_at<NW>(keys, j)));
    if (r != ~0ull) pos[r] = (uint64_t)(base + j);
}
template <int NW>
__global__ void loop_leader_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, uint64_t nk, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                              RemSlots rs, const uint64_t *__restrict__ pos, uint32_t *__restrict__ is_leader) {
    loop_leader<NW>(LocalView{mk, masks, MphfDev(), nullptr, nullptr, rs, pos}, keys, base, n, nk, K, is_leader);
}
template <int NW, int NWS>
__global__ void loop_probe_k(const uint64_t *__restrict__ leaders /*keys*/, int64_t nl, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                             LoopInfo *__restrict__ info, uint32_t *__restrict__ len /*[nl*2]*/) {
    loop_probe<NW, NWS>(LocalView{mk, masks}, leaders, nl, K, info, len);
}
template <int NW, int NWS>
__global__ void loop_write_k(const LoopInfo *__restrict__ info, int64_t nl, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                             const uint32_t *__restrict__ len, const uint64_t *__restrict__ eidx, const uint64_t *__restrict__ eoff, MphfDev mkp,
                             const uint32_t *__restrict__ cov, EdgeOut o, char *__restrict__ scratch, const uint64_t *__restrict__ soff) {
    loop_write<NW, NWS>(LocalView{mk, masks, mkp, cov, o.visited}, info, nl, K, len, eidx, eoff, o, scratch, soff);
}

// ---- host orchestration ----------------------------------------------------------------------------------------------
template <int NW>
KeyParts collect_keys(Ctx *ctx, ChunkStager &src, const FlagLaunch &flags) {
    cudaStream_t st = ctx->stream;
    int64_t mx = 1;
    for (const Chunk &c : src.ks->chunks) mx = std::max(mx, c.n);
    DArr<uint32_t> flag(ctx, (size_t)mx + 1);
    DArr<uint64_t> pos(ctx, (size_t)mx + 1);
    KeyParts kp;
    src.sweep([&](const Chunk &ch, const uint64_t *keys, const uint32_t *) {
        SG_CUDA(cudaMemsetAsync(flag.p + ch.n, 0, 4, st));
        flags(ch, keys, flag.p);
        ctx->launches++;
        exclusive_scan_u32_to_u64(ctx, flag.p, pos.p, (size_t)ch.n + 1);
        uint64_t m = 0;
        SG_CUDA(cudaMemcpyAsync(&m, pos.p + ch.n, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        if (!m) return;
        kp.parts.emplace_back(ctx, (size_t)m * NW);
        kp.sizes.push_back(m);
        kp.total += m;
        compact_keys_k<NW><<<div_up(ch.n, 256), 256, 0, st>>>(flag.p, pos.p, keys, ch.n, kp.parts.back().p);
        ctx->launches++;
    });
    SG_CUDA(cudaStreamSynchronize(st));
    return kp;
}

template <int NW>
KeyParts junction_keys(Ctx *ctx, ChunkStager &kmers, int K, const MphfDev &mk, const uint8_t *masks) {
    return collect_keys<NW>(ctx, kmers, [&](const Chunk &c, const uint64_t *keys, uint32_t *flag) {
        junction_flags_k<NW><<<div_up(c.n, 256), 256, 0, ctx->stream>>>(keys, c.n, K, mk, masks, flag);
    });
}

template <int NW>
void loop_positions(Ctx *ctx, ChunkStager &kmers, const MphfDev &mk, const RemSlots &rs, uint64_t *pos) {
    kmers.sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *) {
        loop_pos_k<NW><<<div_up(c.n, 256), 256, 0, ctx->stream>>>(keys, c.first, c.n, mk, rs, pos);
        ctx->launches++;
    });
}

#define SG_INSTANTIATE_KEYS(NW)                                                                                          \
    template KeyParts collect_keys<NW>(Ctx *, ChunkStager &, const FlagLaunch &);                                        \
    template KeyParts junction_keys<NW>(Ctx *, ChunkStager &, int, const MphfDev &, const uint8_t *);                    \
    template void loop_positions<NW>(Ctx *, ChunkStager &, const MphfDev &, const RemSlots &, uint64_t *);
SG_INSTANTIATE_KEYS(1)
SG_INSTANTIATE_KEYS(2)
SG_INSTANTIATE_KEYS(3)
SG_INSTANTIATE_KEYS(4)

void launch_isolate(Ctx *ctx, uint8_t *masks, const uint8_t *mark, uint64_t n) {
    if (!n) return;
    tc_apply_k<<<div_up((int64_t)n, 256), 256, 0, ctx->stream>>>(masks, mark, n);
    ctx->launches++;
}

void launch_edge_table(Ctx *ctx, const uint32_t *len, const uint64_t *eidx, const uint64_t *eoff, int64_t nslots, uint64_t *out_off, uint32_t *out_len) {
    edge_table_k<<<div_up(nslots, 256), 256, 0, ctx->stream>>>(len, eidx, eoff, nslots, out_off, out_len);
    ctx->launches++;
}

uint64_t masks_clear_visited(Ctx *ctx, uint8_t *masks, const uint8_t *visited, uint64_t n, uint32_t *rem_bits) {
    cudaStream_t st = ctx->stream;
    DArr<unsigned long long> d_rem(ctx, 1);
    SG_CUDA(cudaMemsetAsync(d_rem.p, 0, 8, st));
    masks_clear_visited_k<<<div_up((int64_t)n, 256), 256, 0, st>>>(masks, visited, n, d_rem.p, rem_bits);
    ctx->launches++;
    unsigned long long rem = 0;
    SG_CUDA(cudaMemcpyAsync(&rem, d_rem.p, 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    return rem;
}

void rem_slot_base(Ctx *ctx, const uint32_t *rem_bits, uint64_t nwords, uint64_t *rem_base) {
    cudaStream_t st = ctx->stream;
    DArr<uint32_t> cnt(ctx, nwords + 1);
    SG_CUDA(cudaMemsetAsync(cnt.p + nwords, 0, 4, st));
    popc_words_k<<<div_up((int64_t)nwords, 256), 256, 0, st>>>(rem_bits, nwords, cnt.p);
    ctx->launches++;
    exclusive_scan_u32_to_u64(ctx, cnt.p, rem_base, nwords + 1);
    SG_CUDA(cudaStreamSynchronize(st));
}

// One graph construction: what its phases share (an aggregate: {ctx, g, opt} sets the rest). Only the sweeps read the two sets
// (through a ChunkStager each), so the graph needs the MPHFs, masks and coverage resident, not the sets.
template <int NW, int NWS>
struct GraphBuild {
    Ctx *ctx;
    Graph *g;
    const GraphOptions &opt;
    cudaStream_t st = ctx->stream;
    int K = g->km->K;
    uint64_t nk = (uint64_t)g->km->n;
    bool have_cov = g->mkp && g->kp->has_counts;      // without coverage, g->cov stays unallocated and the kernels get a null pointer
    MphfDev mk = mphf_dev(g->mk), mkp = have_cov ? mphf_dev(g->mkp) : MphfDev();
    std::optional<ChunkStager> kmers;                 // the k-mer set, for every sweep after the masks
    DArr<uint8_t> visited;                            // per k-mer slot: on an edge already (from the unitigs through the loops)
    Trace tr{"sgpu graph", st};
    // kernel launches over every non-empty chunk of the k-mer set: launch(chunk, keys) launches one
    template <class F>
    void kmer_sweep(F &&launch) {
        kmers->sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *) { launch(c, keys); ctx->launches++; });
    }

    // the masks, and the coverage in MPHF order: one sweep over the (k+1)-mers. The resident state first, then the staging
    // buffers of the two sets, one after the other (the (k+1)-mers' stager is gone before the k-mers' is made).
    void masks_coverage() {
        g->masks.alloc(ctx, nk + 8, true);
        SG_CUDA(cudaMemsetAsync(g->masks.p, 0, g->masks.bytes(), st));
        if (have_cov) {
            g->cov.alloc(ctx, (size_t)g->kp->n + 1, true);
            SG_CUDA(cudaMemsetAsync(g->cov.p, 0, g->cov.bytes(), st));
        }
        ChunkStager(g->kp, have_cov).sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *counts) {
            masks_k<NW, NWS><<<div_up(c.n, 256), 256, 0, st>>>(keys, c.n, K, mk, reinterpret_cast<unsigned *>(g->masks.p));
            ctx->launches++;
            if (have_cov) {
                cov_perm_k<NWS><<<div_up(c.n, 256), 256, 0, st>>>(keys, counts, c.n, mkp, g->cov.p);
                ctx->launches++;
            }
        });
        SG_CUDA(cudaStreamSynchronize(st));
        tr.mark("masks + coverage");
        kmers.emplace(g->km, false);
    }

    // The clippers probe every k-mer on a snapshot of the masks (one whole sweep) before any change is applied. Their common
    // tail: IsolateVertex for the marked k-mers, then one tc_links_k sweep (RemoveInconsistentForwardLinks) over the flagged
    // (k-mer, orientation) pairs, which counts the clipped links in stats[links]. Returns the clipper's four counters.
    std::array<unsigned long long, 4> isolate_and_unlink(const uint8_t *mark, const uint8_t *flags, int flags_by_slot, unsigned long long *stats, int links) {
        launch_isolate(ctx, g->masks.p, mark, nk);
        kmer_sweep([&](const Chunk &c, const uint64_t *keys) {
            tc_links_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(keys, c.first, c.n, K, mk, g->masks.p, flags, stats + links, flags_by_slot);
        });
        std::array<unsigned long long, 4> hs;
        SG_CUDA(cudaMemcpyAsync(hs.data(), stats, 32, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        return hs;
    }

    void at_clipper() {
        if (!opt.early_at || !nk) return;
        SG_CHECK(opt.at_min_len <= (uint64_t)K, 2, "early A/T clipper: min_length must not exceed k (the reference indexes kh[k - 1 - i])");
        const AtParams ap = at_params(opt);
        DArr<uint8_t> eflag(ctx, 2 * nk + 8), mark(ctx, nk + 8);
        DArr<uint8_t> rooted(ctx, 2 * nk + 8);
        DArr<unsigned long long> stats(ctx, 4);
        SG_CUDA(cudaMemsetAsync(mark.p, 0, mark.bytes(), st));
        SG_CUDA(cudaMemsetAsync(rooted.p, 0, rooted.bytes(), st));
        SG_CUDA(cudaMemsetAsync(stats.p, 0, 32, st));
        kmer_sweep([&](const Chunk &c, const uint64_t *keys) {
            at_edges_probe_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(keys, c.n, K, mk, g->masks.p, ap, eflag.p, stats.p);
        });
        kmer_sweep([&](const Chunk &c, const uint64_t *keys) {
            at_edges_apply_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(keys, c.n, K, mk, g->masks.p, eflag.p, stats.p);
        });
        kmer_sweep([&](const Chunk &c, const uint64_t *keys) {
            at_tips_probe_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(keys, c.n, K, mk, g->masks.p, ap, mark.p, rooted.p, stats.p);
        });
        const auto hs = isolate_and_unlink(mark.p, rooted.p, 1, stats.p, 3);
        for (int i = 0; i < 4; ++i) g->at_stats[i] = hs[i];
    }

    void tip_clipper() {
        if (!opt.early_tip_length_bound || !nk) return;
        DArr<uint8_t> mark(ctx, nk + 8);
        DArr<uint8_t> tipped(ctx, 2 * nk + 8);
        DArr<unsigned long long> stats(ctx, 4);
        SG_CUDA(cudaMemsetAsync(mark.p, 0, mark.bytes(), st));
        SG_CUDA(cudaMemsetAsync(stats.p, 0, 32, st));
        const uint32_t bound = tip_bound(opt);
        kmer_sweep([&](const Chunk &c, const uint64_t *keys) {
            tc_probe_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(keys, c.first, c.n, K, mk, g->masks.p, bound, mark.p, tipped.p, stats.p);
        });
        const auto hs = isolate_and_unlink(mark.p, tipped.p, 0, stats.p, 2);
        for (int i = 0; i < 3; ++i) g->tc_stats[i] = hs[i];
    }

    // what the reference's extension index holds before the unitig extraction changes it
    void final_masks() {
        g->masks_final.alloc(ctx, nk + 8, true);
        SG_CUDA(cudaMemcpyAsync(g->masks_final.p, g->masks.p, nk, cudaMemcpyDeviceToDevice, st));
        tr.mark("early clippers");
    }

    // the junctions' keys in final_kmers order, so the unitig kernels never reach into the set
    KeyParts junctions() {
        KeyParts jk = junction_keys<NW>(ctx, *kmers, K, mk, g->masks.p);
        tr.mark("junction list");
        return jk;
    }

    // unbranching paths (unitig_batches), in batches sized from the room left
    void unitigs(KeyParts jk) {
        visited.alloc(ctx, nk + 8);
        SG_CUDA(cudaMemsetAsync(visited.p, 0, visited.bytes(), st));
        ctx->times.graph_junction_batches = unitig_batches(
            ctx, g, jk, NW, ctx->budget_left(), tr,
            [&](const uint64_t *bkeys, int64_t nj, uint32_t *len, uint8_t *selfc) {
                unitig_probe_k<NW><<<div_up(nj * 8, 128), 128, 0, st>>>(bkeys, nj, K, mk, g->masks.p, nk, len, selfc);
            },
            [](const uint64_t *, int64_t, const uint32_t *) {},
            [&](const uint64_t *bkeys, int64_t nj, const uint32_t *len, const uint8_t *selfc, const uint64_t *eidx, const uint64_t *eoff, const EdgeBatch &eb) {
                unitig_write_k<NW, NWS><<<div_up(nj * 8, 128), 128, 0, st>>>(bkeys, nj, K, mk, g->masks.p, nk, len, selfc, eidx, eoff, mkp, g->cov.p,
                                                                            eb.out(visited.p));
            });
    }

    // perfect loops: the k-mers that are left with one edge in and one out once the paths are removed
    void loops() {
        const uint64_t nwords = (nk + 31) / 32;
        DArr<uint32_t> rem_bits(ctx, nwords + 1);
        const uint64_t rem = masks_clear_visited(ctx, g->masks.p, visited.p, nk, rem_bits.p);
        if (!rem) return;
        // final_kmers positions of the remaining slots only (RemSlots): the loop kernels never need 8 B per k-mer
        DArr<uint64_t> rem_base(ctx, nwords + 1), rem_pos(ctx, rem);
        rem_slot_base(ctx, rem_bits.p, nwords, rem_base.p);
        RemSlots rs; rs.bits = rem_bits.p; rs.base = rem_base.p;
        loop_positions<NW>(ctx, *kmers, mk, rs, rem_pos.p);
        KeyParts lk = collect_keys<NW>(ctx, *kmers, [&](const Chunk &c, const uint64_t *keys, uint32_t *flag) {
            loop_leader_k<NW><<<div_up(c.n, 128), 128, 0, st>>>(keys, c.first, c.n, nk, K, mk, g->masks.p, rs, rem_pos.p, flag);
        });
        rem_pos.release(); rem_base.release(); rem_bits.release();
        loop_edges(ctx, g, lk, NW, K,
            [&](const uint64_t *leaders, int64_t nl, LoopInfo *info, uint32_t *llen) {
                loop_probe_k<NW, NWS><<<div_up(nl, 64), 64, 0, st>>>(leaders, nl, K, mk, g->masks.p, info, llen);
            },
            [](const uint64_t *, int64_t, const std::vector<uint32_t> &) {},
            [&](const LoopInfo *info, int64_t nl, const uint32_t *llen, const uint64_t *leidx, const uint64_t *leoff, const EdgeBatch &eb, char *scratch,
                const uint64_t *soff) {
                loop_write_k<NW, NWS><<<div_up(nl, 64), 64, 0, st>>>(info, nl, K, mk, g->masks.p, llen, leidx, leoff, mkp, g->cov.p, eb.out(visited.p),
                                                                    scratch, soff);
            });
    }
};

template <int NW, int NWS>
static void graph_build_nw(Ctx *ctx, Graph *g, const GraphOptions &opt) {
    GraphBuild<NW, NWS> b{ctx, g, opt};
    b.masks_coverage();
    b.at_clipper();
    b.tip_clipper();
    b.final_masks();
    if (!b.nk) return;
    b.unitigs(b.junctions());
    if (opt.keep_perfect_loops) b.loops();
}

__global__ void nonzero_flags_k(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i] ? 1u : 0u;
}
void launch_nonzero_flags(Ctx *ctx, const uint32_t *in, uint32_t *out, uint64_t n) {
    if (!n) return;
    nonzero_flags_k<<<div_up((int64_t)n, 256), 256, 0, ctx->stream>>>(in, out, n);
    ctx->launches++;
}

Graph *graph_build(Ctx *ctx, const KSet *kp, const KSet *km, const Mphf *mk, const Mphf *mkp, const GraphOptions &opt) {
    SG_CHECK(kp->K == km->K + 1, 2, "graph: (k+1)-mer / k-mer sets do not match");
    SG_CHECK(mk->n == km->n && mk->B == km->B, 2, "graph: k-mer index does not belong to the k-mer set");
    SG_CHECK(km->K % 2 == 1, 2, "graph: k must be odd (gbuilder.cpp:125)");
    Graph *g = new Graph();
    g->ctx = ctx; g->k = km->K; g->kp = kp; g->km = km; g->mk = mk; g->mkp = mkp;
    ctx->times.stage_h2d_bytes = 0;
    ctx->times.graph_junction_batches = 0;
    try {
        const int nw = km->nw, nws = kp->nw;
        if (nw == 1 && nws == 1) graph_build_nw<1, 1>(ctx, g, opt);
        else if (nw == 1 && nws == 2) graph_build_nw<1, 2>(ctx, g, opt);
        else if (nw == 2 && nws == 2) graph_build_nw<2, 2>(ctx, g, opt);
        else if (nw == 2 && nws == 3) graph_build_nw<2, 3>(ctx, g, opt);
        else if (nw == 3 && nws == 3) graph_build_nw<3, 3>(ctx, g, opt);
        else if (nw == 3 && nws == 4) graph_build_nw<3, 4>(ctx, g, opt);
        else if (nw == 4 && nws == 4) graph_build_nw<4, 4>(ctx, g, opt);
        else throw Error(2, "graph: unsupported word combination");
    } catch (...) { delete g; throw; }
    return g;
}

std::vector<uint64_t> graph_histogram(Ctx *ctx, const Graph *g) {
    if (!g->cov.p) return {};
    return coverage_histogram(ctx, g->cov.p, g->kp->n);
}

void coverage_fill(Ctx *ctx, ChunkStager &kpomers, const Mphf *mkp, uint32_t *cov) {
    SG_CHECK(kpomers.with_counts, 2, "coverage: the (k+1)-mer set carries no multiplicities");
    const MphfDev m = mphf_dev(mkp);
    const int nws = kpomers.ks->nw;
    kpomers.sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *counts) {
        const int grid = div_up(c.n, 256);
        if (nws == 1) cov_perm_k<1><<<grid, 256, 0, ctx->stream>>>(keys, counts, c.n, m, cov);
        else if (nws == 2) cov_perm_k<2><<<grid, 256, 0, ctx->stream>>>(keys, counts, c.n, m, cov);
        else if (nws == 3) cov_perm_k<3><<<grid, 256, 0, ctx->stream>>>(keys, counts, c.n, m, cov);
        else cov_perm_k<4><<<grid, 256, 0, ctx->stream>>>(keys, counts, c.n, m, cov);
        ctx->launches++;
    });
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
}

std::vector<uint64_t> coverage_histogram(Ctx *ctx, const uint32_t *cov, int64_t n) {
    std::vector<uint64_t> h;
    if (n == 0) return h;
    DArr<unsigned> mx(ctx, 1);
    SG_CUDA(cudaMemsetAsync(mx.p, 0, 4, ctx->stream));
    hist_max_k<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(cov, n, mx.p);
    unsigned m = 0;
    SG_CUDA(cudaMemcpyAsync(&m, mx.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (!m) return h;
    DArr<unsigned long long> dh(ctx, m);
    SG_CUDA(cudaMemsetAsync(dh.p, 0, dh.bytes(), ctx->stream));
    hist_fill_k<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(cov, n, dh.p);
    ctx->launches += 2;
    h.resize(m);
    SG_CUDA(cudaMemcpyAsync(h.data(), dh.p, (size_t)m * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
    return h;
}

}  // namespace sg
