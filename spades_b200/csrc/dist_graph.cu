// dist_graph.cu -- the unbranching paths and perfect loops across GPUs (one process per GPU), from each rank's slices of the
// extension masks and coverage (dist_ext.cu). hpcspades condenses the graph on its master from a broadcast extension index
// (GraphCondenser, construction_mpi.cpp:607-632); here every rank walks from the junctions and loop leaders it owns, through the
// indexes, masks, visited flags and coverage of whichever rank owns each k-mer (DistView, graph_dev.cuh): a walk is pointer
// chasing, so it reads the owners' arrays in place over the peer mappings instead of exchanging rounds of lookups. A rank
// allocates only its own slices and the per-bucket tables. Its edges come out in its own final_kmers order, with per-bucket
// counts, so that the host can interleave the ranks' edges into the order one GPU gives over the union.
// The early clippers (graph_dev.cuh) run before the junction list the same way: every rank probes from its own k-mers through the
// owners' indexes and masks, and sets the IsolateVertex and root flags, or clears the mask bits, in the owners' slices. A
// probe's flags are final on every rank before any rank changes a mask, as a snapshot of the masks is on one GPU.
#include <memory>

#include "graph_dev.cuh"

namespace sg {

// ---- kernels: the walks of graph_dev.cuh over a DistView ----------------------------------------------------------------------
template <int NW>
__global__ void dist_unitig_probe_k(DistView v, const uint64_t *__restrict__ jkeys, int64_t njunc, int K, uint64_t nk, uint32_t *__restrict__ len,
                                    uint8_t *__restrict__ selfc) {
    unitig_probe<NW>(v, jkeys, njunc, K, nk, len, selfc);
}
template <int NW, int NWS>
__global__ void dist_unitig_write_k(DistView v, const uint64_t *__restrict__ jkeys, int64_t njunc, int K, uint64_t nk, const uint32_t *__restrict__ len,
                                    const uint8_t *__restrict__ selfc, const uint64_t *__restrict__ eidx, const uint64_t *__restrict__ eoff, EdgeOut o) {
    unitig_write<NW, NWS>(v, jkeys, njunc, K, nk, len, selfc, eidx, eoff, o);
}
// the kept paths of a batch per bucket of their start junction
template <int NW>
__global__ void dist_edge_buckets_k(const uint64_t *__restrict__ jkeys, int64_t njunc, const uint32_t *__restrict__ len, uint32_t B,
                                    unsigned long long *__restrict__ cnt) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= njunc * 8 || !len[tid]) return;
    atomicAdd(&cnt[kmer_bucket<NW>(key_at<NW>(jkeys, tid >> 3), B)], 1ull);
}
template <int NW>
__global__ void dist_loop_leader_k(DistView v, const uint64_t *__restrict__ keys, int64_t base, int64_t n, uint64_t nk, int K, uint32_t *__restrict__ is_leader) {
    loop_leader<NW>(v, keys, base, n, nk, K, is_leader);
}
template <int NW, int NWS>
__global__ void dist_loop_probe_k(DistView v, const uint64_t *__restrict__ leaders, int64_t nl, int K, LoopInfo *__restrict__ info, uint32_t *__restrict__ len) {
    loop_probe<NW, NWS>(v, leaders, nl, K, info, len);
}
template <int NW>
__global__ void dist_tc_probe_k(DistView v, const uint64_t *__restrict__ keys, int64_t base, int64_t n, int K, uint32_t bound, uint8_t *__restrict__ tipped,
                                unsigned long long *__restrict__ stats) {
    tc_probe<NW>(v, keys, base, n, K, bound, tipped, stats);
}
template <int NW>
__global__ void dist_tc_links_k(DistView v, const uint64_t *__restrict__ keys, int64_t base, int64_t n, int K, const uint8_t *__restrict__ tipped,
                                unsigned long long *__restrict__ stat_clipped, int flags_by_slot) {
    tc_links<NW>(v, keys, base, n, K, tipped, stat_clipped, flags_by_slot);
}
template <int NW>
__global__ void dist_at_edges_probe_k(DistView v, const uint64_t *__restrict__ keys, int64_t n, int K, AtParams ap, unsigned long long *__restrict__ stats) {
    at_edges_probe<NW>(v, keys, n, K, ap, stats);
}
template <int NW>
__global__ void dist_at_edges_apply_k(DistView v, const uint64_t *__restrict__ keys, int64_t n, int K, unsigned long long *__restrict__ stats) {
    at_edges_apply<NW>(v, keys, n, K, stats);
}
template <int NW>
__global__ void dist_at_tips_probe_k(DistView v, const uint64_t *__restrict__ keys, int64_t n, int K, AtParams ap, unsigned long long *__restrict__ stats) {
    at_tips_probe<NW>(v, keys, n, K, ap, stats);
}
template <int NW, int NWS>
__global__ void dist_loop_write_k(DistView v, const LoopInfo *__restrict__ info, int64_t nl, int K, const uint32_t *__restrict__ len,
                                  const uint64_t *__restrict__ eidx, const uint64_t *__restrict__ eoff, EdgeOut o, char *__restrict__ scratch,
                                  const uint64_t *__restrict__ soff) {
    loop_write<NW, NWS>(v, info, nl, K, len, eidx, eoff, o, scratch, soff);
}

// ---- state ---------------------------------------------------------------------------------------------------------------
// what a rank publishes: its arena and where each array the walks read lies in it (~0: not allocated)
enum { kDescBits, kDescRanks, kDescDom, kDescWoff, kDescStarts, kDescMasks, kDescVisited, kDescPbits, kDescPranks, kDescPdom, kDescPwoff,
       kDescPstarts, kDescCov, kDescRemBits, kDescRemBase, kDescRemPos, kDescMark, kDescEflag, kDescRooted, kDescArrays };
struct GraphDesc {
    cudaIpcMemHandle_t arena;     // 64 bytes
    uint64_t arena_size;
    uint64_t off[kDescArrays];
    cudaUUID_t device;            // the device that holds the arena (16 bytes)
    uint64_t unused[2];
};
static_assert(sizeof(GraphDesc) == 256, "descriptor layout (SGPU_DIST_GRAPH_IPC_BYTES)");

struct DistGraph {
    Ctx *ctx = nullptr;
    ExtSlices ext;
    GraphOptions opt;
    int K = 0, B = 0, world = 1, rank = 0;
    bool with_cov = false, clip = false;        // clip: an early clipper is on
    uint64_t nk = 0, nk_union = 0, budget = 0;
    std::vector<int> owner, powner;
    std::vector<uint64_t> ustart;                // B: the union's first slot of each k-mer bucket
    DArr<uint8_t> masks, visited;                // this rank's working copy of its mask slice, its visited flags
    DArr<uint32_t> rem_bits;                     // its remaining slots (RemSlots) and their final_kmers positions
    DArr<uint64_t> rem_base, rem_pos;
    DArr<DistPeer> d_peers;
    DArr<int> d_owner, d_powner;
    DArr<uint64_t> dom, woff, lstart, d_ustart, pdom, pwoff, pstart;   // the owners' index rows, per bucket
    bool tables = false;
    DArr<unsigned long long> err;
    DArr<uint8_t> mark, tipped, eflag, rooted;  // the clippers' flags: per owned k-mer, per (position, orientation), per (slot, orientation) twice
    DArr<uint8_t> masks_final;                   // the clipped slice, before the walks change the working copy (only when clip)
    // [0, 4): the A/T clipper's counters, [4, 7): the tip clipper's (sgpu_graph_*_clipper_stats order); [8, 11): mark and root
    // stores and bit clears that landed in another rank's slice (DistView::remote)
    DArr<unsigned long long> cstats;
    std::vector<int> phases;                     // what runs between begin and the unitigs; phases[next] runs next
    size_t next = 0;
    std::unique_ptr<ChunkStager> kmers;
    KeyParts jk;
    Graph edges;                                 // this rank's edges: its unitigs, then its loops
    uint64_t unitig_edges = 0, batches = 0;
    std::vector<uint64_t> ucnt, lcnt;            // B: this rank's unitig edges by start junction's bucket, loop edges by leader's
    // host ms of synchronised work: junction list, unitigs, visited clear, loops, then A/T edges probe, A/T edges apply, A/T tips
    // probe, tip probe, isolate, unlink
    float ms[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    virtual ~DistGraph() = default;
    virtual void junctions() = 0;
    virtual void clip_phase(int p) = 0;
    virtual void unitigs() = 0;
    virtual void clear_visited() = 0;
    virtual void loops() = 0;
    DistView view() const {
        DistView v;
        v.peers = d_peers.p; v.owner = d_owner.p; v.powner = d_powner.p;
        v.dom = dom.p; v.woff = woff.p; v.lstart = lstart.p; v.ustart = d_ustart.p;
        v.pdom = pdom.p; v.pwoff = pwoff.p; v.pstart = pstart.p;
        v.B = (uint32_t)B; v.have_cov = with_cov; v.err = err.p;
        v.self = rank; v.remote = cstats.p + 8;
        return v;
    }
    // fails the call when a walk met a k-mer its owner's index does not hold
    void check_lookups() {
        unsigned long long h = 0;
        SG_CUDA(cudaMemcpyAsync(&h, err.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        SG_CUDA(cudaStreamSynchronize(ctx->stream));
        SG_CHECK(h == 0, 2, "distributed graph: an owner's index rejected a k-mer of a walk (owner tables or sets inconsistent)");
    }
};

template <int NW, int NWS>
struct DistGraphNW : DistGraph {
    void junctions() override { jk = junction_keys<NW>(ctx, *kmers, K, mphf_dev(ext.mk), masks.p); }

    // one phase over this rank's k-mers (the probes and unlinks launch one kernel per chunk of its set)
    void clip_phase(int p) override {
        cudaStream_t st = ctx->stream;
        const DistView v = view();
        const AtParams ap = at_params(opt);
        unsigned long long *s = cstats.p;
        auto sweep = [&](auto &&launch) {
            kmers->sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *) { launch(c, keys); ctx->launches++; });
        };
        switch (p) {
        case kAtEdgesProbe:
            sweep([&](const Chunk &c, const uint64_t *keys) { dist_at_edges_probe_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(v, keys, c.n, K, ap, s); });
            break;
        case kAtEdgesApply:
            sweep([&](const Chunk &c, const uint64_t *keys) { dist_at_edges_apply_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(v, keys, c.n, K, s); });
            break;
        case kAtTipsProbe:
            sweep([&](const Chunk &c, const uint64_t *keys) { dist_at_tips_probe_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(v, keys, c.n, K, ap, s); });
            break;
        case kTipProbe:
            sweep([&](const Chunk &c, const uint64_t *keys) {
                dist_tc_probe_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(v, keys, c.first, c.n, K, tip_bound(opt), tipped.p, s + 4);
            });
            break;
        case kAtIsolate:
        case kTipIsolate:                        // the marks are cleared for the next clipper's probe (after the next barrier)
            launch_isolate(ctx, masks.p, mark.p, nk);
            SG_CUDA(cudaMemsetAsync(mark.p, 0, mark.bytes(), st));
            break;
        case kAtUnlink:
            sweep([&](const Chunk &c, const uint64_t *keys) { dist_tc_links_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(v, keys, c.first, c.n, K, nullptr, s + 3, 1); });
            break;
        case kTipUnlink:
            sweep([&](const Chunk &c, const uint64_t *keys) { dist_tc_links_k<NW><<<div_up(2 * c.n, 128), 128, 0, st>>>(v, keys, c.first, c.n, K, tipped.p, s + 6, 0); });
            break;
        case kJunctions:                         // no peer touches the flags any more
            mark.release(); tipped.release(); eflag.release(); rooted.release();
            masks_final.alloc(ctx, (size_t)nk + 8, true);
            SG_CUDA(cudaMemcpyAsync(masks_final.p, masks.p, (size_t)nk + 8, cudaMemcpyDeviceToDevice, st));
            junctions();
            break;
        }
        check_lookups();
    }

    void unitigs() override {
        cudaStream_t st = ctx->stream;
        const DistView v = view();
        DArr<unsigned long long> cnt(ctx, (size_t)B);
        SG_CUDA(cudaMemsetAsync(cnt.p, 0, cnt.bytes(), st));
        Trace tr("sgpu dist graph", st);
        batches = unitig_batches(
            ctx, &edges, jk, NW, budget ? budget : ctx->budget_left(), tr,
            [&](const uint64_t *bkeys, int64_t nj, uint32_t *len, uint8_t *selfc) {
                dist_unitig_probe_k<NW><<<div_up(nj * 8, 128), 128, 0, st>>>(v, bkeys, nj, K, nk_union, len, selfc);
            },
            [&](const uint64_t *bkeys, int64_t nj, const uint32_t *len) {
                check_lookups();
                dist_edge_buckets_k<NW><<<div_up(nj * 8, 256), 256, 0, st>>>(bkeys, nj, len, (uint32_t)B, cnt.p);
                ctx->launches++;
            },
            [&](const uint64_t *bkeys, int64_t nj, const uint32_t *len, const uint8_t *selfc, const uint64_t *eidx, const uint64_t *eoff, const EdgeBatch &eb) {
                dist_unitig_write_k<NW, NWS><<<div_up(nj * 8, 128), 128, 0, st>>>(v, bkeys, nj, K, nk_union, len, selfc, eidx, eoff, eb.out(nullptr));
            });
        check_lookups();
        unitig_edges = edges.edge_len.size();
        ucnt.assign((size_t)B, 0);
        SG_CUDA(cudaMemcpyAsync(ucnt.data(), cnt.p, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
    }

    void clear_visited() override {
        const uint64_t nwords = (nk + 31) / 32;
        uint64_t rem = 0;
        if (nk) {                                        // a rank may own no k-mer at all (fewer buckets than ranks)
            rem = masks_clear_visited(ctx, masks.p, visited.p, nk, rem_bits.p);
            rem_slot_base(ctx, rem_bits.p, nwords, rem_base.p);
        }
        rem_pos.alloc(ctx, (size_t)std::max<uint64_t>(rem, 1));
        if (rem) loop_positions<NW>(ctx, *kmers, mphf_dev(ext.mk), RemSlots{rem_bits.p, rem_base.p}, rem_pos.p);
        SG_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    void loops() override {
        cudaStream_t st = ctx->stream;
        const DistView v = view();
        KeyParts lk = collect_keys<NW>(ctx, *kmers, [&](const Chunk &c, const uint64_t *keys, uint32_t *flag) {
            dist_loop_leader_k<NW><<<div_up(c.n, 128), 128, 0, st>>>(v, keys, c.first, c.n, nk_union, K, flag);
        });
        check_lookups();
        loop_edges(ctx, &edges, lk, NW, K,
            [&](const uint64_t *leaders, int64_t nl, LoopInfo *info, uint32_t *llen) {
                dist_loop_probe_k<NW, NWS><<<div_up(nl, 64), 64, 0, st>>>(v, leaders, nl, K, info, llen);
            },
            [&](const uint64_t *leaders, int64_t nl, const std::vector<uint32_t> &llen) {
                check_lookups();
                // the loop edges per bucket of their leader (a few keys: counted on the host)
                std::vector<uint64_t> h((size_t)nl * NW);
                SG_CUDA(cudaMemcpy(h.data(), leaders, h.size() * 8, cudaMemcpyDeviceToHost));
                for (int64_t q = 0; q < nl; ++q) {
                    Kmer<NW> k;
                    for (int z = 0; z < NW; ++z) k.w[z] = h[(size_t)q * NW + z];
                    lcnt[kmer_bucket<NW>(k, (uint32_t)B)] += (llen[2 * q] ? 1 : 0) + (llen[2 * q + 1] ? 1 : 0);
                }
            },
            [&](const LoopInfo *info, int64_t nl, const uint32_t *llen, const uint64_t *leidx, const uint64_t *leoff, const EdgeBatch &eb, char *scratch,
                const uint64_t *soff) {
                dist_loop_write_k<NW, NWS><<<div_up(nl, 64), 64, 0, st>>>(v, info, nl, K, llen, leidx, leoff, eb.out(nullptr), scratch, soff);
            });
        check_lookups();
    }
};

// ---- host entries ----------------------------------------------------------------------------------------------------------
DistGraph *dgraph_begin(Ctx *ctx, const ExtDist *e, const int *kmer_owner, const int *kpomer_owner, const uint64_t *kmer_bucket_sizes, uint64_t budget,
                        const GraphOptions &opt) {
    const ExtSlices x = ext_slices(e);
    SG_CHECK(x.ctx == ctx, 2, "distributed graph: the extension index belongs to another context");
    SG_CHECK(x.km->K % 2 == 1, 2, "distributed graph: k must be odd (gbuilder.cpp:125)");
    // on every rank alike, whether it owns k-mers or not (one GPU checks it only for a non-empty set)
    SG_CHECK(!opt.early_at || opt.at_min_len <= (uint64_t)x.km->K, 2, "early A/T clipper: min_length must not exceed k (the reference indexes kh[k - 1 - i])");
    const int B = x.km->B;
    for (int b = 0; b < B; ++b) SG_CHECK(kmer_owner[b] == x.owner[b], 2, "distributed graph: the k-mer owner table is not the extension index's");
    const bool with_cov = x.cov != nullptr;
    SG_CHECK(!with_cov || kpomer_owner, 2, "distributed graph: coverage needs the (k+1)-mer owner table");
    if (with_cov) {
        std::vector<uint8_t> own((size_t)B, 0);
        for (const Chunk &ch : x.kp->chunks) std::fill(own.begin() + ch.b_lo, own.begin() + ch.b_hi, (uint8_t)1);
        for (int b = 0; b < B; ++b) {
            SG_CHECK(kpomer_owner[b] >= 0 && kpomer_owner[b] < x.world, 2, "distributed graph: a (k+1)-mer owner rank outside [0, world)");
            SG_CHECK((kpomer_owner[b] == x.rank) == (own[b] != 0), 2, "distributed graph: the (k+1)-mer owner table does not match this rank's (k+1)-mer set");
        }
    }
    uint64_t nk_union = 0;
    std::vector<uint64_t> ustart((size_t)B);
    for (int b = 0; b < B; ++b) {
        SG_CHECK(x.owner[b] != x.rank || (uint64_t)x.km->bsz[b] == kmer_bucket_sizes[b], 2,
                 "distributed graph: the union's size of a bucket this rank owns is not its own");
        ustart[b] = nk_union;
        nk_union += kmer_bucket_sizes[b];
    }
    const int nw = x.km->nw, nws = x.kp->nw;
    DistGraph *d = nullptr;
    if (nw == 1 && nws == 1) d = new DistGraphNW<1, 1>();
    else if (nw == 1 && nws == 2) d = new DistGraphNW<1, 2>();
    else if (nw == 2 && nws == 2) d = new DistGraphNW<2, 2>();
    else if (nw == 2 && nws == 3) d = new DistGraphNW<2, 3>();
    else if (nw == 3 && nws == 3) d = new DistGraphNW<3, 3>();
    else if (nw == 3 && nws == 4) d = new DistGraphNW<3, 4>();
    else if (nw == 4 && nws == 4) d = new DistGraphNW<4, 4>();
    else throw Error(2, "distributed graph: unsupported word combination");
    d->ctx = ctx; d->ext = x; d->opt = opt;
    d->clip = opt.early_at || opt.early_tip_length_bound;
    if (opt.early_at) d->phases = {kAtEdgesProbe, kAtEdgesApply, kAtTipsProbe, kAtIsolate, kAtUnlink};
    if (opt.early_tip_length_bound) d->phases.insert(d->phases.end(), {kTipProbe, kTipIsolate, kTipUnlink});
    d->phases.push_back(kJunctions);
    d->K = x.km->K; d->B = B; d->world = x.world; d->rank = x.rank; d->with_cov = with_cov;
    d->nk = (uint64_t)x.km->n; d->nk_union = nk_union; d->budget = budget;
    d->owner.assign(kmer_owner, kmer_owner + B);
    if (with_cov) d->powner.assign(kpomer_owner, kpomer_owner + B);
    d->ustart = ustart;
    d->edges.k = d->K;
    d->lcnt.assign((size_t)B, 0);
    d->ucnt.assign((size_t)B, 0);
    ctx->times.stage_h2d_bytes = 0;
    try {
        cudaStream_t st = ctx->stream;
        Stopwatch sw;
        // what peers read first (it stays), then the junction list
        const uint64_t nwords = (d->nk + 31) / 32;
        d->masks.alloc(ctx, (size_t)d->nk + 8, true);
        d->visited.alloc(ctx, (size_t)d->nk + 8, true);
        d->rem_bits.alloc(ctx, (size_t)nwords + 1, true);
        d->rem_base.alloc(ctx, (size_t)nwords + 1, true);
        d->err.alloc(ctx, 1, true);
        d->cstats.alloc(ctx, 11, true);
        SG_CUDA(cudaMemcpyAsync(d->masks.p, x.masks, (size_t)d->nk + 8, cudaMemcpyDeviceToDevice, st));
        SG_CUDA(cudaMemsetAsync(d->visited.p, 0, d->visited.bytes(), st));
        SG_CUDA(cudaMemsetAsync(d->err.p, 0, 8, st));
        SG_CUDA(cudaMemsetAsync(d->cstats.p, 0, d->cstats.bytes(), st));
        // the clippers' flags; peers store into mark and rooted
        if (d->clip) {
            d->mark.alloc(ctx, (size_t)d->nk + 8, true);
            SG_CUDA(cudaMemsetAsync(d->mark.p, 0, d->mark.bytes(), st));
        }
        if (opt.early_tip_length_bound) d->tipped.alloc(ctx, 2 * (size_t)d->nk + 8, true);
        if (opt.early_at) {
            d->eflag.alloc(ctx, 2 * (size_t)d->nk + 8, true);
            d->rooted.alloc(ctx, 2 * (size_t)d->nk + 8, true);
            SG_CUDA(cudaMemsetAsync(d->rooted.p, 0, d->rooted.bytes(), st));
        }
        d->kmers.reset(new ChunkStager(x.km, false));
        if (!d->clip) {                              // the junction list right away: nothing changes the masks before it
            d->junctions();
            d->next = d->phases.size();
        }
        SG_CUDA(cudaStreamSynchronize(st));
        d->ms[0] = sw.ms();
    } catch (...) { delete d; throw; }
    return d;
}

void dgraph_ipc_handle(DistGraph *d, uint8_t *out256) {
    Ctx *ctx = d->ctx;
    GraphDesc ds;
    memset(&ds, 0, sizeof ds);
    const char *what = "distributed graph: an array the peers read did not fit the device memory arena";
    auto off = [&](const void *p) { return p ? ctx->arena_offset(p, what) : ~0ull; };
    const Mphf *mk = d->ext.mk, *mkp = d->ext.mkp;
    ds.off[kDescBits] = off(mk->bits.p); ds.off[kDescRanks] = off(mk->ranks.p);
    ds.off[kDescDom] = off(mk->d_dom.p); ds.off[kDescWoff] = off(mk->d_woff.p); ds.off[kDescStarts] = off(mk->d_starts.p);
    ds.off[kDescMasks] = off(d->masks.p); ds.off[kDescVisited] = off(d->visited.p);
    ds.off[kDescPbits] = off(d->with_cov ? mkp->bits.p : nullptr); ds.off[kDescPranks] = off(d->with_cov ? mkp->ranks.p : nullptr);
    ds.off[kDescPdom] = off(d->with_cov ? mkp->d_dom.p : nullptr); ds.off[kDescPwoff] = off(d->with_cov ? mkp->d_woff.p : nullptr);
    ds.off[kDescPstarts] = off(d->with_cov ? mkp->d_starts.p : nullptr); ds.off[kDescCov] = off(d->ext.cov);
    ds.off[kDescRemBits] = off(d->rem_bits.p); ds.off[kDescRemBase] = off(d->rem_base.p); ds.off[kDescRemPos] = off(d->rem_pos.p);
    ds.off[kDescMark] = off(d->mark.p); ds.off[kDescEflag] = off(d->eflag.p); ds.off[kDescRooted] = off(d->rooted.p);
    cudaDeviceProp prop;
    SG_CUDA(cudaGetDeviceProperties(&prop, ctx->device));
    ds.device = prop.uuid;
    ds.arena_size = ctx->arena_size;
    if (d->world > 1) SG_CUDA(cudaIpcGetMemHandle(&ds.arena, ctx->arena));
    memcpy(out256, &ds, sizeof ds);
}

// the rows of the buckets rank g owns (owner[b] == g) out of its table of `levels` x B entries (as mapped here) into `merged`
static void merge_rows(const uint64_t *peer, int levels, int B, int g, const std::vector<int> &owner, std::vector<uint64_t> &merged) {
    std::vector<uint64_t> h((size_t)levels * B);
    SG_CUDA(cudaMemcpy(h.data(), peer, h.size() * 8, cudaMemcpyDefault));
    for (int l = 0; l < levels; ++l)
        for (int b = 0; b < B; ++b)
            if (owner[b] == g) merged[(size_t)l * B + b] = h[(size_t)l * B + b];
}

// the visible device with this UUID, -1 if none
int device_of(const cudaUUID_t &u) {
    int n = 0;
    SG_CUDA(cudaGetDeviceCount(&n));
    for (int i = 0; i < n; ++i) {
        cudaDeviceProp p;
        SG_CUDA(cudaGetDeviceProperties(&p, i));
        if (!memcmp(&p.uuid, &u, sizeof u)) return i;
    }
    return -1;
}

void dgraph_open_peers(DistGraph *d, const uint8_t *descs) {
    Ctx *ctx = d->ctx;
    const int B = d->B;
    const bool clipping = d->next < d->phases.size() && d->phases[d->next] != kJunctions;
    std::vector<DistPeer> peers((size_t)d->world);
    std::vector<GraphDesc> ds((size_t)d->world);
    for (int g = 0; g < d->world; ++g) memcpy(&ds[g], descs + (size_t)g * sizeof(GraphDesc), sizeof(GraphDesc));
    // the A/T clipper's bit clears are 32-bit atomics on the owners' masks: across devices they need native peer atomics
    if (clipping && d->opt.early_at) {
        const int mine = device_of(ds[d->rank].device);
        for (int g = 0; g < d->world; ++g) {
            const int dev = device_of(ds[g].device);
            if (dev == mine) continue;
            SG_CHECK(dev >= 0, 2, "distributed graph: a peer's device is not visible here, so its peer atomics cannot be checked");
            int native = 0;
            SG_CUDA(cudaDeviceGetP2PAttribute(&native, cudaDevP2PAttrNativeAtomicSupported, ctx->device, dev));
            SG_CHECK(native, 2, "distributed graph: the early A/T clipper needs native atomics between this device and a peer's");
        }
    }
    for (int g = 0; g < d->world; ++g) {
        char *base = ctx->peer_map(d->world, d->rank, g, &ds[g].arena);
        for (int a = 0; a < kDescArrays; ++a)
            SG_CHECK(ds[g].off[a] == ~0ull || ds[g].off[a] < ds[g].arena_size, 2, "bad peer descriptor");
        auto at = [&](int a) { return ds[g].off[a] == ~0ull ? nullptr : (void *)(base + ds[g].off[a]); };
        SG_CHECK(at(kDescBits) && at(kDescMasks) && at(kDescVisited) && at(kDescRemBits) && (!d->with_cov || (at(kDescPbits) && at(kDescCov))), 2,
                 "bad peer descriptor");
        SG_CHECK(!clipping || (at(kDescMark) && (!d->opt.early_at || (at(kDescEflag) && at(kDescRooted)))), 2, "bad peer descriptor");
        peers[g] = DistPeer{(const uint64_t *)at(kDescBits), (const uint64_t *)at(kDescRanks), (uint8_t *)at(kDescMasks),
                            (uint8_t *)at(kDescVisited), (const uint64_t *)at(kDescPbits), (const uint64_t *)at(kDescPranks),
                            (const uint32_t *)at(kDescCov), (const uint32_t *)at(kDescRemBits), (const uint64_t *)at(kDescRemBase),
                            (const uint64_t *)at(kDescRemPos), (uint8_t *)at(kDescMark), (uint8_t *)at(kDescEflag), (uint8_t *)at(kDescRooted)};
    }
    if (!d->tables) {
        // every owner's per-bucket index rows, copied once: a lookup then reads only the owner's bits and ranks remotely
        std::vector<uint64_t> dom((size_t)kLevels * B), woff((size_t)kLevels * B), ls((size_t)B);
        std::vector<uint64_t> pdom, pwoff, ps;
        if (d->with_cov) { pdom.assign((size_t)kLevels * B, 0); pwoff.assign((size_t)kLevels * B, 0); ps.assign((size_t)B, 0); }
        for (int g = 0; g < d->world; ++g) {
            char *base = ctx->peer_map(d->world, d->rank, g, &ds[g].arena);
            auto at = [&](int a) { return (const uint64_t *)(base + ds[g].off[a]); };
            merge_rows(at(kDescDom), kLevels, B, g, d->owner, dom);
            merge_rows(at(kDescWoff), kLevels, B, g, d->owner, woff);
            merge_rows(at(kDescStarts), 1, B, g, d->owner, ls);
            if (d->with_cov) {
                merge_rows(at(kDescPdom), kLevels, B, g, d->powner, pdom);
                merge_rows(at(kDescPwoff), kLevels, B, g, d->powner, pwoff);
                merge_rows(at(kDescPstarts), 1, B, g, d->powner, ps);
            }
        }
        auto up = [&](DArr<uint64_t> &a, const std::vector<uint64_t> &h) {
            a.alloc(ctx, h.size(), true);
            SG_CUDA(cudaMemcpy(a.p, h.data(), h.size() * 8, cudaMemcpyHostToDevice));
        };
        up(d->dom, dom); up(d->woff, woff); up(d->lstart, ls); up(d->d_ustart, d->ustart);
        d->d_owner.alloc(ctx, (size_t)B, true);
        SG_CUDA(cudaMemcpy(d->d_owner.p, d->owner.data(), (size_t)B * sizeof(int), cudaMemcpyHostToDevice));
        if (d->with_cov) {
            up(d->pdom, pdom); up(d->pwoff, pwoff); up(d->pstart, ps);
            d->d_powner.alloc(ctx, (size_t)B, true);
            SG_CUDA(cudaMemcpy(d->d_powner.p, d->powner.data(), (size_t)B * sizeof(int), cudaMemcpyHostToDevice));
        }
        d->d_peers.alloc(ctx, (size_t)d->world, true);
        d->tables = true;
    }
    SG_CUDA(cudaMemcpy(d->d_peers.p, peers.data(), peers.size() * sizeof(DistPeer), cudaMemcpyHostToDevice));
}

static void timed(DistGraph *d, int i, void (DistGraph::*phase)()) {
    Stopwatch sw;
    (d->*phase)();
    d->ms[i] += sw.ms();
}
// the phase of phases[next] when it is one of `a` or `b`
void dgraph_clip_phase(DistGraph *d, int a, int b) {
    SG_CHECK(d->tables, 2, "sgpu_dist_graph_open_peers has not run");
    SG_CHECK(d->next < d->phases.size() && (d->phases[d->next] == a || d->phases[d->next] == b), 2,
             "distributed graph: phase called out of order, or for a clipper that is off");
    const int p = d->phases[d->next];
    static const int slot[] = {4, 5, 6, 8, 9, 7, 8, 9, 0};
    Stopwatch sw;
    d->clip_phase(p);
    d->ms[slot[p]] += sw.ms();
    ++d->next;
}
void dgraph_unitigs(DistGraph *d) {
    SG_CHECK(d->tables, 2, "sgpu_dist_graph_open_peers has not run");
    SG_CHECK(d->next == d->phases.size(), 2, "the early clippers and the junction list have not run");
    SG_CHECK(d->unitig_edges == 0 && d->edges.edge_len.empty() && !d->rem_pos.p, 2, "the unitigs have been extracted already");
    timed(d, 1, &DistGraph::unitigs);
}
void dgraph_clear_visited(DistGraph *d) {
    SG_CHECK(!d->rem_pos.p, 2, "the visited k-mers have been cleared already");
    timed(d, 2, &DistGraph::clear_visited);
}
void dgraph_loops(DistGraph *d) {
    SG_CHECK(d->rem_pos.p, 2, "sgpu_dist_graph_clear_visited has not run");
    SG_CHECK(d->edges.edge_len.size() == d->unitig_edges, 2, "the loops have been extracted already");
    timed(d, 3, &DistGraph::loops);
}
const Graph &dgraph_edges(const DistGraph *d) { return d->edges; }
void dgraph_stats(const DistGraph *d, uint64_t *out4) {
    out4[0] = d->edges.edge_len.size(); out4[1] = d->unitig_edges; out4[2] = d->edges.seq.size(); out4[3] = d->batches;
}
void dgraph_bucket_counts(const DistGraph *d, uint64_t *unitigs, uint64_t *loops) {
    std::copy(d->ucnt.begin(), d->ucnt.end(), unitigs);
    std::copy(d->lcnt.begin(), d->lcnt.end(), loops);
}
void dgraph_times(const DistGraph *d, float *out4) { for (int i = 0; i < 4; ++i) out4[i] = d->ms[i]; }
void dgraph_clip_times(const DistGraph *d, float *out6) { for (int i = 0; i < 6; ++i) out6[i] = d->ms[4 + i]; }
void dgraph_clip_stats(const DistGraph *d, uint64_t *at4, uint64_t *tc3, uint64_t *remote3) {
    unsigned long long h[11];
    SG_CUDA(cudaMemcpy(h, d->cstats.p, sizeof h, cudaMemcpyDeviceToHost));
    for (int i = 0; i < 4; ++i) at4[i] = h[i];
    for (int i = 0; i < 3; ++i) tc3[i] = h[4 + i];
    for (int i = 0; i < 3; ++i) remote3[i] = h[8 + i];
}
void dgraph_masks(const DistGraph *d, uint8_t *out, int64_t n) {
    SG_CHECK(d->next == d->phases.size(), 2, "the early clippers and the junction list have not run");
    SG_CHECK((uint64_t)n == d->nk, 2, "mask array size != number of this rank's k-mers");
    if (n) SG_CUDA(cudaMemcpy(out, d->clip ? d->masks_final.p : d->ext.masks, (size_t)n, cudaMemcpyDeviceToHost));
}
DistGraphInfo dgraph_info(const DistGraph *d) {
    return DistGraphInfo{d->ctx, d->world, d->rank, d->B, d->K, &d->owner, &d->ucnt, &d->lcnt, d->unitig_edges, &d->edges};
}
void dgraph_free(DistGraph *d) { delete d; }

}  // namespace sg
