// dist_edge_index.cu -- the EdgeIndex refill across GPUs (one process per GPU), from each rank's share of a distributed graph
// (dist_graph.cu): what edge_index.cu builds on one GPU over the union, byte for byte.
//   keys   : the distributed canonical count (count.cu, dist_begin_packed) over each rank's own edges, packed as edge_index.cu packs
//            them. For K = k+1 its buckets are the graph's k-mer buckets: they only decide which rank owns a key, the index has one
//            segment as on one GPU; any other K counts into num_buckets buckets, the index's own.
//   index  : ONE index over the union, built by all ranks together and held by every rank. A single-segment boomphf's bits depend
//            on every key, so no rank can build a share of it alone; but a level's bit is set iff exactly one still-unplaced key of
//            the union hashed to it, so every rank inserts its own keys into its copy of a level and the copies are merged through
//            the peer mappings (mphf.cu, MphfPlacer) before anyone filters against it. The geometry comes from the union's bucket
//            sizes, so the bits, ranks and serialized bytes are those of one GPU's index.
//   values : rank r holds the slots [n r / W, n (r+1) / W), one 64-bit word per slot (edge id << 32 | offset). Every rank walks the
//            windows of its own edges (edge_window, as edge_index.cu), looks the slot up in its copy of the index and puts into the
//            owner's word with a system-scope CAS: the first put leaves its value, any further one a tombstone, in any order.
//            Edge ids are the union's: a rank numbers its edges from the all-gathered per-bucket edge counts in the order
//            assemble_graph lays the ranks' edges out.
// Memory: every rank holds the union's index (about 0.65 B per union key at gamma = 4) and, while the levels are placed, the
// level-0 collision and merge words (about 1 B per union key). That departs from the rest of the distributed path, where no rank
// holds memory in proportion to the union; it is the price of a single-segment index.
#include "edge_dev.cuh"

namespace sg {

static const unsigned long long kSlotCleared = ~0ull;                                        // no put yet
static const unsigned long long kSlotTomb = 0xffffffff00000000ull | kEdgeInfoTombstone;      // put more than once
static const uint64_t kMaxUnionEdges = (1ull << 31) - 2;                                     // 3 + 2 e + 1 fits 32 bits

// the owner of slot idx: the last rank whose range starts at or before it
__device__ __forceinline__ int slot_owner(uint64_t idx, uint64_t n, int world) {
    int r = (int)(idx * (uint64_t)world / n);           // its range starts at or before idx
    while (r + 1 < world && dist_slot_lo(n, world, r + 1) <= idx) ++r;
    return r;
}

template <int NW>
__global__ void dist_edge_put_k(UnitigTable u, int K, uint64_t nwork, MphfDev m, const uint32_t *__restrict__ uid, uint64_t *const *__restrict__ slices,
                                int world, uint64_t n, unsigned long long *__restrict__ err) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    uint32_t e, off; int s; Kmer<NW> k;
    if (!edge_window<NW>(u, K, w, &e, &s, &off, &k)) return;
    const uint64_t idx = mphf_lookup_dev<NW>(m, k);
    if (idx >= n) { atomicAdd(err, 1ull); return; }
    const int r = slot_owner(idx, n, world);
    const unsigned long long v = ((unsigned long long)(3u + 2u * uid[e] + (uint32_t)s) << 32) | off;
    unsigned long long *p = (unsigned long long *)(slices[r] + (idx - dist_slot_lo(n, world, r)));
    if (atomicCAS_system(p, kSlotCleared, v) != kSlotCleared) atomicExch_system(p, kSlotTomb);
}

__global__ void dist_edge_expand_k(const uint64_t *__restrict__ slice, uint64_t n, uint64_t *__restrict__ ids, uint32_t *__restrict__ offs) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t v = slice[i];
    if (v == kSlotCleared) { ids[i] = ~0ull; offs[i] = kEdgeInfoCleared; }
    else if (v == kSlotTomb) { ids[i] = ~1ull; offs[i] = kEdgeInfoTombstone; }
    else { ids[i] = v >> 32; offs[i] = (uint32_t)v; }
}

// what a rank publishes: its arena, where its index bits, collision words and slot slice lie in it, and its device
struct DeiDesc {
    cudaIpcMemHandle_t arena;     // 64 bytes
    uint64_t arena_size, off_bits, off_coll, off_slice;
    cudaUUID_t device;            // 16 bytes
    uint64_t unused[2];
};
static_assert(sizeof(DeiDesc) == 128, "descriptor layout (SGPU_DIST_EDGE_INDEX_IPC_BYTES)");

enum { kStepMerge, kStepAdvance, kStepLevelDone, kStepPlaced };

struct DistEdgeIndex {
    Ctx *ctx = nullptr;
    int K = 0, Bc = 0, Bi = 0, world = 1, rank = 0;
    bool single = false;
    EdgePack pack;
    DArr<uint32_t> uid;                  // the union number of each of this rank's edges
    const KSet *ks = nullptr;            // this rank's keys, read until the levels are placed
    Mphf *m = nullptr;                   // the union's index
    MphfPlacer pl;
    DArr<uint64_t> slice;                // this rank's slots; peers put into it
    uint64_t n = 0, lo = 0, hi = 0;
    DArr<const uint64_t *> d_bits, d_coll;
    DArr<uint64_t *> d_slices;
    DArr<unsigned long long> err;
    bool opened = false, ranked = false, filled = false;
    int step = kStepMerge;
    float ms[6] = {0, 0, 0, 0, 0, 0};    // pack, keys, levels, ranks, fill, values
    ~DistEdgeIndex() { delete m; }
};

void dist_edge_numbers(int world, int rank, int B, const int *owner, const uint64_t *ucnt_all, const uint64_t *lcnt_all, uint64_t unitig_edges,
                       uint64_t edges, uint64_t *out) {
    SG_CHECK(world >= 1 && rank >= 0 && rank < world && B >= 1 && unitig_edges <= edges, 2, "edge numbers: bad arguments");
    uint64_t base = 0, cur[2] = {0, unitig_edges};
    const uint64_t *tab[2] = {ucnt_all, lcnt_all};
    for (int t = 0; t < 2; ++t)
        for (int b = 0; b < B; ++b) {
            const int o = owner[b];
            SG_CHECK(o >= 0 && o < world, 2, "edge numbers: a bucket owner outside [0, world)");
            for (int g = 0; g < world; ++g)
                SG_CHECK(g == o || tab[t][(size_t)g * B + b] == 0, 2, "edge numbers: a rank counts edges of a bucket it does not own");
            const uint64_t c = tab[t][(size_t)o * B + b];
            if (o == rank) {
                SG_CHECK(cur[t] + c <= (t == 0 ? unitig_edges : edges), 2, "edge numbers: this rank's bucket counts exceed its edges");
                for (uint64_t i = 0; i < c; ++i) out[cur[t] + i] = base + i;
                cur[t] += c;
            }
            base += c;
        }
    SG_CHECK(cur[0] == unitig_edges && cur[1] == edges, 2, "edge numbers: this rank's bucket counts do not cover its edges");
    SG_CHECK(base <= kMaxUnionEdges, 7, "distributed edge index: more than 2^31 - 2 union edges (edge ids would not fit 32 bits)");
}

DistEdgeIndex *dei_begin(Ctx *ctx, const DistGraph *dg, int K, int num_buckets, const uint64_t *ucnt_all, const uint64_t *lcnt_all) {
    Stopwatch sw;
    const DistGraphInfo gi = dgraph_info(dg);
    SG_CHECK(gi.ctx == ctx, 2, "distributed edge index: the graph belongs to another context");
    if (K == 0) K = gi.k + 1;
    SG_CHECK(K >= 1 && K <= gi.k + 1 && K <= 128, 2, "edge index: K must be in [1, k+1]");
    SG_CHECK(num_buckets >= 1, 2, "edge index: num_buckets must be >= 1");
    const bool kp1 = K == gi.k + 1;
    const int Bc = kp1 ? gi.B : num_buckets;
    SG_CHECK(Bc <= 8192, 2, "distributed edge index: num_buckets must be in [1, 8192] (the distributed count's limit)");
    const Graph *g = gi.edges;
    const size_t E = g->edge_len.size();
    for (int b = 0; b < gi.B; ++b)
        SG_CHECK(ucnt_all[(size_t)gi.rank * gi.B + b] == (*gi.ucnt)[b] && lcnt_all[(size_t)gi.rank * gi.B + b] == (*gi.lcnt)[b], 2,
                 "distributed edge index: this rank's row of the bucket counts is not its graph's");
    std::vector<uint64_t> num(E + 1, 0);
    dist_edge_numbers(gi.world, gi.rank, gi.B, gi.owner->data(), ucnt_all, lcnt_all, gi.unitig_edges, (uint64_t)E, num.data());
    std::vector<uint32_t> num32(E + 1, 0);
    for (size_t i = 0; i < E; ++i) num32[i] = (uint32_t)num[i];
    DistEdgeIndex *d = new DistEdgeIndex();
    d->ctx = ctx; d->K = K; d->Bc = Bc; d->Bi = kp1 ? 1 : num_buckets; d->world = gi.world; d->rank = gi.rank;
    try {
        edge_pack(ctx, g, K, &d->pack);
        d->uid.alloc(ctx, E + 1, true);
        SG_CUDA(cudaMemcpy(d->uid.p, num32.data(), (E + 1) * 4, cudaMemcpyHostToDevice));
        d->err.alloc(ctx, 1, true);
        SG_CUDA(cudaMemset(d->err.p, 0, 8));
    } catch (...) { delete d; throw; }
    d->ms[0] = sw.ms();
    return d;
}

DistState *dei_count_begin(DistEdgeIndex *d, int world, int rank) {
    SG_CHECK(world == d->world && rank == d->rank, 2, "distributed edge index: world / rank differ from the graph's");
    SG_CHECK(!d->m, 2, "distributed edge index: the keys have been given already");
    const EdgePack &p = d->pack;
    return dist_begin_packed(d->ctx, p.words.p, p.nwords, p.woff.p, p.lens.p, p.E, d->K, d->Bc, world, rank);
}

void dei_keys(DistEdgeIndex *d, const KSet *ks, const uint64_t *ubsz, int single) {
    Stopwatch sw;
    Ctx *ctx = d->ctx;
    SG_CHECK(!d->m, 2, "distributed edge index: the keys have been given already");
    SG_CHECK(ks->ctx == ctx && ks->K == d->K && ks->B == d->Bc, 2, "distributed edge index: the key set is not the count over this rank's edges");
    SG_CHECK(!ks->on_host, 7, "distributed edge index: the key set lives in host memory");
    SG_CHECK(!single || d->Bi == 1, 2, "distributed edge index: the single-index flag is for K = k + 1 only");
    uint64_t n = 0;
    for (int b = 0; b < d->Bc; ++b) {
        SG_CHECK((uint64_t)ks->bsz[b] <= ubsz[b], 2, "distributed edge index: a union bucket smaller than this rank's");
        n += ubsz[b];
    }
    std::vector<int64_t> bsz = d->Bi == 1 ? std::vector<int64_t>{(int64_t)n} : std::vector<int64_t>(ubsz, ubsz + d->Bc);
    Mphf *m = new Mphf();
    m->ctx = ctx; m->K = d->K; m->nw = nwords_of(d->K); m->B = d->Bi; m->n = (int64_t)n;
    d->m = m;
    d->ks = ks; d->single = single != 0; d->n = n;
    d->lo = dist_slot_lo(n, d->world, d->rank); d->hi = dist_slot_lo(n, d->world, d->rank + 1);
    const std::vector<uint64_t> level_start = mphf_geometry(ctx, m, bsz);
    d->slice.alloc(ctx, d->hi - d->lo + 1, true);
    SG_CUDA(cudaMemsetAsync(d->slice.p, 0xff, d->slice.bytes(), ctx->stream));
    mphf_place_begin(ctx, m, &d->pl, make_table(ks), (uint64_t)ks->n, level_start);
    d->ms[1] += sw.ms();
}

void dei_ipc_handle(DistEdgeIndex *d, uint8_t *out) {
    Ctx *ctx = d->ctx;
    SG_CHECK(d->m, 2, "sgpu_dist_edge_index_keys has not run");
    DeiDesc ds;
    memset(&ds, 0, sizeof ds);
    const char *what = "distributed edge index: an array the peers read did not fit the device memory arena";
    ds.off_bits = ctx->arena_offset(d->m->bits.p, what);
    ds.off_coll = ctx->arena_offset(d->pl.coll.p, what);
    ds.off_slice = ctx->arena_offset(d->slice.p, what);
    cudaDeviceProp prop;
    SG_CUDA(cudaGetDeviceProperties(&prop, ctx->device));
    ds.device = prop.uuid;
    ds.arena_size = ctx->arena_size;
    if (d->world > 1) SG_CUDA(cudaIpcGetMemHandle(&ds.arena, ctx->arena));
    memcpy(out, &ds, sizeof ds);
}

void dei_open_peers(DistEdgeIndex *d, const uint8_t *descs) {
    Ctx *ctx = d->ctx;
    SG_CHECK(d->m, 2, "sgpu_dist_edge_index_keys has not run");
    std::vector<DeiDesc> ds((size_t)d->world);
    for (int g = 0; g < d->world; ++g) memcpy(&ds[g], descs + (size_t)g * sizeof(DeiDesc), sizeof(DeiDesc));
    // the puts are 64-bit atomics on the owners' slices: across devices they need native peer atomics
    const int mine = device_of(ds[d->rank].device);
    for (int g = 0; g < d->world; ++g) {
        const int dev = device_of(ds[g].device);
        if (dev == mine) continue;
        SG_CHECK(dev >= 0, 2, "distributed edge index: a peer's device is not visible here, so its peer atomics cannot be checked");
        int native = 0;
        SG_CUDA(cudaDeviceGetP2PAttribute(&native, cudaDevP2PAttrNativeAtomicSupported, ctx->device, dev));
        SG_CHECK(native, 2, "distributed edge index: the puts need native atomics between this device and a peer's");
    }
    std::vector<const uint64_t *> bits((size_t)d->world), coll((size_t)d->world);
    std::vector<uint64_t *> slices((size_t)d->world);
    for (int g = 0; g < d->world; ++g) {
        char *base = ctx->peer_map(d->world, d->rank, g, &ds[g].arena);
        SG_CHECK(ds[g].off_bits < ds[g].arena_size && ds[g].off_coll < ds[g].arena_size && ds[g].off_slice < ds[g].arena_size, 2, "bad peer descriptor");
        bits[g] = (const uint64_t *)(base + ds[g].off_bits);
        coll[g] = (const uint64_t *)(base + ds[g].off_coll);
        slices[g] = (uint64_t *)(base + ds[g].off_slice);
    }
    d->d_bits.alloc(ctx, (size_t)d->world, true); d->d_coll.alloc(ctx, (size_t)d->world, true); d->d_slices.alloc(ctx, (size_t)d->world, true);
    SG_CUDA(cudaMemcpy(d->d_bits.p, bits.data(), bits.size() * sizeof(void *), cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d->d_coll.p, coll.data(), coll.size() * sizeof(void *), cudaMemcpyHostToDevice));
    SG_CUDA(cudaMemcpy(d->d_slices.p, slices.data(), slices.size() * sizeof(void *), cudaMemcpyHostToDevice));
    d->opened = true;
}

static void expect_step(const DistEdgeIndex *d, int step) {
    SG_CHECK(d->opened, 2, "sgpu_dist_edge_index_open_peers has not run");
    static const char *what[] = {"distributed edge index: merge called out of order", "distributed edge index: advance called out of order",
                                 "distributed edge index: level_done called out of order", "distributed edge index: the levels are placed already"};
    SG_CHECK(d->step == step, 2, what[d->step == kStepPlaced ? kStepPlaced : step]);
}

void dei_merge(DistEdgeIndex *d) {
    expect_step(d, kStepMerge);
    Stopwatch sw;
    mphf_place_merge(d->ctx, d->m, &d->pl, d->d_bits.p, d->d_coll.p, d->world);
    d->step = kStepAdvance;
    d->ms[2] += sw.ms();
}
uint64_t dei_advance(DistEdgeIndex *d) {
    expect_step(d, kStepAdvance);
    Stopwatch sw;
    const uint64_t live = mphf_place_advance(d->ctx, d->m, &d->pl);
    d->step = kStepLevelDone;
    d->ms[2] += sw.ms();
    return live;
}
int dei_level_done(DistEdgeIndex *d, uint64_t union_live) {
    expect_step(d, kStepLevelDone);
    if (union_live == 0) { d->step = kStepPlaced; return 0; }
    SG_CHECK(d->pl.level < kLevels - 1, 7, "MPHF: keys fell through all 24 bitset levels (reference would use its order-dependent fallback map); unsupported");
    d->step = kStepMerge;
    return 1;
}

void dei_ranks(DistEdgeIndex *d) {
    SG_CHECK(d->m && d->step == kStepPlaced, 2, "distributed edge index: the levels have not all been placed");
    SG_CHECK(!d->ranked, 2, "distributed edge index: the ranks have been computed already");
    Stopwatch sw;
    if (d->n && d->m->total_words) mphf_ranks(d->ctx, d->m);
    // no peer reads the collision words any more (every rank has passed the last merge), and the keys are placed
    d->pl.coll.release(); d->pl.scratch.release(); d->pl.aliveA.release(); d->pl.aliveB.release();
    d->ks = nullptr;
    d->ranked = true;
    d->ms[3] += sw.ms();
}

void dei_fill(DistEdgeIndex *d) {
    SG_CHECK(d->ranked, 2, "sgpu_dist_edge_index_ranks has not run");
    SG_CHECK(!d->filled, 2, "distributed edge index: the values have been filled already");
    Stopwatch sw;
    Ctx *ctx = d->ctx;
    cudaStream_t st = ctx->stream;
    const EdgePack &p = d->pack;
    if (p.nwork && d->n) {
        const UnitigTable u = p.table();
        const MphfDev md = mphf_dev(d->m);
        const int grid = div_up((int64_t)p.nwork, 256);
        switch (nwords_of(d->K)) {
            case 1: dist_edge_put_k<1><<<grid, 256, 0, st>>>(u, d->K, p.nwork, md, d->uid.p, d->d_slices.p, d->world, d->n, d->err.p); break;
            case 2: dist_edge_put_k<2><<<grid, 256, 0, st>>>(u, d->K, p.nwork, md, d->uid.p, d->d_slices.p, d->world, d->n, d->err.p); break;
            case 3: dist_edge_put_k<3><<<grid, 256, 0, st>>>(u, d->K, p.nwork, md, d->uid.p, d->d_slices.p, d->world, d->n, d->err.p); break;
            default: dist_edge_put_k<4><<<grid, 256, 0, st>>>(u, d->K, p.nwork, md, d->uid.p, d->d_slices.p, d->world, d->n, d->err.p); break;
        }
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
    }
    unsigned long long h = 0;
    SG_CUDA(cudaMemcpyAsync(&h, d->err.p, 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    SG_CHECK(h == 0, 6, "internal: a window of an edge is not a key of the union's index");
    d->filled = true;
    d->ms[4] += sw.ms();
}

void dei_values(const DistEdgeIndex *d, uint64_t *ids, uint32_t *offs, int64_t n) {
    SG_CHECK(d->filled, 2, "sgpu_dist_edge_index_fill has not run");
    SG_CHECK((uint64_t)n == d->hi - d->lo, 2, "value array size != this rank's slots");
    if (!n) return;
    Stopwatch sw;
    Ctx *ctx = d->ctx;
    cudaStream_t st = ctx->stream;
    DArr<uint64_t> di(ctx, (size_t)n);
    DArr<uint32_t> dof(ctx, (size_t)n);
    dist_edge_expand_k<<<div_up(n, 256), 256, 0, st>>>(d->slice.p, (uint64_t)n, di.p, dof.p);
    ctx->launches++;
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(ids, di.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(offs, dof.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    const_cast<DistEdgeIndex *>(d)->ms[5] += sw.ms();
}

const Mphf *dei_index(const DistEdgeIndex *d) {
    SG_CHECK(d->ranked, 2, "sgpu_dist_edge_index_ranks has not run");
    return d->m;
}
bool dei_single(const DistEdgeIndex *d) { return d->single; }
int dei_k(const DistEdgeIndex *d) { return d->K; }
void dei_slot_range(const DistEdgeIndex *d, uint64_t *lo, uint64_t *hi) {
    SG_CHECK(d->m, 2, "sgpu_dist_edge_index_keys has not run");
    *lo = d->lo; *hi = d->hi;
}
void dei_times(const DistEdgeIndex *d, float *out6) { for (int i = 0; i < 6; ++i) out6[i] = d->ms[i]; }
void dei_free(DistEdgeIndex *d) { delete d; }

}  // namespace sg
