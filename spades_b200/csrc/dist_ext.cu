// dist_ext.cu -- the extension masks, the (k+1)-mer coverage and its histogram across GPUs (one process per GPU). hpcspades
// fills the masks of every k-mer from each rank's (k+1)-mer buckets and ORs the whole arrays together (ExtensionIndexBuilder,
// FillIndexTask + allreduce(MPI_BOR)), then fills the coverage (PHMCoverageFiller). Here every k-mer bucket has one owner rank
// (the one whose k-mer set holds it), and a rank's arrays are its slices of the union's, in the order of its own indexes:
//   masks     A (k+1)-mer adds one bit to its prefix k-mer and one to its suffix k-mer (masks_dev.cuh); both usually live on
//             other ranks. Per pass (a range of destination buckets), every rank writes its contributions to the pass's buckets
//             into a staging buffer, grouped by owner, and then every owner streams its pieces out of the peers' staging buffers
//             (cudaIpc mappings of their arenas, as the distributed count's exchange does), looks the keys up in its own k-mer
//             index and ORs the bits into its slice. No remote scattered stores, no remote index lookups, no receive buffer.
//   coverage  needs no exchange: a (k+1)-mer is counted exactly at the owner of its bucket, so the coverage slice is the
//             single-GPU fill (cov_perm_k) over this rank's (k+1)-mers against its own (k+1)-mer index, and the histogram of the
//             union is the sum of the ranks' histograms.
// A key's slot in a rank's own index is local_starts[b] + r, where r, its rank inside bucket b, is the same as in the union's
// index (a bucket's MPHF depends only on that bucket's keys): the union's arrays are the owners' bucket runs laid end to end.
#include <memory>

#include "graph.h"
#include "masks_dev.cuh"
#include "mphf_dev.cuh"
#include "pass_plan.h"

namespace sg {

static const int kExtThreads = 256;
static const int kExtMaxBuckets = 8192;      // destination buckets the histogram kernel counts in shared memory
static const int kExtMaxWorld = 255;
static const int kExtMaxPasses = 256;        // every pass sweeps the (k+1)-mers once more

// ---- planning (pure host arithmetic, identical on every rank given the same inputs) ------------------------------------------
// A pass is a range of destination buckets; it is priced by the most records any rank sends or any owner receives in it, at
// 8 NW + 1 bytes a record (key + bit). Nothing a pass makes stays resident (the slices are allocated up front), so the plan
// simulates the job with no outputs.
struct ExtPlan {
    int world = 1, B = 0;
    std::vector<int> owner;          // B: the rank owning k-mer bucket b
    std::vector<uint64_t> sent;      // world x (B+1): records rank s sends to buckets < b
    std::vector<uint64_t> recv;      // world x (B+1): records all ranks send to the buckets < b that rank g owns
    std::vector<uint64_t> cnt_all;   // world x B: records rank s sends to bucket b
    PassPlan passes;
    uint64_t most(int a, int b) const {
        uint64_t m = 0;
        for (int r = 0; r < world; ++r) {
            const size_t o = (size_t)r * (B + 1);
            m = std::max(m, std::max(sent[o + b] - sent[o + a], recv[o + b] - recv[o + a]));
        }
        return m;
    }
    // records rank s sends to owner g in pass p
    uint64_t piece(int p, int s, int g) const {
        uint64_t n = 0;
        for (int b = passes.bounds[p]; b < passes.bounds[p + 1]; ++b)
            if (owner[b] == g) n += cnt_all[(size_t)s * B + b];
        return n;
    }
};

static void ext_plan_tables(ExtPlan &pl, int world, int B, const int *owner, const uint64_t *cnt_all) {
    pl.world = world; pl.B = B;
    pl.owner.assign(owner, owner + B);
    pl.cnt_all.assign(cnt_all, cnt_all + (size_t)world * B);
    pl.sent.assign((size_t)world * (B + 1), 0);
    pl.recv.assign((size_t)world * (B + 1), 0);
    std::vector<uint64_t> before((size_t)B + 1, 0);
    for (int b = 0; b < B; ++b) {
        uint64_t t = 0;
        for (int s = 0; s < world; ++s) {
            const uint64_t c = cnt_all[(size_t)s * B + b];
            const size_t o = (size_t)s * (B + 1);
            pl.sent[o + b + 1] = pl.sent[o + b] + c;
            t += c;
        }
        for (int g = 0; g < world; ++g) {
            const size_t o = (size_t)g * (B + 1);
            pl.recv[o + b + 1] = pl.recv[o + b] + (owner[b] == g ? t : 0);
        }
        before[b + 1] = before[b] + t;
    }
    pl.passes = PassPlan(0, B, std::min(B, kExtMaxPasses), std::move(before));
}

// plans the next pass against budget_bytes (the minimum over the ranks of what they can allocate now); false when every bucket
// has been planned
static bool ext_next_pass(ExtPlan &pl, uint64_t budget_bytes, int record_bytes, uint64_t *most_out) {
    if (pl.passes.done()) return false;
    auto need = [&](int a, int b) { return (double)pl.most(a, b) * record_bytes; };
    if (pl.passes.npass() == 0) pl.passes.aim((double)budget_bytes, false, need, [](int, int) { return 0.0; });
    const int a = pl.passes.bounds.back(), b = pl.passes.next((double)budget_bytes, need);
    *most_out = pl.most(a, b);
    return true;
}

static void check_owner_table(int world, int B, const int *owner) {
    SG_CHECK(world >= 1 && world <= kExtMaxWorld, 2, "distributed extension index: world must be in [1, 255]");
    SG_CHECK(B >= 1 && B <= kExtMaxBuckets, 2, "distributed extension index: num_buckets must be in [1, 8192]");
    for (int b = 0; b < B; ++b) SG_CHECK(owner[b] >= 0 && owner[b] < world, 2, "distributed extension index: an owner rank outside [0, world)");
}

int ext_plan_host(int world, int B, const int *owner, const uint64_t *cnt_all, uint64_t budget_bytes, int record_bytes, int *pass_b, uint64_t *most) {
    check_owner_table(world, B, owner);
    SG_CHECK(record_bytes >= 1, 2, "distributed extension index: bad record size");
    ExtPlan pl;
    ext_plan_tables(pl, world, B, owner, cnt_all);
    uint64_t m = 0, worst = 0;
    while (ext_next_pass(pl, budget_bytes, record_bytes, &m)) worst = std::max(worst, m);
    for (int p = 0; p <= pl.passes.npass(); ++p) pass_b[p] = pl.passes.bounds[p];
    *most = worst;
    return pl.passes.npass();
}

// ---- kernels -------------------------------------------------------------------------------------------------------------
template <int NWS>
__device__ __forceinline__ Kmer<NWS> record_at(const uint64_t *__restrict__ keys, int64_t i) {
    Kmer<NWS> x;
#pragma unroll
    for (int q = 0; q < NWS; ++q) x.w[q] = keys[i * NWS + q];
    return x;
}

// contributions of a chunk's (k+1)-mers per destination k-mer bucket
template <int NW, int NWS>
__global__ void __launch_bounds__(kExtThreads) ext_hist_k(const uint64_t *__restrict__ kp, int64_t n, int K, uint32_t B, unsigned long long *__restrict__ cnt) {
    __shared__ uint32_t s[kExtMaxBuckets];
    for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) s[b] = 0;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const Kmer<NWS> x = record_at<NWS>(kp, i);
        atomicAdd(&s[kmer_bucket<NW>(kpomer_mask_bit<0, NW, NWS>(x, K).key, B)], 1u);
        atomicAdd(&s[kmer_bucket<NW>(kpomer_mask_bit<1, NW, NWS>(x, K).key, B)], 1u);
    }
    __syncthreads();
    for (uint32_t b = threadIdx.x; b < B; b += blockDim.x)
        if (s[b]) atomicAdd(&cnt[b], (unsigned long long)s[b]);
}

// the contributions of a chunk's (k+1)-mers to the buckets [b_lo, b_hi) into the staging buffer, grouped by owner: cursor[g]
// starts at owner g's piece. A warp claims its slots per owner with one shared-memory atomic, a CTA per owner with one global one.
template <int NW, int NWS>
__global__ void __launch_bounds__(kExtThreads) ext_scatter_k(const uint64_t *__restrict__ kp, int64_t n, int K, uint32_t B, uint32_t b_lo, uint32_t b_hi,
                                                             const int *__restrict__ owner, int world, unsigned long long *__restrict__ cursor,
                                                             uint64_t *__restrict__ skeys, uint8_t *__restrict__ sbits) {
    __shared__ unsigned s_cnt[kExtMaxWorld];
    __shared__ unsigned long long s_base[kExtMaxWorld];
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    for (int g = threadIdx.x; g < world; g += blockDim.x) s_cnt[g] = 0;
    __syncthreads();
    MaskBit<NW> c0, c1;
    int g0 = -1, g1 = -1;                       // owner of each contribution, -1 outside the pass
    if (i < n) {
        const Kmer<NWS> x = record_at<NWS>(kp, i);
        c0 = kpomer_mask_bit<0, NW, NWS>(x, K);
        c1 = kpomer_mask_bit<1, NW, NWS>(x, K);
        const uint32_t b0 = kmer_bucket<NW>(c0.key, B), b1 = kmer_bucket<NW>(c1.key, B);
        if (b0 >= b_lo && b0 < b_hi) g0 = owner[b0];
        if (b1 >= b_lo && b1 < b_hi) g1 = owner[b1];
    }
    // the contribution's position among the CTA's contributions to the same owner
    auto claim = [&](int g) {
        const unsigned same = __match_any_sync(0xffffffffu, g);
        const int leader = __ffs(same) - 1;
        unsigned base = 0;
        if (lane == leader && g >= 0) base = atomicAdd(&s_cnt[g], (unsigned)__popc(same));
        return __shfl_sync(0xffffffffu, base, leader) + (unsigned)__popc(same & ((1u << lane) - 1));
    };
    const unsigned r0 = claim(g0), r1 = claim(g1);
    __syncthreads();
    for (int q = threadIdx.x; q < world; q += blockDim.x) s_base[q] = s_cnt[q] ? atomicAdd(&cursor[q], (unsigned long long)s_cnt[q]) : 0ull;
    __syncthreads();
    auto put = [&](int g, unsigned r, const MaskBit<NW> &c) {
        const unsigned long long pos = s_base[g] + r;
#pragma unroll
        for (int q = 0; q < NW; ++q) skeys[pos * NW + q] = c.key.w[q];
        sbits[pos] = (uint8_t)c.bit;
    };
    if (g0 >= 0) put(g0, r0, c0);
    if (g1 >= 0) put(g1, r1, c1);
}

// one peer's piece for this owner, read in place (streaming loads: every record is read once): look the key up in this rank's
// k-mer index and OR the bit into the mask slice. A CTA stages a tile of keys through shared memory so that the remote reads are
// whole lines. miss counts the keys this rank's index rejects (no level holds them). A key absent from an owned bucket may still
// land on a set bit and get a slot, so this catches some inconsistent owner tables or k-mer sets, not all of them.
template <int NW>
__global__ void __launch_bounds__(kExtThreads) ext_apply_k(const uint64_t *__restrict__ keys, const uint8_t *__restrict__ bits, int64_t n, MphfDev mk,
                                                           uint64_t nslots, unsigned *__restrict__ masks32, unsigned long long *__restrict__ miss) {
    __shared__ uint64_t tile[kExtThreads * NW];
    const unsigned long long *src = reinterpret_cast<const unsigned long long *>(keys);
    for (int64_t t0 = (int64_t)blockIdx.x * kExtThreads; t0 < n; t0 += (int64_t)gridDim.x * kExtThreads) {
        const int m = (int)min((int64_t)kExtThreads, n - t0);
        for (int w = threadIdx.x; w < m * NW; w += kExtThreads) tile[w] = __ldcs(src + t0 * NW + w);
        __syncthreads();
        if ((int)threadIdx.x < m) {
            Kmer<NW> k;
#pragma unroll
            for (int q = 0; q < NW; ++q) k.w[q] = tile[threadIdx.x * NW + q];
            const int bit = __ldcs(bits + t0 + threadIdx.x);
            const uint64_t idx = mphf_lookup_dev<NW>(mk, k);
            if (idx < nslots) mask_or(masks32, idx, bit);
            else atomicAdd(miss, 1ull);
        }
        __syncthreads();
    }
}

// ---- state ---------------------------------------------------------------------------------------------------------------
struct ExtPeer { const uint64_t *keys; const uint8_t *bits; };       // a rank's staging buffer, as seen from this GPU

struct ExtDist {
    Ctx *ctx = nullptr;
    const KSet *kp = nullptr, *km = nullptr;
    const Mphf *mkp = nullptr, *mk = nullptr;
    int K = 0, B = 0, nw = 0, world = 1, rank = 0;
    std::vector<int> owner;
    std::vector<uint64_t> local;                 // B: this rank's contributions per destination bucket
    ExtPlan plan;
    bool planned = false;
    DArr<uint8_t> masks;                         // this rank's k-mers + 8 (OR-ed as 32-bit words)
    DArr<uint32_t> cov;                          // this rank's (k+1)-mers + 1, when a (k+1)-mer index was given
    std::vector<uint64_t> hist;                  // this rank's histogram
    DArr<int> d_owner;
    DArr<uint64_t> skeys;                        // staging buffer of the current pass (peers read it)
    DArr<uint8_t> sbits;
    std::vector<ExtPeer> peers;
    std::unique_ptr<ChunkStager> stage;          // the (k+1)-mers' keys, for the histogram and every scatter
    float ms[5] = {0, 0, 0, 0, 0};               // histogram, scatter, apply, coverage fill, coverage histogram (host ms of synchronised work)
    virtual ~ExtDist() = default;
    virtual void histogram() = 0;
    virtual void scatter(int p) = 0;
    virtual void apply(int p) = 0;
    int record_bytes() const { return 8 * nw + 1; }
};

template <int NW, int NWS>
struct ExtDistNW : ExtDist {
    void histogram() override {
        cudaStream_t st = ctx->stream;
        DArr<unsigned long long> cnt(ctx, (size_t)B);
        SG_CUDA(cudaMemsetAsync(cnt.p, 0, cnt.bytes(), st));
        stage->sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *) {
            const int grid = (int)std::min<int64_t>(div_up(c.n, kExtThreads), (int64_t)ctx->num_sms * 8);
            ext_hist_k<NW, NWS><<<grid, kExtThreads, 0, st>>>(keys, c.n, K, (uint32_t)B, cnt.p);
            ctx->launches++;
        });
        local.assign((size_t)B, 0);
        SG_CUDA(cudaMemcpyAsync(local.data(), cnt.p, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
    }

    void scatter(int p) override {
        cudaStream_t st = ctx->stream;
        std::vector<unsigned long long> start((size_t)world + 1, 0);
        for (int g = 0; g < world; ++g) start[g + 1] = start[g] + plan.piece(p, rank, g);
        DArr<unsigned long long> cursor(ctx, (size_t)world);
        SG_CUDA(cudaMemcpyAsync(cursor.p, start.data(), (size_t)world * 8, cudaMemcpyHostToDevice, st));
        const uint32_t b_lo = (uint32_t)plan.passes.bounds[p], b_hi = (uint32_t)plan.passes.bounds[p + 1];
        if (start[world]) {
            stage->sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *) {
                ext_scatter_k<NW, NWS><<<div_up(c.n, kExtThreads), kExtThreads, 0, st>>>(keys, c.n, K, (uint32_t)B, b_lo, b_hi, d_owner.p, world, cursor.p,
                                                                                           skeys.p, sbits.p);
                ctx->launches++;
            });
        }
        // every piece must have been filled exactly: the cursors end where the next owner's piece starts
        std::vector<unsigned long long> end((size_t)world);
        SG_CUDA(cudaMemcpyAsync(end.data(), cursor.p, (size_t)world * 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        for (int g = 0; g < world; ++g) SG_CHECK(end[g] == start[g + 1], 6, "internal: a staging piece does not match its planned size");
    }

    void apply(int p) override {
        cudaStream_t st = ctx->stream;
        const MphfDev m = mphf_dev(mk);
        DArr<unsigned long long> miss(ctx, 1);
        SG_CUDA(cudaMemsetAsync(miss.p, 0, 8, st));
        for (int s = 0; s < world; ++s) {
            uint64_t off = 0;
            for (int g = 0; g < rank; ++g) off += plan.piece(p, s, g);
            const uint64_t n = plan.piece(p, s, rank);
            if (!n) continue;
            const int grid = (int)std::min<uint64_t>((n + kExtThreads - 1) / kExtThreads, (uint64_t)ctx->num_sms * 8);
            ext_apply_k<NW><<<grid, kExtThreads, 0, st>>>(peers[s].keys + off * NW, peers[s].bits + off, (int64_t)n, m, (uint64_t)km->n,
                                                          reinterpret_cast<unsigned *>(masks.p), miss.p);
            ctx->launches++;
            SG_CUDA(cudaGetLastError());
        }
        unsigned long long h = 0;
        SG_CUDA(cudaMemcpyAsync(&h, miss.p, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        SG_CHECK(h == 0, 2, "distributed extension index: this rank's k-mer index rejected a k-mer sent to it (owner table or k-mer set inconsistent)");
    }
};

// ---- host entries ----------------------------------------------------------------------------------------------------------
ExtDist *ext_begin(Ctx *ctx, const KSet *kp, const Mphf *mkp, const KSet *km, const Mphf *mk, const int *owner, int world, int rank) {
    SG_CHECK(kp->ctx == ctx && km->ctx == ctx && mk->ctx == ctx && (!mkp || mkp->ctx == ctx), 2,
             "distributed extension index: a set or an index belongs to another context");
    SG_CHECK(kp->K >= 2 && km->K == kp->K - 1, 2, "distributed extension index: the k-mer set's K must be the (k+1)-mer set's K - 1");
    SG_CHECK(km->B == kp->B, 2, "distributed extension index: the two sets have different bucket counts");
    SG_CHECK(mk->K == km->K && mk->B == km->B && mk->n == km->n, 2, "distributed extension index: the k-mer index does not belong to the k-mer set");
    SG_CHECK(!mkp || (mkp->K == kp->K && mkp->B == kp->B && mkp->n == kp->n), 2,
             "distributed extension index: the (k+1)-mer index does not belong to the (k+1)-mer set");
    SG_CHECK(!mkp || kp->has_counts, 2, "distributed extension index: coverage needs a (k+1)-mer set with multiplicities");
    SG_CHECK(rank >= 0 && rank < world, 2, "bad world/rank");
    check_owner_table(world, km->B, owner);
    std::vector<uint8_t> own((size_t)km->B, 0);
    for (const Chunk &ch : km->chunks) std::fill(own.begin() + ch.b_lo, own.begin() + ch.b_hi, (uint8_t)1);
    for (int b = 0; b < km->B; ++b)
        SG_CHECK((owner[b] == rank) == (own[b] != 0), 2, "distributed extension index: the owner table does not match this rank's k-mer set");
    const int nw = km->nw, nws = kp->nw;
    ExtDist *d = nullptr;
    if (nw == 1 && nws == 1) d = new ExtDistNW<1, 1>();
    else if (nw == 1 && nws == 2) d = new ExtDistNW<1, 2>();
    else if (nw == 2 && nws == 2) d = new ExtDistNW<2, 2>();
    else if (nw == 2 && nws == 3) d = new ExtDistNW<2, 3>();
    else if (nw == 3 && nws == 3) d = new ExtDistNW<3, 3>();
    else if (nw == 3 && nws == 4) d = new ExtDistNW<3, 4>();
    else if (nw == 4 && nws == 4) d = new ExtDistNW<4, 4>();
    else throw Error(2, "distributed extension index: unsupported word combination");
    d->ctx = ctx; d->kp = kp; d->km = km; d->mkp = mkp; d->mk = mk;
    d->K = km->K; d->B = km->B; d->nw = nw; d->world = world; d->rank = rank;
    d->owner.assign(owner, owner + km->B);
    ctx->times.stage_h2d_bytes = 0;
    try {
        cudaStream_t st = ctx->stream;
        // the result slices first (they stay), then the (k+1)-mers' staging buffers
        d->masks.alloc(ctx, (size_t)km->n + 8, true);
        SG_CUDA(cudaMemsetAsync(d->masks.p, 0, d->masks.bytes(), st));
        if (mkp) {
            d->cov.alloc(ctx, (size_t)kp->n + 1, true);
            SG_CUDA(cudaMemsetAsync(d->cov.p, 0, d->cov.bytes(), st));
        }
        d->d_owner.alloc(ctx, (size_t)d->B);
        SG_CUDA(cudaMemcpyAsync(d->d_owner.p, owner, (size_t)d->B * sizeof(int), cudaMemcpyHostToDevice, st));
        if (mkp) {
            // the coverage reads the multiplicities once, through a stager of its own: the passes' stager never holds them
            Stopwatch sc;
            {
                ChunkStager with_counts(kp, true);
                coverage_fill(ctx, with_counts, mkp, d->cov.p);
            }
            d->ms[3] = sc.ms();
            Stopwatch sh;
            d->hist = coverage_histogram(ctx, d->cov.p, kp->n);
            d->ms[4] = sh.ms();
        }
        d->stage.reset(new ChunkStager(kp, false));
        Stopwatch sw;
        d->histogram();
        d->ms[0] = sw.ms();
    } catch (...) { delete d; throw; }
    return d;
}

void ext_local_counts(const ExtDist *d, uint64_t *out) { std::copy(d->local.begin(), d->local.end(), out); }

void ext_plan(ExtDist *d, const uint64_t *cnt_all, uint64_t *total) {
    for (int b = 0; b < d->B; ++b)
        SG_CHECK(cnt_all[(size_t)d->rank * d->B + b] == d->local[b], 2, "distributed extension index: this rank's row of the gathered counts is not its own");
    ext_plan_tables(d->plan, d->world, d->B, d->owner.data(), cnt_all);
    d->planned = true;
    *total = d->plan.passes.before[d->B];
}

uint64_t ext_free_bytes(ExtDist *d) {
    d->skeys.release(); d->sbits.release();
    return (uint64_t)d->ctx->free_bytes();
}

int ext_next_pass(ExtDist *d, uint64_t budget_bytes) {
    SG_CHECK(d->planned, 2, "sgpu_dist_ext_plan has not run");
    d->skeys.release(); d->sbits.release();
    d->peers.clear();
    uint64_t most = 0;
    if (!ext_next_pass(d->plan, budget_bytes, d->record_bytes(), &most)) return -1;
    const int p = d->plan.passes.npass() - 1;
    uint64_t mine = 0;
    for (int g = 0; g < d->world; ++g) mine += d->plan.piece(p, d->rank, g);
    // peers read these two: they must live inside the arena
    d->skeys.alloc(d->ctx, (size_t)mine * d->nw + 2);
    d->sbits.alloc(d->ctx, (size_t)mine + 16);
    return p;
}

// the descriptor a rank publishes for the current pass: its arena and where its staging buffer lies in it
struct ExtDesc {
    cudaIpcMemHandle_t arena;     // 64 bytes
    uint64_t arena_size, off_keys, off_bits, unused;
};
static_assert(sizeof(ExtDesc) == 96, "descriptor layout (SGPU_IPC_BYTES)");

void ext_ipc_handle(ExtDist *d, uint8_t *out96) {
    SG_CHECK(d->skeys.p, 2, "sgpu_dist_ext_next_pass has not planned a pass");
    Ctx *ctx = d->ctx;
    ExtDesc ds;
    memset(&ds, 0, sizeof ds);
    ds.off_keys = ctx->arena_offset(d->skeys.p, "distributed extension index: the staging buffer did not fit the device memory arena");
    ds.off_bits = ctx->arena_offset(d->sbits.p, "distributed extension index: the staging buffer did not fit the device memory arena");
    ds.arena_size = ctx->arena_size;
    if (d->world > 1) SG_CUDA(cudaIpcGetMemHandle(&ds.arena, ctx->arena));
    memcpy(out96, &ds, sizeof ds);
}

void ext_open_peers(ExtDist *d, const uint8_t *descs) {
    d->peers.assign(d->world, ExtPeer{nullptr, nullptr});
    for (int g = 0; g < d->world; ++g) {
        ExtDesc ds;
        memcpy(&ds, descs + (size_t)g * sizeof(ExtDesc), sizeof ds);
        char *base = d->ctx->peer_map(d->world, d->rank, g, &ds.arena);
        SG_CHECK(ds.off_keys < ds.arena_size && ds.off_bits < ds.arena_size, 2, "bad peer descriptor");
        d->peers[g] = ExtPeer{(const uint64_t *)(base + ds.off_keys), (const uint8_t *)(base + ds.off_bits)};
    }
}

static void check_pass(const ExtDist *d, int p) {
    SG_CHECK(d->planned && p >= 0 && p == d->plan.passes.npass() - 1 && d->skeys.p, 2, "bad pass (sgpu_dist_ext_next_pass decides the current one)");
}
void ext_scatter(ExtDist *d, int p) {
    check_pass(d, p);
    Stopwatch sw;
    d->scatter(p);        // synchronised: the staging buffer is complete, peers may read it after the next barrier
    d->ms[1] += sw.ms();
}
void ext_apply(ExtDist *d, int p) {
    check_pass(d, p);
    SG_CHECK((int)d->peers.size() == d->world, 2, "sgpu_dist_ext_open_peers has not run");
    Stopwatch sw;
    d->apply(p);          // synchronised: this rank no longer reads any peer's staging buffer
    d->ms[2] += sw.ms();
}

void ext_masks(const ExtDist *d, uint8_t *out, int64_t n) {
    SG_CHECK(n == d->km->n, 2, "mask array size != number of this rank's k-mers");
    if (n) SG_CUDA(cudaMemcpy(out, d->masks.p, (size_t)n, cudaMemcpyDeviceToHost));
}
void ext_coverage(const ExtDist *d, uint32_t *out, int64_t n) {
    SG_CHECK(d->cov.p, 2, "built without a (k+1)-mer index: no coverage");
    SG_CHECK(n == d->kp->n, 2, "coverage array size != number of this rank's (k+1)-mers");
    if (n) SG_CUDA(cudaMemcpy(out, d->cov.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
}
const std::vector<uint64_t> &ext_histogram(const ExtDist *d) { return d->hist; }
void ext_times(const ExtDist *d, float *out5) { for (int i = 0; i < 5; ++i) out5[i] = d->ms[i]; }
void ext_free(ExtDist *d) { delete d; }
ExtSlices ext_slices(const ExtDist *d) {
    return ExtSlices{d->ctx, d->kp, d->km, d->mkp, d->mk, d->masks.p, d->cov.p, d->owner.data(), d->world, d->rank};
}

}  // namespace sg
