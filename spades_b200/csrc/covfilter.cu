// Coverage pre-filter of the construction stage (SURVEY 8f-3): the pipeline's CoverageFilter phase, stages/construction.cpp:167-198.
//
//   reference                                                         here
//   ----------------------------------------------------------------  -------------------------------------------------------
//   rolling_hash::SymmetricCyclicHash<NDNASeqHash>(k+1)               cyc_* below: fwd/rvs rolled per window, value = fwd + rvs
//     adt/cyclichash.hpp:187-259, character hashes :24-27
//   EstimateCardinalityUpperBound -> hll::hll<24>                     cov_hll_k: atomicMax into 2^24 registers; the estimate is
//     kmer_index/kmer_counting.hpp:215-249, adt/hll.hpp:34-68           finished on the host with the reference's own double sum
//   qf::cqf(maxn): key = hash & (2^(qbits+8) - 1), exact counts       an open-addressing table of (key, count) in HBM; counts
//     adt/cqf.hpp:28-37,57-63; FillCoverageHistogram + CQFProcessor     stop at the threshold like CQFProcessor (:107-120)
//     kmer_counting.hpp:96-121,251-282
//   CovFilteringWrap: median multiplicity of a read's windows >= thr  cov_filter_k: per read, windows below the threshold <= w/2
//     io/reads/coverage_filtering_read_wrapper.hpp:37-124
//
// The counting quotient filter's slot layout is not reproduced: the reference only ever asks it "count(key) >= threshold", and
// a CQF with key_bits = qbits + 8 stores every key exactly (ext/src/gqf/gqf.c:1430-1477: range = 2^key_bits), so an exact
// (key -> count) table answers identically. The hash is symmetric (a window and its reverse complement hash alike), so the
// reference's "windows of reads and their reverse complements that are IsMinimal" is "every window of the forward reads", with
// self-reverse-complementary windows counted twice (they pass the filter on both strands; SURVEY 0.6 has the same doubling).
//
// One thread walks one read (the filter's verdict is per read, and 10^8 reads are parallelism enough); the three passes re-roll
// the hash instead of materialising 8 bytes per window.
#include "sgpu_internal.h"
#include <cmath>
#include <memory>

namespace sg {

namespace {

__device__ __forceinline__ uint64_t cyc_h(int c) {
    // NDNASeqHash(seed 0), cyclichash.hpp:24-27,51
    const uint64_t a = (c & 1) ? 0x3193c18562a02b4cULL : 0x3c8bfbb395c60474ULL;
    const uint64_t b = (c & 1) ? 0x295549f54be24456ULL : 0x20323ed082572324ULL;
    return (c & 2) ? b : a;
}
__device__ __forceinline__ uint64_t rol64d(uint64_t x, unsigned s) { s &= 63; return s ? (x << s) | (x >> (64 - s)) : x; }
__device__ __forceinline__ int base_at(const uint64_t *seq, int i) { return (int)((seq[i >> 5] >> ((i & 31) << 1)) & 3); }

struct CycHash {
    uint64_t fwd, rvs;
    __device__ __forceinline__ uint64_t value() const { return fwd + rvs; }
};
// SymmetricCyclicHash::operator() on the window at base 0 (cyclichash.hpp:231-241)
__device__ __forceinline__ CycHash cyc_init(const uint64_t *seq, int K) {
    CycHash h{0, 0};
    for (int i = 0; i < K; ++i) h.fwd = rol64d(h.fwd, 1) ^ cyc_h(base_at(seq, i));
    for (int i = 0; i < K; ++i) h.rvs = rol64d(h.rvs, 1) ^ cyc_h(3 - base_at(seq, K - 1 - i));
    return h;
}
// hash_update (cyclichash.hpp:250-256): drop `out`, append `in`
__device__ __forceinline__ void cyc_roll(CycHash &h, int out, int in, int K) {
    h.fwd = rol64d(h.fwd, 1) ^ rol64d(cyc_h(out), (unsigned)K) ^ cyc_h(in);
    h.rvs = rol64d(h.rvs, 63) ^ rol64d(cyc_h(3 - out), 63) ^ rol64d(cyc_h(3 - in), (unsigned)(K - 1));
}
// a window equal to its own reverse complement (even K only)
__device__ __forceinline__ bool window_self_rc(const uint64_t *seq, int j, int K) {
    for (int i = 0; 2 * i < K; ++i)
        if (base_at(seq, j + i) != 3 - base_at(seq, j + K - 1 - i)) return false;
    return true;
}
// f(j, h) for every window j of a read of L >= K bases, h its hash
template <class F>
__device__ __forceinline__ void for_each_window(const uint64_t *seq, int L, int K, F &&f) {
    CycHash h = cyc_init(seq, K);
    for (int j = 0;; ++j) {
        f(j, h);
        if (j + K >= L) break;
        cyc_roll(h, base_at(seq, j), base_at(seq, j + K), K);
    }
}

// ---- pass 1: HyperLogLog registers (hll.hpp:34-41) --------------------------------------------------------------------------
__global__ void cov_hll_k(const uint64_t *__restrict__ words, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ lens, int64_t n, int K,
                          uint32_t *__restrict__ reg) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int L = (int)lens[r];
    if (L < K) return;
    for_each_window(words + offs[r], L, K, [&](int, const CycHash &h) {
        const uint64_t d = h.value();
        const uint32_t id = (uint32_t)(d >> 40);
        const uint64_t low = d & ((1ull << 40) - 1);
        const uint32_t rho = (uint32_t)(__clzll((long long)low) - 24 + 1);     // __clzll(0) = 64
        if (reg[id] < rho) atomicMax(&reg[id], rho);
    });
}

// ---- the (key -> count) table --------------------------------------------------------------------------------------------------
// entry = (key + 1) << 16 | count; 0 = empty. key < 2^47.
template <bool SYSTEM>
__device__ __forceinline__ unsigned long long cov_cas(unsigned long long *a, unsigned long long cmp, unsigned long long val) {
    if constexpr (SYSTEM) return atomicCAS_system(a, cmp, val);
    else return atomicCAS(a, cmp, val);
}
struct CovTable {
    unsigned long long *e;
    uint64_t cap;
    uint64_t key_mask;
    unsigned *overflow;         // set when a probe sequence visited every slot (cannot happen while the HLL bound holds; checked on the host)
    __device__ __forceinline__ uint64_t slot_of(uint64_t key) const { return __umul64hi(key * 0x9E3779B97F4A7C15ULL, cap); }
    // CQFProcessor::ProcessKmer: nothing once the count has reached the threshold. SYSTEM: ranks on other GPUs insert into the same
    // table at the same time.
    template <bool SYSTEM>
    __device__ __forceinline__ void add(uint64_t key, unsigned thr) const {
        const unsigned long long tag = (key + 1) << 16;
        uint64_t s = slot_of(key);
        for (uint64_t probes = 0;; ++probes) {
            if (probes > cap) {
                if constexpr (SYSTEM) atomicExch_system(overflow, 1u);
                else *overflow = 1u;
                return;
            }
            unsigned long long cur = e[s];
            if (cur == 0) {
                const unsigned long long old = cov_cas<SYSTEM>(&e[s], 0ull, tag | 1ull);
                if (old == 0) return;
                cur = old;
            }
            if ((cur & ~0xffffull) == tag) {
                while ((cur & 0xffffull) < thr) {
                    const unsigned long long old = cov_cas<SYSTEM>(&e[s], cur, cur + 1);
                    if (old == cur) return;
                    cur = old;
                }
                return;
            }
            if (++s == cap) s = 0;
        }
    }
    __device__ __forceinline__ unsigned count(uint64_t key) const {
        const unsigned long long tag = (key + 1) << 16;
        uint64_t s = slot_of(key);
        for (uint64_t probes = 0; probes <= cap; ++probes) {
            const unsigned long long cur = e[s];
            if (cur == 0) return 0;
            if ((cur & ~0xffffull) == tag) return (unsigned)(cur & 0xffffull);
            if (++s == cap) s = 0;
        }
        return 0;
    }
};

// ---- which table a key's count lives in ----------------------------------------------------------------------------------------
// The owner of a key among `world` tables is the high word of a second multiplicative hash of the masked key scaled by `world`, so it
// does not depend on the slot function inside a table (which takes the high word of key * 0x9E37...).
__host__ __device__ __forceinline__ uint32_t cov_owner(uint64_t key, uint32_t world) {
    const uint64_t h = key * 0xC2B2AE3D27D4EB4FULL;
#ifdef __CUDA_ARCH__
    return (uint32_t)__umul64hi(h, world);
#else
    return (uint32_t)(((unsigned __int128)h * world) >> 64);
#endif
}

// A route gives the key of a window, whether this launch owns the key, the table its count lives in, the scope of the table's atomics
// and whether a read's verdict is split over several launches (`split`: the windows below the threshold are carried in below[r]).

// one table for every key
struct WholeTable {
    CovTable t;
    static constexpr bool system = false, split = false;
    __device__ __forceinline__ uint64_t key(const CycHash &h) const { return h.value() & t.key_mask; }
    __device__ __forceinline__ bool owns(uint64_t) const { return true; }
    __device__ __forceinline__ const CovTable &table(uint64_t) const { return t; }
};

// Key-range passes: a table too large for the device is built and read in P passes over the resident reads. Pass p holds the keys with
// cov_owner(key, P) == p in a table of cov_slice_capacity(bound, P) entries. Every key lands in exactly one pass with all of its
// windows, so its count, each read's number of windows below the threshold and the distinct keys summed over the passes are those of
// the single table. The pass hash composes with the rank owner: floor(h*W*P / 2^64) / P == floor(h*W / 2^64), so
// cov_owner(key, W*P) / P == cov_owner(key, W) and a distributed filter with passes can take id = cov_owner(key, W*P), owner = id / P,
// pass = id % P without changing which rank owns a key.
struct KeyRange {
    CovTable t;
    uint32_t passes, pass;
    static constexpr bool system = false, split = true;
    __device__ __forceinline__ uint64_t key(const CycHash &h) const { return h.value() & t.key_mask; }
    __device__ __forceinline__ bool owns(uint64_t key) const { return cov_owner(key, passes) == pass; }
    __device__ __forceinline__ const CovTable &table(uint64_t) const { return t; }
    __device__ __forceinline__ bool last() const { return pass + 1 == passes; }
};

// The distributed filter: the table is split into one slice per rank, a key lives in its owner's slice. Ranks on other GPUs insert
// into the same slices at the same time (system scope).
struct OwnerSlices {
    const CovTable *slices;
    uint32_t world;
    uint64_t key_mask;
    static constexpr bool system = true, split = false;
    __device__ __forceinline__ uint64_t key(const CycHash &h) const { return h.value() & key_mask; }
    __device__ __forceinline__ bool owns(uint64_t) const { return true; }
    // by value: the compiler cannot tell that `slices` is not written by the CAS of an insert, so a reference would be read again
    // after every CAS (__restrict__ on a member does not change that)
    __device__ __forceinline__ CovTable table(uint64_t key) const { return slices[cov_owner(key, world)]; }
};

// ---- pass 2: counts up to the threshold ------------------------------------------------------------------------------------------
template <class Route>
__global__ void cov_fill_k(const uint64_t *__restrict__ words, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ lens, int64_t n, int K,
                           const Route route, unsigned thr) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int L = (int)lens[r];
    if (L < K) return;
    const uint64_t *seq = words + offs[r];
    for_each_window(seq, L, K, [&](int j, const CycHash &h) {
        const uint64_t key = route.key(h);
        if (!route.owns(key)) return;
        const CovTable &t = route.table(key);
        t.add<Route::system>(key, thr);
        if ((K & 1) == 0 && h.fwd == h.rvs && window_self_rc(seq, j, K)) t.add<Route::system>(key, thr);
    });
}

// ---- pass 3: the verdict per read (coverage_filtering_read_wrapper.hpp:37-72) --------------------------------------------------------
// A split route adds the read's windows of this launch below the threshold to below[r] (one thread per read, no atomics); its last
// pass gives the verdict from the sum. Other routes do not touch below.
template <class Route>
__global__ void cov_filter_k(const uint64_t *__restrict__ words, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ lens, int64_t n, int K,
                             const Route route, unsigned thr, uint32_t *__restrict__ below, uint8_t *__restrict__ keep,
                             uint32_t *__restrict__ keep_words) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int L = (int)lens[r];
    bool k;
    if (L < K) {
        k = thr == 0;                                          // CountMedianMlt returns 0 for a read shorter than K
    } else {
        uint32_t b = 0;
        for_each_window(words + offs[r], L, K, [&](int, const CycHash &h) {
            const uint64_t key = route.key(h);
            if (route.owns(key)) b += route.table(key).count(key) < thr;
        });
        if constexpr (Route::split) {
            if (route.pass) b += below[r];
            if (!route.last()) { below[r] = b; return; }
        }
        k = b <= (uint32_t)(L - K + 1) / 2;                    // element size/2 of the sorted multiplicities >= threshold
    }
    if constexpr (Route::split) {
        if (!route.last()) return;
    }
    keep[r] = k ? 1 : 0;
    keep_words[r] = k ? (uint32_t)((L + 31) >> 5) : 0u;
}

__global__ void cov_keep_count_k(const uint8_t *__restrict__ keep, int64_t n, uint32_t *__restrict__ flag) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) flag[r] = keep[r];
}
// survivors keep their order: read r moves to position new_idx[r], its words to new_off[r]
__global__ void cov_compact_k(const uint64_t *__restrict__ words, const uint64_t *__restrict__ offs, const uint32_t *__restrict__ lens,
                              const uint8_t *__restrict__ keep, const uint64_t *__restrict__ new_idx, const uint64_t *__restrict__ new_off, int64_t n,
                              uint64_t *__restrict__ out_words, uint64_t *__restrict__ out_offs, uint32_t *__restrict__ out_lens) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n || !keep[r]) return;
    const uint32_t L = lens[r];
    const uint64_t d = new_off[r];
    out_offs[new_idx[r]] = d;
    out_lens[new_idx[r]] = L;
    const uint64_t *s = words + offs[r];
    for (uint32_t i = 0; i < ((L + 31) >> 5); ++i) out_words[d + i] = s[i];
}
__global__ void cov_distinct_k(const unsigned long long *__restrict__ e, uint64_t cap, unsigned long long *__restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned c = 0;
    for (; i < cap; i += (uint64_t)gridDim.x * blockDim.x) c += e[i] != 0;
    for (int o = 16; o; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

// HLL registers of the union = element-wise max of the ranks' registers (read through the peers' mapped arenas)
__global__ void cov_hll_merge_k(const uint4 *const *__restrict__ regs, int world, uint4 *__restrict__ out, uint32_t n4) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    uint4 m = regs[0][i];
    for (int g = 1; g < world; ++g) {
        const uint4 r = regs[g][i];
        m.x = max(m.x, r.x); m.y = max(m.y, r.y); m.z = max(m.z, r.z); m.w = max(m.w, r.w);
    }
    out[i] = m;
}

}  // namespace

// hll<24>::cardinality / upper_bound_cardinality (adt/hll.hpp:50-68): same operations in the same order
static double hll_upper_bound(const std::vector<uint32_t> &reg) {
    const uint64_t m = 1ull << 24;
    const double alpha = 0.7213 / (1.0 + 1.079 / (double)m);
    double res = alpha * (double)m * (double)m;
    double E = 0.0;
    uint64_t zeros = 0;
    for (uint64_t i = 0; i < m; ++i) { E += exp2(-(double)reg[i]); zeros += reg[i] == 0; }
    res /= E;
    if (res <= 5.0 * (double)m / 2 && zeros > 0) res = (double)m * (std::log((double)m) - std::log((double)zeros));
    return 1.1 * res;
}

// qf::cqf(maxn) geometry (cqf.hpp:28-37): key bits of the filter for a cardinality bound
static unsigned cov_key_bits(size_t maxn) {
    const unsigned lg = maxn > 1 ? (unsigned)std::ceil(std::log2((double)maxn)) : 0u;     // (no reads: the reference's log2(0) is undefined)
    const unsigned qbits = std::max(7u, lg) + 1;
    const unsigned key_bits = qbits + 8;
    SG_CHECK(key_bits <= 47, 2, "coverage filter: more than 2^38 distinct k-mers estimated");
    return key_bits;
}

// pass 1 over the context's reads into 2^24 device registers (enqueued on the context's stream)
static void cov_hll(Ctx *ctx, int K, uint32_t *reg) {
    cudaStream_t st = ctx->stream;
    const int64_t n = ctx->n_reads;
    SG_CUDA(cudaMemsetAsync(reg, 0, (size_t)4 << 24, st));
    if (n) { cov_hll_k<<<div_up(n, 128), 128, 0, st>>>(ctx->d_words, ctx->d_offs, ctx->d_lens, n, K, reg); ctx->launches++; }
}

struct CovBound {
    size_t maxn = 0;            // cardinality upper bound
    unsigned key_bits = 0;
};
// the bound of 2^24 device registers, once the work enqueued before them is done (synchronises)
static CovBound cov_bound(Ctx *ctx, const uint32_t *reg) {
    std::vector<uint32_t> h_reg((size_t)1 << 24);
    SG_CUDA(cudaMemcpyAsync(h_reg.data(), reg, h_reg.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
    CovBound b;
    b.maxn = (size_t)hll_upper_bound(h_reg);
    b.key_bits = cov_key_bits(b.maxn);
    return b;
}

// What the verdict kernel feeds, and what follows it, in both entry points: the distinct-key counter, where each survivor and its
// words go (order kept), the number kept, the flags for the caller, the statistics and, with apply, the survivors as the context's
// read set (what CovFilteringWrap does to the streams).
struct CovVerdicts {
    Ctx *ctx;
    int64_t n;
    DArr<uint8_t> keep;
    DArr<uint32_t> keep_words, flag;
    DArr<unsigned long long> d_distinct;
    DArr<uint64_t> new_off, new_idx;
    uint64_t kept = 0, kept_words = 0;
    unsigned long long distinct = 0;
    explicit CovVerdicts(Ctx *c) : ctx(c), n(c->n_reads), keep(c, (size_t)c->n_reads + 1), keep_words(c, (size_t)c->n_reads + 1), flag(c, (size_t)c->n_reads + 1),
                                   d_distinct(c, 1) {
        SG_CUDA(cudaMemsetAsync(d_distinct.p, 0, 8, c->stream));
    }
    // adds a table's occupied slots (one pass's, or this rank's slice) to the distinct keys
    void count_distinct(const unsigned long long *e, uint64_t cap) {
        cov_distinct_k<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(e, cap, d_distinct.p);
        ctx->launches++;
    }
    // after the verdict kernel and the distinct counts; a set *overflow (when given) fails the call before any result is written
    void finish(uint8_t *keep_out, const unsigned *overflow, const CovBound &b, uint64_t *stats, int apply) {
        cudaStream_t st = ctx->stream;
        if (n) { cov_keep_count_k<<<div_up(n, 256), 256, 0, st>>>(keep.p, n, flag.p); ctx->launches++; }
        SG_CUDA(cudaMemsetAsync(keep_words.p + n, 0, 4, st));
        SG_CUDA(cudaMemsetAsync(flag.p + n, 0, 4, st));
        new_off.alloc(ctx, (size_t)n + 1); new_idx.alloc(ctx, (size_t)n + 1);
        exclusive_scan_u32_to_u64(ctx, keep_words.p, new_off.p, (size_t)n + 1);
        exclusive_scan_u32_to_u64(ctx, flag.p, new_idx.p, (size_t)n + 1);
        SG_CUDA(cudaMemcpyAsync(&kept, new_idx.p + n, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaMemcpyAsync(&kept_words, new_off.p + n, 8, cudaMemcpyDeviceToHost, st));
        if (keep_out && n) SG_CUDA(cudaMemcpyAsync(keep_out, keep.p, (size_t)n, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaMemcpyAsync(&distinct, d_distinct.p, 8, cudaMemcpyDeviceToHost, st));
        unsigned ovf = 0;
        if (overflow) SG_CUDA(cudaMemcpyAsync(&ovf, overflow, 4, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cudaStreamSynchronize(st));
        SG_CHECK(!ovf, 6, "coverage filter: more distinct keys than the cardinality bound allows (table full)");
        if (stats) { stats[0] = b.maxn; stats[1] = b.key_bits; stats[2] = distinct; stats[3] = kept; }
        if (apply) this->apply();
    }
    void apply() {
        cudaStream_t st = ctx->stream;
        DArr<uint64_t> nw(ctx, kept_words + 4, true), no(ctx, kept + 1, true);
        DArr<uint32_t> nl(ctx, kept + 1, true);
        SG_CUDA(cudaMemsetAsync(nw.p + kept_words, 0, 4 * 8, st));
        if (n) { cov_compact_k<<<div_up(n, 128), 128, 0, st>>>(ctx->d_words, ctx->d_offs, ctx->d_lens, keep.p, new_idx.p, new_off.p, n, nw.p, no.p, nl.p); ctx->launches++; }
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cudaStreamSynchronize(st));
        ctx->h_words.clear(); ctx->h_offs.clear(); ctx->h_lens.clear(); ctx->staged_dirty = false;
        ctx->r_words = std::move(nw); ctx->r_offs = std::move(no); ctx->r_lens = std::move(nl);
        ctx->d_words = ctx->r_words.p; ctx->d_offs = ctx->r_offs.p; ctx->d_lens = ctx->r_lens.p;
        ctx->n_reads = (int64_t)kept; ctx->n_words = kept_words;
    }
};

void cov_filter(Ctx *ctx, int K, unsigned thr, int apply, int passes, uint8_t *keep_out, uint64_t *stats) {
    SG_CHECK(K >= 1 && K <= 128, 2, "K must be in [1,128]");
    SG_CHECK(thr <= 60000u, 2, "coverage threshold must be at most 60000");
    SG_CHECK(passes >= 0 && passes <= kCovMaxPasses, 2, "coverage filter: passes must be in [0, 256] (0 = planned)");
    ensure_reads_on_device(ctx);
    cudaStream_t st = ctx->stream;
    const int64_t n = ctx->n_reads;
    const int T = 128;
    // 1. cardinality upper bound
    CovBound b;
    {
        DArr<uint32_t> reg(ctx, (size_t)1 << 24);
        cov_hll(ctx, K, reg.p);
        b = cov_bound(ctx, reg.p);
    }
    // 2. the table: one, or one per key range when one table does not fit next to the per-read arrays (cov_plan.h)
    const uint64_t budget = ctx->budget_left();
    const CovPassPlan plan = cov_pass_plan(b.maxn, n, budget);
    if (!passes) {
        if (!plan.passes) {
            char m[256];
            snprintf(m, sizeof m, "coverage filter: %llu device bytes needed with %d key-range passes (cardinality bound %zu), %llu left",
                     (unsigned long long)plan.need, kCovMaxPasses, b.maxn, (unsigned long long)budget);
            throw Error(4, m);
        }
        passes = plan.passes;
    }
    CovVerdicts v(ctx);
    DArr<unsigned> d_ovf(ctx, 1);
    DArr<uint32_t> below;
    if (passes > 1) below.alloc(ctx, (size_t)n + 1);
    CovTable t;
    t.cap = cov_pass_capacity(b.maxn, passes);
    t.key_mask = (1ull << b.key_bits) - 1;
    DArr<unsigned long long> table(ctx, t.cap);
    t.e = table.p;
    ctx->times.cov_filter_passes = (uint64_t)passes;
    ctx->times.cov_filter_table_bytes = table.bytes();
    SG_CUDA(cudaMemsetAsync(d_ovf.p, 0, 4, st));
    t.overflow = d_ovf.p;
    // 3. per pass: clear the table, insert the windows' keys, look them up per read
    const auto roll = [&](const auto route) {
        cov_fill_k<<<div_up(n, T), T, 0, st>>>(ctx->d_words, ctx->d_offs, ctx->d_lens, n, K, route, thr);
        cov_filter_k<<<div_up(n, T), T, 0, st>>>(ctx->d_words, ctx->d_offs, ctx->d_lens, n, K, route, thr, below.p, v.keep.p, v.keep_words.p);
        ctx->launches += 2;
    };
    for (int p = 0; p < passes; ++p) {
        SG_CUDA(cudaMemsetAsync(table.p, 0, table.bytes(), st));
        if (n) {
            if (passes == 1) roll(WholeTable{t});
            else roll(KeyRange{t, (uint32_t)passes, (uint32_t)p});
        }
        v.count_distinct(table.p, t.cap);
        if (p + 1 < passes) {                          // the overflow flag is sticky: a full table stops the call before the next pass
            unsigned overflow = 0;
            SG_CUDA(cudaMemcpyAsync(&overflow, d_ovf.p, 4, cudaMemcpyDeviceToHost, st));
            SG_CUDA(cudaGetLastError());
            SG_CUDA(cudaStreamSynchronize(st));
            SG_CHECK(!overflow, 6, "coverage filter: more distinct keys than the cardinality bound allows (table full)");
        }
    }
    table.release();                                   // the scans and the compaction below take its place (same stream)
    below.release();
    v.finish(keep_out, d_ovf.p, b, stats, apply);
}

// ---- distributed filter (sgpu_dist_cov_*): every rank holds a shard of the reads; the result equals cov_filter over the union --------
// A rank's slice holds cov_slice_capacity(bound, world) entries (cov_plan.h).
uint32_t cov_owner_host(uint64_t key, int world) { return cov_owner(key, (uint32_t)world); }

struct CovDist {
    Ctx *ctx = nullptr;
    int K = 0, world = 1, rank = 0;
    unsigned thr = 0;
    DArr<uint32_t> reg;                      // this rank's HLL registers (peers read them in bound)
    DArr<unsigned long long> slice;          // this rank's slice: cap entries, then the overflow flag (peers write both in fill)
    CovBound bound;
    uint64_t cap = 0;
    std::vector<const uint32_t *> peer_reg;  // rank-indexed, as this process sees them
    std::vector<CovTable> peer_slice;
    bool filled = false;
};

// descriptor a rank publishes (all_gather) after begin and again after bound: arena handle + where its registers and slice are
struct CovDesc {
    cudaIpcMemHandle_t arena;
    uint64_t arena_size, off_reg, off_slice, slice_cap;     // slice_cap = 0: no slice yet
};
static_assert(sizeof(CovDesc) == 96, "descriptor layout (SGPU_IPC_BYTES)");

CovDist *dist_cov_begin(Ctx *ctx, int K, unsigned thr, int world, int rank) {
    SG_CHECK(K >= 1 && K <= 128, 2, "K must be in [1,128]");
    SG_CHECK(thr <= 60000u, 2, "coverage threshold must be at most 60000");
    SG_CHECK(world >= 1 && rank >= 0 && rank < world, 2, "bad world / rank");
    ensure_reads_on_device(ctx);
    std::unique_ptr<CovDist> d(new CovDist);
    d->ctx = ctx; d->K = K; d->thr = thr; d->world = world; d->rank = rank;
    d->reg.alloc(ctx, (size_t)1 << 24);
    cov_hll(ctx, K, d->reg.p);
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaStreamSynchronize(ctx->stream));        // the registers are complete before they are published
    return d.release();
}

void dist_cov_ipc_handle(CovDist *d, uint8_t *out96) {
    Ctx *ctx = d->ctx;
    CovDesc ds;
    memset(&ds, 0, sizeof ds);
    ds.arena_size = ctx->arena_size;
    if (d->reg.p) ds.off_reg = ctx->arena_offset(d->reg.p, "distributed coverage filter: the HLL registers did not fit the device memory arena");
    if (d->slice.p) {
        ds.off_slice = ctx->arena_offset(d->slice.p, "distributed coverage filter: the table slice did not fit the device memory arena");
        ds.slice_cap = d->cap;
    }
    if (d->world > 1) SG_CUDA(cudaIpcGetMemHandle(&ds.arena, ctx->arena));
    memcpy(out96, &ds, sizeof ds);
}

void dist_cov_open_peers(CovDist *d, const uint8_t *descs) {
    Ctx *ctx = d->ctx;
    d->peer_reg.assign(d->world, nullptr);
    d->peer_slice.assign(d->world, CovTable{});
    for (int g = 0; g < d->world; ++g) {
        CovDesc ds;
        memcpy(&ds, descs + (size_t)g * sizeof(CovDesc), sizeof ds);
        char *base = ctx->peer_map(d->world, d->rank, g, &ds.arena);
        SG_CHECK(ds.off_reg + ((uint64_t)4 << 24) <= ds.arena_size && ds.off_slice + (ds.slice_cap + 1) * 8 <= ds.arena_size, 2, "bad peer descriptor");
        d->peer_reg[g] = (const uint32_t *)(base + ds.off_reg);
        if (ds.slice_cap) {
            CovTable &t = d->peer_slice[g];
            t.e = (unsigned long long *)(base + ds.off_slice);
            t.cap = ds.slice_cap;
            t.key_mask = (1ull << d->bound.key_bits) - 1;
            t.overflow = (unsigned *)(t.e + t.cap);
        }
    }
}

void dist_cov_bound(CovDist *d) {
    Ctx *ctx = d->ctx;
    SG_CHECK(d->reg.p && (int)d->peer_reg.size() == d->world && !d->slice.p, 2,
             "sgpu_dist_cov_bound runs once, after sgpu_dist_cov_open_peers with the descriptors of sgpu_dist_cov_begin");
    cudaStream_t st = ctx->stream;
    {
        DArr<uint32_t> merged(ctx, (size_t)1 << 24);
        DArr<uint64_t> regs(ctx, (size_t)d->world);
        SG_CUDA(cudaMemcpyAsync(regs.p, d->peer_reg.data(), (size_t)d->world * 8, cudaMemcpyHostToDevice, st));
        const uint32_t n4 = (1u << 24) / 4;
        cov_hll_merge_k<<<div_up(n4, 256), 256, 0, st>>>((const uint4 *const *)regs.p, d->world, (uint4 *)merged.p, n4);
        ctx->launches++;
        d->bound = cov_bound(ctx, merged.p);
    }
    d->cap = cov_slice_capacity(d->bound.maxn, d->world);
    d->slice.alloc(ctx, d->cap + 1);
    SG_CUDA(cudaMemsetAsync(d->slice.p, 0, d->slice.bytes(), st));
    SG_CUDA(cudaStreamSynchronize(st));                 // the slice is empty before it is published
}

void dist_cov_fill(CovDist *d) {
    Ctx *ctx = d->ctx;
    SG_CHECK(d->slice.p && (int)d->peer_slice.size() == d->world && d->peer_slice[d->rank].e == d->slice.p && !d->filled, 2,
             "sgpu_dist_cov_fill runs once, after sgpu_dist_cov_open_peers with the descriptors of sgpu_dist_cov_bound");
    for (const CovTable &t : d->peer_slice) SG_CHECK(t.e, 2, "a peer descriptor carries no table slice");
    d->reg.release();                                   // every rank has finished its bound before it published its slice
    cudaStream_t st = ctx->stream;
    const int64_t n = ctx->n_reads;
    DArr<CovTable> slices(ctx, (size_t)d->world);
    SG_CUDA(cudaMemcpyAsync(slices.p, d->peer_slice.data(), (size_t)d->world * sizeof(CovTable), cudaMemcpyHostToDevice, st));
    if (n) {
        const OwnerSlices route{slices.p, (uint32_t)d->world, (1ull << d->bound.key_bits) - 1};
        cov_fill_k<<<div_up(n, 128), 128, 0, st>>>(ctx->d_words, ctx->d_offs, ctx->d_lens, n, d->K, route, d->thr);
        ctx->launches++;
    }
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaStreamSynchronize(st));                 // this rank inserts nothing more; peers may read after the next barrier
    d->filled = true;
}

void dist_cov_filter(CovDist *d, int apply, uint8_t *keep_out, uint64_t *stats) {
    Ctx *ctx = d->ctx;
    SG_CHECK(d->filled, 2, "sgpu_dist_cov_filter runs after sgpu_dist_cov_fill and a barrier");
    cudaStream_t st = ctx->stream;
    // every rank checks every slice's overflow flag, so all of them fail together
    for (const CovTable &t : d->peer_slice) {
        unsigned overflow = 0;
        SG_CUDA(cudaMemcpy(&overflow, t.overflow, 4, cudaMemcpyDefault));
        SG_CHECK(!overflow, 6, "distributed coverage filter: more distinct keys in a slice than its capacity (table full)");
    }
    const int64_t n = ctx->n_reads;
    DArr<CovTable> slices(ctx, (size_t)d->world);
    SG_CUDA(cudaMemcpyAsync(slices.p, d->peer_slice.data(), (size_t)d->world * sizeof(CovTable), cudaMemcpyHostToDevice, st));
    CovVerdicts v(ctx);
    if (n) {
        const OwnerSlices route{slices.p, (uint32_t)d->world, (1ull << d->bound.key_bits) - 1};
        cov_filter_k<<<div_up(n, 128), 128, 0, st>>>(ctx->d_words, ctx->d_offs, ctx->d_lens, n, d->K, route, d->thr, nullptr, v.keep.p,
                                                     v.keep_words.p);
        ctx->launches++;
    }
    v.count_distinct(d->slice.p, d->cap);
    v.finish(keep_out, nullptr, d->bound, stats, apply);      // synchronises: this rank reads no slice any more
}

void dist_cov_free(CovDist *d) { delete d; }

}  // namespace sg
