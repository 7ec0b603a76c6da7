// sgpu_internal.h -- internal C++ structures behind the C ABI of include/spades_b200.h
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <iterator>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "cov_plan.h"
#include "kmer_dev.cuh"

namespace sg {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

#define SG_CUDA(expr)                                                                                  \
    do {                                                                                               \
        cudaError_t e__ = (expr);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            char b__[512];                                                                             \
            snprintf(b__, sizeof b__, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
            throw sg::Error(5, b__);                                                                   \
        }                                                                                              \
    } while (0)

#define SG_CHECK(cond, code, msg)                                                                      \
    do {                                                                                               \
        if (!(cond)) {                                                                                 \
            char b__[512];                                                                             \
            snprintf(b__, sizeof b__, "%s:%d: %s", __FILE__, __LINE__, (msg));                         \
            throw sg::Error((code), b__);                                                              \
        }                                                                                              \
    } while (0)

// device allocation with byte accounting (so multi-pass planning can see what is resident)
struct Ctx;
template <class T>
struct DArr {
    T *p = nullptr;
    size_t n = 0;
    size_t blk = 0;     // bytes of the underlying block
    Ctx *ctx = nullptr;
    DArr() {}
    DArr(Ctx *c, size_t n_, bool persistent = false) { alloc(c, n_, persistent); }
    DArr(const DArr &) = delete;
    DArr &operator=(const DArr &) = delete;
    DArr(DArr &&o) noexcept { p = o.p; n = o.n; blk = o.blk; ctx = o.ctx; o.p = nullptr; o.n = 0; o.blk = 0; }
    DArr &operator=(DArr &&o) noexcept {
        if (this != &o) { release(); p = o.p; n = o.n; blk = o.blk; ctx = o.ctx; o.p = nullptr; o.n = 0; o.blk = 0; }
        return *this;
    }
    ~DArr() { release(); }
    void alloc(Ctx *c, size_t n_, bool persistent = false);
    void release();
    size_t bytes() const { return n * sizeof(T); }
};

struct PhaseTimes {   // device milliseconds measured with CUDA events on ctx->stream
    float extract_count = 0, extract_scatter = 0, refine = 0, local_sort = 0, compact = 0, mphf = 0, exchange = 0, total = 0;
    uint64_t launches = 0;
    uint64_t instances = 0;       // records written by the partition kernel
    uint64_t passes = 0;
    // paths taken (sgpu_times)
    uint64_t level_a_key_bits = 0, level_a_scatters = 0;
    uint64_t refine_rounds_max = 0, refine_splits_round0 = 0, refine_splits_later = 0;
    uint64_t sort_lsd_fallbacks = 0, sort_oversize_equal = 0;
    // a count whose result goes to host memory: bytes copied there, and host milliseconds spent waiting for those copies
    uint64_t result_d2h_bytes = 0;
    float result_d2h_wait = 0;
    // host-set chunks uploaded by a ChunkStager (reset by sgpu_kmers_from_kpomers_ex, the MPHF build and the graph builds), and
    // the junction batches of the last graph build
    uint64_t stage_h2d_bytes = 0;
    uint64_t graph_junction_batches = 0;
    // the last single-GPU coverage pre-filter: key-range passes, and the bytes of one pass's table
    uint64_t cov_filter_passes = 0, cov_filter_table_bytes = 0;
};

struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy = nullptr;    // non-blocking stream of the copies between host-resident k-mer sets and the device (created at first use)
    cudaStream_t copy_stream() {
        if (!copy) SG_CUDA(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
        return copy;
    }
    int num_sms = 132;
    size_t hbm_budget = 0;       // 0 = use free memory
    size_t allocated = 0, peak = 0;
    int verbose = 0;
    std::string err;
    PhaseTimes times;
    uint64_t launches = 0;
    // reads
    DArr<uint64_t> r_words;      // owned copy (host-appended) ...
    DArr<uint64_t> r_offs;
    DArr<uint32_t> r_lens;
    const uint64_t *d_words = nullptr;   // ... or adopted device pointers
    const uint64_t *d_offs = nullptr;
    const uint32_t *d_lens = nullptr;
    int64_t n_reads = 0;
    uint64_t n_words = 0;
    std::vector<uint64_t> h_words, h_offs;   // host staging until first use
    std::vector<uint32_t> h_lens;
    bool staged_dirty = false;
    // objects created from this context that still hold arena blocks (k-mer sets, indexes, graphs, distributed counts):
    // sgpu_destroy refuses to run while any is alive (their destructors release blocks into this context's arena)
    int live_children = 0;
    bool destroy_pending = false;
    void *owner = nullptr;                   // the sgpu_ctx this context is embedded in
    // multi-GPU: the peers' arenas mapped through cudaIpc, once per process (rank-indexed; own entry unused)
    std::vector<char *> peer_arena;
    std::vector<uint8_t> peer_handle;        // 64 bytes per rank: the handle a mapping was opened from
    void peer_close();
    // the arena of rank g (of `world`) as this process sees it: its own arena, or the peer's opened from `handle` (64 bytes)
    char *peer_map(int world, int rank, int g, const void *handle);
    // offset of a block inside the arena (what a peer adds to its mapping); `what` is the error when the block lies outside it
    uint64_t arena_offset(const void *p, const char *what) const;
    // device memory: one arena reserved from the driver at first use and sub-allocated with a coalescing free list.
    // cudaMalloc/cudaFree of tens of GB cost 100s of ms and a 100 M-read step turns over ~300 GB of buffers; inside the
    // arena an allocation is a map lookup. Short-lived buffers (X/Y ping-pong, scratch) grow from the bottom, long-lived
    // results (k-mer chunks, MPHF, masks) from the top, so the big short-lived blocks keep finding the same hole.
    char *arena = nullptr;
    size_t arena_size = 0;
    std::map<size_t, size_t> arena_free;                     // offset -> size, coalesced
    std::vector<std::pair<void *, size_t>> direct;           // allocations that did not fit the arena
    size_t pool_cached = 0;                                  // free bytes inside the arena
    void arena_init();
    void *pool_alloc(size_t bytes, size_t *blk, bool persistent);
    void pool_release(void *p, size_t blk);
    void pool_trim();
    size_t free_bytes();                                     // allocatable bytes (arena free list)
    // device bytes a pass or step may still plan with: what the HBM budget leaves, or 90 % of the arena's free bytes without one
    size_t budget_left() {
        return hbm_budget ? (hbm_budget > allocated ? hbm_budget - allocated : 0) : (size_t)((double)free_bytes() * 0.90);
    }
};

inline void Ctx::arena_init() {
    if (arena) return;
    size_t f = 0, t = 0;
    cudaMemGetInfo(&f, &t);
    size_t want = hbm_budget ? hbm_budget : (size_t)((double)f * 0.92);
    // SGPU_ARENA_GB: user option, caps the arena (e.g. to leave ncu room for its replay buffers)
    if (const char *e = getenv("SGPU_ARENA_GB")) { const double gb = atof(e); if (gb >= 0.0625) want = std::min(want, (size_t)(gb * (double)(1ull << 30))); }
    want &= ~(size_t)((2u << 20) - 1);
    while (want >= ((size_t)64 << 20)) {
        void *p = nullptr;
        if (cudaMalloc(&p, want) == cudaSuccess) { arena = (char *)p; arena_size = want; break; }
        cudaGetLastError();
        want = (size_t)((double)want * 0.9) & ~(size_t)((2u << 20) - 1);
    }
    if (!arena) throw Error(4, "cannot reserve the device memory arena");
    arena_free.clear();
    arena_free[0] = arena_size;
    pool_cached = arena_size;
}
inline void Ctx::peer_close() {
    for (char *p : peer_arena) if (p) cudaIpcCloseMemHandle(p);
    peer_arena.clear(); peer_handle.clear();
}
inline char *Ctx::peer_map(int world, int rank, int g, const void *handle) {
    if (g == rank) return arena;
    if ((int)peer_arena.size() != world) { peer_close(); peer_arena.assign(world, nullptr); peer_handle.assign((size_t)world * 64, 0); }
    // a peer's arena is mapped once per process; a different handle under the same rank (its context was re-created) remaps
    if (peer_arena[g] && memcmp(&peer_handle[(size_t)g * 64], handle, 64) != 0) {
        cudaIpcCloseMemHandle(peer_arena[g]);
        peer_arena[g] = nullptr;
    }
    if (!peer_arena[g]) {
        cudaIpcMemHandle_t h;
        memcpy(&h, handle, sizeof h);
        void *p = nullptr;
        SG_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        peer_arena[g] = (char *)p;
        memcpy(&peer_handle[(size_t)g * 64], handle, 64);
    }
    return peer_arena[g];
}
inline uint64_t Ctx::arena_offset(const void *p, const char *what) const {
    const char *c = (const char *)p;
    SG_CHECK(arena && c >= arena && c < arena + arena_size, 4, what);
    return (uint64_t)(c - arena);
}
inline void Ctx::pool_trim() {
    peer_close();
    if (arena) cudaFree(arena);
    arena = nullptr; arena_size = 0; arena_free.clear(); pool_cached = 0;
    for (auto &d : direct) cudaFree(d.first);
    direct.clear();
}
inline size_t Ctx::free_bytes() {
    if (!arena) arena_init();
    return pool_cached;
}
inline void *Ctx::pool_alloc(size_t bytes, size_t *blk, bool persistent) {
    if (!arena) arena_init();
    const size_t want = (bytes + 511) & ~(size_t)511;
    if (!persistent) {
        for (auto it = arena_free.begin(); it != arena_free.end(); ++it) {
            if (it->second >= want) {                         // first fit from the bottom
                const size_t off = it->first, sz = it->second;
                arena_free.erase(it);
                if (sz > want) arena_free[off + want] = sz - want;
                pool_cached -= want; *blk = want;
                return arena + off;
            }
        }
    } else {
        for (auto it = arena_free.rbegin(); it != arena_free.rend(); ++it) {
            if (it->second >= want) {                         // last fit, carved from the top end of the hole
                const size_t off = it->first, sz = it->second;
                if (sz == want) arena_free.erase(std::next(it).base());
                else it->second = sz - want;
                pool_cached -= want; *blk = want;
                return arena + off + (sz - want);
            }
        }
    }
    // does not fit (fragmentation or a request beyond the arena): ask the driver directly
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        cudaGetLastError();
        char m[256];
        snprintf(m, sizeof m, "out of device memory: %zu bytes requested, %zu free in the %zu-byte arena (in use %zu)", want, pool_cached, arena_size, allocated);
        throw Error(4, m);
    }
    direct.push_back({p, want});
    *blk = want;
    return p;
}
inline void Ctx::pool_release(void *p, size_t blk) {
    char *c = (char *)p;
    if (arena && c >= arena && c < arena + arena_size) {
        size_t off = (size_t)(c - arena), sz = blk;
        auto nxt = arena_free.lower_bound(off);
        if (nxt != arena_free.end() && off + sz == nxt->first) { sz += nxt->second; nxt = arena_free.erase(nxt); }
        if (nxt != arena_free.begin()) {
            auto prv = std::prev(nxt);
            if (prv->first + prv->second == off) { prv->second += sz; pool_cached += blk; return; }
        }
        arena_free[off] = sz;
        pool_cached += blk;
        return;
    }
    for (size_t i = 0; i < direct.size(); ++i)
        if (direct[i].first == p) { cudaFree(p); direct.erase(direct.begin() + i); return; }
    cudaFree(p);
}
template <class T>
void DArr<T>::alloc(Ctx *c, size_t n_, bool persistent) {
    release();
    ctx = c; n = n_;
    size_t b = (n_ ? n_ : 1) * sizeof(T);
    p = (T *)c->pool_alloc(b, &blk, persistent);
    c->allocated += blk;
    if (c->allocated > c->peak) c->peak = c->allocated;
}
template <class T>
void DArr<T>::release() {
    if (p) {
        ctx->allocated -= blk;
        ctx->pool_release(p, blk);
    }
    p = nullptr; n = 0; blk = 0;
}

// pinned host memory (cudaHostAlloc): copies to and from it run at the full PCIe rate and asynchronously
template <class T>
struct HostArr {
    T *p = nullptr;
    size_t n = 0;
    HostArr() {}
    HostArr(const HostArr &) = delete;
    HostArr &operator=(const HostArr &) = delete;
    HostArr(HostArr &&o) noexcept { p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    HostArr &operator=(HostArr &&o) noexcept {
        if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
        return *this;
    }
    ~HostArr() { release(); }
    void alloc(size_t n_) {
        release();
        void *q = nullptr;
        if (cudaHostAlloc(&q, (n_ ? n_ : 1) * sizeof(T), cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            throw Error(4, "out of pinned host memory for a host-resident k-mer set");
        }
        p = (T *)q; n = n_;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; n = 0; }
};

// A counted k-mer set: what KMerDiskCounter::Count leaves on disk (kmer_index_builder.hpp:306-332), bucket-major, strictly
// increasing inside a bucket. It lives in HBM (keys / counts), or, for a count with SGPU_RESULT_ON_HOST, in pinned host memory
// (h_keys / h_counts; the device arrays are released once the chunk's copy has completed). A set's chunks all live in one place.
struct Chunk {
    DArr<uint64_t> keys;     // n * nw words (records of W = 8*nw bytes, the on-disk record format)
    DArr<uint32_t> counts;   // n (canonical mode) or empty
    HostArr<uint64_t> h_keys;
    HostArr<uint32_t> h_counts;
    int64_t n = 0;
    int b_lo = 0, b_hi = 0;  // buckets [b_lo, b_hi)
    int64_t first = 0;       // index of its first record in final_kmers order
};
// chunks one set may hold: the MPHF build and the graph kernels pass the chunk table by value in their parameter block
// (KeyTable, mphf_dev.cuh), so the count's planner never makes more passes than this
static const int kMaxChunks = 128;
struct KSet {
    Ctx *ctx = nullptr;
    int K = 0, nw = 0, B = 0;
    int64_t n = 0;
    bool has_counts = false;
    bool on_host = false;              // chunks in pinned host memory
    std::vector<Chunk> chunks;
    std::vector<int64_t> bsz;          // B
    std::vector<int64_t> bstart;       // B+1 exclusive prefix (final_kmers order)
};

// A set's chunks on the device, in order. A device set's chunks are read in place, at no cost (no stream, event or buffer). A host
// set's are brought over one at a time, double-buffered: chunk c + 1 is copied on the stager's own stream while chunk c is used on
// the context's stream. acquire(c) makes chunk c readable by work enqueued next on ctx->stream; release(c) marks the end of that
// work (the chunk's buffer may then take chunk c + 2). Chunks are acquired in order, 0 to the last, and a sweep may start again at
// chunk 0. The uploads have a stream of their own so that they do not queue behind a host-memory count's result copies (ctx->copy).
struct ChunkStager {
    Ctx *ctx;
    const KSet *ks;
    bool with_counts;
    DArr<uint64_t> keys[2];
    DArr<uint32_t> counts[2];
    cudaStream_t up = nullptr;
    cudaEvent_t loaded[2] = {nullptr, nullptr}, used[2] = {nullptr, nullptr};
    ChunkStager(const KSet *s, bool counts_too) : ctx(s->ctx), ks(s), with_counts(counts_too && s->has_counts) {
        if (!ks->on_host) return;
        size_t mx = 1;
        for (const Chunk &c : ks->chunks) mx = std::max(mx, (size_t)c.n);
        SG_CUDA(cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            keys[i].alloc(ctx, mx * ks->nw);
            if (with_counts) counts[i].alloc(ctx, mx);
            SG_CUDA(cudaEventCreateWithFlags(&loaded[i], cudaEventDisableTiming));
            SG_CUDA(cudaEventCreateWithFlags(&used[i], cudaEventDisableTiming));
        }
    }
    ~ChunkStager() {
        // the buffers go back to the arena: no copy may still be writing them
        if (up) { cudaStreamSynchronize(up); cudaStreamDestroy(up); }
        for (int i = 0; i < 2; ++i) { if (loaded[i]) cudaEventDestroy(loaded[i]); if (used[i]) cudaEventDestroy(used[i]); }
    }
    ChunkStager(const ChunkStager &) = delete;
    ChunkStager &operator=(const ChunkStager &) = delete;
    void prefetch(size_t c) {
        const Chunk &ch = ks->chunks[c];
        const int s = (int)(c & 1);
        SG_CUDA(cudaStreamWaitEvent(up, used[s], 0));
        if (ch.n) {
            SG_CUDA(cudaMemcpyAsync(keys[s].p, ch.h_keys.p, (size_t)ch.n * ks->nw * 8, cudaMemcpyHostToDevice, up));
            if (with_counts) SG_CUDA(cudaMemcpyAsync(counts[s].p, ch.h_counts.p, (size_t)ch.n * 4, cudaMemcpyHostToDevice, up));
            ctx->times.stage_h2d_bytes += (uint64_t)ch.n * ks->nw * 8 + (with_counts ? (uint64_t)ch.n * 4 : 0);
        }
        SG_CUDA(cudaEventRecord(loaded[s], up));
    }
    void acquire(size_t c, const uint64_t **k, const uint32_t **cnt) {
        if (!ks->on_host) {
            *k = ks->chunks[c].keys.p;
            if (cnt) *cnt = with_counts ? ks->chunks[c].counts.p : nullptr;
            return;
        }
        if (c == 0) prefetch(0);
        const int s = (int)(c & 1);
        SG_CUDA(cudaStreamWaitEvent(ctx->stream, loaded[s], 0));
        if (c + 1 < ks->chunks.size()) prefetch(c + 1);
        *k = keys[s].p;
        if (cnt) *cnt = with_counts ? counts[s].p : nullptr;
    }
    void release(size_t c) { if (ks->on_host) SG_CUDA(cudaEventRecord(used[c & 1], ctx->stream)); }
    // f(chunk, keys, counts) for every non-empty chunk, in order; counts is null without them
    template <class F>
    void sweep(F &&f) {
        for (size_t c = 0; c < ks->chunks.size(); ++c) {
            const uint64_t *k = nullptr;
            const uint32_t *cnt = nullptr;
            acquire(c, &k, &cnt);
            if (ks->chunks[c].n) f(ks->chunks[c], k, cnt);
            release(c);
        }
        SG_CUDA(cudaGetLastError());
    }
};

// SGPU_TRACE (user option, read once per process): wall-clock milliseconds between marks on stderr, one line per mark. A trace
// given a stream (a context's is never null) waits for the work enqueued on it at every mark, so that a mark also times that work.
struct Trace {
    const char *label;
    cudaStream_t st;
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    explicit Trace(const char *l, cudaStream_t s = nullptr) : label(l), st(s) {}
    void mark(const char *what) {
        static const bool on = getenv("SGPU_TRACE") != nullptr;
        if (!on) return;
        if (st) cudaStreamSynchronize(st);
        const auto t = std::chrono::steady_clock::now();
        fprintf(stderr, "[%s] %-28s %9.3f ms\n", label, what, std::chrono::duration<double, std::milli>(t - t0).count());
        t0 = t;
    }
};

// boomphf-compatible index resident in HBM (one mphf per bucket, BooPHF.h / kmer_index.hpp)
static const int kLevels = 25;
struct Mphf {
    Ctx *ctx = nullptr;
    int K = 0, nw = 0, B = 0;
    int64_t n = 0;
    std::vector<uint64_t> dom;         // B*25 hash domains
    std::vector<uint64_t> nchar;       // B*25 words per level (1 + dom/64)
    std::vector<uint64_t> woff;        // B*25 word offset of the level in `bits` (levels padded to 8 words)
    std::vector<uint64_t> lastrank;    // B
    std::vector<int64_t> bsz;          // B
    std::vector<uint64_t> starts;      // B+1, as serialized (last entry not accumulated)
    uint64_t total_words = 0;
    DArr<uint64_t> bits;               // all buckets, all levels
    DArr<uint64_t> ranks;              // one per 8 words
    DArr<uint64_t> d_dom, d_woff, d_starts;   // device copies of the tables
};

// scans / utilities (scan.cu)
void exclusive_scan_u64(Ctx *ctx, const uint64_t *in, uint64_t *out, size_t n);
void exclusive_scan_u32_to_u64(Ctx *ctx, const uint32_t *in, uint64_t *out, size_t n);
void ensure_reads_on_device(Ctx *ctx);

// ingest_gpu.cu
void reads_pack_text(Ctx *ctx, const char *text, uint64_t text_bytes, const uint64_t *seq_off, const uint32_t *seq_len, int64_t n, int longest_valid);
void reads_download(Ctx *ctx, uint64_t *words, uint64_t *offs, uint32_t *lens);
// covfilter.cu; passes = 0: planned against the context's device budget (cov_plan.h), 1: one table, >= 2: that many key-range passes
void cov_filter(Ctx *ctx, int K, unsigned thr, int apply, int passes, uint8_t *keep_out, uint64_t *stats);
// distributed coverage filter (covfilter.cu)
struct CovDist;
CovDist *dist_cov_begin(Ctx *ctx, int K, unsigned thr, int world, int rank);
void dist_cov_ipc_handle(CovDist *d, uint8_t *out96);
void dist_cov_open_peers(CovDist *d, const uint8_t *descs);
void dist_cov_bound(CovDist *d);
void dist_cov_fill(CovDist *d);
void dist_cov_filter(CovDist *d, int apply, uint8_t *keep_out, uint64_t *stats);
void dist_cov_free(CovDist *d);
// pure host arithmetic (exported for CPU tests): a key's owner rank; table capacities and the pass plan are in cov_plan.h
uint32_t cov_owner_host(uint64_t key, int world);

// count.cu
enum CountMode { kCanonical = 0, kAllWindows = 1 };
KSet *count_from_reads(Ctx *ctx, int K, int B, int mode, bool result_on_host = false);
KSet *kmers_from_kpomers(Ctx *ctx, const KSet *kp, int B, bool result_on_host = false);

void kset_checksum(const KSet *ks, uint64_t *out4);

// distributed count (count.cu)
struct DistState;
struct DistPlan;
DistState *dist_begin(Ctx *ctx, int K, int B, int mode, int world, int rank, bool result_on_host = false);
DistState *dist_begin_kpomers(Ctx *ctx, const KSet *kp, int B, int world, int rank, bool result_on_host);
uint32_t dist_num_partitions(const DistState *d);
void dist_local_counts(DistState *d, uint64_t *h_out);
void dist_plan(DistState *d, const uint64_t *cnt_all, uint64_t *total_records);
uint64_t dist_free_bytes(DistState *d);
int dist_next_pass(DistState *d, uint64_t budget_bytes);
void dist_ipc_handle(DistState *d, uint8_t *out96);
void dist_open_peers(DistState *d, const uint8_t *descs);
void dist_scatter(DistState *d, int p);
void dist_exchange(DistState *d, int p);
void dist_sort(DistState *d, int p);
KSet *dist_end(DistState *d);
void dist_free(DistState *d);
// pure host planning (exported for CPU tests): returns npass, fills pass boundaries / owner boundaries / totals
int dist_plan_host(int world, int B, int rA, const uint64_t *cnt_all, uint64_t budget_bytes, int record_bytes, int *pass_b /*B+1 max*/, uint64_t *max_recv);

// mphf.cu
Mphf *mphf_build(Ctx *ctx, const KSet *ks);
size_t mphf_serialized_size(const Mphf *m);
void mphf_serialize_to(const Mphf *m, uint8_t *out, size_t cap);
// the bytes of buckets [b_lo, b_hi) alone: the middle of mphf_serialize_to's image, without num_segments and segment_starts
size_t mphf_serialized_size_buckets(const Mphf *m, int b_lo, int b_hi);
void mphf_serialize_buckets_to(const Mphf *m, int b_lo, int b_hi, uint8_t *out, size_t cap);
void mphf_lookup_host_keys(Ctx *ctx, const Mphf *m, const uint64_t *h_keys, int64_t n, uint64_t *h_out);

static inline int div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace sg
