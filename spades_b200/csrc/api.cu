// api.cu -- the extern "C" boundary (include/spades_b200.h). No exceptions cross it; no CPU fallbacks live behind it.
#include <fcntl.h>
#include <stdio.h>
#include <unistd.h>

#include <string>

#include "../../include/spades_b200.h"
#include "graph.h"
#include "host_par.h"
#include "sgpu_internal.h"

using namespace sg;

struct sgpu_ctx { Ctx c; bool own_stream = true; };

// Lifetime: k-mer sets, indexes, graphs and distributed counts keep blocks of their context's arena. sgpu_destroy() while any of
// them is alive only marks the context; the last child to be freed then tears it down (no use-after-free whatever the order,
// e.g. Python finalisers at interpreter exit).
static void ctx_teardown(sgpu_ctx *ctx) {
    cudaSetDevice(ctx->c.device);
    ctx->c.r_words.release(); ctx->c.r_offs.release(); ctx->c.r_lens.release();
    ctx->c.pool_trim();
    if (ctx->c.copy) cudaStreamDestroy(ctx->c.copy);
    if (ctx->c.stream && ctx->own_stream) cudaStreamDestroy(ctx->c.stream);
    delete ctx;
}
static void child_add(Ctx *c) { c->live_children++; }
static void child_release(Ctx *c) {
    if (--c->live_children == 0 && c->destroy_pending) ctx_teardown(static_cast<sgpu_ctx *>(c->owner));
}
// readers: distributed counts that read this set (sgpu_dist_begin_kpomers); sgpu_kset_free defers the release to the last of them
struct sgpu_kset { KSet *s; mutable int readers = 0; mutable bool free_pending = false; };
struct sgpu_mphf { Mphf *m; };
struct sgpu_graph { Graph *g; };
struct sgpu_edge_index { EdgeIndex *e; };

static int fail(Ctx *c, int code, const std::string &msg) {
    if (c) c->err = msg;
    return code ? code : SGPU_EINTERNAL;
}
#define API_TRY(ctxptr, ...)                                    \
    try { __VA_ARGS__; return SGPU_OK; }                           \
    catch (const sg::Error &e) { return fail((ctxptr), e.code, e.what()); } \
    catch (const std::bad_alloc &) { return fail((ctxptr), SGPU_ENOMEM, "host allocation failed"); } \
    catch (const std::exception &e) { return fail((ctxptr), SGPU_EINTERNAL, e.what()); }

// the entries that predate host sets (sgpu_kmers_from_kpomers, sgpu_graph_build, _ex, _opts) keep refusing them; their _ex /
// _streamed successors take either placement
static void check_device_sets(const sgpu_kset *kpomers, const sgpu_kset *kmers) {
    SG_CHECK(!kpomers->s->on_host && !kmers->s->on_host, SGPU_EUNSUPPORTED,
             "the graph is built from k-mer sets in device memory; this one lives in host memory (SGPU_RESULT_ON_HOST)");
}
static int device_sets_only(Ctx *c, const sgpu_kset *kpomers, const sgpu_kset *kmers) { API_TRY(c, check_device_sets(kpomers, kmers)); }
static int device_kpomers_only(Ctx *c, const sgpu_kset *kpomers) {
    API_TRY(c, SG_CHECK(!kpomers->s->on_host, SGPU_EUNSUPPORTED,
                        "the (k+1)-mer set lives in host memory: the k-mers of the (k+1)-mers read it from the device"));
}

extern "C" {

int sgpu_create(const sgpu_config *cfg, sgpu_ctx **out) {
    if (!out) return SGPU_EINVAL;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return SGPU_ENODEV; }
    int dev = cfg ? cfg->device : 0;
    if (dev < 0 || dev >= ndev) return SGPU_EINVAL;
    if (cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); return SGPU_ENODEV; }
    sgpu_ctx *h = new sgpu_ctx();
    h->c.owner = h;
    h->c.device = dev;
    h->c.hbm_budget = cfg ? (size_t)cfg->hbm_budget_bytes : 0;
    h->c.verbose = cfg ? cfg->verbose : 0;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { cudaGetLastError(); delete h; return SGPU_ECUDA; }
    if (cfg && cfg->stream) { h->c.stream = (cudaStream_t)(uintptr_t)cfg->stream; h->own_stream = false; }
    else if (cudaStreamCreateWithFlags(&h->c.stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); delete h; return SGPU_ECUDA; }
    h->c.num_sms = prop.multiProcessorCount;
    *out = h;
    return SGPU_OK;
}

void sgpu_destroy(sgpu_ctx *ctx) {
    if (!ctx || ctx->c.destroy_pending) return;
    if (ctx->c.live_children > 0) { ctx->c.destroy_pending = true; return; }      // deferred until the last child is freed
    ctx_teardown(ctx);
}

const char *sgpu_last_error(const sgpu_ctx *ctx) { return ctx ? ctx->c.err.c_str() : "no context"; }

int sgpu_get_times(const sgpu_ctx *ctx, sgpu_times *out) {
    if (!ctx || !out) return SGPU_EINVAL;
    const PhaseTimes &t = ctx->c.times;
    out->extract_count_ms = t.extract_count; out->extract_scatter_ms = t.extract_scatter; out->refine_ms = t.refine;
    out->local_sort_ms = t.local_sort; out->compact_ms = t.compact; out->mphf_ms = t.mphf; out->exchange_ms = t.exchange;
    out->instances = t.instances; out->passes = t.passes; out->launches = ctx->c.launches; out->peak_bytes = ctx->c.peak; out->cached_bytes = ctx->c.pool_cached;
    out->level_a_key_bits = t.level_a_key_bits; out->level_a_scatters = t.level_a_scatters;
    out->refine_rounds_max = t.refine_rounds_max; out->refine_splits_round0 = t.refine_splits_round0; out->refine_splits_later = t.refine_splits_later;
    out->sort_lsd_fallbacks = t.sort_lsd_fallbacks; out->sort_oversize_equal = t.sort_oversize_equal;
    out->result_d2h_bytes = t.result_d2h_bytes; out->result_d2h_wait_ms = t.result_d2h_wait;
    out->stage_h2d_bytes = t.stage_h2d_bytes; out->graph_junction_batches = t.graph_junction_batches;
    out->cov_filter_passes = t.cov_filter_passes; out->cov_filter_table_bytes = t.cov_filter_table_bytes;
    return SGPU_OK;
}

int sgpu_reads_clear(sgpu_ctx *ctx) {
    if (!ctx) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        c->h_words.clear(); c->h_offs.clear(); c->h_lens.clear();
        c->r_words.release(); c->r_offs.release(); c->r_lens.release();
        c->d_words = nullptr; c->d_offs = nullptr; c->d_lens = nullptr; c->n_reads = 0; c->n_words = 0; c->staged_dirty = false;
    })
}

int sgpu_reads_append_packed(sgpu_ctx *ctx, const uint64_t *words, uint64_t nwords, const uint64_t *offs, const uint32_t *lens, int64_t nreads) {
    if (!ctx || nreads < 0 || (nreads && (!words || !offs || !lens))) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        const uint64_t base = c->h_words.size();
        for (int64_t r = 0; r < nreads; ++r) {
            const uint64_t need = ((uint64_t)lens[r] + 31) / 32;
            SG_CHECK(offs[r] + need <= nwords, SGPU_EINVAL, "read extends past the word buffer");
            c->h_offs.push_back(base + offs[r]);
            c->h_lens.push_back(lens[r]);
        }
        c->h_words.insert(c->h_words.end(), words, words + nwords);
        c->staged_dirty = true;
    })
}

int sgpu_reads_append_batch(sgpu_ctx *ctx, const sgpu_read_batch *b) {
    if (!ctx || !b) return SGPU_EINVAL;
    return sgpu_reads_append_packed(ctx, sgpu_read_batch_words(b), sgpu_read_batch_num_words(b), sgpu_read_batch_offs(b), sgpu_read_batch_lens(b),
                                    sgpu_read_batch_num_reads(b));
}

int sgpu_reads_upload(sgpu_ctx *ctx, const uint64_t *words, uint64_t nwords, const uint64_t *offs, const uint32_t *lens, int64_t nreads) {
    if (!ctx || nreads < 0 || (nreads && (!words || !offs || !lens))) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        c->h_words.clear(); c->h_offs.clear(); c->h_lens.clear(); c->staged_dirty = false;
        if (c->r_words.n < nwords + 4) c->r_words.alloc(c, nwords + 4, true);
        if (c->r_offs.n < (size_t)nreads + 1) c->r_offs.alloc(c, (size_t)nreads + 1, true);
        if (c->r_lens.n < (size_t)nreads + 1) c->r_lens.alloc(c, (size_t)nreads + 1, true);
        // one asynchronous copy per array on the context's stream (a chunked copy overlapped with the first pass over the reads was
        // slower: the per-chunk launches cost more than the overlap won). The caller's buffers must stay
        // valid and unmodified until the next call that synchronises (sgpu_count / sgpu_dist_begin), see spades_b200.h.
        if (nwords) SG_CUDA(cudaMemcpyAsync(c->r_words.p, words, nwords * 8, cudaMemcpyHostToDevice, c->stream));
        SG_CUDA(cudaMemsetAsync(c->r_words.p + nwords, 0, 4 * 8, c->stream));       // the padding words the window loads may touch
        if (nreads) {
            SG_CUDA(cudaMemcpyAsync(c->r_offs.p, offs, (size_t)nreads * 8, cudaMemcpyHostToDevice, c->stream));
            SG_CUDA(cudaMemcpyAsync(c->r_lens.p, lens, (size_t)nreads * 4, cudaMemcpyHostToDevice, c->stream));
        }
        c->d_words = c->r_words.p; c->d_offs = c->r_offs.p; c->d_lens = c->r_lens.p; c->n_reads = nreads; c->n_words = nwords;
    })
}

int sgpu_reads_pack_text(sgpu_ctx *ctx, const char *text, uint64_t text_bytes, const uint64_t *seq_off, const uint32_t *seq_len, int64_t nreads, int longest_valid) {
    if (!ctx || nreads < 0 || (nreads && (!text || !seq_off || !seq_len))) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); reads_pack_text(c, text, text_bytes, seq_off, seq_len, nreads, longest_valid); })
}
int sgpu_reads_cov_filter(sgpu_ctx *ctx, int K, unsigned threshold, int apply, uint8_t *keep_out, uint64_t *stats) {
    if (!ctx) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); cov_filter(c, K, threshold, apply, 0, keep_out, stats); })
}
int sgpu_reads_cov_filter_ex(sgpu_ctx *ctx, int K, unsigned threshold, int apply, int passes, uint8_t *keep_out, uint64_t *stats) {
    if (!ctx || passes < 0 || passes > kCovMaxPasses) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); cov_filter(c, K, threshold, apply, passes, keep_out, stats); })
}
int sgpu_cov_pass_plan_host(uint64_t cardinality_bound, int64_t nreads, uint64_t budget_bytes, int *passes, uint64_t *pass_capacity) {
    if (nreads < 0 || !passes || !pass_capacity) return SGPU_EINVAL;
    const CovPassPlan pl = cov_pass_plan(cardinality_bound, nreads, budget_bytes);
    *passes = pl.passes;
    *pass_capacity = pl.cap;
    return pl.passes ? SGPU_OK : SGPU_ENOMEM;
}
int sgpu_reads_info(sgpu_ctx *ctx, int64_t *nreads, uint64_t *nwords) {
    if (!ctx || !nreads || !nwords) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); ensure_reads_on_device(c); *nreads = c->n_reads; *nwords = c->n_words; })
}
int sgpu_reads_download(sgpu_ctx *ctx, uint64_t *words, uint64_t *offs, uint32_t *lens) {
    if (!ctx) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); reads_download(c, words, offs, lens); })
}

int sgpu_reads_adopt_device(sgpu_ctx *ctx, const uint64_t *d_words, uint64_t nwords, const uint64_t *d_offs, const uint32_t *d_lens, int64_t nreads) {
    if (!ctx || nreads < 0) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        c->h_words.clear(); c->h_offs.clear(); c->h_lens.clear(); c->staged_dirty = false;
        c->r_words.release(); c->r_offs.release(); c->r_lens.release();
        c->d_words = d_words; c->d_offs = d_offs; c->d_lens = d_lens; c->n_reads = nreads; c->n_words = nwords;
    })
}

int sgpu_count(sgpu_ctx *ctx, int K, int num_buckets, int mode, sgpu_kset **out) {
    if (!ctx || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        const bool on_host = (mode & SGPU_RESULT_ON_HOST) != 0;
        mode &= ~SGPU_RESULT_ON_HOST;
        SG_CHECK(mode == SGPU_CANONICAL || mode == SGPU_ALL_WINDOWS, SGPU_EINVAL, "bad mode");
        SG_CUDA(cudaSetDevice(c->device));
        KSet *s = count_from_reads(c, K, num_buckets, mode, on_host);
        *out = new sgpu_kset{s};
        child_add(c);
    })
}

int sgpu_kmers_from_kpomers_ex(sgpu_ctx *ctx, const sgpu_kset *kpomers, int num_buckets, int mode, sgpu_kset **out) {
    if (!ctx || !kpomers || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CHECK(mode == 0 || mode == SGPU_RESULT_ON_HOST, SGPU_EINVAL, "bad mode");
        SG_CUDA(cudaSetDevice(c->device));
        KSet *s = kmers_from_kpomers(c, kpomers->s, num_buckets, mode == SGPU_RESULT_ON_HOST);
        *out = new sgpu_kset{s};
        child_add(c);
    })
}

int sgpu_kmers_from_kpomers(sgpu_ctx *ctx, const sgpu_kset *kpomers, int num_buckets, sgpu_kset **out) {
    if (!ctx || !kpomers || !out) return SGPU_EINVAL;
    *out = nullptr;
    const int rc = device_kpomers_only(&ctx->c, kpomers);
    return rc != SGPU_OK ? rc : sgpu_kmers_from_kpomers_ex(ctx, kpomers, num_buckets, 0, out);
}

int64_t sgpu_kset_size(const sgpu_kset *s) { return s ? s->s->n : -1; }
int sgpu_kset_k(const sgpu_kset *s) { return s ? s->s->K : -1; }
int sgpu_kset_num_buckets(const sgpu_kset *s) { return s ? s->s->B : -1; }
int sgpu_kset_record_bytes(const sgpu_kset *s) { return s ? 8 * s->s->nw : -1; }
int sgpu_kset_on_host(const sgpu_kset *s) { return s ? (s->s->on_host ? 1 : 0) : -1; }
int sgpu_kset_bucket_sizes(const sgpu_kset *s, int64_t *out) {
    if (!s || !out) return SGPU_EINVAL;
    for (int b = 0; b < s->s->B; ++b) out[b] = s->s->bsz[b];
    return SGPU_OK;
}

}  // extern "C"

// where a chunk's records live: pinned host memory for a host set, HBM otherwise
static const uint64_t *chunk_keys(const Chunk &ch) { return ch.h_keys.p ? ch.h_keys.p : ch.keys.p; }
static const uint32_t *chunk_counts(const Chunk &ch) { return ch.h_counts.p ? ch.h_counts.p : ch.counts.p; }

template <class T, class Get>
static void download_range(const KSet *ks, int64_t first, int64_t n, T *out, size_t per, Get get) {
    SG_CHECK(first >= 0 && n >= 0 && first + n <= ks->n, SGPU_EINVAL, "range outside the k-mer set");
    Ctx *c = ks->ctx;
    SG_CUDA(cudaSetDevice(c->device));
    int64_t done = 0;
    for (const Chunk &ch : ks->chunks) {
        const int64_t lo = std::max(first, ch.first), hi = std::min(first + n, ch.first + ch.n);
        if (lo >= hi) continue;
        T *dst = out + (size_t)(lo - first) * per;
        const T *src = get(ch) + (size_t)(lo - ch.first) * per;
        const size_t bytes = (size_t)(hi - lo) * per * sizeof(T);
        if (ks->on_host) memcpy(dst, src, bytes);
        else SG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
        done += hi - lo;
    }
    SG_CUDA(cudaStreamSynchronize(c->stream));
    SG_CHECK(done == n, SGPU_EINTERNAL, "chunk table does not cover the range");
}

static void write_range(const KSet *ks, int64_t first, int64_t n, FILE *f) {
    const size_t W = (size_t)ks->nw;
    const int64_t step = 1 << 22;
    std::vector<uint64_t> buf;
    for (int64_t o = 0; o < n; o += step) {
        const int64_t m = std::min(step, n - o);
        buf.resize((size_t)m * W);
        download_range<uint64_t>(ks, first + o, m, buf.data(), W, chunk_keys);
        SG_CHECK(fwrite(buf.data(), 8 * W, (size_t)m, f) == (size_t)m, SGPU_EIO, "short write");
    }
}

// the buckets the set's chunks cover: all of them for a single-GPU count, this rank's share of every pass for a distributed one
static std::vector<uint8_t> owned_buckets(const KSet *ks) {
    std::vector<uint8_t> own((size_t)ks->B, 0);
    for (const Chunk &ch : ks->chunks) std::fill(own.begin() + ch.b_lo, own.begin() + ch.b_hi, (uint8_t)1);
    return own;
}

// <prefix>.<b> for every bucket, or for the owned ones only (ranks of a distributed count writing into one directory)
static void write_bucket_files(const KSet *ks, const char *prefix, bool owned_only) {
    const std::vector<uint8_t> own = owned_buckets(ks);
    for (int b = 0; b < ks->B; ++b) {
        if (owned_only && !own[b]) continue;
        std::string p = std::string(prefix) + "." + std::to_string(b);
        FILE *f = fopen(p.c_str(), "wb");
        SG_CHECK(f, SGPU_EIO, "cannot open bucket file for writing");
        try { write_range(ks, ks->bstart[b], ks->bsz[b], f); } catch (...) { fclose(f); throw; }
        fclose(f);
    }
}

extern "C" {

int sgpu_kset_checksum(const sgpu_kset *s, uint64_t *out4) {
    if (!s || !out4) return SGPU_EINVAL;
    Ctx *c = s->s->ctx;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); kset_checksum(s->s, out4); })
}
int sgpu_kset_download_keys(const sgpu_kset *s, int64_t first, int64_t n, uint64_t *out) {
    if (!s || (n && !out)) return SGPU_EINVAL;
    Ctx *c = s->s->ctx;
    API_TRY(c, { download_range<uint64_t>(s->s, first, n, out, (size_t)s->s->nw, chunk_keys); })
}
int sgpu_kset_download_counts(const sgpu_kset *s, int64_t first, int64_t n, uint32_t *out) {
    if (!s || (n && !out)) return SGPU_EINVAL;
    Ctx *c = s->s->ctx;
    API_TRY(c, {
        SG_CHECK(s->s->has_counts, SGPU_EINVAL, "this k-mer set carries no multiplicities");
        download_range<uint32_t>(s->s, first, n, out, 1, chunk_counts);
    })
}

int sgpu_kset_owned_buckets(const sgpu_kset *s, uint8_t *flags) {
    if (!s || !flags) return SGPU_EINVAL;
    const std::vector<uint8_t> own = owned_buckets(s->s);
    memcpy(flags, own.data(), own.size());
    return SGPU_OK;
}
int sgpu_kset_write_buckets(const sgpu_kset *s, const char *prefix) {
    if (!s || !prefix) return SGPU_EINVAL;
    Ctx *c = s->s->ctx;
    API_TRY(c, write_bucket_files(s->s, prefix, false))
}
int sgpu_kset_write_owned_buckets(const sgpu_kset *s, const char *prefix) {
    if (!s || !prefix) return SGPU_EINVAL;
    Ctx *c = s->s->ctx;
    API_TRY(c, write_bucket_files(s->s, prefix, true))
}
int sgpu_kset_write_final(const sgpu_kset *s, const char *path) {
    if (!s || !path) return SGPU_EINVAL;
    Ctx *c = s->s->ctx;
    API_TRY(c, {
        FILE *f = fopen(path, "wb");
        SG_CHECK(f, SGPU_EIO, "cannot open final_kmers for writing");
        try { write_range(s->s, 0, s->s->n, f); } catch (...) { fclose(f); throw; }
        fclose(f);
    })
}
void sgpu_kset_free(sgpu_kset *s) {
    if (!s) return;
    if (s->readers > 0) { s->free_pending = true; return; }       // released by the last sgpu_dist_free that reads it
    if (s->s) { Ctx *c = s->s->ctx; cudaSetDevice(c->device); delete s->s; child_release(c); }
    delete s;
}

int sgpu_mphf_build(sgpu_ctx *ctx, const sgpu_kset *s, sgpu_mphf **out) {
    if (!ctx || !s || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        Mphf *m = mphf_build(c, s->s);
        *out = new sgpu_mphf{m};
        child_add(c);
    })
}
int64_t sgpu_mphf_serialized_size(const sgpu_mphf *m) { return m ? (int64_t)mphf_serialized_size(m->m) : -1; }
int sgpu_mphf_serialize(const sgpu_mphf *m, uint8_t *out, int64_t cap) {
    if (!m || !out || cap < 0) return SGPU_EINVAL;
    Ctx *c = m->m->ctx;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        mphf_serialize_to(m->m, out, (size_t)cap);
    })
}
int64_t sgpu_mphf_serialized_size_buckets(const sgpu_mphf *m, int b_lo, int b_hi) {
    if (!m || b_lo < 0 || b_lo > b_hi || b_hi > m->m->B) return -1;
    return (int64_t)mphf_serialized_size_buckets(m->m, b_lo, b_hi);
}
int sgpu_mphf_serialize_buckets(const sgpu_mphf *m, int b_lo, int b_hi, uint8_t *out, int64_t cap) {
    if (!m || !out || cap < 0) return SGPU_EINVAL;
    Ctx *c = m->m->ctx;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        mphf_serialize_buckets_to(m->m, b_lo, b_hi, out, (size_t)cap);
    })
}
int sgpu_mphf_lookup(const sgpu_mphf *m, const uint64_t *keys, int64_t n, uint64_t *out_idx) {
    if (!m || (n && (!keys || !out_idx))) return SGPU_EINVAL;
    Ctx *c = m->m->ctx;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); mphf_lookup_host_keys(c, m->m, keys, n, out_idx); })
}
void sgpu_mphf_free(sgpu_mphf *m) {
    if (!m) return;
    if (m->m) { Ctx *c = m->m->ctx; cudaSetDevice(c->device); delete m->m; child_release(c); }
    delete m;
}

}  // extern "C"


extern "C" {

// the options of a graph build, refused with SGPU_EINVAL as sgpu_graph_build_opts documents (throws)
static GraphOptions graph_options(const sgpu_graph_options *o) {
    SG_CHECK(!o->early_at_clipper || (o->at_ratio > 0.0 && o->at_ratio <= 1.0 && o->at_max_length >= 1), SGPU_EINVAL, "bad A/T clipper parameters");
    GraphOptions opt;
    opt.keep_perfect_loops = o->keep_perfect_loops != 0;
    opt.early_tip_length_bound = o->early_tip_length_bound;
    opt.early_at = o->early_at_clipper != 0;
    opt.at_ratio = o->at_ratio; opt.at_min_len = o->at_min_length; opt.at_max_len = o->at_max_length;
    return opt;
}

int sgpu_graph_build(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index, const sgpu_mphf *kpomer_index,
                     int keep_perfect_loops, sgpu_graph **out) {
    const sgpu_graph_options o = {keep_perfect_loops, 0, 0, 0.8, 10, 200};
    return sgpu_graph_build_opts(ctx, kpomers, kmers, kmer_index, kpomer_index, &o, out);
}
int sgpu_graph_build_ex(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index, const sgpu_mphf *kpomer_index,
                        int keep_perfect_loops, uint64_t early_tip_length_bound, sgpu_graph **out) {
    const sgpu_graph_options o = {keep_perfect_loops, early_tip_length_bound, 0, 0.8, 10, 200};
    return sgpu_graph_build_opts(ctx, kpomers, kmers, kmer_index, kpomer_index, &o, out);
}
int sgpu_graph_build_opts(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index, const sgpu_mphf *kpomer_index,
                          const sgpu_graph_options *o, sgpu_graph **out) {
    if (!ctx || !kpomers || !kmers || !kmer_index || !o || !out) return SGPU_EINVAL;
    *out = nullptr;
    const int rc = device_sets_only(&ctx->c, kpomers, kmers);
    return rc != SGPU_OK ? rc : sgpu_graph_build_streamed(ctx, kpomers, kmers, kmer_index, kpomer_index, o, out);
}
int sgpu_graph_build_streamed(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_kset *kmers, const sgpu_mphf *kmer_index,
                              const sgpu_mphf *kpomer_index, const sgpu_graph_options *o, sgpu_graph **out) {
    if (!ctx || !kpomers || !kmers || !kmer_index || !o || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        const GraphOptions opt = graph_options(o);
        SG_CUDA(cudaSetDevice(c->device));
        Graph *g = graph_build(c, kpomers->s, kmers->s, kmer_index->m, kpomer_index ? kpomer_index->m : nullptr, opt);
        *out = new sgpu_graph{g};
        child_add(c);
    })
}
int sgpu_graph_at_clipper_stats(const sgpu_graph *g, uint64_t *out4) {
    if (!g || !out4 || !g->g->ctx) return SGPU_EINVAL;
    for (int i = 0; i < 4; ++i) out4[i] = g->g->at_stats[i];
    return SGPU_OK;
}
int sgpu_graph_tip_clipper_stats(const sgpu_graph *g, uint64_t *out3) {
    if (!g || !out3 || !g->g->ctx) return SGPU_EINVAL;
    for (int i = 0; i < 3; ++i) out3[i] = g->g->tc_stats[i];
    return SGPU_OK;
}
int sgpu_graph_masks(const sgpu_graph *g, uint8_t *out, int64_t n) {
    if (!g || (n && !out) || !g->g->ctx) return SGPU_EINVAL;
    Ctx *c = g->g->ctx;
    API_TRY(c, {
        SG_CHECK(n == g->g->km->n, SGPU_EINVAL, "mask array size != number of k-mers");
        SG_CUDA(cudaSetDevice(c->device));
        if (n) SG_CUDA(cudaMemcpy(out, g->g->masks_final.p, (size_t)n, cudaMemcpyDeviceToHost));
    })
}
int sgpu_graph_coverage(const sgpu_graph *g, uint32_t *out, int64_t n) {
    if (!g || (n && !out) || !g->g->ctx) return SGPU_EINVAL;
    Ctx *c = g->g->ctx;
    API_TRY(c, {
        SG_CHECK(g->g->cov.p, SGPU_EINVAL, "graph was built without a (k+1)-mer index: no coverage");
        SG_CHECK(n == g->g->kp->n, SGPU_EINVAL, "coverage array size != number of (k+1)-mers");
        SG_CUDA(cudaSetDevice(c->device));
        if (n) SG_CUDA(cudaMemcpy(out, g->g->cov.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    })
}
int64_t sgpu_graph_histogram(const sgpu_graph *g, uint64_t *out, int64_t cap) {
    if (!g || !g->g->ctx) return -1;
    Ctx *c = g->g->ctx;
    try {
        cudaSetDevice(c->device);
        std::vector<uint64_t> h = graph_histogram(c, g->g);
        if (out) for (int64_t i = 0; i < (int64_t)h.size() && i < cap; ++i) out[i] = h[i];
        return (int64_t)h.size();
    } catch (const std::exception &e) { c->err = e.what(); return -1; }
}
int64_t sgpu_graph_num_unitigs(const sgpu_graph *g) { return g ? (int64_t)g->g->edge_len.size() : -1; }
int64_t sgpu_graph_unitig_bases(const sgpu_graph *g) { return g ? (int64_t)g->g->seq.size() : -1; }
int sgpu_graph_unitigs(const sgpu_graph *g, char *out, uint32_t *lens) {
    if (!g) return SGPU_EINVAL;
    if (out && !g->g->seq.empty()) memcpy(out, g->g->seq.data(), g->g->seq.size());
    if (lens) for (size_t i = 0; i < g->g->edge_len.size(); ++i) lens[i] = g->g->edge_len[i];
    return SGPU_OK;
}
int64_t sgpu_graph_gfa(const sgpu_graph *g, const char *version, char *out, int64_t cap) {
    if (!g) return -1;
    try {
        std::string t = graph_gfa(g->g, version ? version : "SPAdes-4.3.0-dev");
        if (out && (int64_t)t.size() <= cap) memcpy(out, t.data(), t.size());
        return (int64_t)t.size();
    } catch (const std::exception &e) { if (g->g->ctx) g->g->ctx->err = e.what(); return -1; }
}
int sgpu_graph_write_gfa(const sgpu_graph *g, const char *version, const char *path) {
    if (!g || !path) return SGPU_EINVAL;
    Ctx *c = g->g->ctx;
    API_TRY(c, {
        std::vector<std::string> ch = graph_gfa_chunks(g->g, version ? version : "SPAdes-4.3.0-dev");
        // the pieces go to their offsets of the file concurrently (a 5-25 GB text: one writer is the bottleneck of the whole path)
        const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC, 0644);
        SG_CHECK(fd >= 0, SGPU_EIO, "cannot open GFA file for writing");
        std::vector<uint64_t> off(ch.size() + 1, 0);
        for (size_t i = 0; i < ch.size(); ++i) off[i + 1] = off[i] + ch[i].size();
        std::vector<int> okv(ch.size(), 1);
        par_chunks(ch.size(), (int)std::min<size_t>(ch.size(), 32), [&](int, size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) {
                const char *p = ch[i].data();
                uint64_t left = ch[i].size(), at = off[i];
                while (left) {
                    const ssize_t w = pwrite(fd, p, (size_t)std::min<uint64_t>(left, 1ull << 30), (off_t)at);
                    if (w <= 0) { okv[i] = 0; break; }
                    p += w; at += (uint64_t)w; left -= (uint64_t)w;
                }
                std::string().swap(ch[i]);
            }
        });
        bool ok = close(fd) == 0;
        for (int v : okv) ok = ok && v;
        SG_CHECK(ok, SGPU_EIO, "short write");
    })
}
int sgpu_edge_index_build(sgpu_ctx *ctx, const sgpu_graph *g, int K, int num_buckets, sgpu_edge_index **out) {
    if (!ctx || !g || !out) return SGPU_EINVAL;
    *out = nullptr;
    if (!g->g->ctx) return SGPU_EINVAL;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        EdgeIndex *e = edge_index_build(c, g->g, K, num_buckets);
        *out = new sgpu_edge_index{e};
        child_add(c);
    })
}
int sgpu_edge_index_k(const sgpu_edge_index *e) { return e ? e->e->K : -1; }
int64_t sgpu_edge_index_size(const sgpu_edge_index *e) { return e ? e->e->ks->n : -1; }
int64_t sgpu_edge_index_serialized_size(const sgpu_edge_index *e) { return e ? (int64_t)mphf_serialized_size(e->e->m) : -1; }
int sgpu_edge_index_serialize(const sgpu_edge_index *e, uint8_t *out, int64_t cap) {
    if (!e || !out || cap < 0) return SGPU_EINVAL;
    Ctx *c = e->e->ctx;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        mphf_serialize_to(e->e->m, out, (size_t)cap);
        if (e->e->single_segment) memset(out + mphf_serialized_size(e->e->m) - 8, 0, 8);     // see edge_index.cu: segment_starts_[1] of the single-index branch
    })
}
int sgpu_edge_index_values(const sgpu_edge_index *e, uint64_t *edge_ids, uint32_t *offsets, int64_t n) {
    if (!e || (n && (!edge_ids || !offsets))) return SGPU_EINVAL;
    Ctx *c = e->e->ctx;
    API_TRY(c, {
        SG_CHECK(n == e->e->ks->n, SGPU_EINVAL, "value array size != number of K-mers in the edge index");
        SG_CUDA(cudaSetDevice(c->device));
        if (n) {
            SG_CUDA(cudaMemcpy(edge_ids, e->e->edge_id.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
            SG_CUDA(cudaMemcpy(offsets, e->e->offset.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
        }
    })
}
int sgpu_edge_index_lookup(const sgpu_edge_index *e, const uint64_t *keys, int64_t n, uint64_t *out_idx) {
    if (!e || (n && (!keys || !out_idx))) return SGPU_EINVAL;
    Ctx *c = e->e->ctx;
    API_TRY(c, { SG_CUDA(cudaSetDevice(c->device)); mphf_lookup_host_keys(c, e->e->m, keys, n, out_idx); })
}
void sgpu_edge_index_free(sgpu_edge_index *e) {
    if (!e) return;
    if (e->e) { Ctx *c = e->e->ctx; cudaSetDevice(c->device); delete e->e; child_release(c); }
    delete e;
}
void sgpu_graph_free(sgpu_graph *g) {
    if (!g) return;
    if (g->g && !g->g->ctx) delete g->g;                  // a host-only graph (sgpu_graph_from_edges)
    else if (g->g) { Ctx *c = g->g->ctx; cudaSetDevice(c->device); delete g->g; child_release(c); }
    delete g;
}

}  // extern "C"

struct sgpu_dist { DistState *d; Ctx *c; const sgpu_kset *src; };     // src: the (k+1)-mer set read by sgpu_dist_begin_kpomers
extern "C" {
int sgpu_dist_begin(sgpu_ctx *ctx, int K, int num_buckets, int mode, int world, int rank, sgpu_dist **out) {
    if (!ctx || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        const bool on_host = (mode & SGPU_RESULT_ON_HOST) != 0;
        DistState *d = dist_begin(c, K, num_buckets, mode & ~SGPU_RESULT_ON_HOST, world, rank, on_host);
        *out = new sgpu_dist{d, c, nullptr};
        child_add(c);
    })
}
int sgpu_dist_begin_kpomers(sgpu_ctx *ctx, const sgpu_kset *kpomers, int num_buckets, int mode, int world, int rank, sgpu_dist **out) {
    if (!ctx || !kpomers || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CHECK(mode == 0 || mode == SGPU_RESULT_ON_HOST, SGPU_EINVAL, "bad mode");
        SG_CHECK(!kpomers->free_pending, SGPU_EINVAL, "the (k+1)-mer set has been freed");
        SG_CUDA(cudaSetDevice(c->device));
        DistState *d = dist_begin_kpomers(c, kpomers->s, num_buckets, world, rank, mode == SGPU_RESULT_ON_HOST);
        *out = new sgpu_dist{d, c, kpomers};
        kpomers->readers++;
        child_add(c);
    })
}
int64_t sgpu_dist_num_partitions(const sgpu_dist *d) { return d ? (int64_t)dist_num_partitions(d->d) : -1; }
int sgpu_dist_local_counts(sgpu_dist *d, uint64_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_local_counts(d->d, out); })
}
int sgpu_dist_plan(sgpu_dist *d, const uint64_t *all_counts, uint64_t *total_records) {
    if (!d || !all_counts || !total_records) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_plan(d->d, all_counts, total_records); })
}
int sgpu_dist_free_bytes(sgpu_dist *d, uint64_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); *out = dist_free_bytes(d->d); })
}
int sgpu_dist_next_pass(sgpu_dist *d, uint64_t budget_bytes, int *pass) {
    if (!d || !pass) return SGPU_EINVAL;
    *pass = -1;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); *pass = dist_next_pass(d->d, budget_bytes); })
}
int sgpu_dist_ipc_handle(sgpu_dist *d, uint8_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_ipc_handle(d->d, out); })
}
int sgpu_dist_open_peers(sgpu_dist *d, const uint8_t *handles) {
    if (!d || !handles) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_open_peers(d->d, handles); })
}
int sgpu_dist_scatter(sgpu_dist *d, int pass) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_scatter(d->d, pass); })
}
int sgpu_dist_exchange(sgpu_dist *d, int pass) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_exchange(d->d, pass); })
}
int sgpu_dist_sort(sgpu_dist *d, int pass) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_sort(d->d, pass); })
}
int sgpu_dist_end(sgpu_dist *d, sgpu_kset **out) {
    if (!d || !out) return SGPU_EINVAL;
    *out = nullptr;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); KSet *s = dist_end(d->d); *out = new sgpu_kset{s}; child_add(d->c); })
}
void sgpu_dist_free(sgpu_dist *d) {
    if (!d) return;
    Ctx *c = d->c;
    cudaSetDevice(c->device);
    dist_free(d->d);
    const sgpu_kset *src = d->src;
    delete d;
    child_release(c);
    if (src && --src->readers == 0 && src->free_pending) sgpu_kset_free(const_cast<sgpu_kset *>(src));
}
int sgpu_dist_plan_host(int world, int num_buckets, int key_bits_in_partition, const uint64_t *all_counts, uint64_t budget_bytes, int record_bytes,
                        int *pass_bounds, uint64_t *max_recv) {
    if (world < 1 || num_buckets < 1 || !all_counts || !pass_bounds || !max_recv) return -1;
    try { return dist_plan_host(world, num_buckets, key_bits_in_partition, all_counts, budget_bytes, record_bytes, pass_bounds, max_recv); }
    catch (...) { return -1; }
}
}  // extern "C"

struct sgpu_dist_cov { CovDist *d; Ctx *c; };
extern "C" {
int sgpu_dist_cov_begin(sgpu_ctx *ctx, int K, unsigned threshold, int world, int rank, sgpu_dist_cov **out) {
    if (!ctx || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        CovDist *d = dist_cov_begin(c, K, threshold, world, rank);
        *out = new sgpu_dist_cov{d, c};
        child_add(c);
    })
}
int sgpu_dist_cov_ipc_handle(sgpu_dist_cov *d, uint8_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_cov_ipc_handle(d->d, out); })
}
int sgpu_dist_cov_open_peers(sgpu_dist_cov *d, const uint8_t *descriptors) {
    if (!d || !descriptors) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_cov_open_peers(d->d, descriptors); })
}
int sgpu_dist_cov_bound(sgpu_dist_cov *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_cov_bound(d->d); })
}
int sgpu_dist_cov_fill(sgpu_dist_cov *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_cov_fill(d->d); })
}
int sgpu_dist_cov_filter(sgpu_dist_cov *d, int apply, uint8_t *keep_out, uint64_t *stats) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dist_cov_filter(d->d, apply, keep_out, stats); })
}
void sgpu_dist_cov_free(sgpu_dist_cov *d) {
    if (!d) return;
    Ctx *c = d->c;
    cudaSetDevice(c->device);
    dist_cov_free(d->d);
    delete d;
    child_release(c);
}
int sgpu_dist_cov_layout_host(int world, uint64_t cardinality_bound, const uint64_t *keys, int64_t n, uint32_t *owners, uint64_t *slice_capacity) {
    if (world < 1 || n < 0 || (n && (!keys || !owners)) || !slice_capacity) return SGPU_EINVAL;
    for (int64_t i = 0; i < n; ++i) owners[i] = cov_owner_host(keys[i], world);
    *slice_capacity = cov_slice_capacity(cardinality_bound, world);
    return SGPU_OK;
}
}  // extern "C"

struct sgpu_dist_ext { ExtDist *d; Ctx *c; };
extern "C" {
int sgpu_dist_ext_begin(sgpu_ctx *ctx, const sgpu_kset *kpomers, const sgpu_mphf *kpomer_index, const sgpu_kset *kmers, const sgpu_mphf *kmer_index,
                        const int32_t *owners, int world, int rank, sgpu_dist_ext **out) {
    if (!ctx || !kpomers || !kmers || !kmer_index || !owners || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CHECK(world >= 1 && world <= 255 && rank >= 0 && rank < world, SGPU_EINVAL, "bad world/rank");
        SG_CHECK(!kpomers->free_pending && !kmers->free_pending, SGPU_EINVAL, "a k-mer set has been freed");
        SG_CUDA(cudaSetDevice(c->device));
        ExtDist *d = ext_begin(c, kpomers->s, kpomer_index ? kpomer_index->m : nullptr, kmers->s, kmer_index->m, owners, world, rank);
        *out = new sgpu_dist_ext{d, c};
        child_add(c);
    })
}
int sgpu_dist_ext_local_counts(const sgpu_dist_ext *d, uint64_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, ext_local_counts(d->d, out))
}
int sgpu_dist_ext_plan(sgpu_dist_ext *d, const uint64_t *all_counts, uint64_t *total_records) {
    if (!d || !all_counts || !total_records) return SGPU_EINVAL;
    API_TRY(d->c, ext_plan(d->d, all_counts, total_records))
}
int sgpu_dist_ext_free_bytes(sgpu_dist_ext *d, uint64_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); *out = ext_free_bytes(d->d); })
}
int sgpu_dist_ext_next_pass(sgpu_dist_ext *d, uint64_t budget_bytes, int *pass) {
    if (!d || !pass) return SGPU_EINVAL;
    *pass = -1;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); *pass = ext_next_pass(d->d, budget_bytes); })
}
int sgpu_dist_ext_ipc_handle(sgpu_dist_ext *d, uint8_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); ext_ipc_handle(d->d, out); })
}
int sgpu_dist_ext_open_peers(sgpu_dist_ext *d, const uint8_t *descriptors) {
    if (!d || !descriptors) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); ext_open_peers(d->d, descriptors); })
}
int sgpu_dist_ext_scatter(sgpu_dist_ext *d, int pass) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); ext_scatter(d->d, pass); })
}
int sgpu_dist_ext_apply(sgpu_dist_ext *d, int pass) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); ext_apply(d->d, pass); })
}
int sgpu_dist_ext_masks(const sgpu_dist_ext *d, uint8_t *out, int64_t n) {
    if (!d || (n && !out)) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); ext_masks(d->d, out, n); })
}
int sgpu_dist_ext_coverage(const sgpu_dist_ext *d, uint32_t *out, int64_t n) {
    if (!d || (n && !out)) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); ext_coverage(d->d, out, n); })
}
int64_t sgpu_dist_ext_histogram(const sgpu_dist_ext *d, uint64_t *out, int64_t cap) {
    if (!d) return -1;
    const std::vector<uint64_t> &h = ext_histogram(d->d);
    if (out) for (int64_t i = 0; i < (int64_t)h.size() && i < cap; ++i) out[i] = h[i];
    return (int64_t)h.size();
}
int sgpu_dist_ext_times(const sgpu_dist_ext *d, float *out5) {
    if (!d || !out5) return SGPU_EINVAL;
    ext_times(d->d, out5);
    return SGPU_OK;
}
void sgpu_dist_ext_free(sgpu_dist_ext *d) {
    if (!d) return;
    Ctx *c = d->c;
    cudaSetDevice(c->device);
    ext_free(d->d);
    delete d;
    child_release(c);
}
int sgpu_dist_ext_plan_host(int world, int num_buckets, const int32_t *owners, const uint64_t *all_counts, uint64_t budget_bytes, int record_bytes,
                            int *pass_bounds, uint64_t *max_records) {
    if (world < 1 || num_buckets < 1 || !owners || !all_counts || !pass_bounds || !max_records) return -1;
    try { return ext_plan_host(world, num_buckets, owners, all_counts, budget_bytes, record_bytes, pass_bounds, max_records); }
    catch (...) { return -1; }
}
}  // extern "C"

struct sgpu_dist_graph { DistGraph *d; Ctx *c; };
extern "C" {
int sgpu_dist_graph_begin(sgpu_ctx *ctx, const sgpu_dist_ext *ext, const int32_t *kmer_owners, const int32_t *kpomer_owners,
                          const uint64_t *kmer_bucket_sizes, uint64_t budget_bytes, sgpu_dist_graph **out) {
    const sgpu_graph_options o = {1, 0, 0, 0.8, 10, 200};
    return sgpu_dist_graph_begin_opts(ctx, ext, kmer_owners, kpomer_owners, kmer_bucket_sizes, budget_bytes, &o, out);
}
int sgpu_dist_graph_begin_opts(sgpu_ctx *ctx, const sgpu_dist_ext *ext, const int32_t *kmer_owners, const int32_t *kpomer_owners,
                               const uint64_t *kmer_bucket_sizes, uint64_t budget_bytes, const sgpu_graph_options *o, sgpu_dist_graph **out) {
    if (!ctx || !ext || !kmer_owners || !kmer_bucket_sizes || !o || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        const GraphOptions opt = graph_options(o);
        SG_CUDA(cudaSetDevice(c->device));
        DistGraph *d = dgraph_begin(c, ext->d, kmer_owners, kpomer_owners, kmer_bucket_sizes, budget_bytes, opt);
        *out = new sgpu_dist_graph{d, c};
        child_add(c);
    })
}
int sgpu_dist_graph_ipc_handle(sgpu_dist_graph *d, uint8_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_ipc_handle(d->d, out); })
}
int sgpu_dist_graph_open_peers(sgpu_dist_graph *d, const uint8_t *descriptors) {
    if (!d || !descriptors) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_open_peers(d->d, descriptors); })
}
static int dist_graph_phase(sgpu_dist_graph *d, int a, int b) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_clip_phase(d->d, a, b); })
}
int sgpu_dist_graph_at_edges_probe(sgpu_dist_graph *d) { return dist_graph_phase(d, kAtEdgesProbe, kAtEdgesProbe); }
int sgpu_dist_graph_at_edges_apply(sgpu_dist_graph *d) { return dist_graph_phase(d, kAtEdgesApply, kAtEdgesApply); }
int sgpu_dist_graph_at_tips_probe(sgpu_dist_graph *d) { return dist_graph_phase(d, kAtTipsProbe, kAtTipsProbe); }
int sgpu_dist_graph_tip_probe(sgpu_dist_graph *d) { return dist_graph_phase(d, kTipProbe, kTipProbe); }
int sgpu_dist_graph_isolate(sgpu_dist_graph *d) { return dist_graph_phase(d, kAtIsolate, kTipIsolate); }
int sgpu_dist_graph_unlink(sgpu_dist_graph *d) { return dist_graph_phase(d, kAtUnlink, kTipUnlink); }
int sgpu_dist_graph_junctions(sgpu_dist_graph *d) { return dist_graph_phase(d, kJunctions, kJunctions); }
int sgpu_dist_graph_masks(const sgpu_dist_graph *d, uint8_t *out, int64_t n) {
    if (!d || n < 0 || (n && !out)) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_masks(d->d, out, n); })
}
int sgpu_dist_graph_clipper_stats(const sgpu_dist_graph *d, uint64_t *at4, uint64_t *tc3, uint64_t *remote3) {
    if (!d || !at4 || !tc3 || !remote3) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_clip_stats(d->d, at4, tc3, remote3); })
}
int sgpu_dist_graph_clipper_times(const sgpu_dist_graph *d, float *out6) {
    if (!d || !out6) return SGPU_EINVAL;
    dgraph_clip_times(d->d, out6);
    return SGPU_OK;
}
int sgpu_dist_graph_unitigs(sgpu_dist_graph *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_unitigs(d->d); })
}
int sgpu_dist_graph_clear_visited(sgpu_dist_graph *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_clear_visited(d->d); })
}
int sgpu_dist_graph_loops(sgpu_dist_graph *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dgraph_loops(d->d); })
}
int sgpu_dist_graph_stats(const sgpu_dist_graph *d, uint64_t *out4) {
    if (!d || !out4) return SGPU_EINVAL;
    dgraph_stats(d->d, out4);
    return SGPU_OK;
}
int sgpu_dist_graph_edges(const sgpu_dist_graph *d, char *seq, uint32_t *lens, uint64_t *link_start, uint64_t *link_end, uint32_t *raw_cov) {
    if (!d) return SGPU_EINVAL;
    const Graph &g = dgraph_edges(d->d);
    const size_t n = g.edge_len.size();
    if ((n && (!lens || !link_start || !link_end || !raw_cov)) || (!g.seq.empty() && !seq)) return SGPU_EINVAL;
    if (!g.seq.empty()) memcpy(seq, g.seq.data(), g.seq.size());
    if (n) {
        memcpy(lens, g.edge_len.data(), n * 4);
        memcpy(link_start, g.link_start.data(), n * 8);
        memcpy(link_end, g.link_end.data(), n * 8);
        memcpy(raw_cov, g.raw_cov.data(), n * 4);
    }
    return SGPU_OK;
}
int sgpu_dist_graph_bucket_counts(const sgpu_dist_graph *d, uint64_t *unitig_counts, uint64_t *loop_counts) {
    if (!d || !unitig_counts || !loop_counts) return SGPU_EINVAL;
    dgraph_bucket_counts(d->d, unitig_counts, loop_counts);
    return SGPU_OK;
}
int sgpu_dist_graph_times(const sgpu_dist_graph *d, float *out4) {
    if (!d || !out4) return SGPU_EINVAL;
    dgraph_times(d->d, out4);
    return SGPU_OK;
}
void sgpu_dist_graph_free(sgpu_dist_graph *d) {
    if (!d) return;
    Ctx *c = d->c;
    cudaSetDevice(c->device);
    dgraph_free(d->d);
    delete d;
    child_release(c);
}
int sgpu_graph_from_edges(int k, const char *seq, int64_t nbases, const uint32_t *lens, const uint64_t *link_start, const uint64_t *link_end,
                          const uint32_t *raw_cov, int64_t n, sgpu_graph **out) {
    if (!out) return SGPU_EINVAL;
    *out = nullptr;
    if (k < 1 || k > 127 || n < 0 || nbases < 0 || (nbases && !seq) || (n && (!lens || !link_start || !link_end || !raw_cov))) return SGPU_EINVAL;
    uint64_t at = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (lens[i] < (uint32_t)k + 1) return SGPU_EINVAL;                // an edge holds at least one (k+1)-mer
        at += lens[i];
        if (at > (uint64_t)nbases) return SGPU_EINVAL;                    // an edge reaching past the text
    }
    if (at != (uint64_t)nbases) return SGPU_EINVAL;                      // text and lengths disagree
    try {
        Graph *g = new Graph();
        g->k = k;
        g->seq.assign(seq ? seq : "", (size_t)nbases);
        g->edge_len.assign(lens, lens + n);
        g->edge_off.resize((size_t)n);
        for (int64_t i = 0, o = 0; i < n; o += lens[i++]) g->edge_off[i] = (uint64_t)o;
        g->link_start.assign(link_start, link_start + n);
        g->link_end.assign(link_end, link_end + n);
        g->raw_cov.assign(raw_cov, raw_cov + n);
        *out = new sgpu_graph{g};
    } catch (const std::bad_alloc &) { return SGPU_ENOMEM; }
    return SGPU_OK;
}
}  // extern "C"

// ---- self test of kmer_dev.cuh on host and device -----------------------------------------------------------------------
template <int NW>
__host__ __device__ uint64_t selftest_one(int op, int K, uint64_t arg, const uint64_t *key) {
    Kmer<NW> k;
    for (int q = 0; q < NW; ++q) k.w[q] = key[q];
    switch (op) {
        case 0: return xxh3_64<NW>(k);
        case 1: return xxh3_128<NW>(k).lo;
        case 2: return xxh3_128<NW>(k).hi;
        case 3: return kmer_bucket<NW>(k, (uint32_t)arg);
        case 4: return kmer_is_minimal<NW>(k, kmer_rc<NW>(k, K)) ? 1 : 0;
        case 9: return key_bits<NW>(k, K, (int)(arg >> 8), (int)(arg & 255));
        default: {
            int j = op - 5;
            Kmer<NW> r = kmer_rc<NW>(k, K);
            return j < NW ? r.w[j] : 0;
        }
    }
}
// op 10: the rolling window of the level-A kernels against direct extraction. keys = one packed sequence of n*NW words,
// arg = (C << 32) | its length in bases, C = windows per chunk (24 canonical, 12 all-windows; 0 = 24); unit u walks windows
// [C u, C u + C). out[u] = (windows walked << 32) | mismatches.
template <int NW>
__host__ __device__ uint64_t selftest_roll_unit(int K, int L, int C, const uint64_t *seq, int64_t u) {
    const int nwin = L - K + 1;
    const int64_t j0 = u * C;
    if (j0 >= nwin) return 0;
    const int cnt = nwin - j0 < C ? (int)(nwin - j0) : C;
    RollState<NW> st;
    roll_init<NW>(st, seq, (int)j0, K, cnt);
    uint64_t bad = 0;
    for (int s = 0; s < cnt; ++s) {
        if (s) roll_next<NW>(st, K);
        const Kmer<NW> f = kmer_window<NW>(seq, j0 + s, K);
        const Kmer<NW> r = kmer_rc<NW>(f, K);
        if (!kmer_eq<NW>(f, st.f) || !kmer_eq<NW>(r, st.r)) ++bad;
    }
    return ((uint64_t)cnt << 32) | bad;
}
template <int NW>
__global__ void selftest_roll_k(int K, int L, int C, const uint64_t *seq, int64_t n, uint64_t *out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = selftest_roll_unit<NW>(K, L, C, seq, i);
}
template <int NW>
__global__ void selftest_k(int op, int K, uint64_t arg, const uint64_t *keys, int64_t n, uint64_t *out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = selftest_one<NW>(op, K, arg, keys + i * NW);
}
template <int NW>
static void selftest_nw(Ctx *c, int on_device, int op, int K, uint64_t arg, const uint64_t *keys, int64_t n, uint64_t *out) {
    const int64_t L = (int64_t)(uint32_t)arg, C = (arg >> 32) ? (int64_t)(arg >> 32) : 24;
    if (op == 10) SG_CHECK(L >= K && L <= 32 * n * NW && C >= 1 && C <= 33, SGPU_EINVAL, "roll self test: bad sequence length or chunk width");
    if (!on_device) {
        for (int64_t i = 0; i < n; ++i) out[i] = op == 10 ? selftest_roll_unit<NW>(K, (int)L, (int)C, keys, i) : selftest_one<NW>(op, K, arg, keys + i * NW);
        return;
    }
    SG_CHECK(c, SGPU_EINVAL, "device self test needs a context");
    DArr<uint64_t> dk(c, (size_t)n * NW), dout(c, (size_t)n);
    SG_CUDA(cudaMemcpyAsync(dk.p, keys, (size_t)n * NW * 8, cudaMemcpyHostToDevice, c->stream));
    if (op == 10) selftest_roll_k<NW><<<div_up(n, 256), 256, 0, c->stream>>>(K, (int)L, (int)C, dk.p, n, dout.p);
    else selftest_k<NW><<<div_up(n, 256), 256, 0, c->stream>>>(op, K, arg, dk.p, n, dout.p);
    c->launches++;
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(out, dout.p, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
    SG_CUDA(cudaStreamSynchronize(c->stream));
}
extern "C" int sgpu_selftest(sgpu_ctx *ctx, int on_device, int op, int K, uint64_t arg, const uint64_t *keys, int64_t n, uint64_t *out) {
    if (K < 1 || K > 128 || n < 0 || (n && (!keys || !out))) return SGPU_EINVAL;
    Ctx *c = ctx ? &ctx->c : nullptr;
    if (on_device && !c) return SGPU_EINVAL;
    API_TRY(c, {
        if (on_device) SG_CUDA(cudaSetDevice(c->device));
        switch (nwords_of(K)) {
            case 1: selftest_nw<1>(c, on_device, op, K, arg, keys, n, out); break;
            case 2: selftest_nw<2>(c, on_device, op, K, arg, keys, n, out); break;
            case 3: selftest_nw<3>(c, on_device, op, K, arg, keys, n, out); break;
            default: selftest_nw<4>(c, on_device, op, K, arg, keys, n, out); break;
        }
    })
}

struct sgpu_dist_edge_index { DistEdgeIndex *d; Ctx *c; };
extern "C" {
int sgpu_dist_edge_index_begin(sgpu_ctx *ctx, const sgpu_dist_graph *dg, int K, int num_buckets, const uint64_t *unitig_counts_all,
                               const uint64_t *loop_counts_all, sgpu_dist_edge_index **out) {
    if (!ctx || !dg || !unitig_counts_all || !loop_counts_all || !out) return SGPU_EINVAL;
    *out = nullptr;
    Ctx *c = &ctx->c;
    API_TRY(c, {
        SG_CUDA(cudaSetDevice(c->device));
        DistEdgeIndex *d = dei_begin(c, dg->d, K, num_buckets, unitig_counts_all, loop_counts_all);
        *out = new sgpu_dist_edge_index{d, c};
        child_add(c);
    })
}
int sgpu_dist_edge_index_count_begin(sgpu_dist_edge_index *d, int world, int rank, sgpu_dist **out) {
    if (!d || !out) return SGPU_EINVAL;
    *out = nullptr;
    API_TRY(d->c, {
        SG_CUDA(cudaSetDevice(d->c->device));
        DistState *s = dei_count_begin(d->d, world, rank);
        *out = new sgpu_dist{s, d->c, nullptr};
        child_add(d->c);
    })
}
int sgpu_dist_edge_index_keys(sgpu_dist_edge_index *d, const sgpu_kset *keys, const uint64_t *union_bucket_sizes, int single) {
    if (!d || !keys || !union_bucket_sizes) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_keys(d->d, keys->s, union_bucket_sizes, single); })
}
int sgpu_dist_edge_index_ipc_handle(sgpu_dist_edge_index *d, uint8_t *out) {
    if (!d || !out) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_ipc_handle(d->d, out); })
}
int sgpu_dist_edge_index_open_peers(sgpu_dist_edge_index *d, const uint8_t *descriptors) {
    if (!d || !descriptors) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_open_peers(d->d, descriptors); })
}
int sgpu_dist_edge_index_merge(sgpu_dist_edge_index *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_merge(d->d); })
}
int sgpu_dist_edge_index_advance(sgpu_dist_edge_index *d, uint64_t *live) {
    if (!d || !live) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); *live = dei_advance(d->d); })
}
int sgpu_dist_edge_index_level_done(sgpu_dist_edge_index *d, uint64_t union_live, int *more) {
    if (!d || !more) return SGPU_EINVAL;
    API_TRY(d->c, { *more = dei_level_done(d->d, union_live); })
}
int sgpu_dist_edge_index_ranks(sgpu_dist_edge_index *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_ranks(d->d); })
}
int sgpu_dist_edge_index_fill(sgpu_dist_edge_index *d) {
    if (!d) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_fill(d->d); })
}
int sgpu_dist_edge_index_values(const sgpu_dist_edge_index *d, uint64_t *edge_ids, uint32_t *offsets, int64_t n) {
    if (!d || n < 0 || (n && (!edge_ids || !offsets))) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); dei_values(d->d, edge_ids, offsets, n); })
}
int sgpu_dist_edge_index_k(const sgpu_dist_edge_index *d) { return d ? dei_k(d->d) : -1; }
int64_t sgpu_dist_edge_index_size(const sgpu_dist_edge_index *d) {
    if (!d) return -1;
    try { return dei_index(d->d)->n; } catch (const sg::Error &e) { d->c->err = e.what(); return -1; }
}
int sgpu_dist_edge_index_slot_range(const sgpu_dist_edge_index *d, int64_t *lo, int64_t *hi) {
    if (!d || !lo || !hi) return SGPU_EINVAL;
    API_TRY(d->c, {
        uint64_t a = 0, b = 0;
        dei_slot_range(d->d, &a, &b);
        *lo = (int64_t)a; *hi = (int64_t)b;
    })
}
int64_t sgpu_dist_edge_index_serialized_size(const sgpu_dist_edge_index *d) {
    if (!d) return -1;
    try { return (int64_t)mphf_serialized_size(dei_index(d->d)); } catch (const sg::Error &e) { d->c->err = e.what(); return -1; }
}
int sgpu_dist_edge_index_serialize(const sgpu_dist_edge_index *d, uint8_t *out, int64_t cap) {
    if (!d || !out || cap < 0) return SGPU_EINVAL;
    API_TRY(d->c, {
        SG_CUDA(cudaSetDevice(d->c->device));
        const Mphf *m = dei_index(d->d);
        mphf_serialize_to(m, out, (size_t)cap);
        if (dei_single(d->d)) memset(out + mphf_serialized_size(m) - 8, 0, 8);     // segment_starts_[1] of the single-index branch, as sgpu_edge_index_serialize
    })
}
int sgpu_dist_edge_index_lookup(const sgpu_dist_edge_index *d, const uint64_t *keys, int64_t n, uint64_t *out_idx) {
    if (!d || n < 0 || (n && (!keys || !out_idx))) return SGPU_EINVAL;
    API_TRY(d->c, { SG_CUDA(cudaSetDevice(d->c->device)); mphf_lookup_host_keys(d->c, dei_index(d->d), keys, n, out_idx); })
}
int sgpu_dist_edge_index_times(const sgpu_dist_edge_index *d, float *out6) {
    if (!d || !out6) return SGPU_EINVAL;
    dei_times(d->d, out6);
    return SGPU_OK;
}
void sgpu_dist_edge_index_free(sgpu_dist_edge_index *d) {
    if (!d) return;
    Ctx *c = d->c;
    cudaSetDevice(c->device);
    dei_free(d->d);
    delete d;
    child_release(c);
}
int sgpu_dist_edge_numbers_host(int world, int rank, int num_buckets, const int32_t *owners, const uint64_t *unitig_counts_all,
                                const uint64_t *loop_counts_all, uint64_t unitig_edges, uint64_t edges, uint64_t *out) {
    if (!owners || !unitig_counts_all || !loop_counts_all || (edges && !out)) return SGPU_EINVAL;
    try { dist_edge_numbers(world, rank, num_buckets, owners, unitig_counts_all, loop_counts_all, unitig_edges, edges, out); }
    catch (const sg::Error &e) { return e.code; }
    return SGPU_OK;
}
int64_t sgpu_edge_index_vertex_prefix_host(const uint64_t *link_start, const uint64_t *link_end, int64_t n, int num_buckets, uint64_t *out) {
    if (n < 0 || num_buckets < 1 || (n && (!link_start || !link_end)) || !out) return -1;
    try {
        Graph g;
        g.link_start.assign(link_start, link_start + n);
        g.link_end.assign(link_end, link_end + n);
        g.edge_len.assign((size_t)n, 0);
        const std::vector<uint64_t> v = edge_vertex_slots(&g, ((uint64_t)num_buckets + 1) / 2);
        std::copy(v.begin(), v.end(), out);
        return (int64_t)v.size();
    } catch (...) { return -1; }
}
int sgpu_dist_slot_range_host(uint64_t n, int world, int rank, uint64_t *lo, uint64_t *hi) {
    if (world < 1 || rank < 0 || rank >= world || !lo || !hi) return SGPU_EINVAL;
    *lo = dist_slot_lo(n, world, rank); *hi = dist_slot_lo(n, world, rank + 1);
    return SGPU_OK;
}
}  // extern "C"
