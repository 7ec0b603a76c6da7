// mphf.cu -- boomphf-compatible minimal perfect hash, built on the GPU. Replaces
//   KMerIndexBuilder::BuildIndex              (src/common/kmer_index/kmer_mph/kmer_index_builder.hpp:448-498)
//   boomphf::mphf::build / processLevel / ...  (ext/include/boomphf/BooPHF.h:382-755)
//   KMerIndex::serialize / seq_idx             (src/common/kmer_index/kmer_mph/kmer_index.hpp:88-108)
// and produces byte-identical KMerIndex::serialize output.
//
// Why a parallel build is bit-identical: a level's bitset bit is 1 iff exactly one still-unplaced key hashed to
// it (BooPHF.h:633-639 set + :219-229 clearCollisions), which does not depend on insertion order. Level sizes
// come from host libm pow() exactly as BooPHF.h:586-595. Only the level-24 fallback map (:659-678) is order
// dependent; with gamma=4 it is empty in practice (p^24 ~ 2e-16 per key) and a non-empty one is reported as an
// error instead of being emulated.
//
// HBM layout: bitsets are stored LEVEL-MAJOR (all buckets' level 0, then level 1, ...), each (level,bucket)
// piece padded to a multiple of 8 words = one 512-bit rank block, so that one level is one contiguous range
// for the insert / clear kernels and ranks are one u64 per block.
#include <math.h>

#include <algorithm>

#include "mphf_dev.cuh"

namespace sg {

// insert the alive keys of this level (BooPHF.h:633-639); coll is indexed relative to the level start
template <int NW>
__global__ void mphf_insert_k(KeyTable t, const uint64_t *__restrict__ alive, uint64_t n, int level, MphfDev m, uint64_t level_start,
                              uint64_t *__restrict__ coll) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t ki = alive ? (int64_t)alive[i] : (int64_t)i;
    Kmer<NW> k = table_key<NW>(t, ki);
    const uint32_t b = kmer_bucket<NW>(k, m.B);
    uint64_t w;
    const uint64_t pos = level_pos<NW>(m, k, b, level, &w);
    const unsigned long long bit = 1ull << (pos & 63);
    unsigned long long old = atomicOr((unsigned long long *)&m.bits[w], bit);
    if (old & bit) atomicOr((unsigned long long *)&coll[w - level_start], bit);
}

__global__ void mphf_clear_k(uint64_t *__restrict__ bits, uint64_t *__restrict__ coll, uint64_t nwords) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nwords) return;
    uint64_t c = coll[i];
    if (c) { bits[i] &= ~c; coll[i] = 0; }
}

// keys whose bit was cleared stay alive for the next level
template <int NW>
__global__ void mphf_filter_k(KeyTable t, const uint64_t *__restrict__ alive, uint64_t n, int level, MphfDev m, uint64_t *__restrict__ next,
                              uint64_t cap, unsigned long long *__restrict__ next_n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool keep = false;
    int64_t ki = 0;
    if (i < n) {
        ki = alive ? (int64_t)alive[i] : (int64_t)i;
        Kmer<NW> k = table_key<NW>(t, ki);
        const uint32_t b = kmer_bucket<NW>(k, m.B);
        uint64_t w;
        const uint64_t pos = level_pos<NW>(m, k, b, level, &w);
        keep = !((m.bits[w] >> (pos & 63)) & 1ull);
    }
    // block-aggregated append: one global atomic per CTA (a per-warp atomic on the single counter serialises in L2)
    __shared__ unsigned s_warp[8];
    __shared__ unsigned long long s_base;
    const unsigned mask = __ballot_sync(0xffffffffu, keep);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(mask);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned tot = 0;
        for (int w = 0; w < 8; ++w) { unsigned c = s_warp[w]; s_warp[w] = tot; tot += c; }
        s_base = tot ? atomicAdd(next_n, (unsigned long long)tot) : 0ull;
    }
    __syncthreads();
    if (keep) {
        const uint64_t slot = s_base + s_warp[warp] + __popc(mask & ((1u << lane) - 1));
        if (slot < cap) next[slot] = (uint64_t)ki;
    }
}

// fused filter(level) + insert(level+1): a key whose level bit was cleared (it collided) survives; it is appended to the next
// alive list and, in the same thread, inserted into the next level's bitset (BooPHF.h:616-639 getLevel + insertIntoLevel)
template <int NW>
__global__ void mphf_advance_k(KeyTable t, const uint64_t *__restrict__ alive, uint64_t n, int level, MphfDev m, uint64_t *__restrict__ next,
                               uint64_t cap, unsigned long long *__restrict__ next_n, int do_insert, uint64_t next_level_start,
                               uint64_t *__restrict__ coll) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool keep = false;
    int64_t ki = 0;
    if (i < n) {
        ki = alive ? (int64_t)alive[i] : (int64_t)i;
        Kmer<NW> k = table_key<NW>(t, ki);
        const uint32_t b = kmer_bucket<NW>(k, m.B);
        LevelHasher lh(xxh3_128<NW>(k));
        uint64_t h = 0;
        for (int l = 0; l <= level; ++l) h = lh.next();
        size_t p = (size_t)level * m.B + b;
        uint64_t pos = mulhi64(h, m.dom[p]);
        keep = !((m.bits[m.woff[p] + (pos >> 6)] >> (pos & 63)) & 1ull);
        if (keep && do_insert) {
            h = lh.next();
            p += m.B;
            pos = mulhi64(h, m.dom[p]);
            const uint64_t w = m.woff[p] + (pos >> 6);
            const unsigned long long bit = 1ull << (pos & 63);
            unsigned long long old = atomicOr((unsigned long long *)&m.bits[w], bit);
            if (old & bit) atomicOr((unsigned long long *)&coll[w - next_level_start], bit);
        }
    }
    // block-aggregated append: one global atomic per CTA (a per-warp atomic on the single counter serialises in L2)
    __shared__ unsigned s_warp[8];
    __shared__ unsigned long long s_base;
    const unsigned mask = __ballot_sync(0xffffffffu, keep);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(mask);
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned tot = 0;
        for (int w = 0; w < 8; ++w) { unsigned c = s_warp[w]; s_warp[w] = tot; tot += c; }
        s_base = tot ? atomicAdd(next_n, (unsigned long long)tot) : 0ull;
    }
    __syncthreads();
    if (keep) {
        const uint64_t slot = s_base + s_warp[warp] + __popc(mask & ((1u << lane) - 1));
        if (slot < cap) next[slot] = (uint64_t)ki;
    }
}

__global__ void mphf_blockpop_k(const uint64_t *__restrict__ bits, uint64_t nblocks, uint32_t *__restrict__ pop) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nblocks) return;
    const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(bits + i * 8);
    uint32_t s = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) { ulonglong2 v = p[q]; s += __popcll(v.x) + __popcll(v.y); }
    pop[i] = s;
}

// base rank of each (level,bucket) piece = popcount of the bucket's earlier levels (bitVector::build_ranks offset chaining,
// BooPHF.h:431-434)
__global__ void mphf_piecebase_k(const uint64_t *__restrict__ gscan, const uint64_t *__restrict__ woff, uint32_t B, uint64_t total_blocks,
                                 uint64_t *__restrict__ piece_base, uint64_t *__restrict__ lastrank) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    uint64_t run = 0;
    for (int l = 0; l < kLevels; ++l) {
        const size_t p = (size_t)l * B + b;
        const uint64_t blk0 = woff[p] >> 3;
        const uint64_t blk1 = (p + 1 < (size_t)kLevels * B) ? (woff[p + 1] >> 3) : total_blocks;
        piece_base[p] = run;
        run += gscan[blk1] - gscan[blk0];
    }
    lastrank[b] = run;
}
__global__ void mphf_ranks_k(const uint64_t *__restrict__ gscan, const uint64_t *__restrict__ woff, const uint64_t *__restrict__ piece_base,
                             uint32_t npieces, uint64_t nblocks, uint64_t *__restrict__ ranks) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nblocks) return;
    // piece containing block i: largest p with (woff[p]>>3) <= i
    uint32_t lo = 0, hi = npieces - 1;
    while (lo < hi) {
        uint32_t mid = (lo + hi + 1) >> 1;
        if ((woff[mid] >> 3) <= i) lo = mid; else hi = mid - 1;
    }
    ranks[i] = piece_base[lo] + gscan[i] - gscan[woff[lo] >> 3];
}

template <int NW>
__global__ void mphf_lookup_k(MphfDev m, const uint64_t *__restrict__ keys, uint64_t n, uint64_t *__restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Kmer<NW> k;
#pragma unroll
    for (int q = 0; q < NW; ++q) k.w[q] = keys[i * NW + q];
    out[i] = mphf_lookup_dev<NW>(m, k);
}

MphfDev mphf_dev(const Mphf *m) {
    MphfDev d;
    d.dom = m->d_dom.p; d.woff = m->d_woff.p; d.starts = m->d_starts.p; d.bits = m->bits.p; d.ranks = m->ranks.p; d.B = (uint32_t)m->B;
    return d;
}

std::vector<uint64_t> mphf_geometry(Ctx *ctx, Mphf *m, const std::vector<int64_t> &bsz) {
    cudaStream_t st = ctx->stream;
    const int B = m->B;
    // ---- level geometry on the host, same libm as the reference (BooPHF.h:582-595)
    m->dom.assign((size_t)kLevels * B, 0); m->nchar.assign((size_t)kLevels * B, 0); m->woff.assign((size_t)kLevels * B + 1, 0);
    std::vector<uint64_t> level_start(kLevels + 1, 0);
    {
        uint64_t off = 0;
        std::vector<double> pcol(B);
        std::vector<uint64_t> hd(B);
        for (int b = 0; b < B; ++b) {
            uint64_t nb = (uint64_t)bsz[b];
            double gamma = 4.0;
            hd[b] = (uint64_t)ceil((double)nb * gamma);
            pcol[b] = nb ? 1.0 - pow(((gamma * (double)nb - 1) / (gamma * (double)nb)), (double)(nb - 1)) : 0.0;
        }
        for (int l = 0; l < kLevels; ++l) {
            level_start[l] = off;
            for (int b = 0; b < B; ++b) {
                const size_t p = (size_t)l * B + b;
                m->woff[p] = off;
                if (bsz[b] == 0) { m->dom[p] = 64; m->nchar[p] = 0; continue; }   // empty buckets own no words
                uint64_t d = (((uint64_t)((double)hd[b] * pow(pcol[b], l)) + 63) / 64) * 64;
                if (d == 0) d = 64;
                m->dom[p] = d;
                m->nchar[p] = 1 + d / 64;
                off += ((m->nchar[p] + 7) / 8) * 8;
            }
        }
        level_start[kLevels] = off;
        m->woff[(size_t)kLevels * B] = off;
        m->total_words = off;
    }
    m->starts.assign(B + 1, 0);
    for (int b = 0; b < B; ++b) m->starts[b + 1] = (uint64_t)bsz[b];
    for (int i = 1; i < B; ++i) m->starts[i] += m->starts[i - 1];            // kmer_index_builder.hpp:492-493 (stops before B)
    m->bsz = bsz;
    m->lastrank.assign(B, 0);
    const uint64_t total_words = m->total_words;
    const uint64_t nblocks = total_words / 8;
    m->bits.alloc(ctx, total_words + 8, true);
    m->ranks.alloc(ctx, nblocks + 1, true);
    m->d_dom.alloc(ctx, m->dom.size(), true); m->d_woff.alloc(ctx, m->woff.size(), true); m->d_starts.alloc(ctx, m->starts.size(), true);
    SG_CUDA(cudaMemsetAsync(m->bits.p, 0, m->bits.bytes(), st));
    SG_CUDA(cudaMemcpyAsync(m->d_dom.p, m->dom.data(), m->dom.size() * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(m->d_woff.p, m->woff.data(), m->woff.size() * 8, cudaMemcpyHostToDevice, st));
    SG_CUDA(cudaMemcpyAsync(m->d_starts.p, m->starts.data(), m->starts.size() * 8, cudaMemcpyHostToDevice, st));
    return level_start;
}

void mphf_ranks(Ctx *ctx, Mphf *m) {
    cudaStream_t st = ctx->stream;
    const int B = m->B;
    const uint64_t nblocks = m->total_words / 8;
    DArr<uint32_t> pop(ctx, nblocks + 1);
    DArr<uint64_t> gscan(ctx, nblocks + 1), piece_base(ctx, (size_t)kLevels * B), d_last(ctx, B);
    SG_CUDA(cudaMemsetAsync(pop.p + nblocks, 0, 4, st));
    mphf_blockpop_k<<<div_up((int64_t)nblocks, 256), 256, 0, st>>>(m->bits.p, nblocks, pop.p);
    ctx->launches++;
    exclusive_scan_u32_to_u64(ctx, pop.p, gscan.p, nblocks + 1);
    mphf_piecebase_k<<<div_up(B, 128), 128, 0, st>>>(gscan.p, m->d_woff.p, (uint32_t)B, nblocks, piece_base.p, d_last.p);
    mphf_ranks_k<<<div_up((int64_t)nblocks, 256), 256, 0, st>>>(gscan.p, m->d_woff.p, piece_base.p, (uint32_t)(kLevels * B), nblocks, m->ranks.p);
    ctx->launches += 2;
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(m->lastrank.data(), d_last.p, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b) SG_CHECK(m->lastrank[b] == (uint64_t)m->bsz[b], 6, "internal: MPHF is not minimal (rank total != bucket size)");
}

template <int NW>
static void build_nw(Ctx *ctx, const KSet *ks, Mphf *m) {
    cudaStream_t st = ctx->stream;
    const int B = ks->B;
    const uint64_t n = (uint64_t)ks->n;
    const std::vector<uint64_t> level_start = mphf_geometry(ctx, m, ks->bsz);
    if (n == 0 || m->total_words == 0) { SG_CUDA(cudaStreamSynchronize(st)); return; }

    MphfDev md = mphf_dev(m);
    const uint64_t l0_words = level_start[1] - level_start[0];
    DArr<uint64_t> coll(ctx, l0_words + 8);
    SG_CUDA(cudaMemsetAsync(coll.p, 0, coll.bytes(), st));
    DArr<unsigned long long> d_cnt(ctx, 1);
    DArr<uint64_t> aliveA, aliveB;
    // places the n keys of table t, all of buckets [b_lo, b_hi), in every level. A key touches only its own bucket's pieces, so
    // a level's collisions are cleared over the words of those buckets alone, and the bits do not depend on how the set is split.
    // Level 0 takes every key; afterwards one fused kernel per level tests the previous level's bit and inserts the survivors
    // into the next level right away (one key load + one XXH3-128 per key and level instead of two)
    auto place = [&](const KeyTable &t, uint64_t n, int b_lo, int b_hi) {
        auto clear = [&](int l) {
            const uint64_t w0 = m->woff[(size_t)l * B + b_lo], nw = m->woff[(size_t)l * B + b_hi] - w0;
            mphf_clear_k<<<div_up((int64_t)nw, 256), 256, 0, st>>>(m->bits.p + w0, coll.p + (w0 - level_start[l]), nw);
            ctx->launches++;
        };
        const uint64_t *alive = nullptr;
        uint64_t n_alive = n;
        mphf_insert_k<NW><<<div_up((int64_t)n_alive, 256), 256, 0, st>>>(t, alive, n_alive, 0, md, level_start[0], coll.p);
        ctx->launches++;
        clear(0);
        for (int l = 0; l < kLevels - 1 && n_alive; ++l) {
            const bool last = (l == kLevels - 2);              // level 23 has no successor bitset: only count what is left
            DArr<uint64_t> &next = (l & 1) ? aliveA : aliveB;
            uint64_t cap = (l == 0) ? n_alive / 2 + 1024 : n_alive;
            if (next.n < cap) next.alloc(ctx, cap);
            SG_CUDA(cudaMemsetAsync(d_cnt.p, 0, 8, st));
            mphf_advance_k<NW><<<div_up((int64_t)n_alive, 256), 256, 0, st>>>(t, alive, n_alive, l, md, next.p, (uint64_t)next.n, d_cnt.p,
                                                                             last ? 0 : 1, last ? 0 : level_start[l + 1], coll.p);
            ctx->launches++;
            if (!last) clear(l + 1);
            SG_CUDA(cudaGetLastError());
            unsigned long long c = 0;
            SG_CUDA(cudaMemcpyAsync(&c, d_cnt.p, 8, cudaMemcpyDeviceToHost, st));
            SG_CUDA(cudaStreamSynchronize(st));
            SG_CHECK(c <= next.n, 6, "internal: MPHF survivor list overflow");
            alive = next.p;
            n_alive = c;
        }
        SG_CHECK(n_alive == 0, 7, "MPHF: keys fell through all 24 bitset levels (reference would use its order-dependent fallback map); unsupported");
    };
    if (!ks->on_host) {
        place(make_table(ks), n, 0, B);
    } else {
        // a host set is placed chunk by chunk (a chunk is a contiguous bucket range), each chunk uploaded while the one before is placed
        ChunkStager stage(ks, false);
        stage.sweep([&](const Chunk &ch, const uint64_t *keys, const uint32_t *) {
            KeyTable t;
            t.nchunks = 1; t.first[0] = 0; t.first[1] = ch.n; t.keys[0] = keys;
            place(t, (uint64_t)ch.n, ch.b_lo, ch.b_hi);
        });
    }
    mphf_ranks(ctx, m);
}

Mphf *mphf_build(Ctx *ctx, const KSet *ks) {
    Mphf *m = new Mphf();
    m->ctx = ctx; m->K = ks->K; m->nw = ks->nw; m->B = ks->B; m->n = ks->n;
    ctx->times.stage_h2d_bytes = 0;
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a, ctx->stream);
    try {
        switch (ks->nw) {
            case 1: build_nw<1>(ctx, ks, m); break;
            case 2: build_nw<2>(ctx, ks, m); break;
            case 3: build_nw<3>(ctx, ks, m); break;
            default: build_nw<4>(ctx, ks, m); break;
        }
    } catch (...) { cudaEventDestroy(a); cudaEventDestroy(b); delete m; throw; }
    cudaEventRecord(b, ctx->stream);
    cudaEventSynchronize(b);
    float ms = 0; cudaEventElapsedTime(&ms, a, b);
    ctx->times.mphf += ms;
    cudaEventDestroy(a); cudaEventDestroy(b);
    return m;
}

// KMerIndex::serialize (kmer_index.hpp:102-108) -> mphf::save (BooPHF.h:514-535) -> bitVector::save (:316-323).
// The byte image is assembled ON THE DEVICE (piece copies + scalar patches) and leaves in one device->host copy straight
// into the caller's buffer (pinned buffers get the full PCIe rate). Fields are only 4-byte aligned (28-byte bucket header).
struct SerPiece { uint64_t src_word; uint64_t dst_byte; uint64_t nwords; uint32_t from_ranks; uint32_t pad; };
struct SerPatch { uint64_t dst_byte; uint64_t value; uint32_t nbytes; uint32_t pad; };

__global__ void ser_pieces_k(const SerPiece *__restrict__ pieces, const uint64_t *__restrict__ bits, const uint64_t *__restrict__ ranks,
                             uint32_t *__restrict__ img32) {
    const SerPiece p = pieces[blockIdx.x];
    const uint64_t *src = (p.from_ranks ? ranks : bits) + p.src_word;
    uint32_t *dst = img32 + (p.dst_byte >> 2);
    for (uint64_t i = threadIdx.x; i < p.nwords; i += blockDim.x) {
        const uint64_t v = src[i];
        dst[2 * i] = (uint32_t)v;
        dst[2 * i + 1] = (uint32_t)(v >> 32);
    }
}
__global__ void ser_patches_k(const SerPatch *__restrict__ patches, uint64_t n, uint32_t *__restrict__ img32) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SerPatch p = patches[i];
    img32[p.dst_byte >> 2] = (uint32_t)p.value;
    if (p.nbytes == 8) img32[(p.dst_byte >> 2) + 1] = (uint32_t)(p.value >> 32);
}

size_t mphf_serialized_size_buckets(const Mphf *m, int b_lo, int b_hi) {
    const int B = m->B;
    size_t total = 0;
    for (int b = b_lo; b < b_hi; ++b) {
        total += 28 + 8;
        if (m->bsz[b])
            for (int l = 0; l < kLevels; ++l) {
                const size_t p = (size_t)l * B + b;
                total += 16 + 8 * m->nchar[p] + 8 + 8 * ((m->nchar[p] + 7) / 8);
            }
    }
    return total;
}
size_t mphf_serialized_size(const Mphf *m) { return 8 + mphf_serialized_size_buckets(m, 0, m->B) + 8 * ((size_t)m->B + 1); }

// the image of buckets [b_lo, b_hi), with num_segments before and segment_starts after when `whole` (then [b_lo, b_hi) = [0, B))
static void serialize_image(const Mphf *m, int b_lo, int b_hi, bool whole, uint8_t *out, size_t cap) {
    Ctx *ctx = m->ctx;
    const int B = m->B;
    SG_CHECK(b_lo >= 0 && b_lo <= b_hi && b_hi <= B, 2, "bucket range outside the index");
    const size_t total = whole ? mphf_serialized_size(m) : mphf_serialized_size_buckets(m, b_lo, b_hi);
    SG_CHECK(total <= cap, 2, "output buffer too small for the serialized index");
    if (total == 0) return;
    std::vector<SerPiece> pieces;
    std::vector<SerPatch> patches;
    size_t pos = 0;
    auto patch = [&](uint64_t v, uint32_t nbytes) { patches.push_back(SerPatch{pos, v, nbytes, 0}); pos += nbytes; };
    if (whole) patch((uint64_t)B, 8);
    for (int b = b_lo; b < b_hi; ++b) {
        const double gamma = 4.0; uint64_t gbits; memcpy(&gbits, &gamma, 8);
        const uint64_t nelem = (uint64_t)m->bsz[b];
        patch(gbits, 8); patch((uint64_t)kLevels, 4);
        patch(nelem ? m->lastrank[b] : 0, 8);     // the reference leaves this field uninitialised for empty buckets
        patch(nelem, 8);
        if (nelem) {
            for (int l = 0; l < kLevels; ++l) {
                const size_t p = (size_t)l * B + b;
                const uint64_t nr = (m->nchar[p] + 7) / 8;
                patch(m->dom[p], 8); patch(m->nchar[p], 8);
                pieces.push_back(SerPiece{m->woff[p], pos, m->nchar[p], 0, 0}); pos += 8 * m->nchar[p];
                patch(nr, 8);
                pieces.push_back(SerPiece{m->woff[p] >> 3, pos, nr, 1, 0}); pos += 8 * nr;
            }
        }
        patch(0, 8);                                // final-hash map size (must be empty, checked at build time)
    }
    if (whole)
        for (int i = 0; i <= B; ++i) patch(m->starts[i], 8);
    SG_CHECK(pos == total, 6, "internal: serialized size mismatch");
    DArr<uint32_t> img(ctx, total / 4 + 2);
    DArr<SerPiece> dp(ctx, pieces.size() + 1);
    DArr<SerPatch> dq(ctx, patches.size() + 1);
    if (!pieces.empty()) SG_CUDA(cudaMemcpyAsync(dp.p, pieces.data(), pieces.size() * sizeof(SerPiece), cudaMemcpyHostToDevice, ctx->stream));
    SG_CUDA(cudaMemcpyAsync(dq.p, patches.data(), patches.size() * sizeof(SerPatch), cudaMemcpyHostToDevice, ctx->stream));
    if (!pieces.empty()) {
        ser_pieces_k<<<(unsigned)pieces.size(), 256, 0, ctx->stream>>>(dp.p, m->bits.p, m->ranks.p, img.p);
        ctx->launches++;
    }
    ser_patches_k<<<div_up((int64_t)patches.size(), 256), 256, 0, ctx->stream>>>(dq.p, patches.size(), img.p);
    ctx->launches++;
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(out, img.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
}
void mphf_serialize_to(const Mphf *m, uint8_t *out, size_t cap) { serialize_image(m, 0, m->B, true, out, cap); }
void mphf_serialize_buckets_to(const Mphf *m, int b_lo, int b_hi, uint8_t *out, size_t cap) { serialize_image(m, b_lo, b_hi, false, out, cap); }

void mphf_lookup_host_keys(Ctx *ctx, const Mphf *m, const uint64_t *h_keys, int64_t n, uint64_t *h_out) {
    if (n <= 0) return;
    DArr<uint64_t> dk(ctx, (size_t)n * m->nw), dout(ctx, (size_t)n);
    SG_CUDA(cudaMemcpyAsync(dk.p, h_keys, (size_t)n * m->nw * 8, cudaMemcpyHostToDevice, ctx->stream));
    MphfDev md = mphf_dev(m);
    int grid = div_up(n, 256);
    switch (m->nw) {
        case 1: mphf_lookup_k<1><<<grid, 256, 0, ctx->stream>>>(md, dk.p, (uint64_t)n, dout.p); break;
        case 2: mphf_lookup_k<2><<<grid, 256, 0, ctx->stream>>>(md, dk.p, (uint64_t)n, dout.p); break;
        case 3: mphf_lookup_k<3><<<grid, 256, 0, ctx->stream>>>(md, dk.p, (uint64_t)n, dout.p); break;
        default: mphf_lookup_k<4><<<grid, 256, 0, ctx->stream>>>(md, dk.p, (uint64_t)n, dout.p); break;
    }
    ctx->launches++;
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(h_out, dout.p, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
}


// ---- an index over the union of the ranks' keys, placed by every rank together (dist_edge_index.cu drives the steps). A level's
// bit is set iff exactly one still-unplaced key of the union hashed to it: each rank inserts its own keys into its copy of the
// level, then the copies are merged (a bit seen twice, within a rank or across ranks, collides), and every rank filters its keys
// against the merged level before inserting the survivors into the next one.
__global__ void mphf_merge_k(const uint64_t *const *__restrict__ bits, const uint64_t *const *__restrict__ coll, int world, uint64_t w0, uint64_t nwords,
                             uint64_t *__restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nwords) return;
    uint64_t seen = 0, c = 0;
    for (int r = 0; r < world; ++r) {
        const uint64_t s = bits[r][w0 + i];
        c |= coll[r][i] | (seen & s);
        seen |= s;
    }
    out[i] = seen & ~c;
}

void mphf_place_begin(Ctx *ctx, Mphf *m, MphfPlacer *pl, const KeyTable &t, uint64_t n, const std::vector<uint64_t> &level_start) {
    cudaStream_t st = ctx->stream;
    pl->t = t; pl->n_alive = n; pl->alive = nullptr; pl->level = 0; pl->level_start = level_start;
    const uint64_t l0_words = level_start[1] - level_start[0];
    pl->coll.alloc(ctx, l0_words + 8, true);
    pl->scratch.alloc(ctx, l0_words + 8);
    pl->cnt.alloc(ctx, 1);
    SG_CUDA(cudaMemsetAsync(pl->coll.p, 0, pl->coll.bytes(), st));
    if (n) {
        const MphfDev md = mphf_dev(m);
        switch (m->nw) {
            case 1: mphf_insert_k<1><<<div_up((int64_t)n, 256), 256, 0, st>>>(t, nullptr, n, 0, md, level_start[0], pl->coll.p); break;
            case 2: mphf_insert_k<2><<<div_up((int64_t)n, 256), 256, 0, st>>>(t, nullptr, n, 0, md, level_start[0], pl->coll.p); break;
            case 3: mphf_insert_k<3><<<div_up((int64_t)n, 256), 256, 0, st>>>(t, nullptr, n, 0, md, level_start[0], pl->coll.p); break;
            default: mphf_insert_k<4><<<div_up((int64_t)n, 256), 256, 0, st>>>(t, nullptr, n, 0, md, level_start[0], pl->coll.p); break;
        }
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
    }
    SG_CUDA(cudaStreamSynchronize(st));
}

void mphf_place_merge(Ctx *ctx, Mphf *m, MphfPlacer *pl, const uint64_t *const *d_bits, const uint64_t *const *d_coll, int world) {
    cudaStream_t st = ctx->stream;
    const int l = pl->level;
    const uint64_t w0 = pl->level_start[l], nw = pl->level_start[l + 1] - w0;
    if (nw) {
        mphf_merge_k<<<div_up((int64_t)nw, 256), 256, 0, st>>>(d_bits, d_coll, world, w0, nw, pl->scratch.p);
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
    }
    SG_CUDA(cudaStreamSynchronize(st));
}

uint64_t mphf_place_advance(Ctx *ctx, Mphf *m, MphfPlacer *pl) {
    cudaStream_t st = ctx->stream;
    const int l = pl->level;
    const bool last = (l == kLevels - 2);              // level 23 has no successor bitset: only count what is left
    const uint64_t w0 = pl->level_start[l], nw = pl->level_start[l + 1] - w0;
    // the merged level replaces this rank's copy, and its collisions are spent (no peer reads either any more)
    if (nw) SG_CUDA(cudaMemcpyAsync(m->bits.p + w0, pl->scratch.p, nw * 8, cudaMemcpyDeviceToDevice, st));
    SG_CUDA(cudaMemsetAsync(pl->coll.p, 0, pl->coll.bytes(), st));
    const uint64_t n_alive = pl->n_alive;
    uint64_t c = 0;
    if (n_alive) {
        DArr<uint64_t> &next = (l & 1) ? pl->aliveA : pl->aliveB;
        const uint64_t cap = (l == 0) ? n_alive / 2 + 1024 : n_alive;
        if (next.n < cap) next.alloc(ctx, cap);
        SG_CUDA(cudaMemsetAsync(pl->cnt.p, 0, 8, st));
        const MphfDev md = mphf_dev(m);
        const int grid = div_up((int64_t)n_alive, 256);
        const uint64_t nls = last ? 0 : pl->level_start[l + 1];
        switch (m->nw) {
            case 1: mphf_advance_k<1><<<grid, 256, 0, st>>>(pl->t, pl->alive, n_alive, l, md, next.p, (uint64_t)next.n, pl->cnt.p, last ? 0 : 1, nls, pl->coll.p); break;
            case 2: mphf_advance_k<2><<<grid, 256, 0, st>>>(pl->t, pl->alive, n_alive, l, md, next.p, (uint64_t)next.n, pl->cnt.p, last ? 0 : 1, nls, pl->coll.p); break;
            case 3: mphf_advance_k<3><<<grid, 256, 0, st>>>(pl->t, pl->alive, n_alive, l, md, next.p, (uint64_t)next.n, pl->cnt.p, last ? 0 : 1, nls, pl->coll.p); break;
            default: mphf_advance_k<4><<<grid, 256, 0, st>>>(pl->t, pl->alive, n_alive, l, md, next.p, (uint64_t)next.n, pl->cnt.p, last ? 0 : 1, nls, pl->coll.p); break;
        }
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
        unsigned long long h = 0;
        SG_CUDA(cudaMemcpyAsync(&h, pl->cnt.p, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        SG_CHECK(h <= next.n, 6, "internal: MPHF survivor list overflow");
        pl->alive = next.p;
        c = h;
    }
    SG_CUDA(cudaStreamSynchronize(st));
    pl->n_alive = c;
    pl->level = l + 1;
    return c;
}

}  // namespace sg
