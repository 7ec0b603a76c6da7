// graph.cu -- extension masks, coverage, unitigs (unbranching paths + perfect loops), link records. Replaces
//   DeBruijnExtensionIndexBuilder::FillExtensionsFromIndex (src/common/kmer_index/extension_index/kmer_extension_index_builder.hpp:45-60)
//   InOutMask (…/extension_index/inout_mask.hpp:55-221)
//   CoverageHashMapBuilder (src/common/kmer_index/ph_map/coverage_hash_map_builder.hpp:16-57) -- counts come from the sort's run lengths
//   UnbranchingPathExtractor (src/common/assembly_graph/construction/debruijn_graph_constructor.hpp:184-410)
//   FastGraphFromSequencesConstructor::CollectLinkRecords (…:473-487) and GraphCoverageFiller (graph_support/coverage_filling.hpp:52-70)
#include <algorithm>
#include <array>
#include <optional>

#include "graph.h"
#include "masks_dev.cuh"
#include "mphf_dev.cuh"

namespace sg {

__device__ __forceinline__ uint8_t inv_byte(uint8_t a) { return (uint8_t)(__brev((unsigned)a) >> 24); }   // inout_mask.hpp:18-27
__device__ __forceinline__ int uniq4(unsigned m) {           // inout_mask.hpp:61-81 (CheckUnique/GetUnique), -1 if not unique
    return (m && !(m & (m - 1))) ? (__ffs(m) - 1) : -1;
}

template <int NW>
struct CanonIdx { uint64_t idx; bool is_min; };

template <int NW>
__device__ __forceinline__ CanonIdx<NW> canon_lookup(const MphfDev &m, const Kmer<NW> &k, int K) {
    Kmer<NW> r = kmer_rc<NW>(k, K);
    CanonIdx<NW> c;
    c.is_min = kmer_is_minimal<NW>(k, r);          // key_with_hash.hpp:120-128
    c.idx = mphf_lookup_dev<NW>(m, c.is_min ? k : r);
    return c;
}
// get_value(kwh): InvertableStoring::get_value with InOutMask::conjugate (storing_traits.hpp:44-51)
template <int NW>
__device__ __forceinline__ uint8_t oriented_mask(const MphfDev &m, const uint8_t *masks, const Kmer<NW> &k, int K, uint64_t *idx_out = nullptr) {
    CanonIdx<NW> c = canon_lookup<NW>(m, k, K);
    if (idx_out) *idx_out = c.idx;
    uint8_t v = masks[c.idx];
    return c.is_min ? v : inv_byte(v);
}
// prepend nucleotide c, dropping the last (RtSeq::operator>>, rtseq.hpp:569-588)
template <int NW>
__device__ __forceinline__ void kmer_shr(Kmer<NW> &k, int K, int c) {
    uint64_t carry = (uint64_t)c;
#pragma unroll
    for (int j = 0; j < NW; ++j) {
        uint64_t nc = k.w[j] >> 62;
        k.w[j] = (k.w[j] << 2) | carry;
        carry = nc;
    }
    k.w[NW - 1] &= last_word_mask<NW>(K);
}

// record j of a dense key array (a chunk of a k-mer set, or a compacted list of keys)
template <int NW>
__device__ __forceinline__ Kmer<NW> key_at(const uint64_t *__restrict__ keys, int64_t j) {
    Kmer<NW> k;
#pragma unroll
    for (int q = 0; q < NW; ++q) k.w[q] = keys[j * NW + q];
    return k;
}

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

void launch_nonzero_flags(Ctx *ctx, const uint32_t *in, uint32_t *out, uint64_t n);

// walk from `start` along out-edge c until a junction (ConstructSequenceWithEdge :264-273). Calls f(vertex index i>=1, k-mer) per vertex.
template <int NW, class F>
__device__ __forceinline__ uint32_t walk_right(const MphfDev &mk, const uint8_t *masks, int K, const Kmer<NW> &start, int c, uint64_t max_steps, F &&f,
                                               Kmer<NW> *end_out, Kmer<NW> *prev_out) {
    Kmer<NW> prev = start, cur = start;
    kmer_shl<NW>(cur, K, c);
    uint32_t m = 1;
    f(m, cur);
    for (;;) {
        const uint8_t msk = oriented_mask<NW>(mk, masks, cur, K);
        const int uo = uniq4(msk & 15), ui = uniq4(msk >> 4);
        if (uo < 0 || ui < 0) break;
        Kmer<NW> nxt = cur;
        kmer_shl<NW>(nxt, K, uo);
        prev = cur; cur = nxt; ++m;
        f(m, cur);
        if (m > max_steps) break;
    }
    *end_out = cur; *prev_out = prev;
    return m;
}

// probe pass: for junction q and slot s = side*4 + c decide whether the path is emitted and how long it is
template <int NW>
__global__ void unitig_probe_k(const uint64_t *__restrict__ jkeys, int64_t njunc, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                               uint64_t nk, uint32_t *__restrict__ len /*[njunc*8] 0 = none*/, uint8_t *__restrict__ selfc) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= njunc * 8) return;
    const int64_t q = tid >> 3;
    const int side = (int)(tid >> 2) & 1, c = (int)tid & 3;
    const Kmer<NW> key = key_at<NW>(jkeys, q);
    const uint8_t mfw = masks[mphf_lookup_dev<NW>(mk, key)];
    const Kmer<NW> start = side ? kmer_rc<NW>(key, K) : key;          // AddStartDeEdges :214-235
    const uint8_t m = side ? inv_byte(mfw) : mfw;
    len[tid] = 0; selfc[tid] = 0;
    if (!(m & (1u << c))) return;
    Kmer<NW> end, prev;
    auto nop = [](uint32_t, const Kmer<NW> &) {};
    const uint32_t steps = walk_right<NW>(mk, masks, K, start, c, nk + 1, nop, &end, &prev);
    // keep iff !(s < !s)  (:307). s[0..K) = start, (!s)[0..K) = rc(end).
    const Kmer<NW> rcend = kmer_rc<NW>(end, K);
    bool keep, self = false;
    if (kmer_nuc_less<NW>(start, rcend)) keep = false;
    else if (kmer_nuc_less<NW>(rcend, start)) keep = true;
    else {
        // hairpin: first K symbols agree. s[K+i] = last(v_{1+i}); (!s)[K+i] = 3 - first(v_{steps-1-i}), i = 0..steps-1
        keep = true; self = true;
        Kmer<NW> a = start, b = prev;              // a walks forward from v0, b walks backward from v_{steps-1}
        kmer_shl<NW>(a, K, c);
        for (uint32_t i = 0; i < steps; ++i) {
            const int x = kmer_nuc<NW>(a, K - 1), y = 3 - (int)(b.w[0] & 3);
            if (x != y) { keep = x > y; self = false; break; }
            if (i + 1 < steps) {
                const uint8_t ma = oriented_mask<NW>(mk, masks, a, K);
                kmer_shl<NW>(a, K, uniq4(ma & 15));
                if (i + 2 < steps) {                 // b = v_{steps-2-i} is needed next; v_0 = start has no unique-in guarantee, use it directly
                    const uint8_t mb = oriented_mask<NW>(mk, masks, b, K);
                    kmer_shr<NW>(b, K, uniq4(mb >> 4));
                } else b = start;
            }
        }
    }
    if (keep) { len[tid] = (uint32_t)K + steps; selfc[tid] = self ? 1 : 0; }
}

struct EdgeOut {
    char *seq;                 // ASCII bases, all edges concatenated
    uint64_t *link_start;      // LinkRecord hash_and_mask of StartLink / EndLink (:455-471)
    uint64_t *link_end;
    uint32_t *raw_cov;         // sum of (k+1)-mer multiplicities along the edge
    uint8_t *visited;          // per k-mer MPHF index
};

template <int NW, int NWS>
__device__ __forceinline__ uint32_t kpomer_cov(const MphfDev &mkp, const uint32_t *cov, const Kmer<NW> &v, int nextc, int K) {
    Kmer<NWS> x;
#pragma unroll
    for (int q = 0; q < NWS; ++q) x.w[q] = q < NW ? v.w[q] : 0;
    x.w[K >> 5] |= (uint64_t)nextc << ((K & 31) << 1);
    Kmer<NWS> r = kmer_rc<NWS>(x, K + 1);
    return cov[mphf_lookup_dev<NWS>(mkp, kmer_is_minimal<NWS>(x, r) ? x : r)];
}

__device__ __forceinline__ uint64_t link_value(uint64_t idx, bool is_start, bool is_rc) { return (idx << 2) | (is_rc ? 2ull : 0ull) | (is_start ? 1ull : 0ull); }

template <int NW, int NWS>
__global__ void unitig_write_k(const uint64_t *__restrict__ jkeys, int64_t njunc, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                               uint64_t nk, const uint32_t *__restrict__ len, const uint8_t *__restrict__ selfc, const uint64_t *__restrict__ eidx,
                               const uint64_t *__restrict__ eoff, MphfDev mkp, const uint32_t *__restrict__ cov, EdgeOut o) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= njunc * 8) return;
    if (!len[tid]) return;
    const int64_t q = tid >> 3;
    const int side = (int)(tid >> 2) & 1, c = (int)tid & 3;
    const Kmer<NW> key = key_at<NW>(jkeys, q);
    const Kmer<NW> start = side ? kmer_rc<NW>(key, K) : key;
    const uint64_t e = eidx[tid];
    char *out = o.seq + eoff[tid];
    for (int i = 0; i < K; ++i) out[i] = "ACGT"[kmer_nuc<NW>(start, i)];
    uint64_t sidx;
    {
        CanonIdx<NW> ci = canon_lookup<NW>(mk, start, K);
        sidx = ci.idx;
        o.visited[sidx] = 1;
        o.link_start[e] = link_value(sidx, true, !ci.is_min);
    }
    uint32_t raw = 0;
    Kmer<NW> pv = start;
    auto emit = [&](uint32_t i, const Kmer<NW> &v) {
        const int ch = kmer_nuc<NW>(v, K - 1);
        out[K - 1 + i] = "ACGT"[ch];
        uint64_t idx;
        oriented_mask<NW>(mk, masks, v, K, &idx);
        o.visited[idx] = 1;
        if (cov) raw += kpomer_cov<NW, NWS>(mkp, cov, pv, ch, K);
        pv = v;
    };
    Kmer<NW> end, prev;
    walk_right<NW>(mk, masks, K, start, c, nk + 1, emit, &end, &prev);
    if (selfc[tid]) o.link_end[e] = ~0ull;                 // LinkRecord() for self-conjugate edges (:481-484)
    else {
        CanonIdx<NW> ci = canon_lookup<NW>(mk, end, K);
        o.link_end[e] = link_value(ci.idx, false, !ci.is_min);
    }
    o.raw_cov[e] = raw;
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

// ---- early tip clipper -------------------------------------------------------------------------------------------------
// EarlyTipClipperProcessor (assembly_graph/construction/early_simplification.hpp:38-162), run by the pipeline between the
// mask fill and the unitig extraction (stages/construction.cpp:289-302, length bound = read length - k). The reference walks
// the junctions one after the other (or racily from several threads) on the live index; the result does not depend on the
// order (a tip's vertices are reachable from exactly one junction orientation and removals only zero tip vertices -- checked
// against the unmodified reference with 1 and 8 threads and against the oracle's sequential and snapshot modes, tests/), so
// here every (k-mer, orientation) with >= 2 outgoing edges is one thread on a snapshot of the masks:
//   tc_probe_k  FindForward per outgoing edge (:115-125), RemoveTips decision (:133-155), marks the vertices to isolate
//   tc_apply_k  IsolateVertex for the marked vertices
//   tc_links_k  RemoveInconsistentForwardLinks over the tipped junctions (:21-36) on the updated masks
template <int NW, bool MARK>
__device__ __forceinline__ uint32_t tc_find_forward(const MphfDev &mk, const uint8_t *masks, int K, Kmer<NW> kh, uint32_t bound, uint8_t *mark) {
    uint32_t n = 0;
    for (;;) {
        uint64_t idx;
        const uint8_t m = oriented_mask<NW>(mk, masks, kh, K, &idx);
        const int uo = uniq4(m & 15), ui = uniq4(m >> 4);
        if (MARK) mark[idx] = 1;
        if (!(n < bound && ui >= 0 && uo >= 0)) {
            ++n;                                                 // tip.push_back(kh) after the loop (:121)
            return (ui < 0 || (m & 15) != 0) ? 0u : n;           // branching / not a dead end -> not a tip (:122-125)
        }
        ++n;
        kmer_shl<NW>(kh, K, uo);
    }
}
template <int NW>
__global__ void tc_probe_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, uint32_t bound,
                           uint8_t *__restrict__ mark, uint8_t *__restrict__ tipped /*[2 * all k-mers]*/, unsigned long long *__restrict__ stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    tipped += 2 * base;
    const int o = (int)(tid & 1);
    const uint8_t mfw = masks[mphf_lookup_dev<NW>(mk, key)];
    const uint8_t m = o ? inv_byte(mfw) : mfw;
    tipped[tid] = 0;
    if (__popc(m & 15) < 2) return;                              // OutgoingEdgeCount(kh) >= 2 (:72)
    const Kmer<NW> kh = o ? kmer_rc<NW>(key, K) : key;
    uint32_t sz[4] = {0, 0, 0, 0}, mx = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (!(m & (1u << c))) continue;
        Kmer<NW> khc = kh;
        kmer_shl<NW>(khc, K, c);
        sz[c] = tc_find_forward<NW, false>(mk, masks, K, khc, bound, nullptr);
        const uint32_t len = sz[c] ? sz[c] : 0xffffffffu;
        if (len > mx) mx = len;
    }
    uint32_t removed = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (!sz[c] || sz[c] >= mx) continue;                     // RemoveTips: tip.size() < max (:136-141)
        Kmer<NW> khc = kh;
        kmer_shl<NW>(khc, K, c);
        tc_find_forward<NW, true>(mk, masks, K, khc, bound, mark);
        removed += sz[c];
    }
    if (removed) { tipped[tid] = 1; atomicAdd(&stats[0], (unsigned long long)removed); atomicAdd(&stats[1], 1ull); }
}
__global__ void tc_apply_k(uint8_t *__restrict__ masks, const uint8_t *__restrict__ mark, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && mark[i]) masks[i] = 0;
}
template <int NW>
// flags_by_slot = 0: tipped[] is indexed by (k-mer position, orientation), as tc_probe_k writes it; 1: by (MPHF slot, orientation),
// as at_tips_probe_k marks the roots it reaches by walking
__global__ void tc_links_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, int K, MphfDev mk, uint8_t *__restrict__ masks,
                           const uint8_t *__restrict__ tipped, unsigned long long *__restrict__ stat_clipped, int flags_by_slot) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    if (!flags_by_slot && !tipped[2 * base + tid]) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const Kmer<NW> kh = (tid & 1) ? kmer_rc<NW>(key, K) : key;
    const CanonIdx<NW> ci = canon_lookup<NW>(mk, kh, K);
    if (flags_by_slot && !tipped[2 * ci.idx + (uint64_t)(tid & 1)]) return;
    const uint8_t raw = masks[ci.idx];
    const uint8_t m = ci.is_min ? raw : inv_byte(raw);
    const int first = (int)(kh.w[0] & 3);                        // kh[0]
    for (int c = 0; c < 4; ++c) {
        if (!(m & (1u << c))) continue;
        Kmer<NW> nx = kh;
        kmer_shl<NW>(nx, K, c);
        if (!(oriented_mask<NW>(mk, masks, nx, K) & (1u << (4 + first)))) {            // !CheckIncoming(next_kh, kh[0])
            const unsigned bit = 1u << (ci.is_min ? c : 7 - c);                          // DeleteOutgoing(kh, c), inout_mask.hpp:108-114
            atomicAnd(reinterpret_cast<unsigned *>(masks) + (ci.idx >> 2), ~(bit << (8 * (ci.idx & 3))));
            atomicAdd(stat_clipped, 1ull);
        }
    }
}

// ---- early low-complexity (poly A/T) clipper ----------------------------------------------------------------------------------
// EarlyLowComplexityClipperProcessor (assembly_graph/construction/early_simplification.hpp:164-347), the EarlyATClipper phase of the
// RNA pipeline (stages/construction.cpp:317-340,447-448: at_ratio 0.8, min_length 10, max_length 200); runs before the tip clipper.
//   RemoveATEdges (:185-256)  at_edges_probe_k : per (k-mer, orientation) on the untouched masks: junction + low-complexity k-mer ->
//                                                 the outgoing edges of length 1 (next is a junction or a dead end) are flagged
//                             at_edges_apply_k : every flagged link is deleted once (the reference deletes it through whichever of
//                                                 its two representations comes first and skips the other, :237-238: here the
//                                                 representation with the smaller (thread, nucleotide) pair acts)
//   RemoveATTips  (:269-334)  at_tips_probe_k  : per dead end with a unique incoming edge: walk back to the junction (<= max_length),
//                                                 complexity of the tip (+ the root's last nucleotides up to min_length), mark
//                                                 the vertices and the root. The reference isolates tips while other threads
//                                                 walk; the result does not depend on the order (tips are disjoint chains whose
//                                                 decisions read only their own vertices and the root's mask -- checked: unmodified
//                                                 reference with 1 and 8 threads == oracle sequential == oracle snapshot)
//                             tc_apply_k, tc_links_k : IsolateVertex, RemoveInconsistentForwardLinks on the updated masks
__device__ __forceinline__ bool almost_equals_f64(double a, double b) {     // gtest FloatingPoint<double>::AlmostEquals, 4 ULPs (math/xmath.h:283-299)
    if (a != a || b != b) return false;
    const unsigned long long x = (unsigned long long)__double_as_longlong(a), y = (unsigned long long)__double_as_longlong(b);
    const unsigned long long sign = 0x8000000000000000ull;
    const unsigned long long bx = (x & sign) ? (~x + 1ull) : (sign | x), by = (y & sign) ? (~y + 1ull) : (sign | y);
    return (bx >= by ? bx - by : by - bx) <= 4ull;
}
__device__ __forceinline__ bool math_ls(double a, double b) { return !almost_equals_f64(a, b) && a < b; }      // math::ls, xmath.h:300-306
__device__ __forceinline__ bool mask_is_junction(uint8_t m) { return uniq4(m & 15) < 0 || uniq4(m >> 4) < 0; }  // InOutMask::IsJunction

struct AtParams { double ratio; uint32_t min_len, max_len; };

template <int NW>
__global__ void at_edges_probe_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, AtParams ap,
                                 uint8_t *__restrict__ eflag /*[2 * all k-mers]*/, unsigned long long *__restrict__ stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const int o = (int)(tid & 1);
    const uint64_t slot = mphf_lookup_dev<NW>(mk, key);
    const int64_t fid = (int64_t)(2 * slot) + o;                        // flags are indexed by (MPHF slot, orientation), like the masks
    eflag[fid] = 0;
    const uint8_t mfw = masks[slot];
    const uint8_t m = o ? inv_byte(mfw) : mfw;
    if (!mask_is_junction(m)) return;
    const Kmer<NW> kh = o ? kmer_rc<NW>(key, K) : key;
    uint32_t cnt[4] = {0, 0, 0, 0};
    for (int p = 0; p < K; ++p) cnt[kmer_nuc<NW>(kh, p)]++;
    const uint32_t curm = max(max(cnt[0], cnt[1]), max(cnt[2], cnt[3]));
    if (math_ls((double)curm, (double)K * ap.ratio)) return;
    uint8_t f = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (!(m & (1u << c))) continue;
        Kmer<NW> nx = kh;
        kmer_shl<NW>(nx, K, c);
        const uint8_t mn = oriented_mask<NW>(mk, masks, nx, K);
        if (!mask_is_junction(mn) && (mn & 15) != 0) continue;          // an edge of length 1: next is a junction or a dead end
        f |= (uint8_t)(1u << c);
    }
    eflag[fid] = f;
    if (f) atomicAdd(&stats[0], (unsigned long long)__popc(f));
}
__device__ __forceinline__ void mask_clear_bit(uint8_t *masks, uint64_t idx, unsigned bit) {
    atomicAnd(reinterpret_cast<unsigned *>(masks) + (idx >> 2), ~((1u << bit) << (8 * (idx & 3))));
}
template <int NW>
__global__ void at_edges_apply_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, uint8_t *__restrict__ masks, const uint8_t *__restrict__ eflag,
                                 unsigned long long *__restrict__ stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const Kmer<NW> kh = (tid & 1) ? kmer_rc<NW>(key, K) : key;
    const CanonIdx<NW> ci = canon_lookup<NW>(mk, kh, K);
    const int64_t fid = (int64_t)(2 * ci.idx) + (tid & 1);               // kh is the table key (minimal form) iff the orientation bit is 0
    const uint8_t mine = eflag[fid];
    if (!mine) return;
    const int first = (int)(kh.w[0] & 3);                                // kh[0]
    for (int c = 0; c < 4; ++c) {
        if (!(mine & (1u << c))) continue;
        Kmer<NW> nx = kh;
        kmer_shl<NW>(nx, K, c);
        const CanonIdx<NW> cn = canon_lookup<NW>(mk, nx, K);
        // the same link seen from the other strand: (rc(next), complement of kh[0]); rc(next) is the table key iff next is NOT minimal
        const int64_t fid2 = (int64_t)(2 * cn.idx) + (cn.is_min ? 1 : 0);
        const int c2 = 3 - first;
        if ((eflag[fid2] & (1u << c2)) && (fid2 < fid || (fid2 == fid && c2 < c))) continue;
        mask_clear_bit(masks, ci.idx, (unsigned)(ci.is_min ? c : 7 - c));                        // DeleteOutgoing(kh, c)
        mask_clear_bit(masks, cn.idx, (unsigned)(cn.is_min ? 4 + first : 7 - (4 + first)));      // DeleteIncoming(next, kh[0])
        atomicAdd(&stats[1], 2ull);
    }
}
template <int NW>
__global__ void at_tips_probe_k(const uint64_t *__restrict__ keys, int64_t n, int K, MphfDev mk, const uint8_t *__restrict__ masks, AtParams ap,
                                uint8_t *__restrict__ mark, uint8_t *__restrict__ rooted /*[2 * all k-mers]*/, unsigned long long *__restrict__ stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const int o = (int)(tid & 1);
    const uint64_t idx0 = mphf_lookup_dev<NW>(mk, key);
    const uint8_t mfw = masks[idx0];
    const uint8_t m0 = o ? inv_byte(mfw) : mfw;
    if ((m0 & 15) != 0 || uniq4(m0 >> 4) < 0) return;                   // IsDeadEnd && CheckUniqueIncoming
    const Kmer<NW> start = o ? kmer_rc<NW>(key, K) : key;
    Kmer<NW> kh = start;
    uint32_t cnt[4] = {0, 0, 0, 0};
    uint32_t tsz = 0;
    uint8_t m = m0;
    do {                                                                 // walk back to the junction, :292-296
        ++tsz;
        cnt[kmer_nuc<NW>(kh, K - 1)]++;
        kmer_shr<NW>(kh, K, uniq4(m >> 4));
        m = oriented_mask<NW>(mk, masks, kh, K);
    } while (tsz < ap.max_len && !mask_is_junction(m));
    if ((m >> 4) == 0 || !mask_is_junction(m)) return;                   // dead start (isolated short edge) or too long, :301-302
    for (uint32_t p = tsz - 1; p < ap.min_len; ++p) cnt[kmer_nuc<NW>(kh, K - 1 - (int)p)]++;
    const uint32_t curm = max(max(cnt[0], cnt[1]), max(cnt[2], cnt[3]));
    if (math_ls((double)curm, (double)max(tsz, ap.min_len) * ap.ratio)) return;
    // a low-complexity tip: mark its vertices (second walk) and its root
    const CanonIdx<NW> cr = canon_lookup<NW>(mk, kh, K);
    rooted[2 * cr.idx + (cr.is_min ? 0 : 1)] = 1;
    Kmer<NW> w = start;
    uint8_t mw = m0;
    for (uint32_t s2 = 0; s2 < tsz; ++s2) {
        uint64_t idx;
        if (s2) mw = oriented_mask<NW>(mk, masks, w, K, &idx); else idx = idx0;
        mark[idx] = 1;
        kmer_shr<NW>(w, K, uniq4(mw >> 4));
    }
    atomicAdd(&stats[2], (unsigned long long)tsz);
}

// ---- perfect loops (CollectLoops :359-397). Rare; one thread per candidate / per loop is enough. ---------------------
// The final_kmers position of each remaining slot, stored densely: pos[rank of the slot among the remaining ones]. rank() is
// ~0 for a slot that is not remaining. Costs 3/8 B per k-mer plus 8 B per remaining slot.
struct RemSlots {
    const uint32_t *bits;      // one bit per MPHF slot
    const uint64_t *base;      // remaining slots before each 32-slot word (exclusive scan of the words' popcounts)
    __device__ __forceinline__ uint64_t rank(uint64_t slot) const {
        const uint32_t w = bits[slot >> 5], bit = 1u << (slot & 31);
        return (w & bit) ? base[slot >> 5] + (uint64_t)__popc(w & (bit - 1)) : ~0ull;
    }
};
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
// leader of a loop = its vertex with the smallest final_kmers position (that is where the serial scan first meets it)
template <int NW>
// (is_leader: per record of the chunk; nk: all k-mers, the bound of a loop's length)
__global__ void loop_leader_k(const uint64_t *__restrict__ keys, int64_t base, int64_t n, uint64_t nk, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                              RemSlots rs, const uint64_t *__restrict__ pos, uint32_t *__restrict__ is_leader) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    is_leader[j] = 0;
    const Kmer<NW> key = key_at<NW>(keys, j);
    uint64_t idx0;
    uint8_t m = oriented_mask<NW>(mk, masks, key, K, &idx0);
    if (!m || uniq4(m & 15) < 0 || uniq4(m >> 4) < 0) return;
    Kmer<NW> cur = key;
    bool leader = true;
    for (uint64_t it = 0; it <= nk; ++it) {
        kmer_shl<NW>(cur, K, uniq4(m & 15));
        if (kmer_eq<NW>(cur, key)) break;
        uint64_t idx;
        m = oriented_mask<NW>(mk, masks, cur, K, &idx);
        // a loop's vertices are all remaining slots (every other vertex was a junction, a dead end or visited by a path)
        const uint64_t rk = rs.rank(idx);
        if (rk != ~0ull && pos[rk] < (uint64_t)(base + j)) { leader = false; break; }
    }
    is_leader[j] = leader ? 1u : 0u;
}

// per leader: break point (FindMinimalKMerInLoop :252-262), loop length, self-RC split position (ConstructLoopFromVertex :283-293)
struct LoopInfo { uint64_t w[4]; uint32_t nverts; int32_t split; };
template <int NW, int NWS>
__global__ void loop_probe_k(const uint64_t *__restrict__ leaders /*keys*/, int64_t nl, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                             LoopInfo *__restrict__ info, uint32_t *__restrict__ len /*[nl*2]*/) {
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nl) return;
    const Kmer<NW> key = key_at<NW>(leaders, q);
    Kmer<NW> minimal = key, r = kmer_rc<NW>(key, K);
    if (kmer_nuc_less<NW>(r, minimal)) minimal = r;
    Kmer<NW> cur = key;
    uint32_t nv = 0;
    do {
        const uint8_t m = oriented_mask<NW>(mk, masks, cur, K);
        kmer_shl<NW>(cur, K, uniq4(m & 15));
        ++nv;
        if (kmer_eq<NW>(cur, key)) break;
        if (kmer_nuc_less<NW>(cur, minimal)) minimal = cur;
        r = kmer_rc<NW>(cur, K);
        if (kmer_nuc_less<NW>(r, minimal)) minimal = r;
    } while (true);
    // sequence from `minimal`: K + nv symbols; scan its (k+1)-mers for a self-RC one
    int32_t split = -1;
    cur = minimal;
    for (uint32_t i = 0; i < nv; ++i) {
        const uint8_t m = oriented_mask<NW>(mk, masks, cur, K);
        const int ch = uniq4(m & 15);
        Kmer<NWS> x;
#pragma unroll
        for (int z = 0; z < NWS; ++z) x.w[z] = z < NW ? cur.w[z] : 0;
        x.w[K >> 5] |= (uint64_t)ch << ((K & 31) << 1);
        if (kmer_eq<NWS>(x, kmer_rc<NWS>(x, K + 1))) { split = (int32_t)i; break; }
        kmer_shl<NW>(cur, K, ch);
    }
    LoopInfo li;
    for (int z = 0; z < 4; ++z) li.w[z] = z < NW ? minimal.w[z] : 0;
    li.nverts = nv; li.split = split;
    info[q] = li;
    const uint32_t n = (uint32_t)K + nv;
    if (split < 0) { len[2 * q] = n; len[2 * q + 1] = 0; }
    else { len[2 * q] = (uint32_t)K + 1; len[2 * q + 1] = (n - K - (split + 1)) + (split + K); }   // SplitLoop :276-281
}

__device__ __forceinline__ bool ascii_rc_less(const char *s, uint32_t n) {     // s < !s  (Sequence::operator<, sequence.hpp:592-600)
    for (uint32_t i = 0; i < n; ++i) {
        const char a = s[i], b = s[n - 1 - i];
        const char rb = b == 'A' ? 'T' : (b == 'C' ? 'G' : (b == 'G' ? 'C' : 'A'));
        if (a != rb) return a < rb;
    }
    return false;
}
__device__ __forceinline__ void ascii_rc_inplace(char *s, uint32_t n) {
    for (uint32_t i = 0; i < (n + 1) / 2; ++i) {
        const char a = s[i], b = s[n - 1 - i];
        const char ra = a == 'A' ? 'T' : (a == 'C' ? 'G' : (a == 'G' ? 'C' : 'A'));
        const char rb = b == 'A' ? 'T' : (b == 'C' ? 'G' : (b == 'G' ? 'C' : 'A'));
        s[i] = rb; s[n - 1 - i] = ra;
    }
}

template <int NW, int NWS>
__device__ void finish_edge(char *s, uint32_t n, int K, uint64_t e, const MphfDev &mk, const MphfDev &mkp, const uint32_t *cov, EdgeOut &o) {
    if (ascii_rc_less(s, n)) ascii_rc_inplace(s, n);       // keep the larger strand (:383-387)
    // links + coverage from the final string
    auto code = [](char ch) { return ch == 'A' ? 0 : (ch == 'C' ? 1 : (ch == 'G' ? 2 : 3)); };
    Kmer<NW> a, b;
#pragma unroll
    for (int z = 0; z < NW; ++z) { a.w[z] = 0; b.w[z] = 0; }
    for (int i = 0; i < K; ++i) {
        a.w[i >> 5] |= (uint64_t)code(s[i]) << ((i & 31) << 1);
        b.w[i >> 5] |= (uint64_t)code(s[n - K + i]) << ((i & 31) << 1);
    }
    bool self = true;
    for (uint32_t i = 0; i < n; ++i) {
        const char x = s[n - 1 - i];
        const char rx = x == 'A' ? 'T' : (x == 'C' ? 'G' : (x == 'G' ? 'C' : 'A'));
        if (s[i] != rx) { self = false; break; }
    }
    CanonIdx<NW> ca = canon_lookup<NW>(mk, a, K);
    o.link_start[e] = link_value(ca.idx, true, !ca.is_min);
    if (self) o.link_end[e] = ~0ull;
    else {
        CanonIdx<NW> cb = canon_lookup<NW>(mk, b, K);
        o.link_end[e] = link_value(cb.idx, false, !cb.is_min);
    }
    uint32_t raw = 0;
    if (cov) {
        Kmer<NW> v = a;
        for (uint32_t p = (uint32_t)K; p < n; ++p) {
            const int ch = code(s[p]);
            raw += kpomer_cov<NW, NWS>(mkp, cov, v, ch, K);
            kmer_shl<NW>(v, K, ch);
        }
    }
    o.raw_cov[e] = raw;
}

template <int NW, int NWS>
__global__ void loop_write_k(const LoopInfo *__restrict__ info, int64_t nl, int K, MphfDev mk, const uint8_t *__restrict__ masks,
                             const uint32_t *__restrict__ len, const uint64_t *__restrict__ eidx, const uint64_t *__restrict__ eoff, MphfDev mkp,
                             const uint32_t *__restrict__ cov, EdgeOut o, char *__restrict__ scratch, const uint64_t *__restrict__ soff) {
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nl) return;
    const LoopInfo li = info[q];
    Kmer<NW> cur;
#pragma unroll
    for (int z = 0; z < NW; ++z) cur.w[z] = li.w[z];
    const uint32_t n = (uint32_t)K + li.nverts;
    char *s = scratch + soff[q];                              // full loop string
    for (int i = 0; i < K; ++i) s[i] = "ACGT"[kmer_nuc<NW>(cur, i)];
    for (uint32_t i = 0; i < li.nverts; ++i) {
        const uint8_t m = oriented_mask<NW>(mk, masks, cur, K);
        const int ch = uniq4(m & 15);
        s[K + i] = "ACGT"[ch];
        kmer_shl<NW>(cur, K, ch);
    }
    if (li.split < 0) {
        char *d = o.seq + eoff[2 * q];
        for (uint32_t i = 0; i < n; ++i) d[i] = s[i];
        finish_edge<NW, NWS>(d, n, K, eidx[2 * q], mk, mkp, cov, o);
    } else {
        const uint32_t pos = (uint32_t)li.split;
        char *d0 = o.seq + eoff[2 * q];
        for (uint32_t i = 0; i < (uint32_t)K + 1; ++i) d0[i] = s[pos + i];
        finish_edge<NW, NWS>(d0, (uint32_t)K + 1, K, eidx[2 * q], mk, mkp, cov, o);
        char *d1 = o.seq + eoff[2 * q + 1];
        uint32_t w = 0;
        for (uint32_t i = pos + 1; i < n - K; ++i) d1[w++] = s[i];
        for (uint32_t i = 0; i < pos + K; ++i) d1[w++] = s[i];
        finish_edge<NW, NWS>(d1, w, K, eidx[2 * q + 1], mk, mkp, cov, o);
    }
}

// ---- host orchestration ----------------------------------------------------------------------------------------------
// the keys of a sweep's flagged records, in final_kmers order, as one compacted list per chunk that has any (so they are never
// held twice, as a join would)
struct KeyParts {
    std::vector<DArr<uint64_t>> parts;
    std::vector<uint64_t> sizes;
    uint64_t total = 0;
};
// per chunk: flags -> scan -> compacted keys. flags(ch, keys, flag) launches one kernel that fills flag[0, ch.n).
template <int NW, class Flags>
static KeyParts collect_keys(Ctx *ctx, ChunkStager &src, Flags &&flags) {
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

// the text, link records and raw coverage of a batch of edges, as the kernels write them (EdgeOut)
struct EdgeBatch {
    uint64_t n, bases;
    DArr<char> seq;
    DArr<uint64_t> link_start, link_end;
    DArr<uint32_t> raw_cov;
    EdgeBatch(Ctx *ctx, uint64_t n_, uint64_t bases_)
        : n(n_), bases(bases_), seq(ctx, bases_ + 1), link_start(ctx, n_ + 1), link_end(ctx, n_ + 1), raw_cov(ctx, n_ + 1) {}
    EdgeOut out(uint8_t *visited) const { return EdgeOut{seq.p, link_start.p, link_end.p, raw_cov.p, visited}; }
    // appends the batch to g's edges. Its (offset, length) table has n entries, offsets into the batch's text, in device or host
    // memory (cudaMemcpyDefault); the offsets are rebased onto g->seq.
    void append(Graph *g, cudaStream_t st, const uint64_t *off, const uint32_t *len) const {
        const size_t e0 = g->edge_len.size(), b0 = g->seq.size();
        g->edge_off.resize(e0 + n); g->edge_len.resize(e0 + n);
        g->link_start.resize(e0 + n); g->link_end.resize(e0 + n); g->raw_cov.resize(e0 + n);
        g->seq.resize(b0 + bases);
        if (n) {
            SG_CUDA(cudaMemcpyAsync(g->edge_off.data() + e0, off, n * 8, cudaMemcpyDefault, st));
            SG_CUDA(cudaMemcpyAsync(g->edge_len.data() + e0, len, n * 4, cudaMemcpyDefault, st));
            SG_CUDA(cudaMemcpyAsync(g->link_start.data() + e0, link_start.p, n * 8, cudaMemcpyDeviceToHost, st));
            SG_CUDA(cudaMemcpyAsync(g->link_end.data() + e0, link_end.p, n * 8, cudaMemcpyDeviceToHost, st));
            SG_CUDA(cudaMemcpyAsync(g->raw_cov.data() + e0, raw_cov.p, n * 4, cudaMemcpyDeviceToHost, st));
        }
        if (bases) SG_CUDA(cudaMemcpyAsync(&g->seq[b0], seq.p, bases, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        for (size_t e = e0; e < e0 + n; ++e) g->edge_off[e] += b0;
    }
};

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
        tc_apply_k<<<div_up((int64_t)nk, 256), 256, 0, st>>>(g->masks.p, mark, nk);
        ctx->launches++;
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
        AtParams ap; ap.ratio = opt.at_ratio; ap.min_len = (uint32_t)std::min<uint64_t>(opt.at_min_len, 0x7fffffffu); ap.max_len = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(opt.at_max_len, 1), 0x7fffffffu);
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
        const uint32_t bound = (uint32_t)std::min<uint64_t>(opt.early_tip_length_bound, 0x7fffffffu);
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
        KeyParts jk = collect_keys<NW>(ctx, *kmers, [&](const Chunk &c, const uint64_t *keys, uint32_t *flag) {
            junction_flags_k<NW><<<div_up(c.n, 256), 256, 0, st>>>(keys, c.n, K, mk, g->masks.p, flag);
        });
        tr.mark("junction list");
        return jk;
    }

    // unbranching paths, in batches of junctions (never across two chunks' lists) sized from the room left: the 8 slots of a
    // junction cost len + keepf + selfc + eidx + eoff + the compacted (offset, length) = 37 bytes each. The unitig text and link
    // records of a batch depend on its paths' lengths, not on its junctions: they are reckoned at as much again, a heuristic, and a
    // batch whose text needs more still runs (blocks beyond the arena come from the driver). Edge numbers and text offsets carry
    // over from batch to batch.
    void unitigs(KeyParts jk) {
        visited.alloc(ctx, nk + 8);
        SG_CUDA(cudaMemsetAsync(visited.p, 0, visited.bytes(), st));
        const uint64_t per_junc = 2 * 8 * 37;
        const uint64_t jbatch = std::max<uint64_t>(4096, ctx->budget_left() / 2 / per_junc);
        uint64_t batches = 0;
        for (size_t part = 0; part < jk.parts.size(); ++part)
        for (uint64_t q0 = 0, njunc = jk.sizes[part]; q0 < njunc; q0 += jbatch) {
            const uint64_t nj = std::min(jbatch, njunc - q0);
            const uint64_t nslots = nj * 8;
            ++batches;
            DArr<uint32_t> len(ctx, nslots + 1), keepf(ctx, nslots + 1);
            DArr<uint8_t> selfc(ctx, nslots + 1);
            DArr<uint64_t> eidx(ctx, nslots + 1), eoff(ctx, nslots + 1);
            SG_CUDA(cudaMemsetAsync(len.p, 0, len.bytes(), st));
            const uint64_t *bkeys = jk.parts[part].p + q0 * NW;
            unitig_probe_k<NW><<<div_up((int64_t)nslots, 128), 128, 0, st>>>(bkeys, (int64_t)nj, K, mk, g->masks.p, nk, len.p, selfc.p);
            ctx->launches++;
            SG_CUDA(cudaGetLastError());
            exclusive_scan_u32_to_u64(ctx, len.p, eoff.p, nslots + 1);
            // edge index = rank among kept slots
            launch_nonzero_flags(ctx, len.p, keepf.p, nslots + 1);
            exclusive_scan_u32_to_u64(ctx, keepf.p, eidx.p, nslots + 1);
            uint64_t npaths = 0, nbases = 0;
            SG_CUDA(cudaMemcpyAsync(&npaths, eidx.p + nslots, 8, cudaMemcpyDeviceToHost, st));
            SG_CUDA(cudaMemcpyAsync(&nbases, eoff.p + nslots, 8, cudaMemcpyDeviceToHost, st));
            SG_CUDA(cudaStreamSynchronize(st));
            tr.mark("unitig probe + offsets");
            EdgeBatch eb(ctx, npaths, nbases);
            unitig_write_k<NW, NWS><<<div_up((int64_t)nslots, 128), 128, 0, st>>>(bkeys, (int64_t)nj, K, mk, g->masks.p, nk, len.p, selfc.p, eidx.p,
                                                                                 eoff.p, mkp, g->cov.p, eb.out(visited.p));
            ctx->launches++;
            SG_CUDA(cudaGetLastError());
            tr.mark("unitig write");
            // the (offset, length) table is compacted on the device (8 slots per junction, most of them empty)
            DArr<uint64_t> c_off(ctx, npaths + 1);
            DArr<uint32_t> c_len(ctx, npaths + 1);
            edge_table_k<<<div_up((int64_t)nslots, 256), 256, 0, st>>>(len.p, eidx.p, eoff.p, (int64_t)nslots, c_off.p, c_len.p);
            ctx->launches++;
            eb.append(g, st, c_off.p, c_len.p);
            if (q0 + nj == njunc) jk.parts[part].release();
            tr.mark("download + edge table");
        }
        ctx->times.graph_junction_batches = batches;
    }

    // perfect loops: the k-mers that are left with one edge in and one out once the paths are removed
    void loops() {
        DArr<unsigned long long> d_rem(ctx, 1);
        SG_CUDA(cudaMemsetAsync(d_rem.p, 0, 8, st));
        const uint64_t nwords = (nk + 31) / 32;
        DArr<uint32_t> rem_bits(ctx, nwords + 1);
        masks_clear_visited_k<<<div_up((int64_t)nk, 256), 256, 0, st>>>(g->masks.p, visited.p, nk, d_rem.p, rem_bits.p);
        ctx->launches++;
        unsigned long long rem = 0;
        SG_CUDA(cudaMemcpyAsync(&rem, d_rem.p, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        if (!rem) return;
        // final_kmers positions of the remaining slots only (RemSlots): the loop kernels never need 8 B per k-mer
        DArr<uint64_t> rem_base(ctx, nwords + 1), rem_pos(ctx, rem);
        {
            DArr<uint32_t> cnt(ctx, nwords + 1);
            SG_CUDA(cudaMemsetAsync(cnt.p + nwords, 0, 4, st));
            popc_words_k<<<div_up((int64_t)nwords, 256), 256, 0, st>>>(rem_bits.p, nwords, cnt.p);
            ctx->launches++;
            exclusive_scan_u32_to_u64(ctx, cnt.p, rem_base.p, nwords + 1);
            SG_CUDA(cudaStreamSynchronize(st));
        }
        RemSlots rs; rs.bits = rem_bits.p; rs.base = rem_base.p;
        kmer_sweep([&](const Chunk &c, const uint64_t *keys) {
            loop_pos_k<NW><<<div_up(c.n, 256), 256, 0, st>>>(keys, c.first, c.n, mk, rs, rem_pos.p);
        });
        KeyParts lk = collect_keys<NW>(ctx, *kmers, [&](const Chunk &c, const uint64_t *keys, uint32_t *flag) {
            loop_leader_k<NW><<<div_up(c.n, 128), 128, 0, st>>>(keys, c.first, c.n, nk, K, mk, g->masks.p, rs, rem_pos.p, flag);
        });
        rem_pos.release(); rem_base.release(); rem_bits.release();
        const uint64_t nl = lk.total;
        if (!nl) return;
        // the leaders as one list (loops are rare, a few keys)
        DArr<uint64_t> leaders(ctx, (size_t)nl * NW);
        for (size_t i = 0, at = 0; i < lk.parts.size(); at += lk.sizes[i], ++i)
            SG_CUDA(cudaMemcpyAsync(leaders.p + at * NW, lk.parts[i].p, lk.sizes[i] * NW * 8, cudaMemcpyDeviceToDevice, st));
        DArr<LoopInfo> info(ctx, nl);
        DArr<uint32_t> llen(ctx, 2 * nl + 1), lkeep(ctx, 2 * nl + 1), sfull(ctx, nl + 1);
        DArr<uint64_t> leidx(ctx, 2 * nl + 1), leoff(ctx, 2 * nl + 1), soff(ctx, nl + 1);
        SG_CUDA(cudaMemsetAsync(llen.p, 0, llen.bytes(), st));
        loop_probe_k<NW, NWS><<<div_up((int64_t)nl, 64), 64, 0, st>>>(leaders.p, (int64_t)nl, K, mk, g->masks.p, info.p, llen.p);
        ctx->launches++;
        launch_nonzero_flags(ctx, llen.p, lkeep.p, 2 * nl + 1);
        exclusive_scan_u32_to_u64(ctx, llen.p, leoff.p, 2 * nl + 1);
        exclusive_scan_u32_to_u64(ctx, lkeep.p, leidx.p, 2 * nl + 1);
        std::vector<uint32_t> h_llen(2 * nl + 1);
        std::vector<LoopInfo> h_info(nl);
        uint64_t nledges = 0, nlbases = 0;
        SG_CUDA(cudaMemcpyAsync(h_llen.data(), llen.p, (2 * nl + 1) * 4, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaMemcpyAsync(h_info.data(), info.p, nl * sizeof(LoopInfo), cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaMemcpyAsync(&nledges, leidx.p + 2 * nl, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaMemcpyAsync(&nlbases, leoff.p + 2 * nl, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        std::vector<uint64_t> h_soff(nl + 1, 0);
        for (uint64_t q = 0; q < nl; ++q) h_soff[q + 1] = h_soff[q] + (uint64_t)K + h_info[q].nverts;
        SG_CUDA(cudaMemcpyAsync(soff.p, h_soff.data(), (nl + 1) * 8, cudaMemcpyHostToDevice, st));
        DArr<char> scratch(ctx, h_soff[nl] + 1);
        EdgeBatch eb(ctx, nledges, nlbases);
        loop_write_k<NW, NWS><<<div_up((int64_t)nl, 64), 64, 0, st>>>(info.p, (int64_t)nl, K, mk, g->masks.p, llen.p, leidx.p, leoff.p, mkp,
                                                                     g->cov.p, eb.out(visited.p), scratch.p, soff.p);
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
        // the (offset, length) table from the probe's lengths: a loop is one edge, or two where it splits
        std::vector<uint64_t> off;
        std::vector<uint32_t> len;
        for (uint64_t i = 0, at = 0; i < 2 * nl; at += h_llen[i++])
            if (h_llen[i]) { off.push_back(at); len.push_back(h_llen[i]); }
        eb.append(g, st, off.data(), len.data());
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
