// graph_dev.cuh -- the unitig and perfect-loop walks over an index *view*, shared by the single-GPU graph build (graph.cu) and
// the distributed one (dist_graph.cu). A walk needs three things of a k-mer: its slot (through its minimal form), the mask byte
// there, and a place to mark it visited; and the coverage of a (k+1)-mer. A view gives them:
//   LocalView  one GPU: the k-mer index (MphfDev), masks, visited, the (k+1)-mer index and coverage, the remaining-slot tables.
//   DistView   one rank of many: a bucket's owner, the owner's index rows (copied locally) and its arrays as this process maps them.
// The walk bodies are device functions templated on the view; each translation unit wraps them in kernels of its own.
#pragma once
#include <algorithm>
#include <functional>

#include "graph.h"
#include "mphf_dev.cuh"

namespace sg {

__device__ __forceinline__ uint8_t inv_byte(uint8_t a) { return (uint8_t)(__brev((unsigned)a) >> 24); }   // inout_mask.hpp:18-27
__device__ __forceinline__ int uniq4(unsigned m) {           // inout_mask.hpp:61-81 (CheckUnique/GetUnique), -1 if not unique
    return (m && !(m & (m - 1))) ? (__ffs(m) - 1) : -1;
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

// DeleteOutgoing / DeleteIncoming: clears bit `bit` of mask byte idx with a 32-bit atomic on the word that holds it
__device__ __forceinline__ void mask_clear_bit(uint8_t *masks, uint64_t idx, unsigned bit) {
    atomicAnd(reinterpret_cast<unsigned *>(masks) + (idx >> 2), ~((1u << bit) << (8 * (idx & 3))));
}

// ---- views -----------------------------------------------------------------------------------------------------------------
// Ref: where a k-mer's byte lives. slot(key of minimal form) -> Ref; mask / visit / rem_rank / rem_pos read or mark it;
// link_idx(Ref) is the slot a link record carries; upos(Ref, p) turns the final_kmers position p of that k-mer in the set that
// holds it into its position in the union's; lost(m): the walk cannot go on from mask m (only a view that can miss says so).
// The early clippers' flags: mark(Ref) sets a k-mer's IsolateVertex flag, root(Ref, o) / is_root the flag of the (slot,
// orientation) a clipped A/T tip hangs from, eflag / set_eflag the A/T edge flags of a (slot, orientation), clear_bit(Ref, bit)
// deletes one edge of a k-mer's mask.
struct LocalView {
    MphfDev mk;
    const uint8_t *masks;
    MphfDev mkp;
    const uint32_t *cov;       // null: no coverage
    uint8_t *visited;
    RemSlots rs;
    const uint64_t *pos;
    uint8_t *marks;            // the clippers' flags, per slot (marks) or per (slot, orientation)
    uint8_t *eflags;
    uint8_t *roots;
    typedef uint64_t Ref;
    template <int NW>
    __device__ __forceinline__ Ref slot(const Kmer<NW> &key) const { return mphf_lookup_dev<NW>(mk, key); }
    __device__ __forceinline__ uint8_t mask(Ref r) const { return masks[r]; }
    __device__ __forceinline__ uint64_t link_idx(Ref r) const { return r; }
    __device__ __forceinline__ void visit(Ref r) const { visited[r] = 1; }
    __device__ __forceinline__ bool with_cov() const { return cov; }
    template <int NWS>
    __device__ __forceinline__ uint32_t cov_of(const Kmer<NWS> &x) const { return cov[mphf_lookup_dev<NWS>(mkp, x)]; }
    __device__ __forceinline__ uint64_t rem_rank(Ref r) const { return rs.rank(r); }
    __device__ __forceinline__ uint64_t rem_pos(Ref, uint64_t rk) const { return pos[rk]; }
    __device__ __forceinline__ uint64_t upos(Ref, uint64_t p) const { return p; }
    __device__ __forceinline__ bool lost(uint8_t) const { return false; }
    __device__ __forceinline__ void mark(Ref r) const { marks[r] = 1; }
    __device__ __forceinline__ void root(Ref r, int o) const { roots[2 * r + o] = 1; }
    __device__ __forceinline__ bool is_root(Ref r, int o) const { return roots[2 * r + o]; }
    __device__ __forceinline__ uint8_t eflag(Ref r, int o) const { return eflags[2 * r + o]; }
    __device__ __forceinline__ void set_eflag(Ref r, int o, uint8_t f) const { eflags[2 * r + o] = f; }
    // only the clippers clear bits, and their kernels own a writable mask array
    __device__ __forceinline__ void clear_bit(Ref r, unsigned bit) const { mask_clear_bit(const_cast<uint8_t *>(masks), r, bit); }
};

// one rank's arrays as this process maps them (its own arena, or a peer's through cudaIpc)
struct DistPeer {
    const uint64_t *bits, *ranks;          // its k-mer index
    uint8_t *masks;                        // its mask slice (the clippers' and the walks' working copy)
    uint8_t *visited;                      // its visited slice
    const uint64_t *pbits, *pranks;        // its (k+1)-mer index
    const uint32_t *cov;                   // its coverage slice
    const uint32_t *rem_bits;              // its remaining-slot tables (RemSlots) and their final_kmers positions
    const uint64_t *rem_base, *rem_pos;
    uint8_t *mark, *eflag, *rooted;        // its clipper flags: per owned slot, per (owned slot, orientation) twice
};
// A k-mer's bucket b names its owner; the owner's index rows of bucket b (dom, woff for every level, its first slot lstart[b])
// are copied here, so a lookup reads only the owner's bits and ranks remotely. The union's slot and final_kmers position are the
// owner's shifted by ustart[b] - lstart[b]. A lookup no level answers counts in *err and ends the walk. The clippers' stores and
// bit clears act on the owner's slice; those that land in another rank's slice are counted in remote[0, 3) (marks, roots, clears).
struct DistView {
    const DistPeer *peers;
    const int *owner, *powner;             // B: owner of each k-mer bucket, of each (k+1)-mer bucket
    const uint64_t *dom, *woff, *lstart, *ustart;     // k-mer index rows (kLevels x B, B, B)
    const uint64_t *pdom, *pwoff, *pstart;            // (k+1)-mer index rows
    uint32_t B;
    bool have_cov;
    unsigned long long *err;
    int self;                              // this rank
    unsigned long long *remote;
    struct Ref { uint64_t slot; uint32_t b; int g; };   // slot: in the owner's index, ~0 after a miss
    template <int NW>
    __device__ __forceinline__ Ref slot(const Kmer<NW> &key) const {
        Ref r;
        r.b = kmer_bucket<NW>(key, B);
        r.g = owner[r.b];
        const MphfDev m{dom, woff, lstart, const_cast<uint64_t *>(peers[r.g].bits), peers[r.g].ranks, B};
        r.slot = mphf_lookup_dev<NW>(m, key, r.b);
        if (r.slot == ~0ull) atomicAdd(err, 1ull);
        return r;
    }
    __device__ __forceinline__ uint8_t mask(const Ref &r) const { return r.slot == ~0ull ? 0 : peers[r.g].masks[r.slot]; }
    __device__ __forceinline__ uint64_t link_idx(const Ref &r) const { return ustart[r.b] + (r.slot - lstart[r.b]); }
    __device__ __forceinline__ void visit(const Ref &r) const { if (r.slot != ~0ull) peers[r.g].visited[r.slot] = 1; }
    __device__ __forceinline__ bool with_cov() const { return have_cov; }
    template <int NWS>
    __device__ __forceinline__ uint32_t cov_of(const Kmer<NWS> &x) const {
        const uint32_t b = kmer_bucket<NWS>(x, B);
        const int g = powner[b];
        const MphfDev m{pdom, pwoff, pstart, const_cast<uint64_t *>(peers[g].pbits), peers[g].pranks, B};
        const uint64_t s = mphf_lookup_dev<NWS>(m, x, b);
        if (s == ~0ull) { atomicAdd(err, 1ull); return 0; }
        return peers[g].cov[s];
    }
    __device__ __forceinline__ uint64_t rem_rank(const Ref &r) const {
        if (r.slot == ~0ull) return ~0ull;
        const RemSlots rs{peers[r.g].rem_bits, peers[r.g].rem_base};
        return rs.rank(r.slot);
    }
    __device__ __forceinline__ uint64_t rem_pos(const Ref &r, uint64_t rk) const { return upos(r, peers[r.g].rem_pos[rk]); }
    __device__ __forceinline__ uint64_t upos(const Ref &r, uint64_t p) const { return ustart[r.b] + (p - lstart[r.b]); }
    __device__ __forceinline__ bool lost(uint8_t m) const { return uniq4(m & 15) < 0; }
    __device__ __forceinline__ void mark(const Ref &r) const {
        if (r.slot == ~0ull) return;
        peers[r.g].mark[r.slot] = 1;
        if (r.g != self) atomicAdd(&remote[0], 1ull);
    }
    __device__ __forceinline__ void root(const Ref &r, int o) const {
        if (r.slot == ~0ull) return;
        peers[r.g].rooted[2 * r.slot + o] = 1;
        if (r.g != self) atomicAdd(&remote[1], 1ull);
    }
    __device__ __forceinline__ bool is_root(const Ref &r, int o) const { return r.slot != ~0ull && peers[r.g].rooted[2 * r.slot + o]; }
    __device__ __forceinline__ uint8_t eflag(const Ref &r, int o) const { return r.slot == ~0ull ? 0 : peers[r.g].eflag[2 * r.slot + o]; }
    __device__ __forceinline__ void set_eflag(const Ref &r, int o, uint8_t f) const { if (r.slot != ~0ull) peers[r.g].eflag[2 * r.slot + o] = f; }
    // across devices, a 32-bit atomic on a peer's memory needs native peer atomics (dgraph_open_peers checks them)
    __device__ __forceinline__ void clear_bit(const Ref &r, unsigned bit) const {
        if (r.slot == ~0ull) return;
        mask_clear_bit(peers[r.g].masks, r.slot, bit);
        if (r.g != self) atomicAdd(&remote[2], 1ull);
    }
};

// ---- lookups through a view --------------------------------------------------------------------------------------------------
template <class V>
struct CanonIdx { typename V::Ref idx; bool is_min; };

template <int NW, class V>
__device__ __forceinline__ CanonIdx<V> canon_lookup(const V &v, const Kmer<NW> &k, int K) {
    Kmer<NW> r = kmer_rc<NW>(k, K);
    CanonIdx<V> c;
    c.is_min = kmer_is_minimal<NW>(k, r);          // key_with_hash.hpp:120-128
    c.idx = v.template slot<NW>(c.is_min ? k : r);
    return c;
}
// get_value(kwh): InvertableStoring::get_value with InOutMask::conjugate (storing_traits.hpp:44-51)
template <int NW, class V>
__device__ __forceinline__ uint8_t oriented_mask(const V &v, const Kmer<NW> &k, int K, typename V::Ref *idx_out = nullptr) {
    CanonIdx<V> c = canon_lookup<NW>(v, k, K);
    if (idx_out) *idx_out = c.idx;
    uint8_t m = v.mask(c.idx);
    return c.is_min ? m : inv_byte(m);
}
// the coverage of (k+1)-mer v + nextc
template <int NW, int NWS, class V>
__device__ __forceinline__ uint32_t kpomer_cov(const V &vw, const Kmer<NW> &v, int nextc, int K) {
    Kmer<NWS> x;
#pragma unroll
    for (int q = 0; q < NWS; ++q) x.w[q] = q < NW ? v.w[q] : 0;
    x.w[K >> 5] |= (uint64_t)nextc << ((K & 31) << 1);
    Kmer<NWS> r = kmer_rc<NWS>(x, K + 1);
    return vw.template cov_of<NWS>(kmer_is_minimal<NWS>(x, r) ? x : r);
}

__device__ __forceinline__ uint64_t link_value(uint64_t idx, bool is_start, bool is_rc) { return (idx << 2) | (is_rc ? 2ull : 0ull) | (is_start ? 1ull : 0ull); }

struct EdgeOut {
    char *seq;                 // ASCII bases, all edges concatenated
    uint64_t *link_start;      // LinkRecord hash_and_mask of StartLink / EndLink (:455-471)
    uint64_t *link_end;
    uint32_t *raw_cov;         // sum of (k+1)-mer multiplicities along the edge
    uint8_t *visited;          // per k-mer MPHF index (LocalView's)
};

// ---- unbranching paths ---------------------------------------------------------------------------------------------------
// walk from `start` along out-edge c until a junction (ConstructSequenceWithEdge :264-273). Calls f(vertex index i>=1, k-mer) per vertex.
template <int NW, class V, class F>
__device__ __forceinline__ uint32_t walk_right(const V &vw, int K, const Kmer<NW> &start, int c, uint64_t max_steps, F &&f,
                                               Kmer<NW> *end_out, Kmer<NW> *prev_out) {
    Kmer<NW> prev = start, cur = start;
    kmer_shl<NW>(cur, K, c);
    uint32_t m = 1;
    f(m, cur);
    for (;;) {
        const uint8_t msk = oriented_mask<NW>(vw, cur, K);
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
template <int NW, class V>
__device__ __forceinline__ void unitig_probe(V vw, const uint64_t *jkeys, int64_t njunc, int K, uint64_t nk,
                                             uint32_t *len /*[njunc*8] 0 = none*/, uint8_t *selfc) {
    int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= njunc * 8) return;
    const int64_t q = tid >> 3;
    const int side = (int)(tid >> 2) & 1, c = (int)tid & 3;
    const Kmer<NW> key = key_at<NW>(jkeys, q);
    const uint8_t mfw = vw.mask(vw.template slot<NW>(key));
    const Kmer<NW> start = side ? kmer_rc<NW>(key, K) : key;          // AddStartDeEdges :214-235
    const uint8_t m = side ? inv_byte(mfw) : mfw;
    len[tid] = 0; selfc[tid] = 0;
    if (!(m & (1u << c))) return;
    Kmer<NW> end, prev;
    auto nop = [](uint32_t, const Kmer<NW> &) {};
    const uint32_t steps = walk_right<NW>(vw, K, start, c, nk + 1, nop, &end, &prev);
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
                const uint8_t ma = oriented_mask<NW>(vw, a, K);
                kmer_shl<NW>(a, K, uniq4(ma & 15));
                if (i + 2 < steps) {                 // b = v_{steps-2-i} is needed next; v_0 = start has no unique-in guarantee, use it directly
                    const uint8_t mb = oriented_mask<NW>(vw, b, K);
                    kmer_shr<NW>(b, K, uniq4(mb >> 4));
                } else b = start;
            }
        }
    }
    if (keep) { len[tid] = (uint32_t)K + steps; selfc[tid] = self ? 1 : 0; }
}

template <int NW, int NWS, class V>
__device__ __forceinline__ void unitig_write(V vw, const uint64_t *jkeys, int64_t njunc, int K, uint64_t nk,
                                             const uint32_t *len, const uint8_t *selfc, const uint64_t *eidx,
                                             const uint64_t *eoff, const EdgeOut &o) {
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
    {
        CanonIdx<V> ci = canon_lookup<NW>(vw, start, K);
        vw.visit(ci.idx);
        o.link_start[e] = link_value(vw.link_idx(ci.idx), true, !ci.is_min);
    }
    uint32_t raw = 0;
    Kmer<NW> pv = start;
    auto emit = [&](uint32_t i, const Kmer<NW> &v) {
        const int ch = kmer_nuc<NW>(v, K - 1);
        out[K - 1 + i] = "ACGT"[ch];
        typename V::Ref idx;
        oriented_mask<NW>(vw, v, K, &idx);
        vw.visit(idx);
        if (vw.with_cov()) raw += kpomer_cov<NW, NWS>(vw, pv, ch, K);
        pv = v;
    };
    Kmer<NW> end, prev;
    walk_right<NW>(vw, K, start, c, nk + 1, emit, &end, &prev);
    if (selfc[tid]) o.link_end[e] = ~0ull;                 // LinkRecord() for self-conjugate edges (:481-484)
    else {
        CanonIdx<V> ci = canon_lookup<NW>(vw, end, K);
        o.link_end[e] = link_value(vw.link_idx(ci.idx), false, !ci.is_min);
    }
    o.raw_cov[e] = raw;
}

// ---- perfect loops (CollectLoops :359-397). Rare; one thread per candidate / per loop is enough. ---------------------
// leader of a loop = its vertex with the smallest final_kmers position in the union (where the serial scan first meets it)
// (is_leader: per record of the chunk; nk: all k-mers, the bound of a loop's length)
template <int NW, class V>
__device__ __forceinline__ void loop_leader(V vw, const uint64_t *keys, int64_t base, int64_t n, uint64_t nk, int K,
                                            uint32_t *is_leader) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    is_leader[j] = 0;
    const Kmer<NW> key = key_at<NW>(keys, j);
    typename V::Ref idx0;
    uint8_t m = oriented_mask<NW>(vw, key, K, &idx0);
    if (!m || uniq4(m & 15) < 0 || uniq4(m >> 4) < 0) return;
    Kmer<NW> cur = key;
    bool leader = true;
    for (uint64_t it = 0; it <= nk; ++it) {
        kmer_shl<NW>(cur, K, uniq4(m & 15));
        if (kmer_eq<NW>(cur, key)) break;
        typename V::Ref idx;
        m = oriented_mask<NW>(vw, cur, K, &idx);
        if (vw.lost(m)) { leader = false; break; }
        // a loop's vertices are all remaining slots (every other vertex was a junction, a dead end or visited by a path)
        const uint64_t rk = vw.rem_rank(idx);
        if (rk != ~0ull && vw.rem_pos(idx, rk) < vw.upos(idx0, (uint64_t)(base + j))) { leader = false; break; }
    }
    is_leader[j] = leader ? 1u : 0u;
}

// per leader: break point (FindMinimalKMerInLoop :252-262), loop length, self-RC split position (ConstructLoopFromVertex :283-293)
struct LoopInfo { uint64_t w[4]; uint32_t nverts; int32_t split; };
template <int NW, int NWS, class V>
__device__ __forceinline__ void loop_probe(V vw, const uint64_t *leaders /*keys*/, int64_t nl, int K,
                                           LoopInfo *info, uint32_t *len /*[nl*2]*/) {
    int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nl) return;
    const Kmer<NW> key = key_at<NW>(leaders, q);
    Kmer<NW> minimal = key, r = kmer_rc<NW>(key, K);
    if (kmer_nuc_less<NW>(r, minimal)) minimal = r;
    Kmer<NW> cur = key;
    uint32_t nv = 0;
    do {
        const uint8_t m = oriented_mask<NW>(vw, cur, K);
        if (vw.lost(m)) break;
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
        const uint8_t m = oriented_mask<NW>(vw, cur, K);
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

template <int NW, int NWS, class V>
__device__ void finish_edge(char *s, uint32_t n, int K, uint64_t e, const V &vw, const EdgeOut &o) {
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
    CanonIdx<V> ca = canon_lookup<NW>(vw, a, K);
    o.link_start[e] = link_value(vw.link_idx(ca.idx), true, !ca.is_min);
    if (self) o.link_end[e] = ~0ull;
    else {
        CanonIdx<V> cb = canon_lookup<NW>(vw, b, K);
        o.link_end[e] = link_value(vw.link_idx(cb.idx), false, !cb.is_min);
    }
    uint32_t raw = 0;
    if (vw.with_cov()) {
        Kmer<NW> v = a;
        for (uint32_t p = (uint32_t)K; p < n; ++p) {
            const int ch = code(s[p]);
            raw += kpomer_cov<NW, NWS>(vw, v, ch, K);
            kmer_shl<NW>(v, K, ch);
        }
    }
    o.raw_cov[e] = raw;
}

template <int NW, int NWS, class V>
__device__ __forceinline__ void loop_write(V vw, const LoopInfo *info, int64_t nl, int K, const uint32_t *len,
                                           const uint64_t *eidx, const uint64_t *eoff, const EdgeOut &o,
                                           char *scratch, const uint64_t *soff) {
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
        const uint8_t m = oriented_mask<NW>(vw, cur, K);
        const int ch = uniq4(m & 15);
        s[K + i] = "ACGT"[ch];
        kmer_shl<NW>(cur, K, ch);
    }
    if (li.split < 0) {
        char *d = o.seq + eoff[2 * q];
        for (uint32_t i = 0; i < n; ++i) d[i] = s[i];
        finish_edge<NW, NWS>(d, n, K, eidx[2 * q], vw, o);
    } else {
        const uint32_t pos = (uint32_t)li.split;
        char *d0 = o.seq + eoff[2 * q];
        for (uint32_t i = 0; i < (uint32_t)K + 1; ++i) d0[i] = s[pos + i];
        finish_edge<NW, NWS>(d0, (uint32_t)K + 1, K, eidx[2 * q], vw, o);
        char *d1 = o.seq + eoff[2 * q + 1];
        uint32_t w = 0;
        for (uint32_t i = pos + 1; i < n - K; ++i) d1[w++] = s[i];
        for (uint32_t i = 0; i < pos + K; ++i) d1[w++] = s[i];
        finish_edge<NW, NWS>(d1, w, K, eidx[2 * q + 1], vw, o);
    }
}

// ---- early tip clipper -------------------------------------------------------------------------------------------------
// EarlyTipClipperProcessor (assembly_graph/construction/early_simplification.hpp:38-162), run by the pipeline between the
// mask fill and the unitig extraction (stages/construction.cpp:289-302, length bound = read length - k). The reference walks
// the junctions one after the other (or racily from several threads) on the live index; the result does not depend on the
// order (a tip's vertices are reachable from exactly one junction orientation and removals only zero tip vertices -- checked
// against the unmodified reference with 1 and 8 threads and against the oracle's sequential and snapshot modes, tests/), so
// here every (k-mer, orientation) with >= 2 outgoing edges is one thread on a snapshot of the masks:
//   tc_probe   FindForward per outgoing edge (:115-125), RemoveTips decision (:133-155), marks the vertices to isolate
//   tc_apply_k IsolateVertex for the marked vertices (graph.cu, over one array of marks)
//   tc_links   RemoveInconsistentForwardLinks over the tipped junctions (:21-36) on the updated masks
template <int NW, bool MARK, class V>
__device__ __forceinline__ uint32_t tc_find_forward(const V &v, int K, Kmer<NW> kh, uint32_t bound) {
    uint32_t n = 0;
    for (;;) {
        typename V::Ref idx;
        const uint8_t m = oriented_mask<NW>(v, kh, K, &idx);
        const int uo = uniq4(m & 15), ui = uniq4(m >> 4);
        if (MARK) v.mark(idx);
        if (!(n < bound && ui >= 0 && uo >= 0)) {
            ++n;                                                 // tip.push_back(kh) after the loop (:121)
            return (ui < 0 || (m & 15) != 0) ? 0u : n;           // branching / not a dead end -> not a tip (:122-125)
        }
        ++n;
        kmer_shl<NW>(kh, K, uo);
    }
}
// tipped: per (k-mer position of the keys' set, orientation), base = the position of keys[0]
template <int NW, class V>
__device__ __forceinline__ void tc_probe(const V &v, const uint64_t *keys, int64_t base, int64_t n, int K, uint32_t bound, uint8_t *tipped,
                                         unsigned long long *stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    tipped += 2 * base;
    const int o = (int)(tid & 1);
    const uint8_t mfw = v.mask(v.template slot<NW>(key));
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
        sz[c] = tc_find_forward<NW, false>(v, K, khc, bound);
        const uint32_t len = sz[c] ? sz[c] : 0xffffffffu;
        if (len > mx) mx = len;
    }
    uint32_t removed = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (!sz[c] || sz[c] >= mx) continue;                     // RemoveTips: tip.size() < max (:136-141)
        Kmer<NW> khc = kh;
        kmer_shl<NW>(khc, K, c);
        tc_find_forward<NW, true>(v, K, khc, bound);
        removed += sz[c];
    }
    if (removed) { tipped[tid] = 1; atomicAdd(&stats[0], (unsigned long long)removed); atomicAdd(&stats[1], 1ull); }
}
// flags_by_slot = 0: tipped[] is indexed by (k-mer position, orientation), as tc_probe writes it; 1: the view's root flags, by
// (slot, orientation), as at_tips_probe sets them by walking. The bits it clears are those of its own k-mer.
template <int NW, class V>
__device__ __forceinline__ void tc_links(const V &v, const uint64_t *keys, int64_t base, int64_t n, int K, const uint8_t *tipped,
                                         unsigned long long *stat_clipped, int flags_by_slot) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    if (!flags_by_slot && !tipped[2 * base + tid]) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const Kmer<NW> kh = (tid & 1) ? kmer_rc<NW>(key, K) : key;
    const CanonIdx<V> ci = canon_lookup<NW>(v, kh, K);
    if (flags_by_slot && !v.is_root(ci.idx, (int)(tid & 1))) return;
    const uint8_t raw = v.mask(ci.idx);
    const uint8_t m = ci.is_min ? raw : inv_byte(raw);
    const int first = (int)(kh.w[0] & 3);                        // kh[0]
    for (int c = 0; c < 4; ++c) {
        if (!(m & (1u << c))) continue;
        Kmer<NW> nx = kh;
        kmer_shl<NW>(nx, K, c);
        if (!(oriented_mask<NW>(v, nx, K) & (1u << (4 + first)))) {                  // !CheckIncoming(next_kh, kh[0])
            v.clear_bit(ci.idx, (unsigned)(ci.is_min ? c : 7 - c));                  // DeleteOutgoing(kh, c), inout_mask.hpp:108-114
            atomicAdd(stat_clipped, 1ull);
        }
    }
}

// ---- early low-complexity (poly A/T) clipper ----------------------------------------------------------------------------------
// EarlyLowComplexityClipperProcessor (assembly_graph/construction/early_simplification.hpp:164-347), the EarlyATClipper phase of the
// RNA pipeline (stages/construction.cpp:317-340,447-448: at_ratio 0.8, min_length 10, max_length 200); runs before the tip clipper.
//   RemoveATEdges (:185-256)  at_edges_probe : per (k-mer, orientation) on the untouched masks: junction + low-complexity k-mer ->
//                                               the outgoing edges of length 1 (next is a junction or a dead end) are flagged
//                             at_edges_apply : every flagged link is deleted once (the reference deletes it through whichever of
//                                               its two representations comes first and skips the other, :237-238: here the
//                                               representation with the smaller (union slot, orientation, nucleotide) acts)
//   RemoveATTips  (:269-334)  at_tips_probe  : per dead end with a unique incoming edge: walk back to the junction (<= max_length),
//                                               complexity of the tip (+ the root's last nucleotides up to min_length), mark
//                                               the vertices and the root. The reference isolates tips while other threads
//                                               walk; the result does not depend on the order (tips are disjoint chains whose
//                                               decisions read only their own vertices and the root's mask -- checked: unmodified
//                                               reference with 1 and 8 threads == oracle sequential == oracle snapshot)
//                             tc_apply_k, tc_links : IsolateVertex, RemoveInconsistentForwardLinks on the updated masks
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
inline AtParams at_params(const GraphOptions &o) {
    AtParams ap;
    ap.ratio = o.at_ratio;
    ap.min_len = (uint32_t)std::min<uint64_t>(o.at_min_len, 0x7fffffffu);
    ap.max_len = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(o.at_max_len, 1), 0x7fffffffu);
    return ap;
}
inline uint32_t tip_bound(const GraphOptions &o) { return (uint32_t)std::min<uint64_t>(o.early_tip_length_bound, 0x7fffffffu); }

template <int NW, class V>
__device__ __forceinline__ void at_edges_probe(const V &v, const uint64_t *keys, int64_t n, int K, AtParams ap, unsigned long long *stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const int o = (int)(tid & 1);
    const typename V::Ref slot = v.template slot<NW>(key);      // flags are indexed by (slot, orientation), like the masks
    v.set_eflag(slot, o, 0);
    const uint8_t mfw = v.mask(slot);
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
        const uint8_t mn = oriented_mask<NW>(v, nx, K);
        if (!mask_is_junction(mn) && (mn & 15) != 0) continue;          // an edge of length 1: next is a junction or a dead end
        f |= (uint8_t)(1u << c);
    }
    v.set_eflag(slot, o, f);
    if (f) atomicAdd(&stats[0], (unsigned long long)__popc(f));
}
template <int NW, class V>
__device__ __forceinline__ void at_edges_apply(const V &v, const uint64_t *keys, int64_t n, int K, unsigned long long *stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const Kmer<NW> kh = (tid & 1) ? kmer_rc<NW>(key, K) : key;
    const CanonIdx<V> ci = canon_lookup<NW>(v, kh, K);
    const int o = (int)(tid & 1);                                        // kh is the table key (minimal form) iff o == 0
    const int64_t fid = (int64_t)(2 * v.link_idx(ci.idx)) + o;
    const uint8_t mine = v.eflag(ci.idx, o);
    if (!mine) return;
    const int first = (int)(kh.w[0] & 3);                                // kh[0]
    for (int c = 0; c < 4; ++c) {
        if (!(mine & (1u << c))) continue;
        Kmer<NW> nx = kh;
        kmer_shl<NW>(nx, K, c);
        const CanonIdx<V> cn = canon_lookup<NW>(v, nx, K);
        // the same link seen from the other strand: (rc(next), complement of kh[0]); rc(next) is the table key iff next is NOT minimal
        const int o2 = cn.is_min ? 1 : 0;
        const int64_t fid2 = (int64_t)(2 * v.link_idx(cn.idx)) + o2;
        const int c2 = 3 - first;
        if ((v.eflag(cn.idx, o2) & (1u << c2)) && (fid2 < fid || (fid2 == fid && c2 < c))) continue;
        v.clear_bit(ci.idx, (unsigned)(ci.is_min ? c : 7 - c));                        // DeleteOutgoing(kh, c)
        v.clear_bit(cn.idx, (unsigned)(cn.is_min ? 4 + first : 7 - (4 + first)));      // DeleteIncoming(next, kh[0])
        atomicAdd(&stats[1], 2ull);
    }
}
template <int NW, class V>
__device__ __forceinline__ void at_tips_probe(const V &v, const uint64_t *keys, int64_t n, int K, AtParams ap, unsigned long long *stats) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= 2 * n) return;
    const Kmer<NW> key = key_at<NW>(keys, tid >> 1);
    const int o = (int)(tid & 1);
    const typename V::Ref idx0 = v.template slot<NW>(key);
    const uint8_t mfw = v.mask(idx0);
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
        m = oriented_mask<NW>(v, kh, K);
    } while (tsz < ap.max_len && !mask_is_junction(m));
    if ((m >> 4) == 0 || !mask_is_junction(m)) return;                   // dead start (isolated short edge) or too long, :301-302
    for (uint32_t p = tsz - 1; p < ap.min_len; ++p) cnt[kmer_nuc<NW>(kh, K - 1 - (int)p)]++;
    const uint32_t curm = max(max(cnt[0], cnt[1]), max(cnt[2], cnt[3]));
    if (math_ls((double)curm, (double)max(tsz, ap.min_len) * ap.ratio)) return;
    // a low-complexity tip: mark its vertices (second walk) and its root
    const CanonIdx<V> cr = canon_lookup<NW>(v, kh, K);
    v.root(cr.idx, cr.is_min ? 0 : 1);
    Kmer<NW> w = start;
    uint8_t mw = m0;
    for (uint32_t s2 = 0; s2 < tsz; ++s2) {
        typename V::Ref idx;
        if (s2) mw = oriented_mask<NW>(v, w, K, &idx); else idx = idx0;
        v.mark(idx);
        kmer_shr<NW>(w, K, uniq4(mw >> 4));
    }
    atomicAdd(&stats[2], (unsigned long long)tsz);
}

// ---- host pieces shared by both builds (graph.cu) ---------------------------------------------------------------------------
// IsolateVertex for the n marked k-mers of one array of masks (tc_apply_k)
void launch_isolate(Ctx *ctx, uint8_t *masks, const uint8_t *mark, uint64_t n);
// the keys of a sweep's flagged records, in final_kmers order, as one compacted list per chunk that has any (so they are never
// held twice, as a join would)
struct KeyParts {
    std::vector<DArr<uint64_t>> parts;
    std::vector<uint64_t> sizes;
    uint64_t total = 0;
};
// per chunk: flags -> scan -> compacted keys. flags(ch, keys, flag) launches one kernel that fills flag[0, ch.n).
typedef std::function<void(const Chunk &, const uint64_t *, uint32_t *)> FlagLaunch;
template <int NW>
KeyParts collect_keys(Ctx *ctx, ChunkStager &src, const FlagLaunch &flags);
// the junctions' keys of a k-mer set (junction_flags_k over every chunk)
template <int NW>
KeyParts junction_keys(Ctx *ctx, ChunkStager &kmers, int K, const MphfDev &mk, const uint8_t *masks);
// pos[rank of the slot among the remaining ones] = final_kmers position, over every chunk of the set (loop_pos_k)
template <int NW>
void loop_positions(Ctx *ctx, ChunkStager &kmers, const MphfDev &mk, const RemSlots &rs, uint64_t *pos);
void launch_nonzero_flags(Ctx *ctx, const uint32_t *in, uint32_t *out, uint64_t n);
// kept slots -> dense (offset, length) table of the path edges
void launch_edge_table(Ctx *ctx, const uint32_t *len, const uint64_t *eidx, const uint64_t *eoff, int64_t nslots, uint64_t *out_off, uint32_t *out_len);
// RemoveSequences on n mask bytes (the visited ones become 0) and the remaining slots' bits (nwords + 1 words); returns how many
// slots remain
uint64_t masks_clear_visited(Ctx *ctx, uint8_t *masks, const uint8_t *visited, uint64_t n, uint32_t *rem_bits);
// RemSlots::base of the remaining-slot bits (nwords + 1 entries)
void rem_slot_base(Ctx *ctx, const uint32_t *rem_bits, uint64_t nwords, uint64_t *rem_base);

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

// Unbranching paths, in batches of junctions (never across two chunks' lists) sized from `budget` bytes: the 8 slots of a
// junction cost len + keepf + selfc + eidx + eoff + the compacted (offset, length) = 37 bytes each. The unitig text and link
// records of a batch depend on its paths' lengths, not on its junctions: they are reckoned at as much again, a heuristic, and a
// batch whose text needs more still runs (blocks beyond the arena come from the driver). Edge numbers and text offsets carry
// over from batch to batch. probe(keys, nj, len, selfc) and write(keys, nj, len, selfc, eidx, eoff, EdgeBatch) launch the two
// kernels of a batch; probed(keys, nj, len) runs once the probe's lengths are known. Returns the number of batches.
template <class Probe, class Probed, class Write>
uint64_t unitig_batches(Ctx *ctx, Graph *g, KeyParts &jk, int nw, uint64_t budget, Trace &tr, Probe &&probe, Probed &&probed, Write &&write) {
    cudaStream_t st = ctx->stream;
    const uint64_t per_junc = 2 * 8 * 37;
    const uint64_t jbatch = std::max<uint64_t>(4096, budget / 2 / per_junc);
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
        const uint64_t *bkeys = jk.parts[part].p + q0 * nw;
        probe(bkeys, (int64_t)nj, len.p, selfc.p);
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
        probed(bkeys, (int64_t)nj, len.p);
        tr.mark("unitig probe + offsets");
        EdgeBatch eb(ctx, npaths, nbases);
        write(bkeys, (int64_t)nj, len.p, selfc.p, eidx.p, eoff.p, eb);
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
        tr.mark("unitig write");
        // the (offset, length) table is compacted on the device (8 slots per junction, most of them empty)
        DArr<uint64_t> c_off(ctx, npaths + 1);
        DArr<uint32_t> c_len(ctx, npaths + 1);
        launch_edge_table(ctx, len.p, eidx.p, eoff.p, (int64_t)nslots, c_off.p, c_len.p);
        eb.append(g, st, c_off.p, c_len.p);
        if (q0 + nj == njunc) jk.parts[part].release();
        tr.mark("download + edge table");
    }
    return batches;
}

// The perfect loops of the leaders lk (one or two edges each), appended to g. probe(leaders, nl, info, llen) and
// write(info, nl, llen, leidx, leoff, EdgeBatch, scratch, soff) launch the two kernels; probed(leaders, nl, llen on the host) runs
// once the probe's lengths are known.
template <class Probe, class Probed, class Write>
void loop_edges(Ctx *ctx, Graph *g, const KeyParts &lk, int nw, int K, Probe &&probe, Probed &&probed, Write &&write) {
    cudaStream_t st = ctx->stream;
    const uint64_t nl = lk.total;
    if (!nl) return;
    // the leaders as one list (loops are rare, a few keys)
    DArr<uint64_t> leaders(ctx, (size_t)nl * nw);
    for (size_t i = 0, at = 0; i < lk.parts.size(); at += lk.sizes[i], ++i)
        SG_CUDA(cudaMemcpyAsync(leaders.p + at * nw, lk.parts[i].p, lk.sizes[i] * nw * 8, cudaMemcpyDeviceToDevice, st));
    DArr<LoopInfo> info(ctx, nl);
    DArr<uint32_t> llen(ctx, 2 * nl + 1), lkeep(ctx, 2 * nl + 1), sfull(ctx, nl + 1);
    DArr<uint64_t> leidx(ctx, 2 * nl + 1), leoff(ctx, 2 * nl + 1), soff(ctx, nl + 1);
    SG_CUDA(cudaMemsetAsync(llen.p, 0, llen.bytes(), st));
    probe(leaders.p, (int64_t)nl, info.p, llen.p);
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
    probed(leaders.p, (int64_t)nl, h_llen);
    std::vector<uint64_t> h_soff(nl + 1, 0);
    for (uint64_t q = 0; q < nl; ++q) h_soff[q + 1] = h_soff[q] + (uint64_t)K + h_info[q].nverts;
    SG_CUDA(cudaMemcpyAsync(soff.p, h_soff.data(), (nl + 1) * 8, cudaMemcpyHostToDevice, st));
    DArr<char> scratch(ctx, h_soff[nl] + 1);
    EdgeBatch eb(ctx, nledges, nlbases);
    write(info.p, (int64_t)nl, llen.p, leidx.p, leoff.p, eb, scratch.p, soff.p);
    ctx->launches++;
    SG_CUDA(cudaGetLastError());
    // the (offset, length) table from the probe's lengths: a loop is one edge, or two where it splits
    std::vector<uint64_t> off;
    std::vector<uint32_t> len;
    for (uint64_t i = 0, at = 0; i < 2 * nl; at += h_llen[i++])
        if (h_llen[i]) { off.push_back(at); len.push_back(h_llen[i]); }
    eb.append(g, st, off.data(), len.data());
}

}  // namespace sg
