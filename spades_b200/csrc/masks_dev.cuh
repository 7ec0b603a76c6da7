// masks_dev.cuh -- what one (k+1)-mer adds to the extension masks (DeBruijnExtensionIndexBuilder::FillExtensionsFromIndex,
// src/common/kmer_index/extension_index/kmer_extension_index_builder.hpp:45-60, with InOutMask's orientation, inout_mask.hpp:55-221).
// Shared by the single-GPU mask fill (graph.cu) and the distributed one (dist_ext.cu).
#pragma once
#include "kmer_dev.cuh"

namespace sg {

// the minimal form of k-mer k, handed to f: {f(minimal form), whether k is minimal} (KeyWithHash's canonical form)
template <class R>
struct SideResult {
    R value;
    bool is_min;
};
template <int NW, class F>
__device__ __forceinline__ auto min_form_of(const Kmer<NW> &k, int K, F &&f) {
    Kmer<NW> r = kmer_rc<NW>(k, K);
    SideResult<decltype(f(k))> c;
    c.is_min = kmer_is_minimal<NW>(k, r);
    c.value = f(c.is_min ? k : r);
    return c;
}

// SIDE 0: the prefix k-mer of (k+1)-mer x, which gets AddOutgoing(kpomer[K]); SIDE 1: its suffix k-mer, which gets
// AddIncoming(kpomer[0]). f receives the k-mer's minimal form.
template <int SIDE, int NW, int NWS, class F>
__device__ __forceinline__ auto kpomer_side(const Kmer<NWS> &x, int K, F &&f) {
    if (SIDE) return min_form_of<NW>(kmer_suffix<NW, NWS>(x, K), K, f);
    else return min_form_of<NW>(kmer_prefix<NW, NWS>(x, K), K, f);
}
// the nucleotide of that side's edge: kpomer[K] for SIDE 0, kpomer[0] for SIDE 1
template <int SIDE, int NWS>
__device__ __forceinline__ int kpomer_side_nucl(const Kmer<NWS> &x, int K) { return SIDE ? (int)(x.w[0] & 3) : kmer_nuc<NWS>(x, K); }
// the mask bit (0-7) of that edge on the minimal form: mirrored (InOutMask::conjugate) when the k-mer is not minimal
template <int SIDE>
__device__ __forceinline__ int mask_bit(bool is_min, int nucl) { return SIDE ? (is_min ? nucl + 4 : 3 - nucl) : (is_min ? nucl : 7 - nucl); }

// a contribution: the minimal form of the k-mer and the bit (0-7) of its mask that the (k+1)-mer sets
template <int NW>
struct MaskBit {
    Kmer<NW> key;
    int bit;
};
template <int SIDE, int NW, int NWS>
__device__ __forceinline__ MaskBit<NW> kpomer_mask_bit(const Kmer<NWS> &x, int K) {
    const auto c = kpomer_side<SIDE, NW, NWS>(x, K, [](const Kmer<NW> &key) { return key; });
    MaskBit<NW> m;
    m.key = c.value;
    m.bit = mask_bit<SIDE>(c.is_min, kpomer_side_nucl<SIDE, NWS>(x, K));
    return m;
}

// sets bit `bit` of mask byte `idx` (the masks are OR-ed as 32-bit words)
__device__ __forceinline__ void mask_or(unsigned *masks32, uint64_t idx, int bit) {
    atomicOr(&masks32[idx >> 2], (1u << bit) << (8 * (idx & 3)));
}

}  // namespace sg
