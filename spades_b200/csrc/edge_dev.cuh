// edge_dev.cuh -- the edges of a graph as the EdgeIndex refill reads them (edge_index.cu on one GPU, dist_edge_index.cu across
// GPUs): 2-bit packed primary strands on the device and the walk from a work item to its window
#pragma once
#include "graph.h"
#include "mphf_dev.cuh"

namespace sg {

static const uint32_t kEdgeInfoTombstone = 0x7ffffffeu;       // EdgeInfo::TOMBSTONE: -2u without the PicoSpinLock bit (edge_position_index.hpp:29-30)
static const uint32_t kEdgeInfoCleared = 0x7fffffffu;         // EdgeInfo::CLEARED

struct UnitigTable {
    const uint64_t *words;      // 2-bit packed primary strands, each on a word boundary
    const uint64_t *woff;       // [E] first word
    const uint32_t *len;        // [E] nucleotides
    const uint8_t *selfc;       // [E] the edge is its own conjugate
    const uint64_t *wstart;     // [E+1] exclusive prefix of the windows per edge (both strands counted, self-conjugate once)
    int64_t E;
};

// the edges of g packed for the K-mer windows of the refill: the count reads them as "reads" (words / woff / lens), the puts walk
// them through a UnitigTable
struct EdgePack {
    DArr<uint64_t> words, woff, wstart;
    DArr<uint32_t> lens;
    DArr<uint8_t> selfc;
    uint64_t nwords = 0;        // words of the packed text
    uint64_t nwork = 0;         // windows of both strands (self-conjugate edges once)
    int64_t E = 0;
    UnitigTable table() const {
        UnitigTable u;
        u.words = words.p; u.woff = woff.p; u.len = lens.p; u.selfc = selfc.p; u.wstart = wstart.p; u.E = E;
        return u;
    }
};
void edge_pack(Ctx *ctx, const Graph *g, int K, EdgePack *out);

// work item -> (edge, strand, offset); K-mer of the conjugate strand at offset j = rc of the primary window at L - K - j
template <int NW>
__device__ __forceinline__ bool edge_window(const UnitigTable &u, int K, uint64_t w, uint32_t *edge, int *strand, uint32_t *off, Kmer<NW> *k) {
    int64_t lo = 0, hi = u.E - 1;
    while (lo < hi) {                                                   // last edge whose first window index is <= w
        const int64_t mid = (lo + hi + 1) >> 1;
        if (u.wstart[mid] <= w) lo = mid; else hi = mid - 1;
    }
    const uint32_t L = u.len[lo];
    if (L < (uint32_t)K) return false;
    const uint32_t nwin = L - (uint32_t)K + 1;
    uint32_t j = (uint32_t)(w - u.wstart[lo]);
    int s = 0;
    if (j >= nwin) { j -= nwin; s = 1; }
    const uint64_t *seq = u.words + u.woff[lo];
    const Kmer<NW> f = kmer_window<NW>(seq, (int64_t)(s == 0 ? j : nwin - 1 - j), K);
    const Kmer<NW> r = kmer_rc<NW>(f, K);
    *k = s == 0 ? f : r;                                                // the window as it stands on this strand
    *edge = (uint32_t)lo; *strand = s; *off = j;
    return s == 0 ? kmer_is_minimal<NW>(f, r) : kmer_is_minimal<NW>(r, f);      // kwh.is_minimal(): only minimal windows are put
}

}  // namespace sg
