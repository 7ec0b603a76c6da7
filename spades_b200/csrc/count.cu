// count.cu -- k-mer extraction, partition, sort/unique/count. The GPU replacement for
//   KMerSortingSplitter::Split / DumpBuffers   (src/common/kmer_index/kmer_mph/kmer_splitter.hpp:56-179)
//   DeBruijnReadKMerSplitter / DeBruijnKMerKMerSplitter (…/kmer_splitters.hpp:28-207)
//   ParallelSortingSplitter (projects/spades_tools/kmercount.cpp:48-122)
//   KMerDiskCounter::Count / MergeKMers (…/kmer_index_builder.hpp:306-431)
// Output per bucket == the reference's kmers.<b> file: strictly increasing W-byte records, order of
// pdqsort_pod.h:725-734; multiplicities == CoverageHashMapBuilder's second pass (coverage_hash_map_builder.hpp:18-40).
//
// Pipeline (all in HBM, see DESIGN.md "count"):
//   A  level-A partition : records -> (bucket, top rA key bits) partitions. Two kernels over the source with
//      identical static work assignment: per-CTA histograms, then scatter with CTA-private cursors held in
//      shared memory (no global atomics; 16-byte stores merge in L2).
//   B  MSD refinement    : any segment longer than the local-sort capacity is split by its next r key bits by
//      ONE CTA (histogram + scatter through shared-memory cursors), ping-ponging between two buffers; repeated
//      until every segment fits or its key bits are exhausted (then all its records are equal).
//   C  local sort        : one CTA per segment: LSD radix sort in shared memory over the remaining key bits
//      (optimistic 32-bit window + verification, full range on failure), run-length unique/count, written
//      back in place; then a compaction copy into the dense bucket-major result.
#include <algorithm>
#include <chrono>
#include <memory>

#include "pass_plan.h"
#include "sgpu_internal.h"

namespace sg {

// ------------------------------------------------------------------------------------------------------------
// record sources: items are packed sequences (nucleotide i at bits 2(i%32) of word i/32, kmer_dev.cuh) whose K-windows are the
// records. The level-A kernels see an item through first_word / len / words only. kIds: partition ids per chunk (the id row of
// a chunk, a whole number of 16-byte words); kIdLines: 128-byte lines of id rows prefetched for a warp's next tile.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

struct ReadsSrc {
    const uint64_t *words;
    const uint64_t *offs;
    const uint32_t *lens;
    int64_t n;          // items = reads
    uint64_t nwords;    // length of `words`
    int K;
    static constexpr int kIds = 24;         // a chunk's records
    static constexpr int kIdLines = 48;     // 128 chunks: 32 reads of 150 bp at k = 55
    static constexpr bool kSubRanges = true;  // a pass may scatter in partition sub-ranges (levelA_scatter)
    __device__ __forceinline__ uint64_t first_word(int64_t item) const { return offs[item]; }
    __device__ __forceinline__ uint32_t len(int64_t item) const { return lens[item]; }
    // the lengths and offsets of the reads from `item` on, to L2
    __device__ __forceinline__ void prefetch_items(int64_t item, int lane) const {
        if (lane == 0) prefetch_l2(lens + item);
        else if (lane == 1 && item + 16 < n) prefetch_l2(offs + item + 16);
    }
};

// the distinct (K+1)-mers of a k-mer set chunk as reads of K+1 bases at implicit offsets: item i is key words [i * stride, ..).
// Its two windows are the (K+1)-mer's prefix and suffix, and the canonical record of each is what DeBruijnKMerKMerSplitter
// (add_rc + IsMinimal filter) emits. An item is one chunk of two records, so its id row is one 16-byte word.
struct KmerSetSrc {
    const uint64_t *words;
    int64_t n;          // items = (K+1)-mers
    uint64_t nwords;    // n * stride
    int K;              // target K
    uint32_t stride;    // words per key
    static constexpr int kIds = 8;
    static constexpr int kIdLines = 4;      // 32 chunks
    static constexpr bool kSubRanges = false;
    __device__ __forceinline__ uint64_t first_word(int64_t item) const { return (uint64_t)item * stride; }
    __device__ __forceinline__ uint32_t len(int64_t) const { return (uint32_t)K + 1; }
    __device__ __forceinline__ void prefetch_items(int64_t, int) const {}
};

template <int NW>
__device__ __forceinline__ void store_rec(uint64_t *dst, const Kmer<NW> &k) {
    if (NW == 2) {
        *reinterpret_cast<ulonglong2 *>(dst) = make_ulonglong2(k.w[0], k.w[1]);
    } else if (NW == 4) {
        reinterpret_cast<ulonglong2 *>(dst)[0] = make_ulonglong2(k.w[0], k.w[1]);
        reinterpret_cast<ulonglong2 *>(dst)[1] = make_ulonglong2(k.w[2], k.w[3]);
    } else {
#pragma unroll
        for (int q = 0; q < NW; ++q) dst[q] = k.w[q];
    }
}
template <int NW>
__device__ __forceinline__ Kmer<NW> load_rec(const uint64_t *src) {
    Kmer<NW> k;
    if (NW == 2) {
        ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(src);
        k.w[0] = v.x; k.w[1] = v.y;
    } else if (NW == 4) {
        ulonglong2 a = reinterpret_cast<const ulonglong2 *>(src)[0], b = reinterpret_cast<const ulonglong2 *>(src)[1];
        k.w[0] = a.x; k.w[1] = a.y; k.w[2] = b.x; k.w[3] = b.y;
    } else {
#pragma unroll
        for (int q = 0; q < NW; ++q) k.w[q] = src[q];
    }
    return k;
}

// ------------------------------------------------------------------------------------------------------------
// level A
// ------------------------------------------------------------------------------------------------------------
struct LevelA {
    int K;
    uint32_t B;
    uint32_t b_lo, b_hi;    // buckets of this pass
    int rA;                 // key bits folded into the partition id
    uint32_t PA;            // (b_hi-b_lo) << rA
};

// record stores bypass L1 allocation (they are never re-read by this kernel)
template <int NW>
__device__ __forceinline__ void store_rec_stream(uint64_t *dst, const Kmer<NW> &k) {
    if (NW == 2) {
        asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(k.w[0]), "l"(k.w[1]) : "memory");
    } else if (NW == 4) {
        asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(k.w[0]), "l"(k.w[1]) : "memory");
        asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst + 2), "l"(k.w[2]), "l"(k.w[3]) : "memory");
    } else {
#pragma unroll
        for (int q = 0; q < NW; ++q) asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(dst + q), "l"(k.w[q]) : "memory");
    }
}

// the item of unit i: i / uniform when every item has `uniform` units, else the largest t with pref[t] <= i (pref is exclusive)
__device__ __forceinline__ int find_item_u(const uint32_t *pref, int nitems, uint32_t i, uint32_t uniform) {
    if (uniform) return (int)(i / uniform);
    int lo = 0, hi = nitems - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (pref[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
}

template <int NW>
__device__ __forceinline__ bool part_of(const LevelA &p, const Kmer<NW> &k, uint32_t *part) {
    uint32_t b = kmer_bucket<NW>(k, p.B);
    if (b < p.b_lo || b >= p.b_hi) return false;
    *part = ((b - p.b_lo) << p.rA) | key_top_bits<NW>(k, p.K, p.rA);
    return true;
}

// one thread per partition: totals and per-CTA bases. base[g][part] is the running cursor of CTA g.
__global__ void levelA_totals_k(const uint32_t *__restrict__ blk_counts, uint32_t PA, int G, uint64_t *__restrict__ part_total) {
    uint32_t part = blockIdx.x * blockDim.x + threadIdx.x;
    if (part >= PA) return;
    uint64_t s = 0;
    for (int g = 0; g < G; ++g) s += blk_counts[(size_t)g * PA + part];
    part_total[part] = s;
}
__global__ void levelA_bases_k(const uint32_t *__restrict__ blk_counts, uint32_t stride, uint32_t PA, int G,
                               const uint64_t *__restrict__ part_start, uint64_t *__restrict__ base) {
    uint32_t part = blockIdx.x * blockDim.x + threadIdx.x;
    if (part >= PA) return;
    uint64_t run = part_start[part];
    for (int g = 0; g < G; ++g) {
        base[(size_t)g * PA + part] = run;
        run += blk_counts[(size_t)g * stride + part];
    }
}

// ---- level A: rolling kernels ------------------------------------------------------------------------------------------
// The unit of work is a CHUNK of consecutive windows of one item, walked by one thread with a rolling window + rolling reverse
// complement (kmer_dev.cuh roll_*): one shared-memory word load per 32 bases, ~20 integer instructions per window, and in a
// bucket-group pass the windows of other groups cost only the roll. A chunk holds kRollC records: kRollC windows in canonical
// mode (one record per window, the canonical one of its two strands), kRollC / 2 windows in all-windows mode (BOTH: record s
// is window s / 2 and strand s & 1, the roll advances every second record). The 2-byte partition ids of a chunk's records are
// one row of Src::kIds ids: written as 8-byte words by the count pass, fetched as 16-byte loads before the walk starts by every
// scatter pass. (Re-extracting every window from the packed words, the kernels of the first generation, cost a few hundred
// thread instructions per window. Removed.)
static const int kRollC = 24;            // records per chunk
template <bool BOTH> constexpr int kRollWin = BOTH ? kRollC / 2 : kRollC;      // windows per chunk
static_assert(kRollC <= 33 && kRollC % 8 == 0, "roll_init fetches a chunk's bases from two words; an id row is a whole number of 16-byte words");
static_assert(ReadsSrc::kIds == kRollC && KmerSetSrc::kIds % 8 == 0, "an id row holds a chunk's records");
static const int kRollThreads = 512;     // 2-3 CTAs per SM; units of a tile are dealt round-robin to the threads

// The tile of the rolling kernels is a WARP's: 32 consecutive items, staged, scanned and walked by one warp with
// shuffles and __syncwarp only. (The CTA-wide tiles of the first version cost five __syncthreads per 256 reads, and barrier
// and global-load stalls dominated the partition kernel.) A CTA
// still owns a contiguous range of tiles -- the same range in the count and in every scatter launch, which is what makes the
// per-CTA histogram of the count the cursor table of the scatter -- and deals them round-robin to its warps.
static const int kRollTile = 32;                      // items per warp tile
static const int kRollWarps = kRollThreads / 32;
static const int kRollStageWords = 320;               // per warp: 32 reads x 10 words (<= 320 bp each), else global loads
struct RollWarp {
    uint64_t words[kRollStageWords];     // the tile's packed items
    uint32_t pref[kRollTile + 1];        // exclusive prefix of chunks per item
    uint32_t len[kRollTile];             // item lengths
    uint32_t off[kRollTile];             // first staged word of an item
    uint32_t pad_;
};
static_assert(sizeof(RollWarp) % 8 == 0, "per-warp slices stay 8-byte aligned");
static size_t roll_smem_bytes(uint32_t nslots) { return (((size_t)nslots * 4 + 15) & ~(size_t)15) + (size_t)kRollWarps * sizeof(RollWarp); }
__device__ __forceinline__ RollWarp *roll_warp_slice(unsigned char *raw, uint32_t nslots) {
    return reinterpret_cast<RollWarp *>(raw + (((size_t)nslots * 4 + 15) & ~(size_t)15)) + (threadIdx.x >> 5);
}

// one warp: chunk counts of the tile's items -> exclusive prefix, the items' words -> shared memory. Returns the tile's chunk
// total; *uniform = chunks per item when every item has the same (non-zero) count, else 0; *staged = words are in rw.words.
template <bool BOTH, class Src>
__device__ __forceinline__ uint32_t roll_warp_setup(const Src &src, int64_t item0, int nitems, RollWarp &rw, uint32_t *uniform, bool *staged) {
    const int lane = threadIdx.x & 31;
    uint32_t c = 0, L = 0;
    uint64_t a = 0, b = 0;
    if (lane < nitems) {
        L = src.len(item0 + lane);
        a = src.first_word(item0 + lane);
        b = a + (((uint64_t)L + 31) >> 5);
        const uint32_t w = (int)L >= src.K ? (uint32_t)((int)L - src.K + 1) : 0u;
        c = (w + kRollWin<BOTH> - 1) / kRollWin<BOTH>;
    }
    uint32_t inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    rw.len[lane] = L;
    rw.pref[lane] = inc - c;
    const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
    if (lane == 31) rw.pref[kRollTile] = total;
    const uint32_t c0 = __shfl_sync(0xffffffffu, c, 0);
    const bool same = __all_sync(0xffffffffu, lane >= nitems || c == c0);
    *uniform = (same && c0) ? c0 : 0u;
    const uint64_t w0 = __shfl_sync(0xffffffffu, a, 0);
    const bool ok = lane >= nitems || (a >= w0 && b >= a && b - w0 <= (uint64_t)kRollStageWords);
    const bool st = __all_sync(0xffffffffu, ok);
    if (st) {
        rw.off[lane] = (uint32_t)(a - w0);
        uint32_t end = lane < nitems ? (uint32_t)(b - w0) : 0u;
#pragma unroll
        for (int o = 16; o; o >>= 1) end = max(end, __shfl_xor_sync(0xffffffffu, end, o));
        // all loads first, then the stores: the copy costs one memory round trip, not one per 32 words
        uint64_t tmp[kRollStageWords / 32];
#pragma unroll
        for (int j = 0; j < kRollStageWords / 32; ++j) tmp[j] = (uint32_t)(lane + 32 * j) < end ? __ldg(src.words + w0 + lane + 32 * j) : 0ull;
#pragma unroll
        for (int j = 0; j < kRollStageWords / 32; ++j) if ((uint32_t)(lane + 32 * j) < end) rw.words[lane + 32 * j] = tmp[j];
    }
    *staged = st;
    __syncwarp();
    return total;
}

// chunks per warp tile x Src::kIds = ids per tile (rows of the id array: a whole number of 16-byte words per chunk)
template <bool BOTH, class Src>
__global__ void roll_tile_ids_k(Src src, int64_t ntiles, uint32_t *__restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= ntiles) return;
    const int lane = threadIdx.x & 31;
    const int64_t item = t * kRollTile + lane;
    uint32_t s = 0;
    if (item < src.n) {
        const int L = (int)src.len(item);
        const uint32_t w = L >= src.K ? (uint32_t)(L - src.K + 1) : 0u;
        s = (w + kRollWin<BOTH> - 1) / kRollWin<BOTH>;
    }
    for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (lane == 0) out[t] = s * Src::kIds;
}

// geometry of one unit (chunk): which item, which windows (first, count)
struct RollUnit { int it, j0, cnt; };
template <bool BOTH>
__device__ __forceinline__ RollUnit roll_unit(const RollWarp &rw, int nitems, uint32_t u, uint32_t unif, int K) {
    constexpr int C = kRollWin<BOTH>;
    RollUnit q;
    q.it = find_item_u(rw.pref, nitems, u, unif);
    q.j0 = (int)(u - rw.pref[q.it]) * C;
    const int nwin = (int)rw.len[q.it] - K + 1;
    q.cnt = nwin - q.j0 < C ? nwin - q.j0 : C;
    return q;
}

template <int NW, class Src, bool BOTH>
__global__ void __launch_bounds__(kRollThreads, 2) levelA_count_roll_k(Src src, LevelA p, uint32_t *__restrict__ blk_counts,
                                                                      const uint64_t *__restrict__ tile_off, uint16_t *__restrict__ ids) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    uint32_t *hist = reinterpret_cast<uint32_t *>(sm_raw);     // PA
    RollWarp &rw = *roll_warp_slice(sm_raw, p.PA);
    for (uint32_t i = threadIdx.x; i < p.PA; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const int K = p.K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t ntiles = (src.n + kRollTile - 1) / kRollTile;
    const int64_t per = (ntiles + gridDim.x - 1) / gridDim.x;
    const int64_t t0 = (int64_t)blockIdx.x * per, t1 = min(ntiles, t0 + per);
    for (int64_t t = t0 + warp; t < t1; t += kRollWarps) {
        const int64_t item0 = t * kRollTile;
        const int nitems = (int)min((int64_t)kRollTile, src.n - item0);
        uint32_t unif = 0;
        bool staged = false;
        // the warp's next tile is kRollWarps tiles ahead: its item metadata goes to L2 now, its packed items (and id rows) at the
        // end of this tile, when the loads of their addresses issued here have long returned
        const bool has_next = t + kRollWarps < t1;
        const int64_t nx = (t + kRollWarps) * kRollTile;
        uint64_t next_w0 = 0;
        if (has_next) {
            next_w0 = src.first_word(nx);
            src.prefetch_items(nx, lane);
        }
        const uint32_t nunits = roll_warp_setup<BOTH>(src, item0, nitems, rw, &unif, &staged);
        uint64_t *row = ids ? reinterpret_cast<uint64_t *>(ids + tile_off[t]) : nullptr;
        for (uint32_t u = lane; u < nunits; u += 32) {
            const RollUnit q = roll_unit<BOTH>(rw, nitems, u, unif, K);
            const uint64_t *seq = staged ? static_cast<const uint64_t *>(rw.words + rw.off[q.it]) : src.words + src.first_word(item0 + q.it);
            RollState<NW> st;
            roll_init<NW>(st, seq, q.j0, K, q.cnt);
            const int nrec = BOTH ? 2 * q.cnt : q.cnt;
#pragma unroll 1
            for (int g = 0; g < Src::kIds / 4; ++g) {
                uint64_t acc = 0;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int s = 4 * g + e;
                    uint32_t id = 0xffffu;
                    if (s < nrec) {
                        if (s > 0 && !(BOTH && (e & 1))) roll_next<NW>(st, K);
                        const Kmer<NW> k = BOTH ? ((e & 1) ? st.r : st.f) : kmer_is_minimal<NW>(st.f, st.r) ? st.f : st.r;
                        uint32_t part;
                        if (part_of<NW>(p, k, &part)) { atomicAdd(&hist[part], 1u); id = part; }
                    }
                    acc |= (uint64_t)id << (16 * e);
                }
                if (row) row[(size_t)u * (Src::kIds / 4) + g] = acc;
            }
        }
        if (has_next && lane < 10 && next_w0 + 16 * lane < src.nwords) prefetch_l2(src.words + next_w0 + 16 * lane);   // 10 lines = 32 reads x 5 words
        __syncwarp();                                   // the slice is rewritten by the next tile's setup
    }
    __syncthreads();
    uint32_t *out = blk_counts + (size_t)blockIdx.x * p.PA;
    for (uint32_t i = threadIdx.x; i < p.PA; i += blockDim.x) out[i] += hist[i];
}

// base rows are `row_stride` cursors long; a launch handles the partitions [q_lo, q_lo + p.PA) of a row (p.PA = the sub-range's
// size, id_lo = id of its first partition): a bucket-group pass may be split into partition sub-ranges so that the streams a CTA
// has open at any time stay few.
// Records stored one by one as they are rolled leave L2 as partly written sectors: with PA = 640 streams per CTA a stream
// receives a record only every few microseconds, and lone 16-byte stores at 640 streams run at about a ninth of the HBM rate
// (DESIGN.md 6.2). Both scatter kernels therefore collect a CTA's own records in a shared-memory batch and write it out partition
// by partition, consecutive threads storing consecutive records of a run. The order inside a partition is arbitrary.
// (A sector-pairing variant -- two records of a stream leave as one 32-byte store through shared-memory mailboxes -- was
// parity clean but slower: the CAS traffic on the mailboxes cost more than the full sectors won. Removed.)
// Below kABatchMin records at two CTAs per SM, one CTA per SM takes a larger batch. The threshold itself is not tuned; in
// scatter_bench -a 1 (DESIGN.md 6.2) 1024-record batches at two CTAs of 512 run at 546 / 278 GB/s (640 / 2560 streams, 16-byte
// records); the fallback's shape, one CTA of 512 threads per SM with the larger batch, is not in that table.
static const uint32_t kABatchMin = 1024;
// the planned batch hands each warp an equal share of it, and a share must hold one record of each of a warp step's 32 chunks
// (two, one window's both strands, in all-windows mode): else a warp could never advance
static_assert(kABatchMin / kRollWarps >= 32 * 2, "a warp's share of the smallest batch holds one window of a warp step");
// dynamic shared memory: [cursor | batch count] per partition, the warps' RollWarp slices, then the batch
__host__ __device__ __forceinline__ size_t abatch_offset(uint32_t PA) {
    return ((((size_t)2 * PA * 4 + 15) & ~(size_t)15) + (size_t)kRollWarps * sizeof(RollWarp) + 15) & ~(size_t)15;
}
// shared-memory bytes per batched record: the arrival-order batch keeps the record, its tag and a permutation index; the planned
// batch, already in partition order, keeps the record and its 2-byte partition
template <int NW, bool PLANNED>
constexpr size_t abatch_rec_bytes() { return NW * sizeof(uint64_t) + (PLANNED ? sizeof(uint16_t) : sizeof(uint32_t) + sizeof(uint16_t)); }

// ---- the id-less form: an arrival-order batch ---------------------------------------------------------------------------
// Without the id array a record's partition is known only once it is rolled and hashed, so records enter the batch as they come:
// - a warp reserves room for one window step of its lanes with one shared-memory atomic, and a record takes its rank in its
//   partition with another;
// - when a reservation does not fit, the warp stops with that window pending, and every warp meets at the flush: a scan of the
//   batch counts places each partition's run in the batch and claims it from the partition's cursor, an index array permutes
//   the batch into partition order, and consecutive threads store consecutive records of a run;
// - warps without work left, and lanes without a chunk, keep reaching the barriers (__syncthreads_or on "work left").
static const uint32_t kABatchNoTag = 0xffffffffu;      // an arrival slot of the batch that a warp reserved but did not fill
static const int kABatchPartBits = 13;                 // tag = (rank << 13) | partition, partition < kLevelAMaxParts
template <int NW, class Src, bool BOTH>
__global__ void __launch_bounds__(kRollThreads, 2) levelA_scatter_roll_k(Src src, LevelA p, uint64_t *__restrict__ base, uint64_t *__restrict__ out,
                                                                        uint32_t row_stride, uint32_t cap) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    __shared__ uint32_t s_fill;                   // arrival slots reserved in the batch (may run past cap)
    __shared__ uint32_t warp_tot[kRollWarps];
    const uint32_t PA = p.PA;
    // one 32-bit cursor per partition, relative to the first record this launch may write (a CTA's share of a pass is far below
    // 2^32 records); the batch count of a partition in the low 16 bits of cnt, the end of its run in the batch in the high 16
    uint32_t *cur = reinterpret_cast<uint32_t *>(sm_raw);               // PA
    uint32_t *cnt = cur + PA;                                           // PA
    RollWarp &rw = *roll_warp_slice(sm_raw, 2 * PA);
    uint64_t *stage = reinterpret_cast<uint64_t *>(sm_raw + abatch_offset(PA));    // [cap][NW] records in arrival order
    uint32_t *tags = reinterpret_cast<uint32_t *>(stage + (size_t)cap * NW);      // [cap]     (rank << 13) | partition
    uint16_t *idx = reinterpret_cast<uint16_t *>(tags + cap);                     // [cap]     arrival slot of a batch position
    uint64_t *mybase = base + (size_t)blockIdx.x * row_stride;
    const uint64_t region0 = mybase[0];                                 // cursors of a row ascend with the partition
    for (uint32_t i = threadIdx.x; i < PA; i += blockDim.x) { cur[i] = (uint32_t)(mybase[i] - region0); cnt[i] = 0; }
    if (threadIdx.x == 0) s_fill = 0;
    __syncthreads();
    uint64_t *const out0 = out + region0 * NW;
    const int K = p.K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    const int64_t ntiles = (src.n + kRollTile - 1) / kRollTile;
    const int64_t per = (ntiles + gridDim.x - 1) / gridDim.x;
    const int64_t t0 = (int64_t)blockIdx.x * per, t1 = min(ntiles, t0 + per);

    // the warp's tile and the lane's chunk survive a flush: a warp that finds the batch full resumes at its pending window
    int64_t t = t0 + warp;
    bool need_setup = true;
    int nitems = 0;
    uint32_t nunits = 0, unif = 0;
    bool staged = false;
    uint64_t next_w0 = 0;
    int u = 0, s = 0, cnt_w = 0;                  // the lane's chunk, its record (st is at its window), its records
    RollState<NW> st;
    for (;;) {
        while (t < t1) {                          // warp-uniform
            if (need_setup) {
                const int64_t item0 = t * kRollTile;
                nitems = (int)min((int64_t)kRollTile, src.n - item0);
                // the warp's next tile is kRollWarps tiles ahead: its item metadata goes to L2 now, its packed items at the end of
                // this tile, when the loads of their addresses issued here have long returned
                const int64_t nx = (t + kRollWarps) * kRollTile;
                if (t + kRollWarps < t1) {
                    next_w0 = src.first_word(nx);
                    src.prefetch_items(nx, lane);
                }
                nunits = roll_warp_setup<BOTH>(src, item0, nitems, rw, &unif, &staged);
                u = lane - 32; s = cnt_w = 0;
                need_setup = false;
            }
            if (s >= cnt_w && u < (int)nunits) {  // the lane's next chunk
                u += 32;
                if (u < (int)nunits) {
                    const RollUnit q = roll_unit<BOTH>(rw, nitems, (uint32_t)u, unif, K);
                    const uint64_t *seq = staged ? static_cast<const uint64_t *>(rw.words + rw.off[q.it]) : src.words + src.first_word(t * kRollTile + q.it);
                    roll_init<NW>(st, seq, q.j0, K, q.cnt);
                    s = 0; cnt_w = BOTH ? 2 * q.cnt : q.cnt;
                }
            }
            const bool act = s < cnt_w;
            if (!__any_sync(0xffffffffu, act)) {  // the tile is done
                if (t + kRollWarps < t1 && lane < 10 && next_w0 + 16 * lane < src.nwords) prefetch_l2(src.words + next_w0 + 16 * lane);   // 10 lines = 32 reads x 5 words
                __syncwarp();                     // the slice is rewritten by the next tile's setup
                t += kRollWarps;
                need_setup = true;
                continue;
            }
            uint32_t part = 0;
            bool mine = false;
            Kmer<NW> k;
            if (act) {
                // a word-by-word select: `cond ? st.f : st.r` bound to a reference made the compiler keep the roll state in local
                // memory to pick an address
                const bool fwd = BOTH ? !(s & 1) : kmer_is_minimal<NW>(st.f, st.r);
#pragma unroll
                for (int j = 0; j < NW; ++j) k.w[j] = fwd ? st.f.w[j] : st.r.w[j];
                mine = part_of<NW>(p, k, &part);
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, mine);
            if (bal) {
                const uint32_t n = __popc(bal);
                uint32_t b0 = 0;
                if (lane == 0) b0 = atomicAdd(&s_fill, n);
                b0 = __shfl_sync(0xffffffffu, b0, 0);
                if (b0 + n > cap) {               // full: the window stays pending; the slots reserved below cap stay empty
                    if (b0 < cap && (uint32_t)lane < cap - b0) tags[b0 + lane] = kABatchNoTag;
                    break;
                }
                if (mine) {
                    const uint32_t i = b0 + __popc(bal & lt_mask);
                    const uint32_t rank = atomicAdd(&cnt[part], 1u) & 0xffffu;
                    store_rec<NW>(stage + (size_t)i * NW, k);
                    tags[i] = (rank << kABatchPartBits) | part;
                }
            }
            if (act && ++s < cnt_w && (!BOTH || !(s & 1))) roll_next<NW>(st, K);
        }
        const bool more = __syncthreads_or(t < t1);
        // ---- flush: scan of the batch counts (a thread owns a run of consecutive partitions), the runs claimed from the cursors
        const uint32_t nslots = min(s_fill, cap);
        const uint32_t own = (PA + kRollThreads - 1) / kRollThreads;
        const uint32_t j0 = min(PA, threadIdx.x * own), j1 = min(PA, j0 + own);
        uint32_t sum = 0;
        for (uint32_t j = j0; j < j1; ++j) sum += cnt[j] & 0xffffu;
        uint32_t inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        uint32_t wb = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kRollWarps; ++w) { const uint32_t v = warp_tot[w]; if (w < warp) wb += v; total += v; }
        uint32_t o = wb + inc - sum;
        for (uint32_t j = j0; j < j1; ++j) {
            const uint32_t c = cnt[j] & 0xffffu;
            o += c;
            cnt[j] = o << 16;                     // run end; the count starts again at zero
            cur[j] += c;                          // the run takes slots [cur - c, cur)
        }
        if (threadIdx.x == 0) s_fill = 0;
        __syncthreads();
        // rank r of a run goes to position end - 1 - r and slot cur - 1 - r: consecutive positions, consecutive slots
        for (uint32_t i = threadIdx.x; i < nslots; i += kRollThreads) {
            const uint32_t tg = tags[i];
            if (tg == kABatchNoTag) continue;
            idx[(cnt[tg & ((1u << kABatchPartBits) - 1)] >> 16) - 1 - (tg >> kABatchPartBits)] = (uint16_t)i;
        }
        __syncthreads();
        for (uint32_t q = threadIdx.x; q < total; q += kRollThreads) {
            const uint32_t i = idx[q], tg = tags[i];
            const uint32_t slot = cur[tg & ((1u << kABatchPartBits) - 1)] - 1 - (tg >> kABatchPartBits);
            store_rec_stream<NW>(out0 + (size_t)slot * NW, load_rec<NW>(stage + (size_t)i * NW));
        }
        __syncthreads();                          // the next batch overwrites the stage
        if (!more) break;
    }
    for (uint32_t i = threadIdx.x; i < PA; i += blockDim.x) mybase[i] = region0 + cur[i];   // chained launches continue here
}

// ---- the id form: a batch planned from the ids -----------------------------------------------------------------------------
// With the id array a record's partition is known before it is rolled, so the batch is laid out before anything enters it. A
// warp walks its tiles in STEPS of 32 chunks (chunk 32 j + lane of the tile for lane `lane`), and a batch runs in four phases:
// 1. plan: each warp continues where its last batch stopped -- a (tile, step, record) position -- and reads the id rows of its
//    next step (16-byte loads). It takes the step's records window by window as far as its share of the batch (cap /
//    kRollWarps) allows: a popc of a ballot per record index counts the step's own records at that index, and each own id adds
//    one to its partition's batch count. A step that does not fit is taken up to the last window that does, and the warp
//    resumes there in the next batch. Equal shares keep every warp rolling in every batch: a shared reservation of whole steps
//    let the first three of sixteen warps take a batch where every record is own (all-windows mode, one pass).
// 2. claim: a block scan of the batch counts gives each partition its run in the batch, claimed from its cursor.
// 3. roll: each warp rolls exactly what it planned, with no capacity test; an own record takes the next position of its run
//    (one shared-memory atomic) and is written there, with its 2-byte partition next to it: the batch is in partition order.
// 4. flush: consecutive threads store consecutive positions to their partition's slots.
// Per own record that is two shared-memory atomics (the plan's count, the roll's position) and no tag, no permute pass and no
// indirect read in the flush; a foreign window costs the roll and an id test. The flush needs no barrier behind it: the next plan
// touches only the low halves of the batch counts.
// `-Xptxas -v` (at most 64 registers): no stack frame at 1 to 3 words per record; at 4 words of reads a 16-byte frame with 20
// bytes of spill stores, against 56 bytes and 68-84 bytes for the id form of the arrival-order kernel it replaced.
template <int NW, class Src, bool BOTH>
__global__ void __launch_bounds__(kRollThreads, 2) levelA_scatter_plan_k(Src src, LevelA p, uint64_t *__restrict__ base, uint64_t *__restrict__ out,
                                                                        const uint64_t *__restrict__ tile_off, const uint16_t *__restrict__ ids,
                                                                        uint32_t id_lo, uint32_t row_stride, uint32_t q_lo, uint64_t ids_len, uint32_t cap) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    __shared__ uint32_t warp_tot[kRollWarps];
    constexpr int kR = BOTH ? 2 : 1;              // records per window
    constexpr int kRowV = Src::kIds / 8;          // 16-byte words of an id row
    const uint32_t PA = p.PA;
    // one 32-bit cursor per partition, relative to the first record this launch may write; in `run` the partition's batch count
    // (low 16 bits, the plan) and the next position of its run in the batch (high 16 bits, the roll; the run's end at the flush)
    uint32_t *cur = reinterpret_cast<uint32_t *>(sm_raw);               // PA
    uint32_t *run = cur + PA;                                           // PA
    RollWarp &rw = *roll_warp_slice(sm_raw, 2 * PA);
    uint64_t *stage = reinterpret_cast<uint64_t *>(sm_raw + abatch_offset(PA));    // [cap][NW] records in partition order
    uint16_t *ptag = reinterpret_cast<uint16_t *>(stage + (size_t)cap * NW);      // [cap]     partition of a batch position
    uint64_t *mybase = base + (size_t)blockIdx.x * row_stride + q_lo;
    const uint64_t region0 = mybase[0];                                 // cursors of a row ascend with the partition
    for (uint32_t i = threadIdx.x; i < PA; i += blockDim.x) { cur[i] = (uint32_t)(mybase[i] - region0); run[i] = 0; }
    __syncthreads();
    uint64_t *const out0 = out + region0 * NW;
    const int K = p.K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t ntiles = (src.n + kRollTile - 1) / kRollTile;
    const int64_t per = (ntiles + gridDim.x - 1) / gridDim.x;
    const int64_t t0 = (int64_t)blockIdx.x * per, t1 = min(ntiles, t0 + per);
    const uint32_t share = cap / kRollWarps;

    // plan position: tile pt, step pj, record ps of every chunk of the step; pn = the tile's chunks, prow = its id rows
    int64_t pt = t0 + warp;
    int pj = 0, ps = 0;
    uint32_t pn = 0;
    bool p_enter = true;
    const ulonglong2 *prow = nullptr;
    // roll position (the plan position the batch started from) and the tile staged in the warp's slice
    int64_t rt = pt;
    int rj = 0, rs = 0;
    bool need_setup = true;
    int nitems = 0;
    uint32_t nunits = 0, unif = 0;
    bool staged = false;
    uint64_t next_w0 = 0;
    const ulonglong2 *row = nullptr;
    for (;;) {
        // ---- 1. plan
        uint32_t room = share;
        while (pt < t1) {                         // warp-uniform
            if (p_enter) {
                const uint64_t a = tile_off[pt], b = tile_off[pt + 1];
                // the id rows of the warp's next tile go to L2 now, a tile before the plan reads them (Src::kIdLines <= 64 lines)
                if (pt + kRollWarps < t1) {
                    const uint64_t nr = tile_off[pt + kRollWarps];
                    if ((Src::kIdLines >= 32 || lane < Src::kIdLines) && nr + 64 * lane < ids_len) prefetch_l2(ids + nr + 64 * lane);
                    if (lane < Src::kIdLines - 32 && nr + 64 * (32 + lane) < ids_len) prefetch_l2(ids + nr + 64 * (32 + lane));
                }
                pn = (uint32_t)((b - a) / Src::kIds);
                prow = reinterpret_cast<const ulonglong2 *>(ids + a);
                p_enter = false;
            }
            if ((uint32_t)pj * 32 >= pn) {        // the tile is planned
                pt += kRollWarps; pj = 0; ps = 0; p_enter = true;
                continue;
            }
            if (room < 32 * kR) break;            // not even one window of the step fits for sure
            const uint32_t u = (uint32_t)pj * 32 + lane;
            uint64_t idq[Src::kIds / 4];
#pragma unroll
            for (int v = 0; v < kRowV; ++v) {
                ulonglong2 x = make_ulonglong2(~0ull, ~0ull);               // no chunk: foreign ids
                if (u < pn) x = __ldg(prow + (size_t)u * kRowV + v);
                idq[2 * v] = x.x; idq[2 * v + 1] = x.y;
            }
            int end = Src::kIds;                  // records [ps, end) of the step are taken
#pragma unroll
            for (int e = 0; e < Src::kIds; e += kR) {
                uint32_t part[kR];
                bool own[kR];
                uint32_t c = 0;
#pragma unroll
                for (int r = 0; r < kR; ++r) {
                    part[r] = (uint32_t)((idq[(e + r) / 4] >> (16 * ((e + r) % 4))) & 0xffffu) - id_lo;    // 0xffff - id_lo stays >= PA
                    own[r] = e >= ps && part[r] < PA;
                    c += __popc(__ballot_sync(0xffffffffu, own[r]));
                }
                if (c > room) { end = e; break; }
                room -= c;
#pragma unroll
                for (int r = 0; r < kR; ++r) if (own[r]) atomicAdd(&run[part[r]], 1u);
            }
            if (end < Src::kIds) { ps = end; break; }
            ++pj; ps = 0;
        }
        const bool more = __syncthreads_or(pt < t1);
        // ---- 2. claim: scan of the batch counts (a thread owns a run of consecutive partitions), runs claimed from the cursors
        const uint32_t own = (PA + kRollThreads - 1) / kRollThreads;
        const uint32_t j0 = min(PA, threadIdx.x * own), j1 = min(PA, j0 + own);
        uint32_t sum = 0;
        for (uint32_t j = j0; j < j1; ++j) sum += run[j] & 0xffffu;
        uint32_t inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        uint32_t wb = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kRollWarps; ++w) { const uint32_t v = warp_tot[w]; if (w < warp) wb += v; total += v; }
        uint32_t o = wb + inc - sum;
        for (uint32_t j = j0; j < j1; ++j) {
            const uint32_t c = run[j] & 0xffffu;
            run[j] = o << 16;                     // run start; the count starts again at zero
            o += c;
            cur[j] += c;                          // the run takes slots [cur - c, cur)
        }
        __syncthreads();
        // ---- 3. roll: from the roll position up to the plan position
        while (rt < pt || (rt == pt && (rj < pj || (rj == pj && rs < ps)))) {   // warp-uniform
            if (need_setup) {
                const int64_t item0 = rt * kRollTile;
                nitems = (int)min((int64_t)kRollTile, src.n - item0);
                // the warp's next tile is kRollWarps tiles ahead: its item metadata goes to L2 now, its packed items at the end of
                // this tile, when the loads of their addresses issued here have long returned
                const int64_t nx = (rt + kRollWarps) * kRollTile;
                if (rt + kRollWarps < t1) {
                    next_w0 = src.first_word(nx);
                    src.prefetch_items(nx, lane);
                }
                nunits = roll_warp_setup<BOTH>(src, item0, nitems, rw, &unif, &staged);
                row = reinterpret_cast<const ulonglong2 *>(ids + tile_off[rt]);
                need_setup = false;
            }
            if ((uint32_t)rj * 32 >= nunits) {    // the tile is done
                if (rt + kRollWarps < t1 && lane < 10 && next_w0 + 16 * lane < src.nwords) prefetch_l2(src.words + next_w0 + 16 * lane);   // 10 lines = 32 reads x 5 words
                __syncwarp();                     // the slice is rewritten by the next tile's setup
                rt += kRollWarps; rj = 0; rs = 0;
                need_setup = true;
                continue;
            }
            const int end = (rt == pt && rj == pj) ? ps : Src::kIds;
            const int u = rj * 32 + lane;
            if (u < (int)nunits) {
                const RollUnit q = roll_unit<BOTH>(rw, nitems, (uint32_t)u, unif, K);
                const int s_end = min(end, BOTH ? 2 * q.cnt : q.cnt);
                if (rs < s_end) {
                    uint64_t idq[Src::kIds / 4];
#pragma unroll
                    for (int v = 0; v < kRowV; ++v) {
                        const ulonglong2 x = __ldg(row + (size_t)u * kRowV + v);
                        idq[2 * v] = x.x; idq[2 * v + 1] = x.y;
                    }
                    // the id queue from record rs on (whole words moved register to register, then the rest of a word)
                    for (int w = 0; w < rs / 4; ++w) {
#pragma unroll
                        for (int v = 0; v + 1 < Src::kIds / 4; ++v) idq[v] = idq[v + 1];
                    }
                    idq[0] >>= 16 * (rs & 3);
                    const uint64_t *seq = staged ? static_cast<const uint64_t *>(rw.words + rw.off[q.it]) : src.words + src.first_word(rt * kRollTile + q.it);
                    RollState<NW> st;
                    roll_init<NW>(st, seq, q.j0 + rs / kR, K, q.cnt - rs / kR);
                    for (int s = rs;;) {
                        const uint32_t part = (uint32_t)(idq[0] & 0xffffu) - id_lo;
                        if (part < PA) {
                            // a word-by-word select: `cond ? st.f : st.r` bound to a reference made the compiler keep the roll
                            // state in local memory to pick an address
                            const bool fwd = BOTH ? !(s & 1) : kmer_is_minimal<NW>(st.f, st.r);
                            Kmer<NW> k;
#pragma unroll
                            for (int j = 0; j < NW; ++j) k.w[j] = fwd ? st.f.w[j] : st.r.w[j];
                            const uint32_t pos = atomicAdd(&run[part], 1u << 16) >> 16;
                            store_rec<NW>(stage + (size_t)pos * NW, k);
                            ptag[pos] = (uint16_t)part;
                        }
                        if (++s >= s_end) break;
                        if (!BOTH || !(s & 1)) roll_next<NW>(st, K);
                        if ((s & 3) == 0) {
#pragma unroll
                            for (int v = 0; v + 1 < Src::kIds / 4; ++v) idq[v] = idq[v + 1];
                        } else {
                            idq[0] >>= 16;
                        }
                    }
                }
            }
            if (end == Src::kIds) { ++rj; rs = 0; } else rs = end;
        }
        __syncthreads();
        // ---- 4. flush: position q of a run ending at e goes to slot cur - e + q
        for (uint32_t q = threadIdx.x; q < total; q += kRollThreads) {
            const uint32_t part = ptag[q];
            const uint32_t slot = cur[part] - (run[part] >> 16) + q;
            store_rec_stream<NW>(out0 + (size_t)slot * NW, load_rec<NW>(stage + (size_t)q * NW));
        }
        if (!more) break;
    }
    for (uint32_t i = threadIdx.x; i < PA; i += blockDim.x) mybase[i] = region0 + cur[i];   // chained launches continue here
}
// Measured (H100 80GB HBM3, 700 W, 40 M x 150 bp, k = 55, 4 passes, PA = 640, two CTAs per SM): the planned batch (3488 records
// at 16 bytes) takes 114.8-114.9 ms per step against 128.3-129.0 ms for the arrival-order batch (2848 records) in the same form,
// which took 129 ms against 189 ms for the form that stored each record as it was rolled. (A third generation of
// this kernel -- id sweep, 32-bit keys collected without atomics, ballot-ranked LSD sort of the batch in shared memory,
// run-by-run flush -- was parity clean and slower than the store-as-you-go form: about twice the thread instructions per
// record. Removed.)

// ------------------------------------------------------------------------------------------------------------
// segments
// ------------------------------------------------------------------------------------------------------------
struct Seg {
    uint64_t start;     // record index in its buffer
    uint64_t len;
    uint32_t bits;      // key bits already fixed by partitioning
    uint32_t bb;        // (bucket << 1) | buffer
};

__global__ void seg_init_k(const uint64_t *__restrict__ part_start, const uint64_t *__restrict__ part_total, uint32_t PA, int rA,
                           uint32_t b_lo, Seg *__restrict__ segs) {
    uint32_t part = blockIdx.x * blockDim.x + threadIdx.x;
    if (part >= PA) return;
    Seg s;
    s.start = part_start[part]; s.len = part_total[part]; s.bits = (uint32_t)rA; s.bb = ((b_lo + (part >> rA)) << 1) | 0u;
    segs[part] = s;
}

// ---- CTA-major staging of the level-A output ------------------------------------------------------------------------------
// Level A writes CTA-major: CTA g owns one contiguous region of the staging
// buffer, partitioned inside ([g][partition]); a partition is then G pieces, and the FIRST refinement round reads its
// segment piece by piece (sequential runs: one page at a time) and writes the children partition-major into the partner
// buffer -- the gather costs no extra pass over the data. Partitions that need no refinement take the same kernel with
// r = 0 (a copy into the partner buffer).
// The layout is not what sets the partition kernel's store rate: in scripts/microbench/scatter_bench.cu, CTA-major and
// partition-major outputs run within 6 % of each other at every stream count, and confining a CTA's stores to 2 MB slices of
// its 57 MB region at a time changes nothing (DESIGN.md 6.2). The rate falls with the open streams per CTA, and at 512 to
// 1024 streams it doubles with 32-byte instead of 16-byte stores.
struct Pieces {
    const uint64_t *pbase;     // [G][PA]  first record of piece (g, partition) in the staging buffer
    const uint32_t *cnt;       // blk_counts + p_lo: cnt[g * cnt_stride + partition]
    uint32_t cnt_stride, PA;
    int G;
};
static const int kMaxPieces = 1024;       // CTAs of the level-A grid (G <= 1024)

// row g of cnt -> exclusive prefix inside the row (rel) and the row total
__global__ void stage_rows_k(const uint32_t *__restrict__ cnt, uint32_t cnt_stride, uint32_t PA, uint64_t *__restrict__ rel, uint64_t *__restrict__ row_total) {
    __shared__ uint64_t wsum[8];
    __shared__ uint64_t carry_s;
    const uint32_t *row = cnt + (size_t)blockIdx.x * cnt_stride;
    uint64_t *out = rel + (size_t)blockIdx.x * PA;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;       // 256 threads
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (uint32_t b = 0; b < PA; b += blockDim.x) {
        const uint32_t i = b + threadIdx.x;
        const uint64_t v = i < PA ? row[i] : 0;
        uint64_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        uint64_t wb = 0, all = 0;
        for (int w = 0; w < 8; ++w) { if (w < warp) wb += wsum[w]; all += wsum[w]; }
        const uint64_t carry = carry_s;
        if (i < PA) out[i] = carry + wb + inc - v;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + all;
        __syncthreads();
    }
    if (threadIdx.x == 0) row_total[blockIdx.x] = carry_s;
}
__global__ void stage_add_k(uint64_t *__restrict__ rel, const uint64_t *__restrict__ row_start, uint32_t PA, int G) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)G * PA) return;
    rel[i] += row_start[i / PA];
}

struct RefinePlan { uint32_t cap, target, rmax; int total_bits; };
__device__ __forceinline__ int plan_r(const RefinePlan &rp, uint64_t len, uint32_t bits) {
    if (len <= rp.cap) return 0;
    int rem = rp.total_bits - (int)bits;
    if (rem <= 0) return 0;
    uint64_t want = (len + rp.target - 1) / rp.target;
    int r = 1;
    while (r < (int)rp.rmax && (1ull << r) < want) ++r;
    return r < rem ? r : rem;
}
// children[i] = 2^r or 1 ; work flag
__global__ void refine_plan_k(const Seg *__restrict__ segs, uint64_t n, RefinePlan rp, uint32_t *__restrict__ nchild, uint32_t *__restrict__ isw, int force_all) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int r = plan_r(rp, segs[i].len, segs[i].bits);
    nchild[i] = r ? (1u << r) : 1u;
    isw[i] = (r || force_all) ? 1u : 0u;      // force_all: staged level-A output, every segment is gathered by the refinement kernel
}
__global__ void refine_copy_k(const Seg *__restrict__ segs, uint64_t n, const uint32_t *__restrict__ isw, const uint64_t *__restrict__ child_base,
                              const uint64_t *__restrict__ work_pos, Seg *__restrict__ nsegs, uint64_t *__restrict__ worklist) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (isw[i]) worklist[work_pos[i]] = i;
    else nsegs[child_base[i]] = segs[i];
}

static const int kRThreads = 1024;
static const int kRWarps = kRThreads / 32;
static const int kRMaxBins = 2048;
// The scatter sweep collects a batch of records per CTA in shared memory and writes it out bin by bin. A thread holds a batch's
// share in registers between its loads and the permute: 128 bytes of records at 1 and 2 words (16384 / 8192 records, 4 per bin
// on average at 2048 bins for 16-byte records), 96 at 3 and 4 words, where 128 spill in the gather (64 registers at one CTA of
// 1024 threads per SM). At 8-byte records the batch is capped at 12 per thread so that it and its slot array fit shared memory.
template <int NW> struct RBatch {
    static const int RPT = NW == 1 ? 12 : NW == 2 ? 8 : NW == 3 ? 4 : 3;                              // records per thread
    static const int N = RPT * kRThreads;                                                                  // records per batch
    static constexpr size_t smem() { return (size_t)N * (NW * sizeof(uint64_t) + sizeof(uint32_t)); }
};

// one CTA splits one oversize segment by its next r key bits: buf[bb&1] -> buf[(bb&1)^1]
// PIECED: the segments are level-A partitions whose records lie in G pieces of the CTA-major staging buffer (buf0); segment
// index == partition. A warp streams the pieces g = warp, warp + 32, ... one after the other; the children are written
// contiguously into buf1.
// Two sweeps over the segment: a histogram of the r-bit digits (-> the children's ranges), then the scatter. At 2048 bins a bin
// receives a record only every few microseconds, so records stored one by one as they arrive leave L2 as partly written sectors
// that each cost a fill read. The scatter therefore works in batches of RBatch<NW>::N records: every record takes a rank in its
// bin with one shared-memory atomic, a block scan of the batch counts gives each bin's run in the batch, the owner thread of a
// bin (2 bins per thread, as in the segment scan) claims the run from the bin's cursor, which it keeps in registers, and the batch
// is permuted into bin order in shared memory and flushed with consecutive threads storing consecutive records of a run. The
// next batch's loads are issued before the flush. The order inside a child is arbitrary, as it was with atomic slots.
template <int NW, bool PIECED>
__global__ void __launch_bounds__(kRThreads) refine_k(const Seg *__restrict__ segs, const uint64_t *__restrict__ worklist, uint64_t nwork,
                                                     const uint64_t *__restrict__ child_base, RefinePlan rp, int K,
                                                     uint64_t *__restrict__ buf0, uint64_t *__restrict__ buf1, Seg *__restrict__ nsegs,
                                                     unsigned long long *__restrict__ work_counter, Pieces pc) {
    constexpr int RPT = RBatch<NW>::RPT, N = RBatch<NW>::N;
    __shared__ uint32_t hist[kRMaxBins];        // segment histogram, then the batch counts
    __shared__ uint32_t run_off[kRMaxBins];     // a bin's first position in the batch
    __shared__ uint32_t run_slot[kRMaxBins];    // ... and its first slot in the child
    __shared__ uint32_t warp_tot[kRWarps];
    __shared__ unsigned long long s_w;
    __shared__ uint64_t pc_start[PIECED ? kMaxPieces : 1];
    __shared__ uint32_t pc_len[PIECED ? kMaxPieces : 1];
    extern __shared__ uint64_t sm_refine_dyn[];
    uint64_t *stage = sm_refine_dyn;                                                    // [N][NW] the batch in bin order
    uint32_t *stage_slot = reinterpret_cast<uint32_t *>(stage + (size_t)N * NW);         // [N]     their slots in the segment
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (threadIdx.x == 0) s_w = atomicAdd(work_counter, 1ull);
        __syncthreads();
        const uint64_t wi = s_w;
        __syncthreads();
        if (wi >= nwork) return;
        const uint64_t si = worklist[wi];
        const Seg s = segs[si];
        const int r = plan_r(rp, s.len, s.bits);
        const uint32_t nb = 1u << r;
        const uint64_t *src = ((s.bb & 1) ? buf1 : buf0) + s.start * NW;
        uint64_t *dst = ((s.bb & 1) ? buf0 : buf1) + s.start * NW;
        if (PIECED) {
            for (int g = threadIdx.x; g < pc.G; g += blockDim.x) {
                pc_start[g] = pc.pbase[(size_t)g * pc.PA + si];
                pc_len[g] = pc.cnt[(size_t)g * pc.cnt_stride + si];
            }
        }
        for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        if (PIECED) {
            // a WARP streams a piece (a few thousand consecutive records), four independent 512-byte loads in flight per warp:
            // with the whole CTA striding over one piece at a time a thread had a single 16-byte load outstanding
            for (int g = warp; g < pc.G; g += kRWarps) {
                const uint64_t *ps = buf0 + pc_start[g] * NW;
                const uint32_t n = pc_len[g];
                uint32_t i = lane;
                for (; i + 96 < n; i += 128) {
                    const Kmer<NW> k0 = load_rec<NW>(ps + (uint64_t)i * NW), k1 = load_rec<NW>(ps + (uint64_t)(i + 32) * NW);
                    const Kmer<NW> k2 = load_rec<NW>(ps + (uint64_t)(i + 64) * NW), k3 = load_rec<NW>(ps + (uint64_t)(i + 96) * NW);
                    atomicAdd(&hist[key_bits<NW>(k0, K, (int)s.bits, r)], 1u);
                    atomicAdd(&hist[key_bits<NW>(k1, K, (int)s.bits, r)], 1u);
                    atomicAdd(&hist[key_bits<NW>(k2, K, (int)s.bits, r)], 1u);
                    atomicAdd(&hist[key_bits<NW>(k3, K, (int)s.bits, r)], 1u);
                }
                for (; i < n; i += 32) {
                    const Kmer<NW> k = load_rec<NW>(ps + (uint64_t)i * NW);
                    atomicAdd(&hist[key_bits<NW>(k, K, (int)s.bits, r)], 1u);
                }
            }
        } else {
            // (Four loads in flight for the contiguous form too -- second-level splits, the multi-GPU path -- need 57 instead of 32
            // registers, which halves its residency: no gain with 2 GPUs, slower on one. Not kept.)
            for (uint64_t i = threadIdx.x; i < s.len; i += blockDim.x) {
                Kmer<NW> k = load_rec<NW>(src + i * NW);
                atomicAdd(&hist[key_bits<NW>(k, K, (int)s.bits, r)], 1u);
            }
        }
        __syncthreads();
        // exclusive scan of hist[0..nb) (nb <= 2048 = 2 per thread)
        uint32_t a = 0, b = 0;
        const uint32_t i0 = 2 * threadIdx.x;
        if (i0 < nb) { a = hist[i0]; hist[i0] = 0; }          // the owner's bins: the batch counts start at zero (the scan's
        if (i0 + 1 < nb) { b = hist[i0 + 1]; hist[i0 + 1] = 0; }   // barriers order this before the first batch's atomics)
        uint32_t v = a + b, inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) warp_tot[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = warp_tot[lane], winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
                if (lane >= o) winc += t;
            }
            warp_tot[lane] = winc - w;
        }
        __syncthreads();
        const uint32_t ex = warp_tot[warp] + inc - v;
        const uint64_t cb = child_base[si];
        if (i0 < nb) {
            Seg c; c.start = s.start + ex; c.len = a; c.bits = s.bits + (uint32_t)r; c.bb = s.bb ^ 1u;
            nsegs[cb + i0] = c;
        }
        if (i0 + 1 < nb) {
            Seg c; c.start = s.start + ex + a; c.len = b; c.bits = s.bits + (uint32_t)r; c.bb = s.bb ^ 1u;
            nsegs[cb + i0 + 1] = c;
        }
        uint32_t cur0 = ex, cur1 = ex + a;                            // the owner's two bins: next free slot in the child

        // ---- scatter sweep, batch by batch
        Kmer<NW> rec[RPT];
        uint32_t have = 0;                        // bit j: rec[j] holds a record
        int pg = warp;                            // PIECED: the warp's piece ...
        uint32_t ppos = 0;                        // ... and its next record (warp-uniform)
        uint64_t cpos = 0;                        // contiguous: the batch's first record
        auto load_batch = [&]() {
            have = 0;
            if (PIECED) {
                while (pg < pc.G && ppos >= pc_len[pg]) { pg += kRWarps; ppos = 0; }
                if (pg < pc.G) {
                    const uint64_t *ps = buf0 + pc_start[pg] * NW;
                    const uint32_t n = pc_len[pg];
#pragma unroll
                    for (int j = 0; j < RPT; ++j) {
                        const uint32_t i = ppos + lane + 32 * j;
                        if (i < n) { rec[j] = load_rec<NW>(ps + (uint64_t)i * NW); have |= 1u << j; }
                    }
                    ppos += 32 * RPT;
                }
            } else {
#pragma unroll
                for (int j = 0; j < RPT; ++j) {
                    const uint64_t i = cpos + threadIdx.x + (uint64_t)kRThreads * j;
                    if (i < s.len) { rec[j] = load_rec<NW>(src + i * NW); have |= 1u << j; }
                }
                cpos += N;
            }
        };
        load_batch();
        for (;;) {
            uint32_t tag[RPT];                    // (rank in its bin's run << 11) | bin
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
                if (have >> j & 1u) {
                    const uint32_t bin = key_bits<NW>(rec[j], K, (int)s.bits, r);
                    tag[j] = (atomicAdd(&hist[bin], 1u) << 11) | bin;
                }
            }
            if (!__syncthreads_or(have)) break;
            // block scan of the batch counts; the owner claims each of its bins' runs and clears the count for the next batch
            const uint32_t c0 = i0 < nb ? hist[i0] : 0u, c1 = i0 + 1 < nb ? hist[i0 + 1] : 0u;
            const uint32_t bv = c0 + c1;
            uint32_t binc = bv;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, binc, o);
                if (lane >= o) binc += t;
            }
            if (lane == 31) warp_tot[warp] = binc;
            __syncthreads();
            uint32_t w = warp_tot[lane], winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
                if (lane >= o) winc += t;
            }
            const uint32_t total = __shfl_sync(0xffffffffu, winc, 31);
            const uint32_t off = __shfl_sync(0xffffffffu, winc - w, warp) + binc - bv;
            if (i0 < nb) { run_off[i0] = off; run_slot[i0] = cur0; hist[i0] = 0; cur0 += c0; }
            if (i0 + 1 < nb) { run_off[i0 + 1] = off + c0; run_slot[i0 + 1] = cur1; hist[i0 + 1] = 0; cur1 += c1; }
            __syncthreads();
            // permute into bin order, then put the next batch's loads in flight before the flush
#pragma unroll
            for (int j = 0; j < RPT; ++j) {
                if (have >> j & 1u) {
                    const uint32_t bin = tag[j] & (kRMaxBins - 1), rank = tag[j] >> 11;
                    const uint32_t p = run_off[bin] + rank;
                    store_rec<NW>(stage + (size_t)p * NW, rec[j]);
                    stage_slot[p] = run_slot[bin] + rank;
                }
            }
            load_batch();
            __syncthreads();
            for (uint32_t p = threadIdx.x; p < total; p += kRThreads)
                store_rec_stream<NW>(dst + (uint64_t)stage_slot[p] * NW, load_rec<NW>(stage + (size_t)p * NW));
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// local sort + unique + count
// ------------------------------------------------------------------------------------------------------------
template <int NW> struct SortCfg { static const int CAP = NW <= 2 ? 2048 : 1024; };
static const int kSThreads = 512;     // two CTAs of 16 warps per SM: room for a second segment buffer at every record width
static const int kSWarps = kSThreads / 32;

// stable LSD pass over key bits [pos, pos+width) : A -> Bf
template <int NW>
__device__ __forceinline__ void lsd_pass(const uint64_t *A, uint64_t *Bf, uint32_t n, int K, int pos, int width, uint32_t *cnt /*[kSWarps][256]*/,
                                         uint32_t *tot /*[256 / 32]*/) {
    static_assert(kSThreads >= 256, "one thread per digit");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk = ((n + kSWarps * 32 - 1) / (kSWarps * 32)) * 32;   // items per warp, multiple of 32
    const uint32_t w0 = warp * chunk;
    for (int i = threadIdx.x; i < kSWarps * 256; i += kSThreads) cnt[i] = 0;
    __syncthreads();
    for (uint32_t r = 0; r < chunk; r += 32) {
        const uint32_t i = w0 + r + lane;
        uint32_t d = 256;
        if (i < n) d = key_bits<NW>(load_rec<NW>(A + (size_t)i * NW), K, pos, width);
        const uint32_t m = __match_any_sync(0xffffffffu, d);
        if (d < 256 && (int)(__ffs(m) - 1) == lane) cnt[warp * 256 + d] += __popc(m);
        __syncwarp();
    }
    __syncthreads();
    // per digit (threads 0..255, one digit each): warp prefix + digit totals
    {
        const uint32_t d = threadIdx.x;
        uint32_t run = 0, inc = 0;
        if (d < 256) {
#pragma unroll
            for (int w = 0; w < kSWarps; ++w) { uint32_t t = cnt[w * 256 + d]; cnt[w * 256 + d] = run; run += t; }
            // exclusive scan of run over 256 digits
            inc = run;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (lane == 31) tot[warp] = inc;
        }
        __syncthreads();
        if (d < 256) {
            uint32_t wb = 0;
            for (int w = 0; w < warp; ++w) wb += tot[w];
            const uint32_t ex = wb + inc - run;
#pragma unroll
            for (int w = 0; w < kSWarps; ++w) cnt[w * 256 + d] += ex;
        }
    }
    __syncthreads();
    for (uint32_t r = 0; r < chunk; r += 32) {
        const uint32_t i = w0 + r + lane;
        uint32_t d = 256;
        Kmer<NW> k;
        if (i < n) { k = load_rec<NW>(A + (size_t)i * NW); d = key_bits<NW>(k, K, pos, width); }
        const uint32_t m = __match_any_sync(0xffffffffu, d);
        uint32_t rank = 0;
        if (d < 256) rank = cnt[warp * 256 + d] + __popc(m & ((1u << lane) - 1));
        __syncwarp();
        if (d < 256) {
            store_rec<NW>(Bf + (size_t)rank * NW, k);
            if ((int)(__ffs(m) - 1) == lane) cnt[warp * 256 + d] += __popc(m);
        }
        __syncwarp();
    }
    __syncthreads();
}

// sort A[0..n) by key bits [lo, hi) (MSB-first positions). Result may end up in A or Bf; returns pointer.
template <int NW>
__device__ __forceinline__ uint64_t *lsd_sort_range(uint64_t *A, uint64_t *Bf, uint32_t n, int K, int lo, int hi, uint32_t *cnt, uint32_t *tot) {
    int p = hi;
    while (p > lo) {
        int w = p - lo >= 8 ? 8 : p - lo;
        lsd_pass<NW>(A, Bf, n, K, p - w, w, cnt, tot);
        uint64_t *t = A; A = Bf; Bf = t;
        p -= w;
    }
    return A;
}

// exclusive scan of one value per thread over the CTA; `all` receives the total. One barrier; `tot` is free again only after the
// next barrier.
__device__ __forceinline__ uint32_t cta_exscan(uint32_t v, uint32_t *tot, uint32_t &all) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) tot[warp] = inc;
    __syncthreads();
    uint32_t wb = 0;
    all = 0;
#pragma unroll
    for (int w = 0; w < kSWarps; ++w) { const uint32_t t = tot[w]; if (w < warp) wb += t; all += t; }
    return wb + inc - v;
}

// +1 on the 16-bit counter c[i] (two counters share a 32-bit word; no counter exceeds CAP), returns its old value
__device__ __forceinline__ uint32_t atomic_inc_u16(uint16_t *c, uint32_t i) {
    const int sh = (i & 1) * 16;
    return (atomicAdd(reinterpret_cast<uint32_t *>(c) + (i >> 1), 1u << sh) >> sh) & 0xffffu;
}

// asynchronous global -> shared copy of a segment's records by the whole CTA (cp.async; completes at cp_async_wait_all). Records
// of an even number of words start on a 16-byte boundary and go as 16-byte copies; 8- and 24-byte records may start on an 8-byte
// boundary and go as 8-byte copies. Empty and oversize segments are never loaded.
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }
template <int NW, int CAP>
__device__ __forceinline__ void prefetch_segment(uint64_t *dst, const uint64_t *src, uint64_t len) {
    if (len == 0 || len > (uint64_t)CAP) return;
    const uint32_t sdst = (uint32_t)__cvta_generic_to_shared(dst);
    if (NW % 2 == 0) {
        for (uint32_t q = threadIdx.x; q < (uint32_t)len * NW / 2; q += kSThreads)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sdst + 16 * q), "l"(src + 2 * q) : "memory");
    } else {
        for (uint32_t q = threadIdx.x; q < (uint32_t)len * NW; q += kSThreads)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(sdst + 8 * q), "l"(src + q) : "memory");
    }
}

// ---- local sort: representative + residual -----------------------------------------------------------------------------
// After level A + MSD refinement a segment holds ~CAP*3/4 records that agree on their first `bits` key bits. Most of them are
// copies of a few keys (a genomic (k+1)-mer is seen ~coverage times) plus error singletons. Earlier generations (a full LSD
// radix sort per segment; one counting pass into 2^11 bins with one thread collapsing each bin; one thread per bin
// deduplicating its residual records and writing the bin) were replaced by the kernel below; the LSD passes above survive as its
// exact fallback.
static const int kSortBinBits = 11;   // bins per segment = 2^11: fewer bins = less per-segment bookkeeping (init + two scans over the bins) but more
                                      // keys sharing a bin (2^10 bins gave no gain)

// Every bin elects a representative (any one of its records: a plain shared-memory store per record); records equal to it only
// bump a counter. A bin holding records that differ from its representative gets a run of slots in a small residual buffer:
// the representative first, then those records. Every residual slot then finds by itself, comparing within its bin's few
// slots, whether it holds its key's first copy and how many copies there are, and every distinct key takes its rank in the
// bin from the same compares, so each output record has its position without a thread walking a bin. Anything unusual
// (residual overflow, a bin with more than kBinSlotsMax slots or more than kBinDistinctMax keys) falls back to the exact LSD
// radix path, which uses the segment's region in the partner buffer as scratch.
// The CTAs are persistent and load one segment ahead: while segment i is sorted, segment i+1 arrives in the second buffer by
// cp.async, and the claim of segment i+2 is in flight.
static const int kResCap = 512;
static const int kBinSlotsMax = 128;
static const int kBinDistinctMax = 16;

template <int NW, int kBinBits, int CAP>
struct SortSmem {
    static constexpr int kBins = 1 << kBinBits;
    // two segment buffers, the residual records, rep/repcnt/rhist/dres and rstart (u16 per bin), rcnt/rbin (u16 per residual slot)
    static constexpr size_t bytes = ((size_t)2 * CAP + kResCap) * NW * sizeof(uint64_t) + ((size_t)5 * kBins + 2 + 2 * kResCap) * sizeof(uint16_t);
};

template <int NW, int kBinBits, int CAP>
__device__ __forceinline__ void sort_segment(const uint64_t si, const Seg s, uint64_t *A, uint64_t *R, uint16_t *rep, uint16_t *rcnt, uint16_t *rbin,
                                             uint32_t *lsdcnt, uint32_t *tot, int *s_flag, int K, uint64_t *buf0, uint64_t *buf1,
                                             uint32_t *ndist, unsigned long long *stats) {
    constexpr int kBins = 1 << kBinBits;
    constexpr int BPT = kBins / kSThreads;
    constexpr int IPT = CAP / kSThreads;                  // records per thread
    uint16_t *repcnt = rep + kBins;                       // copies of the representative besides itself
    uint16_t *rhist = repcnt + kBins;                     // residual records -> slot cursor -> output offset of the bin
    uint16_t *dres = rhist + kBins;                       // distinct keys in the bin's residual slots
    uint16_t *rstart = dres + kBins;                      // kBins+1 first residual slot of the bin
    const int total_bits = 2 * K;
    uint64_t *gsrc = ((s.bb & 1) ? buf1 : buf0) + s.start * NW;
    uint64_t *gpartner = ((s.bb & 1) ? buf0 : buf1) + s.start * NW;
    uint32_t *gcnt = reinterpret_cast<uint32_t *>(gpartner);
    if (s.len == 0) { if (threadIdx.x == 0) ndist[si] = 0; return; }
    if (s.len > (uint64_t)CAP) {
        if (threadIdx.x == 0) {
            gcnt[0] = (uint32_t)s.len; ndist[si] = 1;
            atomicAdd(&stats[s.bits < (uint32_t)total_bits ? 0 : 2], 1ull);     // [0] is an internal error, [2] an equal-key segment
        }
        return;
    }
    const uint32_t n = (uint32_t)s.len;
    const int lo = (int)s.bits;
    const int r2 = (total_bits - lo) < kBinBits ? (total_bits - lo) : kBinBits;
    const uint32_t nb = 1u << r2;
    {   // rep = 0xffff (empty bin), repcnt = rhist = dres = 0: the four tables are contiguous, two bins per word
        uint32_t *w = reinterpret_cast<uint32_t *>(rep);
        const uint32_t nw = (nb + 1) / 2;
        for (uint32_t i = threadIdx.x; i < nw; i += kSThreads) { w[i] = 0xffffffffu; w[kBins / 2 + i] = 0; w[kBins + i] = 0; w[3 * kBins / 2 + i] = 0; }
        if (threadIdx.x == 0) *s_flag = 0;
    }
    __syncthreads();
    // ---- P1: elect representatives
    uint32_t dig[IPT];
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
        const uint32_t i = threadIdx.x + j * kSThreads;
        dig[j] = 0;
        if (i < n) {
            dig[j] = r2 ? key_bits<NW>(load_rec<NW>(A + (size_t)i * NW), K, lo, r2) : 0u;
            rep[dig[j]] = (uint16_t)i;
        }
    }
    __syncthreads();
    // ---- P2: copies of the representative only count; everything else is residual
    uint32_t resmask = 0, repmask = 0;
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
        const uint32_t i = threadIdx.x + j * kSThreads;
        if (i < n) {
            const uint32_t r = rep[dig[j]];
            if (r == i) repmask |= 1u << j;
            else if (kmer_eq<NW>(load_rec<NW>(A + (size_t)i * NW), load_rec<NW>(A + (size_t)r * NW))) atomic_inc_u16(repcnt, dig[j]);
            else { atomic_inc_u16(rhist, dig[j]); resmask |= 1u << j; }
        }
    }
    __syncthreads();
    // ---- P3: residual slots of every bin (its representative + its residual records), exclusive scan
    const uint32_t b0 = threadIdx.x * BPT;
    uint32_t loc[BPT];
    uint32_t sum = 0;
    bool big = false;
#pragma unroll
    for (int q = 0; q < BPT; ++q) {
        const uint32_t h = (b0 + q < nb) ? rhist[b0 + q] : 0u;
        loc[q] = h ? h + 1 : 0u;
        big |= loc[q] > (uint32_t)kBinSlotsMax;
        sum += loc[q];
    }
    if (big) *s_flag = 1;
    uint32_t rtotal;
    {
        uint32_t run = cta_exscan(sum, tot, rtotal);
#pragma unroll
        for (int q = 0; q < BPT; ++q) {
            if (b0 + q < nb) { rstart[b0 + q] = (uint16_t)run; rhist[b0 + q] = (uint16_t)(run + 1); }
            run += loc[q];
        }
        if (threadIdx.x == kSThreads - 1) rstart[nb] = (uint16_t)rtotal;
    }
    __syncthreads();
    bool bad = rtotal > (uint32_t)kResCap || *s_flag;
    if (!bad) {
        // ---- P4: the representative of every bin with residual records takes the bin's first slot, the residual records the rest
#pragma unroll
        for (int j = 0; j < IPT; ++j) {
            const uint32_t i = threadIdx.x + j * kSThreads;
            uint32_t pos = 0xffffffffu;
            if (resmask & (1u << j)) pos = atomic_inc_u16(rhist, dig[j]);
            else if ((repmask & (1u << j)) && rstart[dig[j] + 1] != rstart[dig[j]]) pos = rstart[dig[j]];
            if (pos != 0xffffffffu) { store_rec<NW>(R + (size_t)pos * NW, load_rec<NW>(A + (size_t)i * NW)); rbin[pos] = (uint16_t)dig[j]; }
        }
        __syncthreads();
        // ---- P5: one thread per slot: first copy of its key in the bin? how many copies? (a residual record never equals the
        //          representative in its bin's first slot). rcnt = multiplicity at a key's first slot, 0 elsewhere.
        for (uint32_t p = threadIdx.x; p < rtotal; p += kSThreads) {
            const uint32_t b = rbin[p], bs = rstart[b], be = rstart[b + 1];
            uint32_t c = 0;
            bool head = true;
            if (p == bs) c = repcnt[b] + 1u;
            else {
                const Kmer<NW> key = load_rec<NW>(R + (size_t)p * NW);
                for (uint32_t z = bs + 1; z < be; ++z) {
                    if (kmer_eq<NW>(load_rec<NW>(R + (size_t)z * NW), key)) { ++c; head = head && z >= p; }
                }
            }
            rcnt[p] = head ? (uint16_t)c : (uint16_t)0;
            if (head && atomic_inc_u16(dres, b) >= (uint32_t)kBinDistinctMax) *s_flag = 1;
        }
        __syncthreads();
        bad = *s_flag;
    }
    if (bad) {
        // exact fallback: LSD radix over every remaining key bit (scratch = the partner buffer's region, which no other segment's
        // records share, the next segment's included), run-length unique
        if (threadIdx.x == 0) atomicAdd(&stats[1], 1ull);
        uint64_t *S = lsd_sort_range<NW>(A, gpartner, n, K, lo, total_bits, lsdcnt, tot);
        if (S != A) {
            for (uint32_t i = threadIdx.x; i < n * NW; i += kSThreads) A[i] = S[i];
            __syncthreads();
        }
        uint32_t *heads = lsdcnt;   // the sort is done: its counters (>= CAP+1 u32) are free
        const uint32_t per = (n + kSThreads - 1) / kSThreads;
        const uint32_t i0 = threadIdx.x * per, i1 = min(n, i0 + per);
        uint32_t nh = 0;
        for (uint32_t i = i0; i < i1; ++i)
            if (i == 0 || kmer_word_cmp<NW>(load_rec<NW>(A + (size_t)(i - 1) * NW), load_rec<NW>(A + (size_t)i * NW)) != 0) ++nh;
        uint32_t all;
        uint32_t j = cta_exscan(nh, tot, all);
        for (uint32_t i = i0; i < i1; ++i)
            if (i == 0 || kmer_word_cmp<NW>(load_rec<NW>(A + (size_t)(i - 1) * NW), load_rec<NW>(A + (size_t)i * NW)) != 0) heads[j++] = i;
        if (threadIdx.x == 0) { heads[all] = n; ndist[si] = all; }
        __syncthreads();
        for (uint32_t q = threadIdx.x; q < all; q += kSThreads) {
            const uint32_t h = heads[q];
            store_rec<NW>(gsrc + (size_t)q * NW, load_rec<NW>(A + (size_t)h * NW));
            gcnt[q] = heads[q + 1] - h;
        }
        return;
    }
    // ---- P6: output offset of every bin (exclusive scan of its distinct keys over the occupied bins), then every distinct key
    //          is stored at its bin's offset + its rank in the bin
    uint32_t dsum = 0;
#pragma unroll
    for (int q = 0; q < BPT; ++q) {
        loc[q] = (b0 + q < nb && rep[b0 + q] != 0xffffu) ? (dres[b0 + q] ? (uint32_t)dres[b0 + q] : 1u) : 0u;
        dsum += loc[q];
    }
    uint32_t all;
    {
        uint32_t run = cta_exscan(dsum, tot, all);
#pragma unroll
        for (int q = 0; q < BPT; ++q) {
            if (b0 + q < nb) rhist[b0 + q] = (uint16_t)run;      // rhist is free after P4: output offset of the bin
            run += loc[q];
        }
    }
    __syncthreads();
    // a bin without residual slots: its representative is its only key
#pragma unroll
    for (int j = 0; j < IPT; ++j) {
        if (!(repmask & (1u << j)) || rstart[dig[j] + 1] != rstart[dig[j]]) continue;
        const uint32_t i = threadIdx.x + j * kSThreads, o = rhist[dig[j]];
        store_rec<NW>(gsrc + (size_t)o * NW, load_rec<NW>(A + (size_t)i * NW));
        gcnt[o] = repcnt[dig[j]] + 1u;
    }
    // a key's first slot: rank among the first slots of its bin
    for (uint32_t p = threadIdx.x; p < rtotal; p += kSThreads) {
        const uint32_t c = rcnt[p];
        if (!c) continue;
        const uint32_t b = rbin[p], bs = rstart[b], be = rstart[b + 1];
        const Kmer<NW> key = load_rec<NW>(R + (size_t)p * NW);
        uint32_t o = rhist[b];
        for (uint32_t z = bs; z < be; ++z)
            if (rcnt[z] && kmer_word_cmp<NW>(load_rec<NW>(R + (size_t)z * NW), key) < 0) ++o;
        store_rec<NW>(gsrc + (size_t)o * NW, key);
        gcnt[o] = c;
    }
    if (threadIdx.x == 0) ndist[si] = all;
}

template <int NW, int kBinBits, int CAP>
__global__ void __launch_bounds__(kSThreads, 2) local_sort3_k(const Seg *__restrict__ segs, uint64_t nsegs, int K, uint64_t *__restrict__ buf0,
                                                             uint64_t *__restrict__ buf1, uint32_t *__restrict__ ndist,
                                                             unsigned long long *__restrict__ work_counter, unsigned long long *__restrict__ stats) {
    constexpr int kBins = 1 << kBinBits;
    static_assert(kBins % kSThreads == 0, "bins: a multiple of the CTA size");
    static_assert(CAP % kSThreads == 0 && CAP <= SortCfg<NW>::CAP && CAP < 0xffff, "segment capacity: a multiple of the CTA size, at most the default");
    static_assert((size_t)kResCap * NW * 8 + (size_t)4 * kBins * 2 >= (size_t)4 * (CAP + 1) && (size_t)kResCap * NW * 8 + (size_t)4 * kBins * 2 >= (size_t)4 * 256 * kSWarps,
                  "the residual records and the bin tables double as scratch of the LSD fallback");
    extern __shared__ __align__(16) uint64_t sm64[];
    uint64_t *Abuf = sm64;                                // 2 x CAP*NW: the segment being sorted, the next one arriving
    uint64_t *R = Abuf + (size_t)2 * CAP * NW;            // kResCap*NW residual slots, grouped by bin
    uint16_t *rep = reinterpret_cast<uint16_t *>(R + (size_t)kResCap * NW);   // 4 x kBins + kBins+2, see sort_segment
    uint16_t *rcnt = rep + 5 * kBins + 2;                 // kResCap multiplicity at a key's first slot
    uint16_t *rbin = rcnt + kResCap;                      // kResCap bin of the slot
    uint32_t *lsdcnt = reinterpret_cast<uint32_t *>(R);   // fallback only
    __shared__ uint32_t tot[kSWarps];
    __shared__ unsigned long long s_claim[2];
    __shared__ int s_flag;
    // claims run two segments ahead: s_claim[(it + 1) & 1] holds the segment after the current one when iteration `it` starts,
    // and thread 0 stores the claim of the one after that into s_claim[it & 1] at the end of the iteration
    if (threadIdx.x == 0) s_claim[0] = atomicAdd(work_counter, 1ull);
    __syncthreads();
    uint64_t si = s_claim[0];
    if (threadIdx.x == 0) s_claim[1] = atomicAdd(work_counter, 1ull);
    Seg s = {0, 0, 0, 0};
    if (si < nsegs) {
        s = segs[si];
        prefetch_segment<NW, CAP>(Abuf, ((s.bb & 1) ? buf1 : buf0) + s.start * NW, s.len);
    }
    cp_async_commit();
    for (uint32_t it = 0;; ++it) {
        cp_async_wait_all();
        __syncthreads();              // segment si is in A; every thread is done with the other buffer and with s_claim[(it + 1) & 1]'s writer
        if (si >= nsegs) return;      // claims only grow: no copy was issued after this one
        uint64_t *A = Abuf + (size_t)(it & 1) * CAP * NW;
        const uint64_t ni = s_claim[(it + 1) & 1];
        Seg ns = {0, 0, 0, 0};
        if (ni < nsegs) {
            ns = segs[ni];
            // the next segment's records [start, start+len) are disjoint from this segment's in both buffers, so the sort's
            // scratch (partner region) and output (source region) below never touch what the copy reads
            prefetch_segment<NW, CAP>(Abuf + (size_t)((it + 1) & 1) * CAP * NW, ((ns.bb & 1) ? buf1 : buf0) + ns.start * NW, ns.len);
        }
        cp_async_commit();
        unsigned long long claim = 0;
        if (threadIdx.x == 0) claim = atomicAdd(work_counter, 1ull);
        sort_segment<NW, kBinBits, CAP>(si, s, A, R, rep, rcnt, rbin, lsdcnt, tot, &s_flag, K, buf0, buf1, ndist, stats);
        if (threadIdx.x == 0) s_claim[it & 1] = claim;
        si = ni;
        s = ns;
    }
}

// (A fourth generation -- (21-bit digit | index) keys sorted with three ballot-ranked 7-bit LSD passes, equal records found as
// neighbours, no shared-memory atomics at all -- was parity clean and slower than the kernel above. Removed together with the
// sort primitive.)

// compaction: one warp per segment copies its distinct records / counts to the dense output
template <int NW>
__global__ void compact_k(const Seg *__restrict__ segs, uint64_t nsegs, const uint32_t *__restrict__ ndist, const uint64_t *__restrict__ dbase,
                          const uint64_t *__restrict__ buf0, const uint64_t *__restrict__ buf1, int K, int want_counts, int double_selfrc,
                          uint64_t *__restrict__ out_keys, uint32_t *__restrict__ out_counts, unsigned long long *__restrict__ bucket_sizes) {
    const uint64_t wid = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (wid >= nsegs) return;
    const Seg s = segs[wid];
    const uint32_t nd = ndist[wid];
    if (nd == 0) return;
    const uint64_t *src = ((s.bb & 1) ? buf1 : buf0) + s.start * NW;
    const uint32_t *csrc = reinterpret_cast<const uint32_t *>(((s.bb & 1) ? buf0 : buf1) + s.start * NW);
    const uint64_t ob = dbase[wid];
    for (uint32_t q = lane; q < nd; q += 32) {
        Kmer<NW> k = load_rec<NW>(src + (size_t)q * NW);
        store_rec<NW>(out_keys + (ob + q) * NW, k);
        if (want_counts) {
            uint32_t c = csrc[q];
            if (double_selfrc && kmer_eq<NW>(k, kmer_rc<NW>(k, K))) c *= 2u;   // SURVEY 0.6: a self-RC (k+1)-mer is seen in the read and in its RC
            out_counts[ob + q] = c;
        }
    }
    if (lane == 0) atomicAdd(&bucket_sizes[s.bb >> 1], (unsigned long long)nd);
}

// ------------------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------------------
struct Timer {
    cudaEvent_t a, b; cudaStream_t s;
    Timer(cudaStream_t st) : s(st) { cudaEventCreate(&a); cudaEventCreate(&b); }
    ~Timer() { cudaEventDestroy(a); cudaEventDestroy(b); }
    void start() { cudaEventRecord(a, s); }
    float stop() { cudaEventRecord(b, s); cudaEventSynchronize(b); float ms = 0; cudaEventElapsedTime(&ms, a, b); return ms; }
};

// Environment, read ONCE per process and clamped to what the kernels support. User options: SGPU_ARENA_GB and SGPU_TRACE
// (sgpu_internal.h). Tuning knobs kept for A/B runs on the GPU box:
//   SGPU_PA_MAX   level-A partitions for the whole job (default 4096; every (CTA, partition) pair is an open write stream)
//   SGPU_RMAX     key bits per refinement round (default 11 = 2048 bins per CTA)
//   SGPU_A_SUB    partition sub-ranges per level-A scatter pass (default 0 = automatic)
struct Tuning {
    uint32_t pa_max = 4096;
    uint32_t rmax = 11;
    int a_sub = 0;
};
static const Tuning &tuning() {
    static const Tuning t = [] {
        Tuning x;
        if (const char *e = getenv("SGPU_PA_MAX")) x.pa_max = (uint32_t)std::min(8192, std::max(1, atoi(e)));
        if (const char *e = getenv("SGPU_RMAX")) x.rmax = (uint32_t)std::min(11, std::max(1, atoi(e)));
        if (const char *e = getenv("SGPU_A_SUB")) x.a_sub = std::min(64, std::max(0, atoi(e)));
        return x;
    }();
    return t;
}

static int ilog2_floor(uint64_t v) { int r = 0; while (v >>= 1) ++r; return r; }

static const int kLevelAMaxParts = 8192;      // partitions one level-A launch can address (shared-memory histogram / cursor tables)

// mean segment length the refinement aims for: 3/4 of the local-sort capacity
template <int NW> static uint32_t sort_target() { return (uint32_t)SortCfg<NW>::CAP * 6 / 8; }

// Copies a count's finished chunks to pinned host memory behind the next pass (SGPU_RESULT_ON_HOST). One chunk is in flight at
// a time, on the context's copy stream. Its device arrays stay allocated until the copy has completed: the arena is host
// bookkeeping, so a block released early could be handed to the next pass's buffers while the copy still reads it.
struct ResultSink {
    Ctx *ctx;
    KSet *ks;
    int inflight = -1;                       // index in ks->chunks of the chunk being copied
    cudaEvent_t compacted = nullptr, copied = nullptr;
    ResultSink(Ctx *c, KSet *s) : ctx(c), ks(s) {
        SG_CUDA(cudaEventCreateWithFlags(&compacted, cudaEventDisableTiming));
        SG_CUDA(cudaEventCreateWithFlags(&copied, cudaEventDisableTiming));
    }
    ~ResultSink() {
        if (inflight >= 0) cudaEventSynchronize(copied);
        cudaEventDestroy(compacted); cudaEventDestroy(copied);
    }
    ResultSink(const ResultSink &) = delete;
    ResultSink &operator=(const ResultSink &) = delete;
    // the last chunk of the set has just been compacted on ctx->stream: start its copy and return
    void push() {
        drain();
        Chunk &ch = ks->chunks.back();
        const size_t kb = (size_t)ch.n * ks->nw * 8, cb = ks->has_counts ? (size_t)ch.n * 4 : 0;
        ch.h_keys.alloc((size_t)ch.n * ks->nw);
        if (ks->has_counts) ch.h_counts.alloc((size_t)ch.n);
        cudaStream_t cs = ctx->copy_stream();
        SG_CUDA(cudaEventRecord(compacted, ctx->stream));
        SG_CUDA(cudaStreamWaitEvent(cs, compacted, 0));
        if (kb) SG_CUDA(cudaMemcpyAsync(ch.h_keys.p, ch.keys.p, kb, cudaMemcpyDeviceToHost, cs));
        if (cb) SG_CUDA(cudaMemcpyAsync(ch.h_counts.p, ch.counts.p, cb, cudaMemcpyDeviceToHost, cs));
        SG_CUDA(cudaEventRecord(copied, cs));
        ctx->times.result_d2h_bytes += kb + cb;
        inflight = (int)ks->chunks.size() - 1;
    }
    // wait for the chunk in flight, then give its device arrays back
    void drain() {
        if (inflight < 0) return;
        const auto t0 = std::chrono::steady_clock::now();
        SG_CUDA(cudaEventSynchronize(copied));
        ctx->times.result_d2h_wait += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        Chunk &ch = ks->chunks[(size_t)inflight];
        ch.keys.release(); ch.counts.release();
        inflight = -1;
    }
};

// Puts a counted set together pass by pass: every pass appends one chunk, in bucket order, compact_k adds each bucket's records
// to d_bsz, and finish() fills in the bucket sizes and hands the set over. With SGPU_RESULT_ON_HOST every chunk is copied to host
// memory behind the next pass (ResultSink).
struct KSetBuilder {
    Ctx *ctx;
    std::unique_ptr<KSet> ks;                // the set under construction, deleted with the builder unless finish() handed it over
    DArr<unsigned long long> d_bsz;          // records per bucket
    int64_t first = 0;                       // records in the chunks appended so far
    bool double_selfrc;                      // canonical count at even K: a self-RC (k+1)-mer is seen in the read and in its RC
    std::unique_ptr<ResultSink> sink;        // declared after `ks`, so destroyed first: no copy outlives the set
    KSetBuilder(Ctx *c, int K, int nw, int B, bool counts, bool double_selfrc_, bool on_host) : ctx(c), ks(new KSet()), double_selfrc(double_selfrc_) {
        ks->ctx = c; ks->K = K; ks->nw = nw; ks->B = B; ks->has_counts = counts; ks->on_host = on_host;
        if (on_host) sink.reset(new ResultSink(c, ks.get()));
        d_bsz.alloc(c, (size_t)B);
        SG_CUDA(cudaMemsetAsync(d_bsz.p, 0, (size_t)B * 8, c->stream));
    }
    // the chunk of the next pass, n records of buckets [b_lo, b_hi); the previous chunk's copy is drained first
    Chunk &open(int b_lo, int b_hi, uint64_t n) {
        if (sink) sink->drain();
        ks->chunks.emplace_back();
        Chunk &ch = ks->chunks.back();
        ch.n = (int64_t)n; ch.b_lo = b_lo; ch.b_hi = b_hi; ch.first = first;
        ch.keys.alloc(ctx, (size_t)n * ks->nw + 2, true);
        if (ks->has_counts) ch.counts.alloc(ctx, (size_t)n + 1, true);
        return ch;
    }
    // the chunk open() returned has been compacted on ctx->stream
    void close() {
        first += ks->chunks.back().n;
        if (sink) sink->push();
    }
    KSet *finish() {
        if (sink) { sink->drain(); sink.reset(); }
        const int B = ks->B;
        std::vector<unsigned long long> hb(B);
        SG_CUDA(cudaMemcpyAsync(hb.data(), d_bsz.p, (size_t)B * 8, cudaMemcpyDeviceToHost, ctx->stream));
        SG_CUDA(cudaStreamSynchronize(ctx->stream));
        ks->bsz.assign(B, 0); ks->bstart.assign(B + 1, 0);
        for (int b = 0; b < B; ++b) { ks->bsz[b] = (int64_t)hb[b]; ks->bstart[b + 1] = ks->bstart[b] + ks->bsz[b]; }
        ks->n = first;
        SG_CHECK(ks->bstart[B] == ks->n, 6, "internal: bucket sizes do not add up");
        return ks.release();
    }
};

// refinement + local sort + compaction of one pass into the next chunk of `set`: X holds the level-A output (CTA-major pieces when
// `pieces` is given, else partition-major with the given starts/totals), Y is the ping-pong partner of the same size
template <int NW>
static void sort_pass(Ctx *ctx, int K, DArr<uint64_t> &X, DArr<uint64_t> &Y, const uint64_t *part_start_p, const uint64_t *part_total_p, uint32_t PA,
                      int rA_, uint32_t b_lo, int b_hi, KSetBuilder &set, Timer &tm, Trace &tr, const Pieces *pieces = nullptr) {
    constexpr int CAP = SortCfg<NW>::CAP;
    const int total_bits = 2 * K;
    cudaStream_t st = ctx->stream;
    // ---- segments + refinement rounds
    uint64_t nsegs = PA;
    DArr<Seg> segs(ctx, nsegs);
    seg_init_k<<<div_up(PA, 256), 256, 0, st>>>(part_start_p, part_total_p, PA, rA_, b_lo, segs.p);
    ctx->launches++;
    RefinePlan rp; rp.cap = CAP; rp.target = sort_target<NW>(); rp.total_bits = total_bits;
    rp.rmax = tuning().rmax;
    DArr<unsigned long long> wcounter(ctx, 4);
    tm.start();
    uint64_t rounds = 0;
    for (int round = 0; round < 300; ++round) {
        DArr<uint32_t> nchild(ctx, nsegs + 1), isw(ctx, nsegs + 1);
        DArr<uint64_t> cbase(ctx, nsegs + 1), wpos(ctx, nsegs + 1);
        SG_CUDA(cudaMemsetAsync(nchild.p + nsegs, 0, 4, st));
        SG_CUDA(cudaMemsetAsync(isw.p + nsegs, 0, 4, st));
        const bool pieced = pieces && round == 0;       // X holds the CTA-major staging buffer: round 0 gathers every partition
        refine_plan_k<<<div_up(nsegs, 256), 256, 0, st>>>(segs.p, nsegs, rp, nchild.p, isw.p, pieced ? 1 : 0);
        ctx->launches++;
        exclusive_scan_u32_to_u64(ctx, nchild.p, cbase.p, nsegs + 1);
        exclusive_scan_u32_to_u64(ctx, isw.p, wpos.p, nsegs + 1);
        uint64_t tot[2];
        SG_CUDA(cudaMemcpyAsync(&tot[0], cbase.p + nsegs, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaMemcpyAsync(&tot[1], wpos.p + nsegs, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        if (tot[1] == 0) break;
        DArr<Seg> nsegs_arr(ctx, tot[0]);
        DArr<uint64_t> worklist(ctx, tot[1]);
        refine_copy_k<<<div_up(nsegs, 256), 256, 0, st>>>(segs.p, nsegs, isw.p, cbase.p, wpos.p, nsegs_arr.p, worklist.p);
        ctx->launches++;
        SG_CUDA(cudaMemsetAsync(wcounter.p, 0, 8, st));
        const int grid = (int)std::min<uint64_t>(tot[1], (uint64_t)ctx->num_sms);     // one CTA per SM: the batch fills shared memory
        const size_t sm = RBatch<NW>::smem();
        if (pieced) {
            SG_CUDA(cudaFuncSetAttribute(refine_k<NW, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
            refine_k<NW, true><<<grid, kRThreads, sm, st>>>(segs.p, worklist.p, tot[1], cbase.p, rp, K, X.p, Y.p, nsegs_arr.p, wcounter.p, *pieces);
        } else {
            SG_CUDA(cudaFuncSetAttribute(refine_k<NW, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
            refine_k<NW, false><<<grid, kRThreads, sm, st>>>(segs.p, worklist.p, tot[1], cbase.p, rp, K, X.p, Y.p, nsegs_arr.p, wcounter.p, Pieces());
        }
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
        tr.mark("refine round");
        (round == 0 ? ctx->times.refine_splits_round0 : ctx->times.refine_splits_later) += tot[0] - nsegs;
        ++rounds;
        segs = std::move(nsegs_arr);
        nsegs = tot[0];
    }
    ctx->times.refine_rounds_max = std::max(ctx->times.refine_rounds_max, rounds);
    ctx->times.refine += tm.stop();
    // ---- local sort
    DArr<uint32_t> ndist(ctx, nsegs + 1);
    DArr<unsigned long long> stats(ctx, 4);
    SG_CUDA(cudaMemsetAsync(ndist.p, 0, ndist.bytes(), st));
    SG_CUDA(cudaMemsetAsync(stats.p, 0, 32, st));
    SG_CUDA(cudaMemsetAsync(wcounter.p, 0, 8, st));
    tm.start();
    {
        auto launch = [&](auto kernel, size_t smem) {
            SG_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int occ = 1;
            SG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kSThreads, smem));
            if (occ < 1) occ = 1;
            int grid = (int)std::min<uint64_t>(nsegs, (uint64_t)ctx->num_sms * occ);
            if (grid < 1) grid = 1;
            kernel<<<grid, kSThreads, smem, st>>>(segs.p, nsegs, K, X.p, Y.p, ndist.p, wcounter.p, stats.p);
        };
        launch(local_sort3_k<NW, kSortBinBits, CAP>, SortSmem<NW, kSortBinBits, CAP>::bytes);
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
    }
    DArr<uint64_t> dbase(ctx, nsegs + 1);
    exclusive_scan_u32_to_u64(ctx, ndist.p, dbase.p, nsegs + 1);
    uint64_t D = 0;
    unsigned long long h_stats[4];
    SG_CUDA(cudaMemcpyAsync(&D, dbase.p + nsegs, 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaMemcpyAsync(h_stats, stats.p, 32, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    ctx->times.local_sort += tm.stop();
    tr.mark("local sort");
    SG_CHECK(h_stats[0] == 0, 6, "internal: oversize segment with unfixed key bits reached the local sort");
    ctx->times.sort_lsd_fallbacks += h_stats[1];
    ctx->times.sort_oversize_equal += h_stats[2];
    // ---- compaction into the dense chunk
    Chunk &ch = set.open((int)b_lo, b_hi, D);
    tm.start();
    if (nsegs) {
        compact_k<NW><<<div_up((int64_t)nsegs * 32, 256), 256, 0, st>>>(segs.p, nsegs, ndist.p, dbase.p, X.p, Y.p, K, set.ks->has_counts ? 1 : 0,
                                                                     set.double_selfrc ? 1 : 0, ch.keys.p, ch.counts.p, set.d_bsz.p);
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
    }
    ctx->times.compact += tm.stop();
    tr.mark("compact");
    set.close();
}

// ---- level A as a job: one histogram (+ partition id) pass over the source, then one scatter per bucket-group pass -----------
// Shared by the single-GPU count and the multi-GPU count (where a "pass" scatters this rank's shard for the pass's buckets).
template <int NW, class Src, bool BOTH>
struct LevelAJob {
    Ctx *ctx = nullptr;
    std::vector<Src> srcs;
    int K = 0, B = 0, rA = 0, G = 0;
    int s_lo = 0, s_hi = 0;               // buckets covered by this job (one histogram super-range)
    uint32_t PA_all = 0;                  // (s_hi - s_lo) << rA
    bool use_ids = false;
    DArr<uint32_t> blk_counts;            // [G][PA_all] records of (CTA, partition)
    DArr<uint64_t> part_total_all;        // [PA_all]
    std::vector<DArr<uint64_t>> tile_off; // per source: first id of every tile
    std::vector<DArr<uint16_t>> ids;      // per source: 2-byte partition id per record slot
    std::vector<uint64_t> h_part;         // host copy of part_total_all
    ChunkStager *stage = nullptr;         // the set whose chunks are the sources (null for the reads): each launch reads what it hands over
    // runs launch(si, src) for every non-empty source, in order; a host set's chunk is uploaded behind the launches of the one before
    template <class F>
    void for_each_src(F &&launch) const {
        if (stage)
            stage->sweep([&](const Chunk &ch, const uint64_t *keys, const uint32_t *) {
                const size_t si = (size_t)(&ch - stage->ks->chunks.data());
                Src src = srcs[si];
                src.words = keys;
                launch(si, src);
            });
        else
            for (size_t si = 0; si < srcs.size(); ++si)
                if (srcs[si].n) launch(si, srcs[si]);
    }
    uint64_t bucket_records(int b) const {
        uint64_t s = 0;
        for (uint32_t q = 0; q < (1u << rA); ++q) s += h_part[((size_t)(b - s_lo) << rA) + q];
        return s;
    }
};

// total fan-out bits wanted for est_records, minus what the bucket function provides, clamped to the tables
// CTAs of the level-A grid per SM: the two that are resident. (More waves -- 3, 4, 6 per SM -- for tail balance gained a few
// per cent at best, with 3x smaller pieces for the gather. Not kept.)
static int levelA_ctas_per_sm() { return 2; }
// dynamic shared memory of one level-A scatter launch over PA partitions, and its batch capacity in records: the batch takes
// what the tables and warp slices leave of an SM's share for the two CTAs per SM the grid is sized for (2 x 113 KB of the
// 228 KB of an H100 SM). Where the largest tables would leave less than kABatchMin records, the batch takes what a single CTA
// may opt into, and one CTA per SM is resident. PLANNED: levelA_scatter_plan_k's batch, else levelA_scatter_roll_k's.
template <int NW, bool PLANNED>
static size_t levelA_batch_smem(uint32_t PA, uint32_t *cap) {
    static_assert(kLevelAMaxParts <= (1 << kABatchPartBits) && kLevelAMaxParts <= 0xffff, "a batch tag holds the partition");
    int dev = 0, per_sm = 0, per_cta = 0, reserved = 0;
    SG_CUDA(cudaGetDevice(&dev));
    SG_CUDA(cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    SG_CUDA(cudaDeviceGetAttribute(&per_cta, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    SG_CUDA(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
    const size_t rec = abatch_rec_bytes<NW, PLANNED>(), fixed = abatch_offset(PA), kStatic = 128;   // s_fill, warp_tot
    size_t room = (size_t)per_sm / levelA_ctas_per_sm() - (size_t)reserved - kStatic;
    if (room < fixed + kABatchMin * rec) room = (size_t)per_cta - kStatic;
    SG_CHECK(room >= fixed + kABatchMin * rec, 6, "internal: level-A batch does not fit shared memory");
    *cap = (uint32_t)std::min<size_t>((room - fixed) / rec, 32768) & ~31u;     // positions in a batch are 16-bit
    // the planned batch: a warp's share holds one window of each chunk of a warp step, else the warp could never advance
    SG_CHECK(!PLANNED || *cap / kRollWarps >= 32 * 2, 6, "internal: level-A warp share below one window step");
    return fixed + (size_t)*cap * rec;
}
static int levelA_key_bits(uint64_t est_records, int B, int total_bits, uint32_t target, uint32_t pa_max) {
    const int want = ilog2_floor(est_records / target + 1) + 1;
    const int bbits = ilog2_floor((uint64_t)B) + (((1u << ilog2_floor((uint64_t)B)) < (uint32_t)B) ? 1 : 0);
    int rA = want - bbits;
    if (rA < 0) rA = 0;
    while (rA > 0 && ((uint64_t)B << rA) > pa_max) --rA;
    if (rA > total_bits) rA = total_bits;
    if (rA > 13) rA = 13;                 // a histogram super-range holds at least one bucket: (1 << rA) <= kLevelAMaxParts
    return rA;
}

template <int NW, class Src, bool BOTH>
static void levelA_count(LevelAJob<NW, Src, BOTH> &job, Timer &tm, Trace &tr) {
    Ctx *ctx = job.ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t PA_all = job.PA_all;
    const int G = job.G;
    SG_CHECK(PA_all >= 1 && PA_all <= (uint32_t)kLevelAMaxParts, 6, "internal: level-A partition table too large");
    LevelA pa_all;
    pa_all.K = job.K; pa_all.B = (uint32_t)job.B; pa_all.b_lo = (uint32_t)job.s_lo; pa_all.b_hi = (uint32_t)job.s_hi; pa_all.rA = job.rA; pa_all.PA = PA_all;
    job.blk_counts.alloc(ctx, (size_t)G * PA_all);
    job.part_total_all.alloc(ctx, (size_t)PA_all + 1);
    job.h_part.assign(PA_all, 0);
    SG_CUDA(cudaMemsetAsync(job.blk_counts.p, 0, job.blk_counts.bytes(), st));
    job.tile_off.clear(); job.ids.clear();
    job.tile_off.resize(job.srcs.size()); job.ids.resize(job.srcs.size());
    // per-record partition ids (2 bytes per id slot, Src::kIds slots per chunk): only when they fit comfortably next to the
    // sort buffers. The id rows of the tiles are laid out first; their total is the id array's size.
    const double free0 = (double)ctx->free_bytes();
    std::vector<uint64_t> nslots(job.srcs.size(), 0);
    uint64_t all_slots = 0;
    for (size_t si = 0; si < job.srcs.size(); ++si) {
        const Src &src = job.srcs[si];
        if (src.n == 0) continue;
        const int64_t ntiles = (src.n + kRollTile - 1) / kRollTile;
        DArr<uint32_t> ttot(ctx, (size_t)ntiles + 1);
        job.tile_off[si].alloc(ctx, (size_t)ntiles + 1);
        SG_CUDA(cudaMemsetAsync(ttot.p + ntiles, 0, 4, st));
        roll_tile_ids_k<BOTH><<<div_up(ntiles, 8), 256, 0, st>>>(src, ntiles, ttot.p);
        ctx->launches++;
        exclusive_scan_u32_to_u64(ctx, ttot.p, job.tile_off[si].p, (size_t)ntiles + 1);
        SG_CUDA(cudaMemcpyAsync(&nslots[si], job.tile_off[si].p + ntiles, 8, cudaMemcpyDeviceToHost, st));
        SG_CUDA(cudaStreamSynchronize(st));
        all_slots += nslots[si];
    }
    job.use_ids = PA_all < 0xffffu && (double)all_slots * 2.0 < free0 * 0.20;
    for (size_t si = 0; si < job.srcs.size(); ++si) {
        if (!job.use_ids) job.tile_off[si] = DArr<uint64_t>();
        else if (job.srcs[si].n) job.ids[si].alloc(ctx, (size_t)nslots[si] + 8);
    }
    tm.start();
    SG_CUDA(cudaFuncSetAttribute(levelA_count_roll_k<NW, Src, BOTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)roll_smem_bytes(PA_all)));
    job.for_each_src([&](size_t si, const Src &src) {
        levelA_count_roll_k<NW, Src, BOTH><<<G, kRollThreads, roll_smem_bytes(PA_all), st>>>(src, pa_all, job.blk_counts.p, job.tile_off[si].p, job.ids[si].p);
        ctx->launches++;
    });
    SG_CUDA(cudaGetLastError());
    levelA_totals_k<<<div_up(PA_all, 256), 256, 0, st>>>(job.blk_counts.p, PA_all, G, job.part_total_all.p);
    ctx->launches++;
    SG_CUDA(cudaMemcpyAsync(job.h_part.data(), job.part_total_all.p, (size_t)PA_all * 8, cudaMemcpyDeviceToHost, st));
    SG_CUDA(cudaStreamSynchronize(st));
    ctx->times.extract_count += tm.stop();
    tr.mark("A1 count+totals");
}

// Scatter the records of buckets [b_lo, b_hi) into X, CTA-major (see `Pieces`): CTA g of the level-A grid owns one contiguous
// region, partitioned inside. pbase_buf ([G][PA], caller-owned) receives the first record of every (CTA, partition) piece.
// I_pass / total_records only steer the number of partition sub-ranges.
template <int NW, class Src, bool BOTH>
static void levelA_scatter(LevelAJob<NW, Src, BOTH> &job, int b_lo, int b_hi, uint64_t I_pass, uint64_t total_records, uint64_t *X, uint64_t *pbase_buf,
                           Pieces &pcs, Timer &tm, Trace &tr) {
    Ctx *ctx = job.ctx;
    cudaStream_t st = ctx->stream;
    const int G = job.G;
    const uint32_t PA_all = job.PA_all;
    const uint32_t p_lo = (uint32_t)(b_lo - job.s_lo) << job.rA;
    LevelA pa;
    pa.K = job.K; pa.B = (uint32_t)job.B; pa.b_lo = (uint32_t)b_lo; pa.b_hi = (uint32_t)b_hi; pa.rA = job.rA; pa.PA = (uint32_t)(b_hi - b_lo) << job.rA;
    const uint32_t PA = pa.PA;
    SG_CHECK(PA >= 1 && PA <= (uint32_t)kLevelAMaxParts && G <= kMaxPieces, 6, "internal: level-A pass geometry");
    DArr<uint64_t> base(ctx, (size_t)G * PA);
    {
        DArr<uint64_t> row_total(ctx, (size_t)G + 1), row_start(ctx, (size_t)G + 1);
        SG_CUDA(cudaMemsetAsync(row_total.p + G, 0, 8, st));
        stage_rows_k<<<G, 256, 0, st>>>(job.blk_counts.p + p_lo, PA_all, PA, base.p, row_total.p);
        exclusive_scan_u64(ctx, row_total.p, row_start.p, (size_t)G + 1);
        stage_add_k<<<div_up((int64_t)G * PA, 256), 256, 0, st>>>(base.p, row_start.p, PA, G);
        ctx->launches += 2;
        SG_CUDA(cudaMemcpyAsync(pbase_buf, base.p, (size_t)G * PA * 8, cudaMemcpyDeviceToDevice, st));   // the scatter advances `base`
    }
    pcs.pbase = pbase_buf; pcs.cnt = job.blk_counts.p + p_lo; pcs.cnt_stride = PA_all; pcs.PA = PA; pcs.G = G;
    tm.start();
    // partition sub-ranges (only with the id array, where a foreign window costs just the roll): fewer streams open per CTA. A
    // sub-range costs one more roll over ALL windows of the source: worth it when the pass holds most of the job's records (a
    // single-pass job gains from 4 sub-ranges, a job of several passes loses from even 2). Measured for canonical reads only, so
    // the all-windows count and the k-mer set source scatter once per pass (a (k+1)-mer rolled again for its two records made
    // 4 sub-ranges slower than one, DESIGN.md 6.2).
    int nsub_auto = (int)(4.0 * (double)I_pass / (double)std::max<uint64_t>(1, total_records) + 0.5);
    nsub_auto = std::min(4, std::max(1, nsub_auto));
    uint32_t nsub = job.use_ids && !BOTH && Src::kSubRanges ? (uint32_t)(tuning().a_sub ? tuning().a_sub : nsub_auto) : 1u;
    if (nsub > PA) nsub = PA;
    for (uint32_t sb = 0; sb < nsub; ++sb) {
        const uint32_t q_lo = (uint32_t)((uint64_t)PA * sb / nsub), q_hi = (uint32_t)((uint64_t)PA * (sb + 1) / nsub);
        if (q_hi == q_lo) continue;
        LevelA pa_sub = pa;
        pa_sub.PA = q_hi - q_lo;
        uint32_t cap = 0;
        const size_t smem = job.use_ids ? levelA_batch_smem<NW, true>(pa_sub.PA, &cap) : levelA_batch_smem<NW, false>(pa_sub.PA, &cap);
        if (job.use_ids) SG_CUDA(cudaFuncSetAttribute(levelA_scatter_plan_k<NW, Src, BOTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        else SG_CUDA(cudaFuncSetAttribute(levelA_scatter_roll_k<NW, Src, BOTH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        job.for_each_src([&](size_t si, const Src &src) {
            if (job.use_ids)
                levelA_scatter_plan_k<NW, Src, BOTH><<<G, kRollThreads, smem, st>>>(src, pa_sub, base.p, X, job.tile_off[si].p, job.ids[si].p, p_lo + q_lo, PA, q_lo, (uint64_t)job.ids[si].n, cap);
            else
                levelA_scatter_roll_k<NW, Src, BOTH><<<G, kRollThreads, smem, st>>>(src, pa, base.p, X, PA, cap);
            ctx->launches++; ctx->times.level_a_scatters++;
        });
    }
    SG_CUDA(cudaGetLastError());
    ctx->times.extract_scatter += tm.stop();       // synchronises: `base` may go out of scope
    tr.mark("A2 scatter");
}

// what one pass needs next to what is already resident: X + Y + its own output (distinct/instances <= 0.6 assumed, checked
// against the arena when the output is allocated)
static double pass_bytes_needed(uint64_t recs, size_t W) { return (double)recs * W * 2.0 + (double)recs * (W + 4) * 0.6 + (64 << 20); }

template <int NW, bool BOTH, class Src>
static void run_count(Ctx *ctx, const std::vector<Src> &srcs, int K, uint64_t est_records, KSetBuilder &set, ChunkStager *stage = nullptr) {
    const int total_bits = 2 * K, B = set.ks->B;
    const size_t W = 8 * NW;
    cudaStream_t st = ctx->stream;
    Timer tm(st);
    Trace tr("sgpu count", st);

    // ---- level-A geometry for the whole job. Partition id = (bucket, top rA key bits). ONE histogram pass over the
    // source serves every bucket-group pass (the groups are contiguous partition ranges), so a multi-pass job hashes
    // the source once, and passes are planned from exact per-bucket record counts.
    const int rA = levelA_key_bits(est_records, B, total_bits, sort_target<NW>(), tuning().pa_max);
    ctx->times.level_a_key_bits = (uint64_t)rA;
    const int SR = std::max(1, kLevelAMaxParts >> rA);      // buckets per histogram super-range
    // every pass becomes one chunk of the set, and a set holds at most kMaxChunks of them: each super-range may use an equal
    // share of the chunks still free. There are at most 128 super-ranges (B <= 2^20 with SR = 8192 when rA = 0, a single one
    // when rA > 0), so every share is at least one pass.
    const int n_ranges = (B + SR - 1) / SR;
    for (int s_lo = 0; s_lo < B; s_lo += SR) {
        const int share = (kMaxChunks - (int)set.ks->chunks.size()) / (n_ranges - s_lo / SR);
        LevelAJob<NW, Src, BOTH> job;
        job.ctx = ctx; job.srcs = srcs; job.K = K; job.B = B; job.rA = rA; job.G = ctx->num_sms * levelA_ctas_per_sm(); job.stage = stage;
        job.s_lo = s_lo; job.s_hi = std::min(B, s_lo + SR);
        job.PA_all = (uint32_t)(job.s_hi - job.s_lo) << rA;
        levelA_count(job, tm, tr);
        // bucket-group passes against what the budget leaves now. Blocks beyond the arena come from the driver, so a pass may go
        // above the budget; a device that really lacks the memory fails with SGPU_ENOMEM.
        std::vector<uint64_t> before(job.s_hi - job.s_lo + 1, 0);
        for (int b = job.s_lo; b < job.s_hi; ++b) before[b - job.s_lo + 1] = before[b - job.s_lo] + job.bucket_records(b);
        PassPlan plan(job.s_lo, job.s_hi, share, std::move(before));
        const uint64_t total_records = plan.records(job.s_lo, job.s_hi);
        auto need = [&](int a, int b) { return pass_bytes_needed(plan.records(a, b), W); };
        // a set that goes to host memory keeps only the previous pass's output on the device, while it is copied
        plan.aim((double)ctx->budget_left(), set.sink != nullptr, need, [&](int a, int b) { return (double)plan.records(a, b) * (W + 4) * 0.5; });
        while (!plan.done()) {
            const int b_lo = plan.bounds.back(), b_hi = plan.next((double)ctx->budget_left(), need);
            const uint64_t I = plan.records(b_lo, b_hi);
            const uint32_t p_lo = (uint32_t)(b_lo - job.s_lo) << rA;
            const uint32_t PA = (uint32_t)(b_hi - b_lo) << rA;
            DArr<uint64_t> part_total(ctx, PA + 1), part_start(ctx, PA + 1);
            SG_CUDA(cudaMemcpyAsync(part_total.p, job.part_total_all.p + p_lo, (size_t)PA * 8, cudaMemcpyDeviceToDevice, st));
            SG_CUDA(cudaMemsetAsync(part_total.p + PA, 0, 8, st));
            exclusive_scan_u64(ctx, part_total.p, part_start.p, PA + 1);
            ctx->times.passes++;
            ctx->times.instances += I;
            DArr<uint64_t> X(ctx, (size_t)I * NW + 2), Y(ctx, (size_t)I * NW + 2);
            DArr<uint64_t> pbase(ctx, (size_t)job.G * PA);
            Pieces pcs;
            levelA_scatter(job, b_lo, b_hi, I, total_records, X.p, pbase.p, pcs, tm, tr);
            sort_pass<NW>(ctx, K, X, Y, part_start.p, part_total.p, PA, rA, (uint32_t)b_lo, b_hi, set, tm, tr, &pcs);
        }
    }
}

__global__ void count_windows_k(const uint32_t *__restrict__ lens, int64_t n, int K, unsigned long long *__restrict__ out) {
    unsigned long long s = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int L = (int)lens[i];
        if (L >= K) s += (unsigned long long)(L - K + 1);
    }
    for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// windows of the context's read set (exact), for the level-A geometry
static uint64_t count_windows(Ctx *ctx, int K) {
    DArr<unsigned long long> d_w(ctx, 1);
    SG_CUDA(cudaMemsetAsync(d_w.p, 0, 8, ctx->stream));
    if (ctx->n_reads) {
        count_windows_k<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(ctx->d_lens, ctx->n_reads, K, d_w.p);
        ctx->launches++;
    }
    unsigned long long wn = 0;
    SG_CUDA(cudaMemcpyAsync(&wn, d_w.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
    return (uint64_t)wn;
}

static ReadsSrc reads_source(Ctx *ctx, int K) {
    ReadsSrc src;
    src.words = ctx->d_words; src.offs = ctx->d_offs; src.lens = ctx->d_lens; src.n = ctx->n_reads; src.nwords = ctx->n_words; src.K = K;
    return src;
}

template <int NW>
static KSet *count_reads_nw(Ctx *ctx, int K, int B, int mode, bool on_host) {
    ensure_reads_on_device(ctx);
    const uint64_t wn = count_windows(ctx, K);
    std::vector<ReadsSrc> srcs{reads_source(ctx, K)};
    const bool canonical = mode == kCanonical;
    KSetBuilder set(ctx, K, NW, B, canonical, canonical && K % 2 == 0, on_host);
    if (canonical) run_count<NW, false>(ctx, srcs, K, wn, set);
    else run_count<NW, true>(ctx, srcs, K, wn * 2, set);
    return set.finish();
}

KSet *count_from_reads(Ctx *ctx, int K, int B, int mode, bool result_on_host) {
    SG_CHECK(K >= 1 && K <= 128, 2, "K must be in [1,128]");
    SG_CHECK(B >= 1 && B <= (1 << 20), 2, "num_buckets must be in [1, 2^20]");
    ctx->times = PhaseTimes();
    switch (nwords_of(K)) {
        case 1: return count_reads_nw<1>(ctx, K, B, mode, result_on_host);
        case 2: return count_reads_nw<2>(ctx, K, B, mode, result_on_host);
        case 3: return count_reads_nw<3>(ctx, K, B, mode, result_on_host);
        default: return count_reads_nw<4>(ctx, K, B, mode, result_on_host);
    }
}

// one source per chunk of a (k+1)-mer set; the launches read the words a ChunkStager over the set hands over
static std::vector<KmerSetSrc> kpomer_sources(const KSet *kp) {
    std::vector<KmerSetSrc> srcs;
    for (const Chunk &c : kp->chunks) {
        KmerSetSrc s; s.words = c.keys.p; s.n = c.n; s.nwords = (uint64_t)c.n * kp->nw; s.K = kp->K - 1; s.stride = (uint32_t)kp->nw;
        srcs.push_back(s);
    }
    return srcs;
}
static void check_kpomer_source(const KSet *kp) {
    SG_CHECK(kp->K >= 2, 2, "source k-mers too short");
    SG_CHECK(kp->nw == nwords_of(kp->K), 2, "unsupported k-mer word combination");
}

template <int NW>
static KSet *kmers_from_kpomers_nw(Ctx *ctx, const KSet *kp, int B, bool on_host) {
    const int K = kp->K - 1;
    // allocated before the passes are planned, so the planner sees a host set's two staging buffers
    ChunkStager stage(kp, false);
    KSetBuilder set(ctx, K, NW, B, false, false, on_host);
    run_count<NW, false>(ctx, kpomer_sources(kp), K, (uint64_t)kp->n * 2, set, &stage);
    return set.finish();
}

KSet *kmers_from_kpomers(Ctx *ctx, const KSet *kp, int B, bool result_on_host) {
    check_kpomer_source(kp);
    SG_CHECK(B >= 1 && B <= (1 << 20), 2, "num_buckets must be in [1, 2^20]");
    ctx->times = PhaseTimes();
    switch (nwords_of(kp->K - 1)) {
        case 1: return kmers_from_kpomers_nw<1>(ctx, kp, B, result_on_host);
        case 2: return kmers_from_kpomers_nw<2>(ctx, kp, B, result_on_host);
        case 3: return kmers_from_kpomers_nw<3>(ctx, kp, B, result_on_host);
        default: return kmers_from_kpomers_nw<4>(ctx, kp, B, result_on_host);
    }
}

// checksums of a counted set (bench / multi-GPU self check): out = { n, sum of all key words, xor of all key words rotated by
// their word index, sum of multiplicities } -- order independent, so per-rank values of disjoint bucket sets add / xor up
__global__ void kset_checksum_k(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ counts, uint64_t n, int nw,
                                unsigned long long *__restrict__ out) {
    unsigned long long s = 0, x = 0, c = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        for (int q = 0; q < nw; ++q) {
            const unsigned long long w = keys[i * nw + q];
            s += w * (unsigned long long)(2 * q + 1);
            x ^= (w << (7 * q + 1)) | (w >> (64 - (7 * q + 1)));
        }
        if (counts) c += counts[i];
    }
    for (int o = 16; o; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        x ^= __shfl_down_sync(0xffffffffu, x, o);
        c += __shfl_down_sync(0xffffffffu, c, o);
    }
    if ((threadIdx.x & 31) == 0) { atomicAdd(&out[1], s); atomicXor(&out[2], x); atomicAdd(&out[3], c); }
}
void kset_checksum(const KSet *ks, uint64_t *out4) {
    Ctx *ctx = ks->ctx;
    DArr<unsigned long long> d(ctx, 4);
    SG_CUDA(cudaMemsetAsync(d.p, 0, 32, ctx->stream));
    ChunkStager stage(ks, true);                 // a host set streams through the device
    stage.sweep([&](const Chunk &c, const uint64_t *keys, const uint32_t *counts) {
        kset_checksum_k<<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(keys, counts, (uint64_t)c.n, ks->nw, d.p);
        ctx->launches++;
    });
    unsigned long long h[4];
    SG_CUDA(cudaMemcpyAsync(h, d.p, 32, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
    out4[0] = (uint64_t)ks->n; out4[1] = h[1]; out4[2] = h[2]; out4[3] = h[3];
}

// ------------------------------------------------------------------------------------------------------------
// multi-GPU count (SURVEY 8e; replaces projects/hpcspades/mpi/stages/construction_mpi.cpp:222-300). Buckets are the unit of
// independence (KMerSegmentPolicy is a pure function of the k-mer), so every bucket has one owner GPU. Each rank histograms its
// own read shard once with the same rolling kernel as the single-GPU count (2-byte partition ids included); the per-partition
// totals are all-gathered (host plumbing, torch.distributed). Per pass every rank scatters its shard's records of the pass's
// buckets into a local staging buffer (CTA-major pieces, like the single-GPU count), and then ONE kernel on the owner does the
// exchange AND the merge: it pulls every (source rank, level-A CTA, partition) piece out of the sources' staging buffers through
// NVLink peer mappings (cudaIpc: every rank maps the peers' memory ARENAS once per process; buffers are offsets inside them) with
// coalesced 16-byte loads and lays the pieces of a partition next to each other, ready for the ordinary refinement / local sort
// / compaction. (A first version pushed each 16-byte record to its owner from inside the partition kernel; remote scattered
// stores are not write-combined and ran at ~1 GB/s.)
// ------------------------------------------------------------------------------------------------------------
struct DistPlan {
    int world = 1, rank = 0, B = 0, rA = 0;
    uint32_t PA_all = 0;
    PassPlan passes;                           // over all B buckets
    std::vector<uint64_t> tot;                 // PA_all: records per partition summed over ranks
    std::vector<uint64_t> Tb;                  // B+1: records in buckets < b, all ranks
    std::vector<uint64_t> Ps;                  // world x (B+1): records of rank s in buckets < b
    int npass() const { return passes.npass(); }
    int pass_lo(int p) const { return passes.bounds[p]; }
    static int own_lo_of(int b_lo, int b_hi, int world, int g) { return b_lo + (int)((int64_t)(b_hi - b_lo) * g / world); }
    int own_lo(int p, int g) const { return own_lo_of(pass_lo(p), pass_lo(p + 1), world, g); }
    // largest number of records an owner receives / a rank sends if [b_lo, b_hi) is one pass
    void maxima(int b_lo, int b_hi, uint64_t *mx, uint64_t *ms) const {
        *mx = 0; *ms = 0;
        for (int g = 0; g < world; ++g) *mx = std::max(*mx, Tb[own_lo_of(b_lo, b_hi, world, g + 1)] - Tb[own_lo_of(b_lo, b_hi, world, g)]);
        for (int s = 0; s < world; ++s) *ms = std::max(*ms, Ps[(size_t)s * (B + 1) + b_hi] - Ps[(size_t)s * (B + 1) + b_lo]);
    }
};

static const double kDistHeadroom = 1.05;      // staging / merged buffers are sized 5 % above the planned maximum

// device bytes one pass needs next to what is already resident: staging buffer (doubles as the sort's ping-pong partner, so
// >= recv), merged buffer, its own output (distinct/instances <= 0.6 assumed, like the single-GPU planner) and the per-pass tables
static double dist_pass_bytes(uint64_t mx, uint64_t ms, size_t W, uint64_t fixed_bytes) {
    return ((double)std::max(mx, ms) + (double)mx) * W * (kDistHeadroom + 0.03) + (double)mx * (W + 4) * 0.6 + (double)fixed_bytes;
}

// pure host functions (also exported for the CPU/gloo tests): identical on every rank given the same inputs
void dist_plan_tables(DistPlan &pl, int world, int rank, int B, int rA, const uint64_t *cnt_all) {
    SG_CHECK(rA >= 0 && ((uint64_t)B << rA) <= (uint64_t)kLevelAMaxParts, 2, "distributed count: more level-A partitions than one launch can address");
    pl.world = world; pl.rank = rank; pl.B = B; pl.rA = rA; pl.PA_all = (uint32_t)B << rA;
    pl.tot.assign(pl.PA_all, 0);
    pl.Tb.assign((size_t)B + 1, 0);
    pl.Ps.assign((size_t)world * (B + 1), 0);
    for (int s = 0; s < world; ++s) {
        for (uint32_t q = 0; q < pl.PA_all; ++q) pl.tot[q] += cnt_all[(size_t)s * pl.PA_all + q];
        for (int b = 0; b < B; ++b) {
            uint64_t t = 0;
            for (uint32_t q = (uint32_t)b << rA; q < ((uint32_t)(b + 1) << rA); ++q) t += cnt_all[(size_t)s * pl.PA_all + q];
            pl.Ps[(size_t)s * (B + 1) + b + 1] = pl.Ps[(size_t)s * (B + 1) + b] + t;
        }
    }
    for (int b = 0; b <= B; ++b) {           // Tb = sum over ranks of Ps
        uint64_t t = 0;
        for (int s = 0; s < world; ++s) t += pl.Ps[(size_t)s * (B + 1) + b];
        pl.Tb[b] = t;
    }
    pl.passes = PassPlan(0, B, kMaxChunks, pl.Tb);
}
// plan the next pass against `budget_bytes` = what every rank can allocate NOW (minimum over ranks). Returns false when all
// buckets are done. The first call also fixes the pass size aimed for by simulating the whole job (outputs of earlier passes
// stay resident: ~half a record's bytes per record, as measured on read sets with errors).
bool dist_next_pass(DistPlan &pl, uint64_t budget_bytes, size_t W, uint64_t fixed_bytes, uint64_t *mx_out, uint64_t *ms_out) {
    if (pl.passes.done()) return false;
    auto need = [&](int a, int b) { uint64_t mx, ms; pl.maxima(a, b, &mx, &ms); return dist_pass_bytes(mx, ms, W, fixed_bytes); };
    if (pl.npass() == 0)
        pl.passes.aim((double)budget_bytes, false, need, [&](int a, int b) { uint64_t mx, ms; pl.maxima(a, b, &mx, &ms); return (double)mx * (W + 4) * 0.5; });
    const int b_lo = pl.passes.bounds.back(), b_hi = pl.passes.next((double)budget_bytes, need);
    pl.maxima(b_lo, b_hi, mx_out, ms_out);
    return true;
}

struct PullSrc { const uint64_t *sbuf; const uint64_t *pbase; const uint32_t *blk; };     // one source rank, as seen from this GPU

struct DistState {
    Ctx *ctx = nullptr;
    int K = 0, B = 0, nw = 0, G = 0;
    DistPlan plan;
    std::vector<uint64_t> h_cnt_all;         // world x PA_all
    DArr<uint64_t> sbuf, xbuf;               // staging buffer (peers read it; later the ping-pong partner) and the merged buffer
    DArr<uint64_t> pbase;                    // [G][max partitions of a pass]: piece starts of the current pass (peers read it)
    std::vector<PullSrc> peers;              // world entries (own entry = local pointers)
    std::unique_ptr<KSetBuilder> set;        // this rank's buckets, until sgpu_dist_end hands them over
    std::unique_ptr<ChunkStager> stage;      // a (k+1)-mer source: the histogram and every scatter read its chunks through it
    virtual ~DistState() = default;
    virtual void begin() = 0;
    virtual void local_counts(uint64_t *h_out) = 0;
    virtual const uint32_t *blk_counts_ptr() = 0;
    virtual void scatter(int p) = 0;
    virtual void pull(int p) = 0;
    virtual void sort(int p) = 0;
};

// exchange + merge in one kernel. Work item = (owned partition q, source rank s): the CTA fetches the source's G piece
// descriptors (start in its staging buffer, record count) with one parallel remote read, then streams the pieces into the
// merged buffer back to back with 16-byte loads over NVLink.
static const int kPullThreads = 512;
template <int NW>
__global__ void __launch_bounds__(kPullThreads) dist_pull_k(const PullSrc *__restrict__ srcs, int world, int G, uint32_t PA_all, uint32_t PAp, uint32_t pq0,
                                                            uint32_t q0, uint32_t nq, const uint64_t *__restrict__ dst_off, uint64_t *__restrict__ out,
                                                            unsigned long long *__restrict__ work_counter) {
    __shared__ unsigned long long s_w;
    __shared__ uint64_t p_start[kMaxPieces];      // source record index of piece g
    __shared__ uint64_t p_dst[kMaxPieces + 1];    // destination record index of piece g (exclusive prefix of the counts)
    __shared__ uint32_t wsum[kPullThreads / 32];
    const uint64_t nwork = (uint64_t)nq * (uint64_t)world;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (;;) {
        if (threadIdx.x == 0) s_w = atomicAdd(work_counter, 1ull);
        __syncthreads();
        const uint64_t w = s_w;
        __syncthreads();
        if (w >= nwork) return;
        const uint32_t q = q0 + (uint32_t)(w / (uint64_t)world);
        const int s = (int)(w % (uint64_t)world);
        const PullSrc ps = srcs[s];
        // piece counts -> exclusive prefix (G <= kMaxPieces = 2 * kPullThreads: two per thread)
        uint32_t c0 = 0, c1 = 0;
        const int g0 = 2 * threadIdx.x;
        if (g0 < G) { c0 = ps.blk[(size_t)g0 * PA_all + q]; p_start[g0] = ps.pbase[(size_t)g0 * PAp + (q - pq0)]; }
        if (g0 + 1 < G) { c1 = ps.blk[(size_t)(g0 + 1) * PA_all + q]; p_start[g0 + 1] = ps.pbase[(size_t)(g0 + 1) * PAp + (q - pq0)]; }
        uint32_t v = c0 + c1, inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        uint32_t wb = 0;
        for (int x = 0; x < warp; ++x) wb += wsum[x];
        const uint64_t d0 = dst_off[w] + (uint64_t)(wb + inc - v);
        if (g0 < G) p_dst[g0] = d0;
        if (g0 + 1 < G) p_dst[g0 + 1] = d0 + c0;
        if (g0 + 2 >= G && g0 < G) p_dst[G] = d0 + v;      // the thread holding the last piece(s) also writes the end
        __syncthreads();
        for (int g = 0; g < G; ++g) {
            const uint64_t n = p_dst[g + 1] - p_dst[g];
            if (n == 0) continue;
            const uint64_t *src = ps.sbuf + p_start[g] * NW;
            uint64_t *dst = out + p_dst[g] * NW;
            const uint64_t nwords = n * NW;
            if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
                const ulonglong2 *s2 = reinterpret_cast<const ulonglong2 *>(src);
                ulonglong2 *d2 = reinterpret_cast<ulonglong2 *>(dst);
                const uint64_t n2 = nwords / 2;
                uint64_t i = threadIdx.x;
                for (; i + 3ull * kPullThreads < n2; i += 4ull * kPullThreads) {       // four loads in flight per thread
                    const ulonglong2 a = s2[i], b = s2[i + kPullThreads], c = s2[i + 2 * kPullThreads], e = s2[i + 3 * kPullThreads];
                    d2[i] = a; d2[i + kPullThreads] = b; d2[i + 2 * kPullThreads] = c; d2[i + 3 * kPullThreads] = e;
                }
                for (; i < n2; i += kPullThreads) d2[i] = s2[i];
                if ((nwords & 1) && threadIdx.x == 0) dst[nwords - 1] = src[nwords - 1];
            } else {
                for (uint64_t i = threadIdx.x; i < nwords; i += kPullThreads) dst[i] = src[i];
            }
        }
        __syncthreads();      // p_start / p_dst are rewritten by the next work item
    }
}

// Src: the context's reads (ReadsSrc), or the chunks of this rank's (k+1)-mer set (KmerSetSrc), set in job.srcs before begin()
template <int NW, class Src, bool BOTH>
struct DistStateNW : DistState {
    LevelAJob<NW, Src, BOTH> job;

    void begin() override {
        Timer tm(ctx->stream);
        Trace tr("sgpu count", ctx->stream);
        job.ctx = ctx; job.K = K; job.B = B; job.rA = plan.rA; job.G = G; job.stage = stage.get();
        job.s_lo = 0; job.s_hi = B; job.PA_all = plan.PA_all;
        levelA_count(job, tm, tr);
    }
    void local_counts(uint64_t *h_out) override { memcpy(h_out, job.h_part.data(), (size_t)plan.PA_all * 8); }
    const uint32_t *blk_counts_ptr() override { return job.blk_counts.p; }

    void scatter(int p) override {
        // local partition of this rank's shard for the pass's buckets into the staging buffer (CTA-major pieces)
        Timer tm(ctx->stream);
        Trace tr("sgpu count", ctx->stream);
        const int b_lo = plan.pass_lo(p), b_hi = plan.pass_lo(p + 1);
        uint64_t I = 0, total = 0;
        for (uint32_t q = 0; q < plan.PA_all; ++q) {
            const uint64_t c = h_cnt_all[(size_t)plan.rank * plan.PA_all + q];
            total += c;
            if (q >= ((uint32_t)b_lo << plan.rA) && q < ((uint32_t)b_hi << plan.rA)) I += c;
        }
        SG_CHECK((I * NW + 2) <= sbuf.n, 6, "internal: staging buffer smaller than the pass");
        Pieces pcs;
        levelA_scatter(job, b_lo, b_hi, I, total, sbuf.p, pbase.p, pcs, tm, tr);
        SG_CUDA(cudaStreamSynchronize(ctx->stream));
    }

    void pull(int p) override {
        cudaStream_t st = ctx->stream;
        const int world = plan.world;
        const uint32_t pq0 = (uint32_t)plan.pass_lo(p) << plan.rA;
        const uint32_t PAp = (uint32_t)(plan.pass_lo(p + 1) - plan.pass_lo(p)) << plan.rA;
        const uint32_t q0 = (uint32_t)plan.own_lo(p, plan.rank) << plan.rA, q1 = (uint32_t)plan.own_lo(p, plan.rank + 1) << plan.rA;
        const uint32_t nq = q1 - q0;
        if (nq == 0) return;
        // destination of (q, s): partitions in order, inside a partition the sources in rank order
        std::vector<uint64_t> dst_off((size_t)nq * world);
        uint64_t run = 0;
        for (uint32_t q = q0; q < q1; ++q)
            for (int s = 0; s < world; ++s) {
                dst_off[(size_t)(q - q0) * world + s] = run;
                run += h_cnt_all[(size_t)s * plan.PA_all + q];
            }
        SG_CHECK(run * NW + 2 <= xbuf.n, 6, "internal: merged buffer smaller than the pass");
        if (run == 0) return;
        DArr<uint64_t> d_off(ctx, dst_off.size());
        DArr<PullSrc> d_src(ctx, (size_t)world);
        DArr<unsigned long long> wc(ctx, 1);
        SG_CUDA(cudaMemcpyAsync(d_off.p, dst_off.data(), dst_off.size() * 8, cudaMemcpyHostToDevice, st));
        SG_CUDA(cudaMemcpyAsync(d_src.p, peers.data(), (size_t)world * sizeof(PullSrc), cudaMemcpyHostToDevice, st));
        SG_CUDA(cudaMemsetAsync(wc.p, 0, 8, st));
        Timer tm(st);
        tm.start();
        const uint64_t nwork = (uint64_t)nq * world;
        const int grid = (int)std::min<uint64_t>(nwork, (uint64_t)ctx->num_sms * 4);
        dist_pull_k<NW><<<grid, kPullThreads, 0, st>>>(d_src.p, world, G, plan.PA_all, PAp, pq0, q0, nq, d_off.p, xbuf.p, wc.p);
        ctx->launches++;
        SG_CUDA(cudaGetLastError());
        ctx->times.exchange += tm.stop();
    }

    void sort(int p) override {
        cudaStream_t st = ctx->stream;
        const int my_lo = plan.own_lo(p, plan.rank), my_hi = plan.own_lo(p, plan.rank + 1);
        const uint32_t PA = (uint32_t)(my_hi - my_lo) << plan.rA;
        const size_t Q0 = (size_t)my_lo << plan.rA;
        std::vector<uint64_t> tot(PA + 1, 0), start(PA + 1, 0);
        for (uint32_t q = 0; q < PA; ++q) { tot[q] = plan.tot[Q0 + q]; start[q + 1] = start[q] + tot[q]; }
        ctx->times.passes++;
        ctx->times.instances += start[PA];
        if (PA && start[PA]) {
            DArr<uint64_t> d_tot(ctx, PA + 1), d_start(ctx, PA + 1);
            SG_CUDA(cudaMemcpyAsync(d_tot.p, tot.data(), (size_t)(PA + 1) * 8, cudaMemcpyHostToDevice, st));
            SG_CUDA(cudaMemcpyAsync(d_start.p, start.data(), (size_t)(PA + 1) * 8, cudaMemcpyHostToDevice, st));
            Timer tm(st);
            Trace tr("sgpu count", st);
            sort_pass<NW>(ctx, K, xbuf, sbuf, d_start.p, d_tot.p, PA, plan.rA, (uint32_t)my_lo, my_hi, *set, tm, tr);
        } else {
            set->open(my_lo, my_hi, 0);          // nothing arrived: the pass still has its (empty) chunk
            set->close();
        }
    }
};

template <int NW, class Src, bool BOTH>
static DistState *dist_state_of(std::vector<Src> srcs) {
    auto *d = new DistStateNW<NW, Src, BOTH>();
    d->job.srcs = std::move(srcs);
    return d;
}
template <int NW>
static DistState *dist_state_new(Ctx *ctx, int K, int mode) {
    std::vector<ReadsSrc> srcs{reads_source(ctx, K)};
    return mode == kAllWindows ? dist_state_of<NW, ReadsSrc, true>(srcs) : dist_state_of<NW, ReadsSrc, false>(srcs);
}
template <int NW>
static DistState *dist_state_kpomers(const KSet *kp) { return dist_state_of<NW, KmerSetSrc, false>(kpomer_sources(kp)); }

// geometry, set and level-A histogram of a distributed count whose sources d already holds (`counts`, `double_selfrc`: as
// KSetBuilder's; `src_set`: the (k+1)-mer set whose chunks are the sources, null for the reads); d is deleted on failure
static DistState *dist_start(DistState *d, Ctx *ctx, int K, int B, int world, int rank, bool counts, bool double_selfrc, bool result_on_host,
                             const KSet *src_set) {
    d->ctx = ctx; d->K = K; d->B = B; d->nw = nwords_of(K);
    d->G = ctx->num_sms * levelA_ctas_per_sm();
    // every rank must use the same geometry, so it depends on B only. As many level-A partitions as the shared-memory tables allow:
    // an owner's segment is the union of all ranks' records of a partition, so finer partitions keep refinement at one round
    int rA = 0;
    while (rA < 8 && ((uint64_t)B << (rA + 1)) <= (uint64_t)kLevelAMaxParts && rA + 1 <= 2 * K) ++rA;
    d->plan.world = world; d->plan.rank = rank; d->plan.B = B; d->plan.rA = rA; d->plan.PA_all = (uint32_t)B << rA;
    ctx->times.level_a_key_bits = (uint64_t)rA;
    try {
        // a host source's staging buffers are allocated before the histogram, so sgpu_dist_free_bytes sees them from the first pass
        if (src_set) d->stage.reset(new ChunkStager(src_set, false));
        d->set.reset(new KSetBuilder(ctx, K, d->nw, B, counts, double_selfrc, result_on_host));
        d->begin();
    } catch (...) { delete d; throw; }
    return d;
}

static void check_dist_args(int B, int world, int rank) {
    SG_CHECK(B >= 1 && B <= kLevelAMaxParts, 2, "distributed count: num_buckets must be in [1, 8192]");
    SG_CHECK(world >= 1 && world <= 255 && rank >= 0 && rank < world, 2, "bad world/rank");
}

DistState *dist_begin(Ctx *ctx, int K, int B, int mode, int world, int rank, bool result_on_host) {
    SG_CHECK(K >= 1 && K <= 128, 2, "K must be in [1,128]");
    check_dist_args(B, world, rank);
    SG_CHECK(mode == kCanonical || mode == kAllWindows, 2, "bad mode");
    ensure_reads_on_device(ctx);
    ctx->times = PhaseTimes();
    DistState *d = nullptr;
    switch (nwords_of(K)) {
        case 1: d = dist_state_new<1>(ctx, K, mode); break;
        case 2: d = dist_state_new<2>(ctx, K, mode); break;
        case 3: d = dist_state_new<3>(ctx, K, mode); break;
        default: d = dist_state_new<4>(ctx, K, mode); break;
    }
    return dist_start(d, ctx, K, B, world, rank, mode == kCanonical, mode == kCanonical && K % 2 == 0, result_on_host, nullptr);
}

// the k-mers of this rank's (k+1)-mer set, bucket-owned like dist_begin's count; the records are those of kmers_from_kpomers
// (no multiplicities). The ranks' sets may overlap: every owner's sort removes the duplicates its pieces bring.
DistState *dist_begin_kpomers(Ctx *ctx, const KSet *kp, int B, int world, int rank, bool result_on_host) {
    check_kpomer_source(kp);
    SG_CHECK(kp->ctx == ctx, 2, "the (k+1)-mer set belongs to another context");
    check_dist_args(B, world, rank);
    ctx->times = PhaseTimes();
    const int K = kp->K - 1;
    DistState *d = nullptr;
    switch (nwords_of(K)) {
        case 1: d = dist_state_kpomers<1>(kp); break;
        case 2: d = dist_state_kpomers<2>(kp); break;
        case 3: d = dist_state_kpomers<3>(kp); break;
        default: d = dist_state_kpomers<4>(kp); break;
    }
    return dist_start(d, ctx, K, B, world, rank, false, false, result_on_host, kp);
}
uint32_t dist_num_partitions(const DistState *d) { return d->plan.PA_all; }
void dist_local_counts(DistState *d, uint64_t *h_out) { d->local_counts(h_out); }

static const uint64_t kDistFixedBytes = (uint64_t)192 << 20;      // per-pass tables (segments, work lists, scans) next to the big buffers

void dist_plan(DistState *d, const uint64_t *cnt_all, uint64_t *total_records) {
    dist_plan_tables(d->plan, d->plan.world, d->plan.rank, d->B, d->plan.rA, cnt_all);
    d->h_cnt_all.assign(cnt_all, cnt_all + (size_t)d->plan.world * d->plan.PA_all);
    *total_records = d->plan.Tb[d->B];
}

// bytes this rank could allocate for the next pass (the previous pass's staging / merged buffers are given back first)
uint64_t dist_free_bytes(DistState *d) {
    d->sbuf.release(); d->xbuf.release(); d->pbase.release();
    return (uint64_t)d->ctx->free_bytes();
}

// plan the next pass against budget_bytes (the minimum of dist_free_bytes over the ranks, so that every rank takes the same
// decision) and allocate its buffers. Returns the pass index, or -1 when every bucket has been processed.
int dist_next_pass(DistState *d, uint64_t budget_bytes) {
    Ctx *ctx = d->ctx;
    const size_t W = (size_t)8 * d->nw;
    d->sbuf.release(); d->xbuf.release(); d->pbase.release();
    uint64_t mx = 0, ms = 0;
    if (!dist_next_pass(d->plan, budget_bytes, W, kDistFixedBytes, &mx, &ms)) return -1;
    const int p = d->plan.npass() - 1;
    // buffers the peers read must live inside the arena (one driver allocation, mapped by the peers as a whole)
    const uint32_t pa = (uint32_t)(d->plan.pass_lo(p + 1) - d->plan.pass_lo(p)) << d->plan.rA;
    d->sbuf.alloc(ctx, (size_t)((double)std::max(mx, ms) * kDistHeadroom) * d->nw + 16);
    d->xbuf.alloc(ctx, (size_t)((double)mx * kDistHeadroom) * d->nw + 16);
    d->pbase.alloc(ctx, (size_t)d->G * pa);
    d->peers.clear();
    return p;
}

// descriptor a rank publishes (all_gather) after dist_plan: arena handle + where its peer-readable buffers are inside the arena
struct DistDesc {
    cudaIpcMemHandle_t arena;     // 64 bytes
    uint64_t arena_size, off_sbuf, off_pbase, off_blk;
};
static_assert(sizeof(cudaIpcMemHandle_t) == 64 && sizeof(DistDesc) == 96, "descriptor layout (SGPU_IPC_BYTES)");

void dist_ipc_handle(DistState *d, uint8_t *out96) {
    Ctx *ctx = d->ctx;
    DistDesc ds;
    memset(&ds, 0, sizeof ds);
    ds.off_sbuf = ctx->arena_offset(d->sbuf.p, "distributed count: the staging buffer did not fit the device memory arena");
    ds.off_pbase = ctx->arena_offset(d->pbase.p, "distributed count: the piece table did not fit the device memory arena");
    ds.off_blk = ctx->arena_offset(d->blk_counts_ptr(), "distributed count: the level-A count table did not fit the device memory arena");
    ds.arena_size = ctx->arena_size;
    if (d->plan.world > 1) SG_CUDA(cudaIpcGetMemHandle(&ds.arena, ctx->arena));
    memcpy(out96, &ds, sizeof ds);
}

void dist_open_peers(DistState *d, const uint8_t *descs) {
    Ctx *ctx = d->ctx;
    const int world = d->plan.world;
    d->peers.assign(world, PullSrc{nullptr, nullptr, nullptr});
    for (int g = 0; g < world; ++g) {
        DistDesc ds;
        memcpy(&ds, descs + (size_t)g * sizeof(DistDesc), sizeof ds);
        char *base = ctx->peer_map(world, d->plan.rank, g, &ds.arena);
        SG_CHECK(ds.off_sbuf < ds.arena_size && ds.off_pbase < ds.arena_size && ds.off_blk < ds.arena_size, 2, "bad peer descriptor");
        d->peers[g] = PullSrc{(const uint64_t *)(base + ds.off_sbuf), (const uint64_t *)(base + ds.off_pbase), (const uint32_t *)(base + ds.off_blk)};
    }
}

void dist_scatter(DistState *d, int p) {
    SG_CHECK(p >= 0 && p == d->plan.npass() - 1 && d->sbuf.p, 2, "bad pass (sgpu_dist_next_pass decides the current one)");
    d->scatter(p);
    SG_CUDA(cudaStreamSynchronize(d->ctx->stream));        // the staging buffer is complete; peers may read it after the next barrier
}
void dist_exchange(DistState *d, int p) {
    SG_CHECK(p >= 0 && p == d->plan.npass() - 1 && d->sbuf.p, 2, "bad pass (sgpu_dist_next_pass decides the current one)");
    SG_CHECK((int)d->peers.size() == d->plan.world, 2, "sgpu_dist_open_peers has not run");
    d->pull(p);
    SG_CUDA(cudaStreamSynchronize(d->ctx->stream));        // this rank no longer reads any peer's staging buffer
}
void dist_sort(DistState *d, int p) {
    SG_CHECK(p >= 0 && p == d->plan.npass() - 1 && d->sbuf.p, 2, "bad pass (sgpu_dist_next_pass decides the current one)");
    d->sort(p);
    SG_CUDA(cudaStreamSynchronize(d->ctx->stream));
}
KSet *dist_end(DistState *d) {
    SG_CHECK(d->set, 2, "sgpu_dist_end has already run");
    KSet *ks = d->set->finish();
    d->set.reset();
    return ks;
}
void dist_free(DistState *d) { delete d; }

// the whole pass sequence for a FIXED budget (CPU tests): every pass is planned against the budget minus the estimated outputs of
// the passes before it
int dist_plan_host(int world, int B, int rA, const uint64_t *cnt_all, uint64_t budget_bytes, int record_bytes, int *pass_b, uint64_t *max_recv) {
    DistPlan pl;
    dist_plan_tables(pl, world, 0, B, rA, cnt_all);
    double lim = (double)budget_bytes;
    uint64_t mx = 0, ms = 0, worst = 0;
    while (dist_next_pass(pl, (uint64_t)std::max(0.0, lim), (size_t)record_bytes, 0, &mx, &ms)) {
        worst = std::max(worst, mx);
        lim -= (double)mx * (record_bytes + 4) * 0.5;
    }
    for (int p = 0; p <= pl.npass(); ++p) pass_b[p] = pl.pass_lo(p);
    *max_recv = worst;
    return pl.npass();
}

}  // namespace sg
