// cov_plan.h -- how the coverage pre-filter sizes its counting table: one slice per rank of the distributed filter, or one table per
// key-range pass on one GPU. Pure host arithmetic without CUDA, so CPU programs compile it too.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cmath>

namespace sg {

// Entries of the single table: 1.5 x the cardinality bound.
inline uint64_t cov_table_capacity(uint64_t maxn) { return std::max<uint64_t>(1024, maxn + maxn / 2); }

// Entries of a table that holds the keys of one of `parts` owners (a rank's slice, or a pass's key range): 1.5 x an even share of
// the bound, like the single table, plus 8 standard deviations of a binomial owner load (at most sqrt(share)) for the unevenness of
// the owner hash. Such a table overflows only when its distinct keys exceed the capacity.
inline uint64_t cov_slice_capacity(uint64_t maxn, int parts) {
    const uint64_t share = (maxn + (uint64_t)parts - 1) / (uint64_t)parts;
    return std::max<uint64_t>(1024, share + share / 2 + 8 * (uint64_t)std::ceil(std::sqrt((double)share)));
}

// Every pass rolls every read twice (fill, then lookup), so a table that needs more passes than this is refused.
static const int kCovMaxPasses = 256;

// device bytes of a block of `bytes` (the arena hands out 512-byte multiples)
inline uint64_t cov_block_bytes(uint64_t bytes) { return (std::max<uint64_t>(bytes, 1) + 511) & ~(uint64_t)511; }

// Device bytes the filter holds next to its table over n reads: for n + 1 entries the verdict (1 byte), the words kept, the scan
// flag and the windows below the threshold of the pass path (4 bytes each), then the distinct-key counter and the overflow flag.
inline uint64_t cov_resident_bytes(int64_t n) {
    const uint64_t m = (uint64_t)n + 1;
    return cov_block_bytes(m) + 3 * cov_block_bytes(4 * m) + cov_block_bytes(8) + cov_block_bytes(4);
}

struct CovPassPlan {
    int passes = 0;        // 0: not even kCovMaxPasses passes fit
    uint64_t cap = 0;      // entries of one pass table (of the kCovMaxPasses-pass table when nothing fits)
    uint64_t need = 0;     // cov_resident_bytes + the pass table's block
};

// Entries of one table of a P-pass filter: the single table at P = 1, a key range's share of it (cov_slice_capacity) above.
inline uint64_t cov_pass_capacity(uint64_t maxn, int passes) { return passes == 1 ? cov_table_capacity(maxn) : cov_slice_capacity(maxn, passes); }

// The smallest number of key-range passes whose table fits `budget` device bytes next to the filter's resident bytes. The
// capacity does not grow with P, so a smaller budget never plans fewer passes.
inline CovPassPlan cov_pass_plan(uint64_t maxn, int64_t n, uint64_t budget) {
    CovPassPlan pl;
    for (int p = 1; p <= kCovMaxPasses; ++p) {
        pl.cap = cov_pass_capacity(maxn, p);
        pl.need = cov_resident_bytes(n) + cov_block_bytes(8 * pl.cap);
        if (pl.need <= budget) { pl.passes = p; break; }
    }
    return pl;
}

}  // namespace sg
