// pass_plan.h -- how a count splits a bucket range into passes. Pure host arithmetic without CUDA, so CPU programs compile it too.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <utility>
#include <vector>

namespace sg {

// The bucket-group passes of one bucket range [lo, hi). A pass takes whole buckets in order and becomes one chunk of the counted
// set. The caller prices a candidate pass [a, b) with two functions: need(a, b), the device bytes it needs next to what is already
// resident, and out(a, b), the bytes its output leaves resident.
//
// aim() simulates the greedy plan "as many whole buckets as fit" against a budget, with the outputs of earlier passes resident (or,
// for a set copied to host memory behind the next pass, only the one in flight), to learn how many passes the range needs. The
// passes then aim for equal sizes, because a tiny last pass still costs a full sweep of the source, and there are at most `share`
// of them. next() plans one pass against the budget as it is now: whole buckets while they fit and stay within the size aimed for.
// When the budget would need more passes than the share, or this is the share's last pass, the pass takes at least an even split of
// the buckets left, above the budget if need be: the budget is a planning target, not a hard limit.
struct PassPlan {
    int lo = 0, hi = 0, share = 1;
    std::vector<uint64_t> before;    // before[b - lo]: records in buckets [lo, b), for b in [lo, hi]
    std::vector<int> bounds;         // bucket boundaries of the passes planned so far, starting with lo
    uint64_t target = 0;             // records per pass aimed for
    bool capped = false;             // the budget needs more passes than the share

    PassPlan() {}
    PassPlan(int lo_, int hi_, int share_, std::vector<uint64_t> before_)
        : lo(lo_), hi(hi_), share(share_), before(std::move(before_)), bounds(1, lo_) {}
    int npass() const { return (int)bounds.size() - 1; }
    bool done() const { return bounds.back() >= hi; }
    uint64_t records(int a, int b) const { return before[b - lo] - before[a - lo]; }

    template <class Need, class Out>
    void aim(double budget, bool only_inflight, Need need, Out out) {
        double lim = budget, inflight = 0;
        int n = 0;
        for (int b = lo; b < hi; ++n) {
            const int e = greedy(b, 1, lim, inflight, 0, need);
            if (only_inflight) inflight = out(b, e);
            else lim -= out(b, e);
            b = e;
        }
        capped = n > share;
        const uint64_t total = records(lo, hi);
        target = total / (uint64_t)std::min(n, share) + total / 64 + 1;
    }
    // plans the next pass and returns its end
    template <class Need>
    int next(double budget, Need need) {
        const int b_lo = bounds.back(), left = share - npass();
        const int min_b = (capped || left == 1) ? (hi - b_lo + left - 1) / left : 1;
        bounds.push_back(greedy(b_lo, min_b, budget, 0, target, need));
        return bounds.back();
    }
    // the pass from b_lo: at least min_b buckets, then more while need + extra stays within the budget and the records within
    // max_records (0 = no limit)
    template <class Need>
    int greedy(int b_lo, int min_b, double budget, double extra, uint64_t max_records, Need need) const {
        int b = b_lo;
        while (b < hi && (b - b_lo < min_b || (need(b_lo, b + 1) + extra <= budget && (!max_records || records(b_lo, b + 1) <= max_records)))) ++b;
        return b;
    }
};

}  // namespace sg
