// CPU check of the count's pass planner (spades_b200/csrc/pass_plan.h). Reads one case per line from stdin:
//     lo hi share budget sink seed
// draws the records of buckets [lo, hi) from `seed` (some buckets empty), plans the range against a fixed budget and prints
//     capped npass bound_0 ... bound_npass
// A pass of r records needs 32 r + 4096 bytes and leaves 10 r resident. tests/test_pass_plan.py checks the plans.
#include <stdint.h>
#include <stdio.h>

#include <random>
#include <vector>

#include "../../spades_b200/csrc/pass_plan.h"

int main() {
    int lo, hi, share, sink;
    double budget;
    unsigned long long seed;
    while (scanf("%d %d %d %lf %d %llu", &lo, &hi, &share, &budget, &sink, &seed) == 6) {
        std::mt19937_64 rng(seed);
        std::vector<uint64_t> before(hi - lo + 1, 0);
        for (int b = lo; b < hi; ++b) before[b - lo + 1] = before[b - lo] + (rng() % 4 == 0 ? 0 : rng() % 100000);
        sg::PassPlan plan(lo, hi, share, before);
        auto need = [&](int a, int b) { return 32.0 * (double)plan.records(a, b) + 4096.0; };
        plan.aim(budget, sink != 0, need, [&](int a, int b) { return 10.0 * (double)plan.records(a, b); });
        while (!plan.done()) plan.next(budget, need);
        printf("%d %d", plan.capped ? 1 : 0, plan.npass());
        for (int b : plan.bounds) printf(" %d", b);
        printf("\n");
    }
    return 0;
}
