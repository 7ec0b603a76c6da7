"""CPU test of the count's pass planner (spades_b200/csrc/pass_plan.h), through tests/host/pass_plan_check.cpp: passes take whole
buckets in order, never more passes than the share of chunks, one bucket per pass under a near-zero budget when the share allows
it, and an even split of the buckets when the budget would need more passes than the share."""
import os
import random
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "pass_plan_check.cpp")
HDR = os.path.join(ROOT, "spades_b200", "csrc", "pass_plan.h")
BIN = os.path.join(ROOT, "tests", "host", "_build", "pass_plan_check")


def _plans(cases):
    """cases: (lo, hi, share, budget, sink, seed) -> [(capped, bounds)]"""
    if not (os.path.exists(BIN) and os.path.getmtime(BIN) > max(os.path.getmtime(SRC), os.path.getmtime(HDR))):
        os.makedirs(os.path.dirname(BIN), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", SRC, "-o", BIN])
    text = "".join("%d %d %d %r %d %d\n" % c for c in cases)
    out = subprocess.run([BIN], input=text, capture_output=True, text=True, timeout=120, check=True).stdout.splitlines()
    assert len(out) == len(cases)
    plans = []
    for line in out:
        v = [int(x) for x in line.split()]
        assert len(v) == v[1] + 3
        plans.append((bool(v[0]), v[2:]))
    return plans


def test_whole_buckets_in_order_within_the_share():
    rng = random.Random(5)
    cases = []
    for i in range(600):
        lo = rng.choice([0, 0, rng.randrange(1, 5000)])
        nb = rng.choice([1, 2, 3, rng.randrange(1, 200), rng.randrange(1, 8193)])
        share = rng.choice([1, 2, rng.randrange(1, 129), 128])
        budget = 10.0 ** rng.uniform(3.5, 11)          # from below one bucket to the whole range
        cases.append((lo, lo + nb, share, budget, rng.randrange(2), i))
    for (lo, hi, share, _, _, _), (capped, b) in zip(cases, _plans(cases)):
        assert b[0] == lo and b[-1] == hi
        assert all(x < y for x, y in zip(b, b[1:])), b
        assert len(b) - 1 <= share


def test_one_bucket_per_pass_under_a_near_zero_budget():
    cases = [(lo, lo + nb, share, 1.0, sink, 7 * nb + sink) for lo in (0, 300) for nb, share in ((1, 1), (5, 5), (37, 128), (128, 128))
             for sink in (0, 1)]
    for (lo, hi, _, _, _, _), (capped, b) in zip(cases, _plans(cases)):
        assert not capped
        assert b == list(range(lo, hi + 1))


def test_even_split_when_capped():
    cases = [(lo, lo + nb, share, 1.0, sink, nb) for lo in (0, 1000) for nb, share in ((300, 128), (129, 128), (1000, 7), (8192, 128), (50, 1))
             for sink in (0, 1)]
    for (lo, hi, share, _, _, _), (capped, b) in zip(cases, _plans(cases)):
        assert capped
        assert len(b) - 1 == share
        sizes = {y - x for x, y in zip(b, b[1:])}
        nb = hi - lo
        assert sizes <= {nb // share, -(-nb // share)}, sizes
