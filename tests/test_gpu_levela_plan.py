"""The planned batch of the level-A partition kernel at its edges, against the C oracle (run with -m gpu on an H100).

With the partition-id array, levelA_scatter_plan_k lays out each batch from the ids before it rolls anything: a warp takes its
next steps of 32 chunks window by window up to its share of the batch, and resumes in the next batch at the first window that
did not fit, possibly in the middle of a chunk and of a tile. The cases, each asserted through the path counters to reach the
id path:
  - steps that never fit a warp's share: single-pass, single-sub-range counts (SGPU_A_SUB = 1) where every id is own, so a
    step of 32 chunks of 150 bp reads holds more records than a share and every warp resumes mid-step, batch after batch;
  - the smallest batch: 8192 partitions (SGPU_PA_MAX = 8192, B = 8192), one CTA per SM;
  - most ids foreign: a multi-pass count under a small HBM budget with three partition sub-ranges per pass (SGPU_A_SUB = 3), so a
    launch owns about a tenth of the records and a warp plans many steps, across tiles, per batch;
  - the all-windows count (a window's two strands are taken together) and the k-mers of the (k+1)-mers (KmerSetSrc);
  - ragged reads -- shorter than K, of exactly K bases, of 150 and of more than 320 bases -- at 1 to 4 words per record, in
    canonical and all-windows mode.
SGPU_PA_MAX and SGPU_A_SUB are read once per process, so each group runs in a child process of its own (this file, run as a
script)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from spades_b200.packing import pack_reads, synthetic_reads  # noqa: E402

pytestmark = pytest.mark.gpu

ARENA_GB = 2
MULTIPASS_BUDGET_MB = 128

# H100 (sm_90): shared memory per SM, opt-in limit per CTA, reserved per CTA; the kernel's static shared memory (count.cu)
SM_PER_SM, SM_OPTIN, SM_RESERVED, SM_STATIC = 233472, 232448, 1024, 128
ROLL_WARP_BYTES, ROLL_WARPS, CTAS_PER_SM = 2952, 16, 2
IDS_PER_CHUNK = 24           # records of a chunk of reads (count.cu: kRollC)

# (name, group, source, K, B, reads): source "canon" = canonical count of the reads at K, "allwin" = all-windows count,
# "kpomers" = k-mers of their (K+1)-mers
CASES = [
    ("canon_k55", "single", "canon", 55, 16, "uniform"),
    ("allwin_k55", "single", "allwin", 55, 16, "uniform"),
    ("kpomers_k21", "single", "kpomers", 21, 16, "uniform"),
    ("kpomers_k99", "single", "kpomers", 99, 16, "uniform"),
] + [("ragged_canon_k%d" % K, "single", "canon", K, 16, "ragged%d" % K) for K in (21, 55, 77, 99)] + [
    ("ragged_allwin_k%d" % K, "single", "allwin", K, 16, "ragged%d" % K) for K in (33, 97)] + [
    ("pa8192_k55", "pa8192", "canon", 55, 8192, "uniform"),
    ("multipass_k55", "multipass", "canon", 55, 16, "multipass"),
]
GROUPS = {"single": {"SGPU_A_SUB": "1"}, "pa8192": {"SGPU_A_SUB": "1", "SGPU_PA_MAX": "8192"}, "multipass": {"SGPU_A_SUB": "3"}}


def plan_cap(PA, K):
    """records in one batch of levelA_scatter_plan_k (levelA_batch_smem<NW, true>, count.cu)"""
    rec = 8 * ((K + 31) // 32) + 2
    fixed = (((2 * PA * 4 + 15) & ~15) + ROLL_WARPS * ROLL_WARP_BYTES + 15) & ~15
    room = SM_PER_SM // CTAS_PER_SM - SM_RESERVED - SM_STATIC
    if room < fixed + 1024 * rec:
        room = SM_OPTIN - SM_STATIC
    return min((room - fixed) // rec, 32768) & ~31


def reads_of(name):
    if name == "uniform":
        return synthetic_reads(40_000, 150, 200_000, 0.01, seed=3801)       # ~3.8 M windows at K = 55
    if name == "multipass":
        return synthetic_reads(60_000, 150, 200_000, 0.01, seed=3802)
    K = int(name[len("ragged"):])
    reads = synthetic_reads(20_000, 150, 60_000, 0.01, seed=3803)
    reads += synthetic_reads(5_000, K, 60_000, 0.01, seed=3804)
    reads += synthetic_reads(2_000, K - 1, 60_000, 0.01, seed=3805)
    reads += synthetic_reads(2_000, 400, 60_000, 0.01, seed=3806)
    reads += synthetic_reads(300, 1000, 60_000, 0.01, seed=3807)
    order = np.random.default_rng(3808 + K).permutation(len(reads))
    return [reads[i] for i in order]


def _counters(c):
    t = c.times()
    return {f: int(t[f]) for f in ("passes", "level_a_key_bits", "level_a_scatters")}


def worker(out_path, group):
    from spades_b200.kmer_index import (Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter,
                                        ParallelSortingSplitter)
    out, info = {}, {}
    c = Context(0, hbm_budget_bytes=MULTIPASS_BUDGET_MB << 20) if group == "multipass" else Context(0)
    try:
        for name, g, source, K, B, inp in CASES:
            if g != group:
                continue
            c.set_reads(*pack_reads(reads_of(inp)))
            if source == "canon":
                st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
                info[name] = _counters(c)
            elif source == "allwin":
                st = KMerDiskCounter(c, ParallelSortingSplitter(K)).Count(B)
                info[name] = _counters(c)
            else:
                kp = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K + 1)).Count(B)
                info[name + "/kp"] = _counters(c)
                try:
                    st = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(K, kp)).Count(B)
                    info[name] = _counters(c)
                finally:
                    kp.free()
            try:
                out[name + "/keys"], out[name + "/bsz"] = st.kmers(), st.bucket_sizes()
            finally:
                st.free()
    finally:
        c.close()
    out["info"] = np.frombuffer(json.dumps(info).encode(), np.uint8)
    np.savez(out_path, **out)


_RESULTS = {}


def _run(group, tmp_path):
    if group in _RESULTS:
        return _RESULTS[group]
    import gpu_util
    gpu_util.release()
    env = {k: v for k, v in os.environ.items() if k not in ("SGPU_PA_MAX", "SGPU_A_SUB", "SGPU_ARENA_GB")}
    env.update(GROUPS[group])
    if group != "multipass":
        env["SGPU_ARENA_GB"] = str(ARENA_GB)
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    out = tmp_path / ("levela_plan_%s.npz" % group)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out), group], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, "worker failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-3000:])
    with np.load(out) as z:
        got = {k: z[k] for k in z.files}
    _RESULTS[group] = got
    return got


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_planned_batch_matches_oracle(case, tmp_path):
    import oracle as O
    name, group, source, K, B, inp = case
    got = _run(group, tmp_path)
    info = json.loads(got["info"].tobytes())
    cnt = info[name]
    PA = B << cnt["level_a_key_bits"]
    if group == "multipass":
        # three sub-range launches per pass: only the id path takes partition sub-ranges
        assert cnt["passes"] >= 2 and cnt["level_a_scatters"] == 3 * cnt["passes"], "expected a multi-pass count in sub-ranges: %s" % info
    else:
        nsrc = info[name + "/kp"]["passes"] if source == "kpomers" else 1
        assert cnt["passes"] == 1 and cnt["level_a_scatters"] == nsrc, "expected one scatter launch over every record: %s" % info
    if group == "pa8192":
        assert PA == 8192, "partitions of the launch: %s" % info
    if source != "kpomers" and group != "multipass":
        # every id of a single-pass launch is own: a step of 32 chunks of 150 bp reads holds more records than a warp's share
        assert 32 * IDS_PER_CHUNK > plan_cap(PA, K) // ROLL_WARPS
    words, offs, lens = pack_reads(reads_of(inp))
    if source == "kpomers":
        want = O.kmers_from_kpomers(O.count(words, offs, lens, K + 1, B, 0), B)
    else:
        want = O.count(words, offs, lens, K, B, 1 if source == "allwin" else 0)
    np.testing.assert_array_equal(got[name + "/bsz"], want.bsz)
    np.testing.assert_array_equal(got[name + "/keys"], want.keys)


if __name__ == "__main__":
    worker(sys.argv[1], sys.argv[2])
