"""The level-A partition kernel's shared-memory batch at its edges, against the C oracle (run with -m gpu on an H100).

levelA_scatter_roll_k collects a CTA's own windows in a batch and writes it out partition by partition when it is full; a warp
that finds the batch full waits at its pending window and resumes after the flush. Every case runs as ONE single-pass scatter
launch (SGPU_A_SUB = 1, asserted through the path counters), so every window of a CTA's tiles is its own, and each case holds
enough windows that every CTA but the last fills its batch at least twice (checked from the input against the batch capacity
that the library computes for an H100). The cases:
  - 150 bp reads at K = 55;
  - one partition (SGPU_PA_MAX = 1, B = 1): one run spans every batch;
  - 8192 partitions (B = 8192): the largest tables and the smallest batch for them, which leave too little room for two CTAs per
    SM, so one CTA per SM takes its batch from the per-CTA opt-in limit;
  - ragged tiles: reads shorter than K, of exactly K bases, of 150 bases and of more than 320 bases shuffled together, so that
    warps and lanes reach the flushes with different amounts of work left, at 1 to 4 words per record.
SGPU_PA_MAX and SGPU_A_SUB are read once per process, so each setting runs in a child process of its own (this file, run as a
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

# (name, reads, K, B, SGPU_PA_MAX or None)
CASES = [
    ("full_k55", "uniform", 55, 16, None),
    ("pa1_k55", "uniform", 55, 1, "1"),
    ("pa8192_k55", "uniform", 55, 8192, "8192"),
] + [("ragged_k%d" % K, "ragged%d" % K, K, 16, None) for K in (21, 55, 77, 99)]


# H100 (sm_90): shared memory per SM, opt-in limit per CTA, reserved per CTA; the kernel's static shared memory (count.cu)
SM_PER_SM, SM_OPTIN, SM_RESERVED, SM_STATIC = 233472, 232448, 1024, 128
ROLL_WARP_BYTES, ROLL_WARPS, ROLL_TILE, CTAS_PER_SM = 2952, 16, 32, 2


def batch_cap(PA, K):
    """records in one batch of levelA_scatter_roll_k (levelA_batch_smem, count.cu)"""
    nw = (K + 31) // 32
    rec = 8 * nw + 4 + 2
    fixed = (((2 * PA * 4 + 15) & ~15) + ROLL_WARPS * ROLL_WARP_BYTES + 15) & ~15
    room = SM_PER_SM // CTAS_PER_SM - SM_RESERVED - SM_STATIC
    if room < fixed + 1024 * rec:
        room = SM_OPTIN - SM_STATIC
    return min((room - fixed) // rec, 32768) & ~31


def windows_per_cta(lens, K, G):
    """own windows of every CTA of the level-A grid (static tile ranges) in a single-pass, single-sub-range launch"""
    w = np.maximum(lens.astype(np.int64) - K + 1, 0)
    ntiles = (len(w) + ROLL_TILE - 1) // ROLL_TILE
    per = (ntiles + G - 1) // G
    tile_w = np.add.reduceat(w, np.arange(0, len(w), ROLL_TILE))
    return [int(tile_w[g * per:(g + 1) * per].sum()) for g in range(G) if g * per < ntiles]


def reads_of(name):
    if name == "uniform":
        return synthetic_reads(40_000, 150, 200_000, 0.01, seed=3101)       # ~3.8 M windows at K = 55
    K = int(name[len("ragged"):])
    reads = synthetic_reads(40_000, 150, 60_000, 0.01, seed=3102)
    reads += synthetic_reads(10_000, K, 60_000, 0.01, seed=3103)
    reads += synthetic_reads(3_000, K - 1, 60_000, 0.01, seed=3104)
    reads += synthetic_reads(3_000, 400, 60_000, 0.01, seed=3105)
    reads += synthetic_reads(600, 1000, 60_000, 0.01, seed=3106)
    order = np.random.default_rng(3107 + K).permutation(len(reads))
    return [reads[i] for i in order]


def worker(out_path, pa_max):
    from spades_b200.kmer_index import Context, DeBruijnReadKMerSplitter, KMerDiskCounter
    out, info = {}, {}
    c = Context(0)
    try:
        for name, inp, K, B, pa in CASES:
            if pa != pa_max:
                continue
            c.set_reads(*pack_reads(reads_of(inp)))
            st = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K)).Count(B)
            try:
                t = c.times()
                info[name] = {f: int(t[f]) for f in ("passes", "level_a_key_bits", "level_a_scatters")}
                out[name + "/keys"], out[name + "/counts"], out[name + "/bsz"] = st.kmers(), st.counts(), st.bucket_sizes()
            finally:
                st.free()
    finally:
        c.close()
    out["info"] = np.frombuffer(json.dumps(info).encode(), np.uint8)
    np.savez(out_path, **out)


_RESULTS = {}


def _run(pa_max, tmp_path):
    if pa_max in _RESULTS:
        return _RESULTS[pa_max]
    import gpu_util
    gpu_util.release()
    env = {k: v for k, v in os.environ.items() if k not in ("SGPU_PA_MAX", "SGPU_A_SUB")}
    env["SGPU_A_SUB"] = "1"
    if pa_max is not None:
        env["SGPU_PA_MAX"] = pa_max
    env["SGPU_ARENA_GB"] = str(ARENA_GB)
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    out = tmp_path / ("levela_batch_%s.npz" % (pa_max or "default"))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out), pa_max or ""], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "worker failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-3000:])
    with np.load(out) as z:
        got = {k: z[k] for k in z.files}
    _RESULTS[pa_max] = got
    return got


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_levela_batch_matches_oracle(case, tmp_path):
    import oracle as O
    name, inp, K, B, pa_max = case
    got = _run(pa_max, tmp_path)
    info = json.loads(got["info"].tobytes())[name]
    assert info["passes"] == 1 and info["level_a_scatters"] == 1, "expected one scatter launch over every window: %s" % info
    PA = B << info["level_a_key_bits"]
    if pa_max is not None:
        assert PA == int(pa_max), "partitions of the launch: %s" % info
    words, offs, lens = pack_reads(reads_of(inp))
    import torch
    G = CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count
    per_cta = windows_per_cta(lens, K, G)
    cap = batch_cap(PA, K)
    assert min(per_cta[:-1]) > 2 * cap, "the batch (%d records) must overflow at least twice in every CTA: %d" % (cap, min(per_cta[:-1]))
    want = O.count(words, offs, lens, K, B, 0)
    np.testing.assert_array_equal(got[name + "/bsz"], want.bsz)
    np.testing.assert_array_equal(got[name + "/keys"], want.keys)
    np.testing.assert_array_equal(got[name + "/counts"], want.counts)


if __name__ == "__main__":
    worker(sys.argv[1], sys.argv[2] or None)
