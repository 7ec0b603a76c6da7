"""The level-A rolling kernels over their other sources, against the C oracle (run with -m gpu on an H100).

levelA_count_roll_k / levelA_scatter_roll_k serve three inputs: canonical counts of reads (test_gpu_levela_batch.py), the
all-windows count of reads (spades-kmercount: a chunk is 12 windows x 2 strands) and the k-mers of the (k+1)-mers (a k-mer set
read as sequences of K+1 bases, two windows per item). The cases here take the last two to the kernels' edges:
  - chunk geometry: all-windows counts at every word boundary of K, over reads shorter than K, of exactly K bases, of 150 bases
    and of more than 320 bases (a warp tile that no longer fits its staging slice);
  - full batches: single-pass, single-sub-range launches (SGPU_A_SUB = 1) in which every CTA but the last fills its batch at
    least twice, for the all-windows count and for the graph path's k-mers of the (k+1)-mers at k = 21, 55 and 99;
  - the id-less scatter: a budgeted context in which the partition-id array does not fit (its size, computed from the input,
    is more than the fifth of the arena the count allows it), over several passes. These sources scatter once per pass and
    source whatever SGPU_A_SUB says (partition sub-ranges are taken by canonical counts only), which SGPU_A_SUB = 3 checks.
SGPU_A_SUB is read once per process, so each setting runs in a child process of its own (this file, run as a script)."""
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
from test_gpu_levela_batch import CTAS_PER_SM, ROLL_TILE, batch_cap, windows_per_cta  # noqa: E402

pytestmark = pytest.mark.gpu

ARENA_GB = 2
B_FULL = 16
IDLESS_BUDGET_MB = 200
IDS_PER_KPOMER, IDS_PER_ALLWIN_CHUNK, ALLWIN_CHUNK = 8, 24, 12     # partition-id slots (count.cu: KmerSetSrc::kIds, kRollC)

# (name, source, K, reads): source "allwin" = all-windows count of the reads at K, "kpomers" = k-mers of their (K+1)-mers
FULL_CASES = [("allwin_k55", "allwin", 55, "full")] + [("kpomers_k%d" % k, "kpomers", k, "full") for k in (21, 55, 99)]
IDLESS_CASES = [("allwin_k55", "allwin", 55, "idless_allwin"), ("kpomers_k55", "kpomers", 55, "idless_kpomers")]


def reads_of(name):
    if name == "full":
        return synthetic_reads(40_000, 150, 200_000, 0.01, seed=3201)
    if name == "idless_allwin":
        return synthetic_reads(120_000, 150, 200_000, 0.001, seed=3202)     # 23 M records, 46 MB of ids
    return synthetic_reads(72_000, 150, 200_000, 0.01, seed=3203)             # ~3 M (k+1)-mers, ~50 MB of ids


def ragged_reads(K):
    reads = synthetic_reads(300, 150, 3000, 0.01, seed=3300 + K)
    reads += synthetic_reads(100, K, 3000, 0.01, seed=3400 + K)
    reads += synthetic_reads(100, K - 1, 3000, 0.01, seed=3500 + K)
    reads += synthetic_reads(60, 400, 3000, 0.01, seed=3600 + K)
    order = np.random.default_rng(3700 + K).permutation(len(reads))
    return [reads[i] for i in order]


@pytest.mark.parametrize("K", [21, 32, 33, 64, 65, 96, 97, 128])
def test_all_windows_chunk_geometry_matches_oracle(K):
    import oracle as O
    from gpu_util import gpu_count_artifacts
    reads = ragged_reads(K)
    art, st = gpu_count_artifacts(reads, K, 7)
    st.free()
    words, offs, lens = pack_reads(reads)
    want = O.count(words, offs, lens, K, 7, 1)
    np.testing.assert_array_equal(art["bsz"], want.bsz)
    np.testing.assert_array_equal(art["final_kmers"], want.keys)


def _counters(c):
    t = c.times()
    return {f: int(t[f]) for f in ("passes", "level_a_key_bits", "level_a_scatters")}


def worker(out_path, group):
    from spades_b200.kmer_index import (Context, DeBruijnKMerKMerSplitter, DeBruijnReadKMerSplitter, KMerDiskCounter,
                                        ParallelSortingSplitter)
    cases = FULL_CASES if group == "full" else IDLESS_CASES
    out, info = {}, {}
    c = Context(0) if group == "full" else Context(0, hbm_budget_bytes=IDLESS_BUDGET_MB << 20)
    try:
        for name, source, K, inp in cases:
            c.set_reads(*pack_reads(reads_of(inp)))
            if source == "allwin":
                st = KMerDiskCounter(c, ParallelSortingSplitter(K)).Count(B_FULL)
                info[name] = _counters(c)
            else:
                kp = KMerDiskCounter(c, DeBruijnReadKMerSplitter(K + 1)).Count(B_FULL)
                info[name + "/kp"] = _counters(c)
                info[name + "/kp"]["n"] = int(kp.total_kmers())
                try:
                    st = KMerDiskCounter(c, DeBruijnKMerKMerSplitter(K, kp)).Count(B_FULL)
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
    env["SGPU_A_SUB"] = "1" if group == "full" else "3"
    if group == "full":
        env["SGPU_ARENA_GB"] = str(ARENA_GB)
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    out = tmp_path / ("levela_sources_%s.npz" % group)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out), group], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, "worker failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-3000:])
    with np.load(out) as z:
        got = {k: z[k] for k in z.files}
    _RESULTS[group] = got
    return got


def _oracle(source, K, inp):
    import oracle as O
    words, offs, lens = pack_reads(reads_of(inp))
    if source == "allwin":
        return O.count(words, offs, lens, K, B_FULL, 1), (words, offs, lens)
    kp = O.count(words, offs, lens, K + 1, B_FULL, 0)
    return O.kmers_from_kpomers(kp, B_FULL), kp


def _check(got, name, want):
    np.testing.assert_array_equal(got[name + "/bsz"], want.bsz)
    np.testing.assert_array_equal(got[name + "/keys"], want.keys)


@pytest.mark.parametrize("case", FULL_CASES, ids=[c[0] for c in FULL_CASES])
def test_full_batches_match_oracle(case, tmp_path):
    import torch
    name, source, K, inp = case
    got = _run("full", tmp_path)
    info = json.loads(got["info"].tobytes())
    cnt = info[name]
    assert cnt["passes"] == 1 and cnt["level_a_scatters"] == 1, "expected one scatter launch over every record: %s" % info
    want, aux = _oracle(source, K, inp)
    G = CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count
    if source == "allwin":
        per_cta = [2 * w for w in windows_per_cta(aux[2], K, G)]
    else:
        assert info[name + "/kp"]["passes"] == 1, "the (k+1)-mers must be one chunk: %s" % info
        n = info[name + "/kp"]["n"]
        assert n == aux.n
        per = ((n + ROLL_TILE - 1) // ROLL_TILE + G - 1) // G * ROLL_TILE          # items of a CTA's tile range
        per_cta = [2 * min(per, n - g * per) for g in range(G) if g * per < n]
    cap = batch_cap(B_FULL << cnt["level_a_key_bits"], K)
    assert min(per_cta[:-1]) > 2 * cap, "the batch (%d records) must overflow at least twice in every CTA: %d" % (cap, min(per_cta[:-1]))
    _check(got, name, want)


@pytest.mark.parametrize("case", IDLESS_CASES, ids=[c[0] for c in IDLESS_CASES])
def test_idless_scatter_matches_oracle(case, tmp_path):
    name, source, K, inp = case
    got = _run("idless", tmp_path)
    info = json.loads(got["info"].tobytes())
    cnt = info[name]
    want, aux = _oracle(source, K, inp)
    # the id array (2 bytes per slot) takes more than the fifth of the arena that the count allows it
    if source == "allwin":
        w = np.maximum(aux[2].astype(np.int64) - K + 1, 0)
        slots = int(((w + ALLWIN_CHUNK - 1) // ALLWIN_CHUNK).sum()) * IDS_PER_ALLWIN_CHUNK
        nsrc = 1
    else:
        slots = info[name + "/kp"]["n"] * IDS_PER_KPOMER
        nsrc = info[name + "/kp"]["passes"]             # every pass of the (k+1)-mer count is one chunk, one source
    assert 2 * slots > 0.2 * (IDLESS_BUDGET_MB << 20), slots
    assert cnt["passes"] >= 2, "expected a multi-pass count: %s" % info
    assert cnt["level_a_scatters"] == cnt["passes"] * nsrc, "expected one scatter launch per pass and source: %s" % info
    _check(got, name, want)


if __name__ == "__main__":
    worker(sys.argv[1], sys.argv[2])
