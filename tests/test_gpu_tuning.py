"""The count under every setting of its tuning knobs, against the C oracle (run with -m gpu on an H100).

SGPU_PA_MAX (level-A partitions), SGPU_RMAX (refinement key bits per round) and SGPU_A_SUB (level-A partition sub-ranges per pass)
are user settings, read once per process. Each setting therefore runs in a child process of its own (tests/tuning_worker.py)
over the same seeded inputs; this process never sets them. The settings drive the refinement and the local sort to depths the
suite's inputs reach nowhere else: a partition that is a whole bucket (PA_MAX = 1), 2-bin refinement rounds until every key bit is
fixed (RMAX = 1), partition sub-ranges combined with pass offsets (A_SUB > 1 on a multi-pass count).

Every case is compared with the oracle: keys, multiplicities, bucket sizes, the device checksum and the serialized KMerIndex, and
every artefact of the graph path. The context's path counters are asserted too, so that a setting or an input that stops reaching
its path fails instead of quietly testing the common path again. A clamped knob value must give the outputs and the counters of
the value it is clamped to."""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import golden_util as G
import gpu_util
import oracle as O
import tuning_worker as W
from spades_b200.packing import pack_reads
from test_gpu_parity import _compare, _oracle_art

pytestmark = pytest.mark.gpu

ARENA_GB = 2                     # the worker's arena (SGPU_ARENA_GB): the largest case needs ~0.2 GB
NEED_BYTES = (ARENA_GB << 30) + (3 << 29)      # arena + what a process costs on the device next to it
KNOBS = ("SGPU_PA_MAX", "SGPU_RMAX", "SGPU_A_SUB")

# every value in range that changes a code path
SETTINGS = {
    "default": {},
    "rmax1": {"SGPU_RMAX": "1"},
    "rmax3": {"SGPU_RMAX": "3"},
    "rmax7_pa1280": {"SGPU_RMAX": "7", "SGPU_PA_MAX": "1280"},
    "pa1": {"SGPU_PA_MAX": "1"},
    "pa8192": {"SGPU_PA_MAX": "8192"},
    "asub3": {"SGPU_A_SUB": "3"},
    "asub64": {"SGPU_A_SUB": "64"},
}
# out-of-range values and the setting they are clamped to
CLAMPED = {
    "rmax0": ({"SGPU_RMAX": "0"}, "rmax1"),
    "rmax99": ({"SGPU_RMAX": "99"}, "default"),
    "pa0": ({"SGPU_PA_MAX": "0"}, "pa1"),
    "pa100000": ({"SGPU_PA_MAX": "100000"}, "pa8192"),
    "asub-5": ({"SGPU_A_SUB": "-5"}, "default"),
}


def knobs(env):
    """(pa_max, rmax, a_sub) as the library reads and clamps them (count.cu, tuning())"""
    pa = min(8192, max(1, int(env.get("SGPU_PA_MAX", 4096))))
    rmax = min(11, max(1, int(env.get("SGPU_RMAX", 11))))
    asub = min(64, max(0, int(env.get("SGPU_A_SUB", 0))))
    return pa, rmax, asub


def cap(K):
    """local-sort capacity (records of one segment) and the segment length the refinement aims for"""
    return (2048, 1536) if K <= 64 else (1024, 768)


def expected_key_bits(est, B, K, pa_max):
    """levelA_key_bits (count.cu): level-A key bits for `est` records"""
    target = cap(K)[1]
    want = (est // target + 1).bit_length()
    bbits = (B - 1).bit_length()
    rA = max(0, want - bbits)
    while rA > 0 and (B << rA) > pa_max:
        rA -= 1
    return min(rA, 2 * K, 13)


# ---- oracle: one result per case, shared by every setting ----------------------------------------------------------------------
_READS, _ORACLE, _COUNTERS = {}, {}, {}


def _packed(inp):
    if inp not in _READS:
        reads = W.reads_of(inp)
        _READS[inp] = (reads, pack_reads(reads))
    return _READS[inp]


def _oracle(case):
    name, inp, K, B, mode, _ = case
    if name not in _ORACLE:
        reads, (words, offs, lens) = _packed(inp)
        if mode == "graph":
            want = _oracle_art(reads, K, B)
            _ORACLE[name] = dict(art=want, n_kp=int(want["oracle"]["kp"].n),
                                 windows=int(np.maximum(lens.astype(np.int64) - K, 0).sum()))
        else:
            ks = O.count(words, offs, lens, K, B, mode)
            wsum = int((ks.keys * (2 * np.arange(ks.nw, dtype=np.uint64) + 1)[None, :]).sum(dtype=np.uint64))
            xr = 0
            for q in range(ks.nw):
                col, rot = ks.keys[:, q], np.uint64(7 * q + 1)
                xr ^= int(np.bitwise_xor.reduce((col << rot) | (col >> (np.uint64(64) - rot))))
            csum = 0 if ks.counts is None else int(ks.counts.astype(np.uint64).sum())
            _ORACLE[name] = dict(keys=ks.keys, counts=ks.counts, bsz=ks.bsz, checksum=[int(ks.n), wsum, xr, csum],
                                 index=O.Mphf(ks).serialize(), windows=int(np.maximum(lens.astype(np.int64) - K + 1, 0).sum()),
                                 max_count=0 if ks.counts is None or ks.n == 0 else int(ks.counts.max()))
    return _ORACLE[name]


def _want_graph_file(tmp_path):
    path = tmp_path / "want_graph.npz"
    want = {}
    for case in W.CASES:
        if case[4] == "graph":
            art = _oracle(case)["art"]
            want[case[0] + "/kpomers"], want[case[0] + "/kmers"] = art["kpomers"], art["kmers"]
    np.savez(path, **want)
    return path


# ---- one setting in a child process ---------------------------------------------------------------------------------------------
def _run_setting(setting, env_knobs, tmp_path):
    """run tuning_worker.py under the given knobs; returns (mismatches per case, counters per case)"""
    gpu_util.release()               # the session's shared context holds most of the device memory
    import torch
    free, total = torch.cuda.mem_get_info(0)
    if free < NEED_BYTES:
        pytest.skip("device 0 has %.2f GiB free of %.2f GiB; the worker needs %.2f GiB" % (free / 2**30, total / 2**30, NEED_BYTES / 2**30))
    want_path = _want_graph_file(tmp_path)
    out = tmp_path / ("%s.npz" % setting)
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(env_knobs)
    env["SGPU_ARENA_GB"] = str(ARENA_GB)
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    t0 = time.time()
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tuning_worker.py"), str(out), str(want_path)],
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "worker failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-3000:])
    got = np.load(out)
    try:
        counters = json.loads(got["counters"].tobytes())
        errors = json.loads(got["errors"].tobytes())
        bad = {}
        for case in W.CASES:
            name = case[0]
            if name in errors:
                bad[name] = [errors[name]]
                continue
            m = _mismatches(case, got)
            if m:
                bad[name] = m
    finally:
        got.close()
        out.unlink()
    _print_table(setting, env_knobs, counters, time.time() - t0)
    return bad, counters


def _mismatches(case, got):
    name, _, K, B, mode, _ = case
    want = _oracle(case)
    if mode == "graph":
        if name + "/gfa" not in got.files:
            return ["sets differ from the oracle's: no graph built"]
        art = {key: got[name + "/" + key] for key in ("kpomers", "kp_bsz", "kmers", "masks", "cov", "hist", "kp_counts")}
        art["kmer_index"], art["kpomer_index"] = got[name + "/kmer_index"].tobytes(), got[name + "/kpomer_index"].tobytes()
        u = got[name + "/unitigs"].tobytes().decode()
        art["unitigs"] = u.split("\n") if u else []
        art["gfa"] = got[name + "/gfa"].tobytes().decode()
        return _compare(art, want["art"], B)
    bad = []
    if not np.array_equal(got[name + "/keys"].ravel(), want["keys"].ravel()):
        bad.append("keys")
    if mode == W.CANON and not np.array_equal(got[name + "/counts"], want["counts"]):
        bad.append("counts")
    if not np.array_equal(got[name + "/bsz"], want["bsz"]):
        bad.append("bucket sizes")
    if [int(x) for x in got[name + "/checksum"]] != want["checksum"]:
        bad.append("checksum")
    if name + "/index" not in got.files:
        bad.append("records not strictly increasing: no index built")
    elif not G.index_equal(want["index"], got[name + "/index"].tobytes(), B):
        bad.append("index")
    return bad


def _print_table(setting, env_knobs, counters, secs):
    print("\n%s %s (%.1f s)" % (setting, " ".join("%s=%s" % kv for kv in sorted(env_knobs.items())) or "(defaults)", secs))
    print("  %-16s %4s %8s %6s %8s %8s %6s %6s %6s" % ("case", "rA", "scatters", "rounds", "split0", "split1+", "lsd", "equal", "passes"))
    for name, cnt in counters.items():
        for part, c in ([("", cnt)] if "kp" not in cnt else [("/" + p, cnt[p]) for p in ("kp", "km") if p in cnt]):
            print("  %-16s %4d %8d %6d %8d %8d %6d %6d %6d" % (name + part, c["level_a_key_bits"], c["level_a_scatters"], c["refine_rounds_max"],
                                                            c["refine_splits_round0"], c["refine_splits_later"], c["sort_lsd_fallbacks"],
                                                            c["sort_oversize_equal"], c["passes"]))


def _path_failures(setting, env_knobs, counters):
    """the paths each case was built to reach, under the given knobs"""
    pa_max, rmax, a_sub = knobs(env_knobs)
    fail = []

    def need(ok, name, what):
        if not ok:
            fail.append("%s: %s" % (name, what))

    for case in W.CASES:
        name, inp, K, B, mode, budget = case
        if name not in counters:
            continue
        want = _oracle(case)
        if mode == "graph":
            kp, km = counters[name].get("kp"), counters[name].get("km")
            need(kp and kp["level_a_key_bits"] == expected_key_bits(want["windows"], B, K + 1, pa_max), name, "(k+1)-mer count rA")
            need(km and km["level_a_key_bits"] == expected_key_bits(2 * want["n_kp"], B, K, pa_max), name, "k-mer count rA")
            need(km and km["level_a_scatters"] == km["passes"], name, "one scatter per pass for the (k+1)-mer source")
            continue
        c = counters[name]
        est = want["windows"] * (2 if mode == W.ALL else 1)
        rA = expected_key_bits(est, B, K, pa_max)
        need(c["level_a_key_bits"] == rA, name, "rA %d, expected %d" % (c["level_a_key_bits"], rA))
        need(c["passes"] == (B if budget else 1), name, "passes %d" % c["passes"])
        PA = (1 if budget else B) << rA              # partitions of one pass
        if mode == W.ALL:
            need(c["level_a_scatters"] == c["passes"], name, "one scatter per pass")
        elif a_sub or not budget:
            nsub = min(a_sub or 4, PA)
            need(c["level_a_scatters"] == c["passes"] * nsub, name, "scatters %d, expected %d per pass" % (c["level_a_scatters"], nsub))
        if mode == W.CANON and inp == "mix":
            # a key with more copies than a segment holds: its segment is refined until every key bit is fixed, at most rmax bits a round
            assert (want["max_count"] + 1) // 2 > cap(K)[0]
            need(c["sort_oversize_equal"] > 0, name, "no oversize equal-key segment")
            need(c["refine_rounds_max"] >= math.ceil((2 * K - rA) / rmax), name,
                 "%d refinement rounds, at least %d needed" % (c["refine_rounds_max"], math.ceil((2 * K - rA) / rmax)))
        if inp.startswith("polyA"):
            need(c["sort_lsd_fallbacks"] > 0, name, "no LSD fallback")
        if pa_max == 1 and inp == "mix" and mode == W.CANON:
            need(c["refine_splits_round0"] > 0, name, "no round-0 split")
    if pa_max > 4096:
        # the only case whose level A wants more than the default 4096 partitions
        c = counters["all70"]
        need(10 << c["level_a_key_bits"] > 4096, "all70", "%d level-A partitions" % (10 << c["level_a_key_bits"]))
    if pa_max == 1:
        # B = 2, whole buckets as partitions: ~1 M records each, split by r >= 10 bits in the gather round (the bench's shape)
        need(counters["k56_b2"]["refine_splits_round0"] >= 2 * 1023, "k56_b2", "round-0 splits %d" % counters["k56_b2"]["refine_splits_round0"])
    return fail


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_count_under_tuning_knobs_matches_oracle(setting, tmp_path):
    bad, counters = _run_setting(setting, SETTINGS[setting], tmp_path)
    _COUNTERS[setting] = counters
    assert bad == {}
    assert _path_failures(setting, SETTINGS[setting], counters) == []


@pytest.mark.parametrize("setting", list(CLAMPED))
def test_clamped_tuning_knob_acts_as_its_clamp(setting, tmp_path):
    env_knobs, clamp = CLAMPED[setting]
    bad, counters = _run_setting(setting, env_knobs, tmp_path)
    assert bad == {}
    if clamp not in _COUNTERS:
        bad_clamp, _COUNTERS[clamp] = _run_setting(clamp, SETTINGS[clamp], tmp_path)
        assert bad_clamp == {}
    # every counter but the LSD fallbacks: which record of a local-sort bin is its representative depends on the order the atomic
    # scatter of the refinement left, and with it how many records of the bin are residual
    for c in (counters, _COUNTERS[clamp]):
        for cnt in c.values():
            for x in (cnt.values() if "kp" in cnt else [cnt]):
                x.pop("sort_lsd_fallbacks", None)
    assert counters == _COUNTERS[clamp]
