"""Host-side mirror of the reference's k-mer index interface, over the C ABI (no torch types, no CPU fallback).

Names and argument meaning follow the reference so the parity tests read like its own:
  KMerDiskCounter.Count / CountAll     src/common/kmer_index/kmer_mph/kmer_index_builder.hpp:284-340
  KMerDiskStorage                      …/kmer_index_builder.hpp:47-256
  KMerIndexBuilder.BuildIndex          …/kmer_index_builder.hpp:448-514
  KMerIndex.serialize / seq_idx        …/kmer_index.hpp:88-108
  DeBruijnReadKMerSplitter / ParallelSortingSplitter / DeBruijnKMerKMerSplitter  (the `splitter` argument of a counter)
"""
import ctypes as C

import numpy as np

from . import _lib

SGPU_CANONICAL, SGPU_ALL_WINDOWS = 0, 1
SGPU_RESULT_ON_HOST = 0x100      # OR-ed into a count's mode: the set is returned in pinned host memory


class SpadesGpuError(RuntimeError):
    pass


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class Context:
    """One GPU context (one per process per GPU)."""

    def __init__(self, device=0, hbm_budget_bytes=0, verbose=0, stream=0):
        self.L = _lib.load()
        cfg = _lib.SgpuConfig(device, hbm_budget_bytes, verbose, stream)
        h = C.c_void_p()
        rc = self.L.sgpu_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise SpadesGpuError(f"sgpu_create failed with code {rc} (3 = no CUDA device): this path has no CPU fallback")
        self.h = h

    def check(self, rc):
        if rc != 0:
            raise SpadesGpuError(f"[{rc}] " + self.L.sgpu_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.sgpu_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    # reads -------------------------------------------------------------------------------------------------
    def set_reads(self, words, offs, lens):
        """Host buffers in the layout of spades_b200.packing.pack_reads (H2D happens at first use)."""
        words = np.ascontiguousarray(words, np.uint64); offs = np.ascontiguousarray(offs, np.uint64); lens = np.ascontiguousarray(lens, np.uint32)
        self.check(self.L.sgpu_reads_clear(self.h))
        self.check(self.L.sgpu_reads_append_packed(self.h, _p(words), len(words), _p(offs), _p(lens), len(lens)))

    def upload_reads(self, words_ptr, nwords, offs_ptr, lens_ptr, nreads):
        """Raw host pointers (e.g. pinned torch tensors) copied straight to the device."""
        self.check(self.L.sgpu_reads_upload(self.h, C.c_void_p(words_ptr), nwords, C.c_void_p(offs_ptr), C.c_void_p(lens_ptr), nreads))

    def adopt_device_reads(self, d_words_ptr, nwords, d_offs_ptr, d_lens_ptr, nreads):
        self.check(self.L.sgpu_reads_adopt_device(self.h, C.c_void_p(d_words_ptr), nwords, C.c_void_p(d_offs_ptr), C.c_void_p(d_lens_ptr), nreads))

    def times(self):
        t = _lib.SgpuTimes()
        self.L.sgpu_get_times(self.h, C.byref(t))
        return {f[0]: getattr(t, f[0]) for f in _lib.SgpuTimes._fields_}


class KMerDiskStorage:
    """Result of a count: B buckets of strictly increasing records, resident in HBM or, for a count with result_on_host, in pinned
    host memory (every accessor and KMerIndexBuilder work on both; the graph path needs sets in HBM)."""

    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h
        L = ctx.L
        self._k = L.sgpu_kset_k(h)
        self._B = L.sgpu_kset_num_buckets(h)
        self._n = L.sgpu_kset_size(h)
        self.nw = L.sgpu_kset_record_bytes(h) // 8

    def k(self):
        return self._k

    def num_buckets(self):
        return self._B

    def total_kmers(self):
        return self._n

    def on_host(self):
        return self.ctx.L.sgpu_kset_on_host(self.h) == 1

    def bucket_sizes(self):
        out = np.zeros(self._B, np.int64)
        self.ctx.check(self.ctx.L.sgpu_kset_bucket_sizes(self.h, _p(out)))
        return out

    def bucket_size(self, i):
        return int(self.bucket_sizes()[i])

    def kmers(self, first=0, n=None):
        """final_kmers order records as u64 [n, nw]."""
        n = self._n - first if n is None else n
        out = np.zeros((max(n, 1), self.nw), np.uint64)
        self.ctx.check(self.ctx.L.sgpu_kset_download_keys(self.h, first, n, _p(out)))
        return out[:n]

    def download_keys_into(self, host_ptr, n, first=0):
        """records [first, first+n) of final_kmers order copied to caller memory (e.g. a pinned buffer of n * nw u64)"""
        self.ctx.check(self.ctx.L.sgpu_kset_download_keys(self.h, first, n, C.c_void_p(host_ptr)))

    def counts(self, first=0, n=None):
        n = self._n - first if n is None else n
        out = np.zeros(max(n, 1), np.uint32)
        self.ctx.check(self.ctx.L.sgpu_kset_download_counts(self.h, first, n, _p(out)))
        return out[:n]

    def checksum(self):
        """(n, weighted sum of the record words, xor of the rotated record words, sum of multiplicities), computed on the device."""
        out = np.zeros(4, np.uint64)
        self.ctx.check(self.ctx.L.sgpu_kset_checksum(self.h, _p(out)))
        return [int(x) for x in out]

    def write_buckets(self, prefix):
        self.ctx.check(self.ctx.L.sgpu_kset_write_buckets(self.h, str(prefix).encode()))

    def owned_buckets(self):
        """bool [B]: the buckets this set holds (all of them, or this rank's share of a distributed count)"""
        out = np.zeros(self._B, np.uint8)
        self.ctx.check(self.ctx.L.sgpu_kset_owned_buckets(self.h, _p(out)))
        return out.astype(bool)

    def write_owned_buckets(self, prefix):
        """prefix.<b> for the owned buckets only: the ranks of a distributed count writing into one directory leave every bucket file once"""
        self.ctx.check(self.ctx.L.sgpu_kset_write_owned_buckets(self.h, str(prefix).encode()))

    def merge(self, path):
        """KMerDiskStorage::merge -> final_kmers file."""
        self.ctx.check(self.ctx.L.sgpu_kset_write_final(self.h, str(path).encode()))

    def free(self):
        if self.h:
            self.ctx.L.sgpu_kset_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeBruijnReadKMerSplitter:
    """reads (+RC) -> canonical K-mers (StoringTypeFilter<InvertableStoring>)."""
    mode = SGPU_CANONICAL

    def __init__(self, K):
        self.K = K


class ParallelSortingSplitter(DeBruijnReadKMerSplitter):
    """spades-kmercount: every window of read and RC, unfiltered."""
    mode = SGPU_ALL_WINDOWS


class DeBruijnKMerKMerSplitter:
    """distinct (K+1)-mers -> canonical K-mers."""

    def __init__(self, K_target, kpomers: KMerDiskStorage):
        assert kpomers.k() == K_target + 1
        self.K, self.source = K_target, kpomers


class KMerDiskCounter:
    """result_on_host: the counted set goes to pinned host memory, pass by pass behind the next one, so it may exceed HBM. The
    (k+1)-mers of a DeBruijnKMerKMerSplitter may live in either place."""

    def __init__(self, ctx: Context, splitter, result_on_host=False):
        self.ctx, self.splitter, self.result_on_host = ctx, splitter, result_on_host

    def Count(self, num_buckets, num_threads=0):
        h = C.c_void_p()
        if isinstance(self.splitter, DeBruijnKMerKMerSplitter):
            mode = SGPU_RESULT_ON_HOST if self.result_on_host else 0
            rc = self.ctx.L.sgpu_kmers_from_kpomers_ex(self.ctx.h, self.splitter.source.h, num_buckets, mode, C.byref(h))
        else:
            mode = self.splitter.mode | (SGPU_RESULT_ON_HOST if self.result_on_host else 0)
            rc = self.ctx.L.sgpu_count(self.ctx.h, self.splitter.K, num_buckets, mode, C.byref(h))
        self.ctx.check(rc)
        return KMerDiskStorage(self.ctx, h)

    def CountAll(self, num_buckets, num_threads=0, merge_to=None):
        st = self.Count(num_buckets, num_threads)
        if merge_to:
            st.merge(merge_to)
        return st


class KMerIndex:
    def __init__(self, ctx, h, storage):
        self.ctx, self.h, self.storage = ctx, h, storage

    def serialize(self) -> bytes:
        n = self.ctx.L.sgpu_mphf_serialized_size(self.h)
        if n < 0:
            raise SpadesGpuError(self.ctx.L.sgpu_last_error(self.ctx.h).decode())
        buf = np.zeros(n, np.uint8)
        self.ctx.check(self.ctx.L.sgpu_mphf_serialize(self.h, _p(buf), n))
        return buf.tobytes()

    def serialized_size(self) -> int:
        return int(self.ctx.L.sgpu_mphf_serialized_size(self.h))

    def serialize_buckets(self, b_lo, b_hi) -> bytes:
        """the serialized buckets [b_lo, b_hi) alone, as they appear inside serialize()"""
        n = self.ctx.L.sgpu_mphf_serialized_size_buckets(self.h, b_lo, b_hi)
        if n < 0:
            raise ValueError("bucket range [%d, %d) outside the index" % (b_lo, b_hi))
        buf = np.zeros(max(n, 1), np.uint8)
        self.ctx.check(self.ctx.L.sgpu_mphf_serialize_buckets(self.h, b_lo, b_hi, _p(buf), n))
        return buf[:n].tobytes()

    def serialize_into(self, host_ptr, cap):
        """KMerIndex::serialize bytes written to caller memory (e.g. a pinned buffer); returns the size."""
        n = self.serialized_size()
        self.ctx.check(self.ctx.L.sgpu_mphf_serialize(self.h, C.c_void_p(host_ptr), cap))
        return n

    def seq_idx(self, keys):
        keys = np.ascontiguousarray(keys, np.uint64).reshape(-1, self.storage.nw)
        out = np.zeros(max(len(keys), 1), np.uint64)
        self.ctx.check(self.ctx.L.sgpu_mphf_lookup(self.h, _p(keys), len(keys), _p(out)))
        return out[: len(keys)]

    def free(self):
        if self.h:
            self.ctx.L.sgpu_mphf_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class KMerIndexBuilder:
    def __init__(self, ctx: Context):
        self.ctx = ctx

    def BuildIndex(self, storage: KMerDiskStorage) -> KMerIndex:
        h = C.c_void_p()
        self.ctx.check(self.ctx.L.sgpu_mphf_build(self.ctx.h, storage.h, C.byref(h)))
        return KMerIndex(self.ctx, h, storage)
