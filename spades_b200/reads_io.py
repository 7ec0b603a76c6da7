"""Host-side mirror of the reference's read front end over the C ABI (pure host code: works without a GPU).

  read_fastx      io::FastaFastqGzParser (kseq + zlib) + io::LongestValid     src/common/io/reads/fasta_fastq_gz_parser.hpp:25-150,
                                                                              longest_valid_wrapper.hpp:16-53, io_helper.cpp:21-35
  read_seqfile    io::BinaryFileSingleStream over <prefix>.seq / .off          io/reads/binary_streams.hpp:54-140
  write_seqfile   io::BinaryWriter::ToBinary (single reads)                   io/reads/binary_converter.cpp:84-145
"""
import ctypes as C

import numpy as np

from . import _lib


class ReadBatch:
    """2-bit packed reads (words, offs, lens) in the layout Context.set_reads / sgpu_reads_append_packed take."""

    def __init__(self, h):
        self.h = h
        L = _lib.load()
        n, nw = L.sgpu_read_batch_num_reads(h), L.sgpu_read_batch_num_words(h)
        self.words = np.ctypeslib.as_array(C.cast(L.sgpu_read_batch_words(h), C.POINTER(C.c_uint64)), shape=(nw,)).copy() if nw else np.zeros(0, np.uint64)
        self.offs = np.ctypeslib.as_array(C.cast(L.sgpu_read_batch_offs(h), C.POINTER(C.c_uint64)), shape=(n,)).copy() if n else np.zeros(0, np.uint64)
        self.lens = np.ctypeslib.as_array(C.cast(L.sgpu_read_batch_lens(h), C.POINTER(C.c_uint32)), shape=(n,)).copy() if n else np.zeros(0, np.uint32)
        st = np.zeros(3, np.uint64)
        L.sgpu_read_batch_stats(h, st.ctypes.data_as(C.c_void_p))
        self.records, self.trimmed, self.dropped = (int(x) for x in st)

    def __len__(self):
        return len(self.lens)

    def strings(self):
        out = []
        for o, l in zip(self.offs, self.lens):
            w = self.words[int(o):int(o) + (int(l) + 31) // 32]
            codes = ((w[:, None] >> (np.arange(32, dtype=np.uint64) * np.uint64(2))) & np.uint64(3)).astype(np.uint8).ravel()[:int(l)]
            out.append(np.frombuffer(b"ACGT", np.uint8)[codes].tobytes().decode())
        return out

    def write_seqfile(self, prefix):
        rc = _lib.load().sgpu_read_batch_write_seqfile(self.h, str(prefix).encode())
        if rc:
            raise IOError("cannot write %s.seq/.off (error %d)" % (prefix, rc))

    def free(self):
        if self.h:
            _lib.load().sgpu_read_batch_free(self.h); self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _parse(fn, *args):
    L = _lib.load()
    h = C.c_void_p()
    rc = fn(*args, C.byref(h))
    if rc:
        msg = L.sgpu_read_batch_error(h).decode() if h else "error %d" % rc
        if h:
            L.sgpu_read_batch_free(h)
        raise IOError(msg)
    return ReadBatch(h)


def read_fastx(path, longest_valid=True, threads=0) -> ReadBatch:
    """threads: 0 = all hardware threads for uncompressed files (exact: pieces are only accepted where the sequential parser
    provably stands at the same place), 1 = sequential"""
    return _parse(_lib.load().sgpu_fastx_parse_threads, str(path).encode(), 1 if longest_valid else 0, int(threads))


def read_seqfile(prefix) -> ReadBatch:
    return _parse(_lib.load().sgpu_seqfile_parse, str(prefix).encode())


def index_text(data: bytes):
    """host side of the GPU packer: (offsets u64[n], lengths u32[n]) of every read's sequence inside a strictly 2-line FASTA / 4-line FASTQ
    text, or None when the text is not in that layout (multi-line records, junk: use read_fastx, which has kseq's general semantics)"""
    L = _lib.load()
    cap = data.count(b"\n") // 2 + 2
    off = np.zeros(cap, np.uint64); ln = np.zeros(cap, np.uint32)
    n = L.sgpu_text_index_fastx(data, len(data), off.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), cap)
    if n < 0:
        return None
    return off[:n], ln[:n]


def pack_text_on_gpu(ctx, data: bytes, longest_valid=True):
    """FASTA/FASTQ text -> the context's packed read set with trimming (LongestValid) and 2-bit packing done by CUDA kernels
    (sgpu_reads_pack_text); the host only locates the sequence lines. Returns the number of reads (zero-length ones included)."""
    idx = index_text(data)
    if idx is None:
        raise IOError("not a strict 2-line FASTA / 4-line FASTQ text: use read_fastx")
    off, ln = idx
    ctx.check(ctx.L.sgpu_reads_pack_text(ctx.h, data, len(data), off.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), len(ln),
                                         1 if longest_valid else 0))
    return len(ln)


def download_reads(ctx):
    """the context's packed read set as host arrays (words, offs, lens)"""
    n, nw = C.c_int64(), C.c_uint64()
    ctx.check(ctx.L.sgpu_reads_info(ctx.h, C.byref(n), C.byref(nw)))
    words = np.zeros(max(nw.value, 1), np.uint64); offs = np.zeros(max(n.value, 1), np.uint64); lens = np.zeros(max(n.value, 1), np.uint32)
    ctx.check(ctx.L.sgpu_reads_download(ctx.h, words.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p)))
    return words[: nw.value], offs[: n.value], lens[: n.value]


def CovFilteringWrap(ctx, k_plus_one, threshold, apply=True, passes=0):
    """The construction stage's coverage pre-filter (stages/construction.cpp:167-198: EstimateCardinalityUpperBound -> qf::cqf ->
    FillCoverageHistogram -> io::CovFilteringWrap, io/reads/coverage_filtering_read_wrapper.hpp:100-122) on the context's read set:
    a read survives iff the median multiplicity of its (k+1)-mers reaches `threshold`. Returns (keep flags of the reads as they were,
    {"cardinality_upper_bound", "key_bits", "distinct_keys", "kept"}); with apply the survivors become the context's read set.
    passes: 0 = one counting table, or key-range passes when it does not fit the device memory left; 1 = one table; 2 .. 256 = that
    many key-range passes. The result is the same for every value; Context.times() reports the passes taken."""
    n, nw = C.c_int64(), C.c_uint64()
    ctx.check(ctx.L.sgpu_reads_info(ctx.h, C.byref(n), C.byref(nw)))
    keep = np.zeros(max(n.value, 1), np.uint8)
    stats = np.zeros(4, np.uint64)
    args = (int(k_plus_one), int(threshold), 1 if apply else 0)
    out = (keep.ctypes.data_as(C.c_void_p), stats.ctypes.data_as(C.c_void_p))
    if passes == 0:
        ctx.check(ctx.L.sgpu_reads_cov_filter(ctx.h, *args, *out))
    else:
        ctx.check(ctx.L.sgpu_reads_cov_filter_ex(ctx.h, *args, int(passes), *out))
    return keep[: n.value], {"cardinality_upper_bound": int(stats[0]), "key_bits": int(stats[1]), "distinct_keys": int(stats[2]), "kept": int(stats[3])}
