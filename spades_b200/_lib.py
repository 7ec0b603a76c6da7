"""ctypes binding of libspades_b200.so (C ABI declared in include/spades_b200.h).

There is NO fallback: if the CUDA library is missing or no GPU is visible the product path raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libspades_b200.so")

# every symbol include/spades_b200.h declares (tests check that the library exports exactly these)
SYMBOLS = [
    "sgpu_create", "sgpu_destroy", "sgpu_last_error", "sgpu_get_times",
    "sgpu_reads_clear", "sgpu_reads_append_packed", "sgpu_reads_upload", "sgpu_reads_adopt_device", "sgpu_reads_pack_text", "sgpu_reads_info",
    "sgpu_reads_download", "sgpu_text_index_fastx", "sgpu_reads_cov_filter", "sgpu_reads_cov_filter_ex", "sgpu_cov_pass_plan_host",
    "sgpu_fastx_parse", "sgpu_fastx_parse_threads", "sgpu_seqfile_parse", "sgpu_read_batch_write_seqfile", "sgpu_read_batch_num_reads", "sgpu_read_batch_num_words",
    "sgpu_read_batch_words", "sgpu_read_batch_offs", "sgpu_read_batch_lens", "sgpu_read_batch_stats", "sgpu_read_batch_error", "sgpu_read_batch_free",
    "sgpu_reads_append_batch",
    "sgpu_count", "sgpu_kmers_from_kpomers", "sgpu_kmers_from_kpomers_ex",
    "sgpu_kset_size", "sgpu_kset_k", "sgpu_kset_num_buckets", "sgpu_kset_record_bytes", "sgpu_kset_on_host", "sgpu_kset_bucket_sizes",
    "sgpu_kset_checksum", "sgpu_kset_download_keys", "sgpu_kset_download_counts", "sgpu_kset_write_buckets", "sgpu_kset_write_final", "sgpu_kset_free",
    "sgpu_kset_owned_buckets", "sgpu_kset_write_owned_buckets",
    "sgpu_mphf_build", "sgpu_mphf_serialized_size", "sgpu_mphf_serialize", "sgpu_mphf_lookup", "sgpu_mphf_free",
    "sgpu_mphf_serialized_size_buckets", "sgpu_mphf_serialize_buckets",
    "sgpu_graph_build", "sgpu_graph_build_ex", "sgpu_graph_build_opts", "sgpu_graph_build_streamed", "sgpu_graph_at_clipper_stats", "sgpu_graph_tip_clipper_stats", "sgpu_graph_masks", "sgpu_graph_coverage", "sgpu_graph_histogram", "sgpu_graph_num_unitigs",
    "sgpu_graph_unitig_bases", "sgpu_graph_unitigs", "sgpu_graph_gfa", "sgpu_graph_write_gfa", "sgpu_graph_free",
    "sgpu_edge_index_build", "sgpu_edge_index_k", "sgpu_edge_index_size", "sgpu_edge_index_serialized_size", "sgpu_edge_index_serialize",
    "sgpu_edge_index_values", "sgpu_edge_index_lookup", "sgpu_edge_index_free",
    "sgpu_dist_begin", "sgpu_dist_begin_kpomers", "sgpu_dist_num_partitions", "sgpu_dist_local_counts", "sgpu_dist_plan", "sgpu_dist_free_bytes", "sgpu_dist_next_pass", "sgpu_dist_ipc_handle",
    "sgpu_dist_open_peers", "sgpu_dist_scatter", "sgpu_dist_exchange", "sgpu_dist_sort", "sgpu_dist_end", "sgpu_dist_free", "sgpu_dist_plan_host",
    "sgpu_dist_cov_begin", "sgpu_dist_cov_ipc_handle", "sgpu_dist_cov_open_peers", "sgpu_dist_cov_bound", "sgpu_dist_cov_fill", "sgpu_dist_cov_filter",
    "sgpu_dist_cov_free", "sgpu_dist_cov_layout_host",
    "sgpu_dist_ext_begin", "sgpu_dist_ext_local_counts", "sgpu_dist_ext_plan", "sgpu_dist_ext_free_bytes", "sgpu_dist_ext_next_pass",
    "sgpu_dist_ext_ipc_handle", "sgpu_dist_ext_open_peers", "sgpu_dist_ext_scatter", "sgpu_dist_ext_apply", "sgpu_dist_ext_masks",
    "sgpu_dist_ext_coverage", "sgpu_dist_ext_histogram", "sgpu_dist_ext_times", "sgpu_dist_ext_free", "sgpu_dist_ext_plan_host",
    "sgpu_dist_graph_begin", "sgpu_dist_graph_ipc_handle", "sgpu_dist_graph_open_peers", "sgpu_dist_graph_unitigs", "sgpu_dist_graph_clear_visited",
    "sgpu_dist_graph_loops", "sgpu_dist_graph_stats", "sgpu_dist_graph_edges", "sgpu_dist_graph_bucket_counts", "sgpu_dist_graph_times",
    "sgpu_dist_graph_free", "sgpu_graph_from_edges",
    "sgpu_dist_graph_begin_opts", "sgpu_dist_graph_at_edges_probe", "sgpu_dist_graph_at_edges_apply", "sgpu_dist_graph_at_tips_probe",
    "sgpu_dist_graph_tip_probe", "sgpu_dist_graph_isolate", "sgpu_dist_graph_unlink", "sgpu_dist_graph_junctions", "sgpu_dist_graph_masks",
    "sgpu_dist_graph_clipper_stats", "sgpu_dist_graph_clipper_times",
    "sgpu_dist_edge_index_begin", "sgpu_dist_edge_index_count_begin", "sgpu_dist_edge_index_keys", "sgpu_dist_edge_index_ipc_handle",
    "sgpu_dist_edge_index_open_peers", "sgpu_dist_edge_index_merge", "sgpu_dist_edge_index_advance", "sgpu_dist_edge_index_level_done",
    "sgpu_dist_edge_index_ranks", "sgpu_dist_edge_index_fill", "sgpu_dist_edge_index_values", "sgpu_dist_edge_index_k", "sgpu_dist_edge_index_size",
    "sgpu_dist_edge_index_slot_range", "sgpu_dist_edge_index_serialized_size", "sgpu_dist_edge_index_serialize", "sgpu_dist_edge_index_lookup",
    "sgpu_dist_edge_index_times", "sgpu_dist_edge_index_free", "sgpu_dist_edge_numbers_host", "sgpu_edge_index_vertex_prefix_host",
    "sgpu_dist_slot_range_host",
    "sgpu_selftest",
    "sgpu_graph_fastg", "sgpu_graph_write_fastg", "sgpu_graph_unitigs_fasta", "sgpu_graph_write_unitigs_fasta", "sgpu_graph_format_stats",
    "sgpu_format_coverage",
]


class SgpuConfig(C.Structure):
    _fields_ = [("device", C.c_int), ("hbm_budget_bytes", C.c_uint64), ("verbose", C.c_int), ("stream", C.c_uint64)]


class SgpuGraphOptions(C.Structure):
    _fields_ = [("keep_perfect_loops", C.c_int), ("early_tip_length_bound", C.c_uint64), ("early_at_clipper", C.c_int), ("at_ratio", C.c_double),
                ("at_min_length", C.c_uint64), ("at_max_length", C.c_uint64)]


class SgpuTimes(C.Structure):
    _fields_ = [("extract_count_ms", C.c_float), ("extract_scatter_ms", C.c_float), ("refine_ms", C.c_float),
                ("local_sort_ms", C.c_float), ("compact_ms", C.c_float), ("mphf_ms", C.c_float), ("exchange_ms", C.c_float),
                ("instances", C.c_uint64), ("passes", C.c_uint64), ("launches", C.c_uint64), ("peak_bytes", C.c_uint64), ("cached_bytes", C.c_uint64),
                ("level_a_key_bits", C.c_uint64), ("level_a_scatters", C.c_uint64), ("refine_rounds_max", C.c_uint64),
                ("refine_splits_round0", C.c_uint64), ("refine_splits_later", C.c_uint64), ("sort_lsd_fallbacks", C.c_uint64),
                ("sort_oversize_equal", C.c_uint64), ("result_d2h_bytes", C.c_uint64), ("result_d2h_wait_ms", C.c_float),
                ("stage_h2d_bytes", C.c_uint64), ("graph_junction_batches", C.c_uint64),
                ("cov_filter_passes", C.c_uint64), ("cov_filter_table_bytes", C.c_uint64)]


class SgpuFormatStats(C.Structure):
    _fields_ = [("runs", C.c_uint64), ("records", C.c_uint64), ("bytes", C.c_uint64), ("format_ms", C.c_float), ("d2h_ms", C.c_float),
                ("write_ms", C.c_float), ("vertices_ms", C.c_float), ("sizes_ms", C.c_float)]


_lib = None


def load():
    """Load the CUDA library; raises if it has not been built (run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: the CUDA extension was not built; there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, i64, i32, u64 = C.c_void_p, C.c_int64, C.c_int, C.c_uint64
    pp = C.POINTER(vp)
    L.sgpu_create.restype = i32; L.sgpu_create.argtypes = [C.POINTER(SgpuConfig), pp]
    L.sgpu_destroy.restype = None; L.sgpu_destroy.argtypes = [vp]
    L.sgpu_last_error.restype = C.c_char_p; L.sgpu_last_error.argtypes = [vp]
    L.sgpu_get_times.restype = i32; L.sgpu_get_times.argtypes = [vp, C.POINTER(SgpuTimes)]
    L.sgpu_reads_clear.restype = i32; L.sgpu_reads_clear.argtypes = [vp]
    L.sgpu_reads_append_packed.restype = i32; L.sgpu_reads_append_packed.argtypes = [vp, vp, u64, vp, vp, i64]
    L.sgpu_reads_upload.restype = i32; L.sgpu_reads_upload.argtypes = [vp, vp, u64, vp, vp, i64]
    L.sgpu_reads_pack_text.restype = i32; L.sgpu_reads_pack_text.argtypes = [vp, vp, u64, vp, vp, i64, i32]
    L.sgpu_reads_info.restype = i32; L.sgpu_reads_info.argtypes = [vp, C.POINTER(i64), C.POINTER(u64)]
    L.sgpu_reads_download.restype = i32; L.sgpu_reads_download.argtypes = [vp, vp, vp, vp]
    L.sgpu_reads_cov_filter.restype = i32; L.sgpu_reads_cov_filter.argtypes = [vp, i32, C.c_uint, i32, vp, vp]
    L.sgpu_reads_cov_filter_ex.restype = i32; L.sgpu_reads_cov_filter_ex.argtypes = [vp, i32, C.c_uint, i32, i32, vp, vp]
    L.sgpu_cov_pass_plan_host.restype = i32; L.sgpu_cov_pass_plan_host.argtypes = [u64, i64, u64, C.POINTER(i32), C.POINTER(u64)]
    L.sgpu_text_index_fastx.restype = i64; L.sgpu_text_index_fastx.argtypes = [vp, u64, vp, vp, i64]
    L.sgpu_reads_adopt_device.restype = i32; L.sgpu_reads_adopt_device.argtypes = [vp, vp, u64, vp, vp, i64]
    L.sgpu_fastx_parse.restype = i32; L.sgpu_fastx_parse.argtypes = [C.c_char_p, i32, pp]
    L.sgpu_fastx_parse_threads.restype = i32; L.sgpu_fastx_parse_threads.argtypes = [C.c_char_p, i32, i32, pp]
    L.sgpu_seqfile_parse.restype = i32; L.sgpu_seqfile_parse.argtypes = [C.c_char_p, pp]
    L.sgpu_read_batch_write_seqfile.restype = i32; L.sgpu_read_batch_write_seqfile.argtypes = [vp, C.c_char_p]
    L.sgpu_read_batch_num_reads.restype = i64; L.sgpu_read_batch_num_reads.argtypes = [vp]
    L.sgpu_read_batch_num_words.restype = u64; L.sgpu_read_batch_num_words.argtypes = [vp]
    L.sgpu_read_batch_words.restype = vp; L.sgpu_read_batch_words.argtypes = [vp]
    L.sgpu_read_batch_offs.restype = vp; L.sgpu_read_batch_offs.argtypes = [vp]
    L.sgpu_read_batch_lens.restype = vp; L.sgpu_read_batch_lens.argtypes = [vp]
    L.sgpu_read_batch_stats.restype = i32; L.sgpu_read_batch_stats.argtypes = [vp, vp]
    L.sgpu_read_batch_error.restype = C.c_char_p; L.sgpu_read_batch_error.argtypes = [vp]
    L.sgpu_read_batch_free.restype = None; L.sgpu_read_batch_free.argtypes = [vp]
    L.sgpu_reads_append_batch.restype = i32; L.sgpu_reads_append_batch.argtypes = [vp, vp]
    L.sgpu_count.restype = i32; L.sgpu_count.argtypes = [vp, i32, i32, i32, pp]
    L.sgpu_kmers_from_kpomers.restype = i32; L.sgpu_kmers_from_kpomers.argtypes = [vp, vp, i32, pp]
    L.sgpu_kmers_from_kpomers_ex.restype = i32; L.sgpu_kmers_from_kpomers_ex.argtypes = [vp, vp, i32, i32, pp]
    L.sgpu_kset_size.restype = i64; L.sgpu_kset_size.argtypes = [vp]
    L.sgpu_kset_k.restype = i32; L.sgpu_kset_k.argtypes = [vp]
    L.sgpu_kset_num_buckets.restype = i32; L.sgpu_kset_num_buckets.argtypes = [vp]
    L.sgpu_kset_record_bytes.restype = i32; L.sgpu_kset_record_bytes.argtypes = [vp]
    L.sgpu_kset_on_host.restype = i32; L.sgpu_kset_on_host.argtypes = [vp]
    L.sgpu_kset_bucket_sizes.restype = i32; L.sgpu_kset_bucket_sizes.argtypes = [vp, vp]
    L.sgpu_kset_checksum.restype = i32; L.sgpu_kset_checksum.argtypes = [vp, vp]
    L.sgpu_kset_download_keys.restype = i32; L.sgpu_kset_download_keys.argtypes = [vp, i64, i64, vp]
    L.sgpu_kset_download_counts.restype = i32; L.sgpu_kset_download_counts.argtypes = [vp, i64, i64, vp]
    L.sgpu_kset_write_buckets.restype = i32; L.sgpu_kset_write_buckets.argtypes = [vp, C.c_char_p]
    L.sgpu_kset_owned_buckets.restype = i32; L.sgpu_kset_owned_buckets.argtypes = [vp, vp]
    L.sgpu_kset_write_owned_buckets.restype = i32; L.sgpu_kset_write_owned_buckets.argtypes = [vp, C.c_char_p]
    L.sgpu_kset_write_final.restype = i32; L.sgpu_kset_write_final.argtypes = [vp, C.c_char_p]
    L.sgpu_kset_free.restype = None; L.sgpu_kset_free.argtypes = [vp]
    L.sgpu_mphf_build.restype = i32; L.sgpu_mphf_build.argtypes = [vp, vp, pp]
    L.sgpu_mphf_serialized_size.restype = i64; L.sgpu_mphf_serialized_size.argtypes = [vp]
    L.sgpu_mphf_serialize.restype = i32; L.sgpu_mphf_serialize.argtypes = [vp, vp, i64]
    L.sgpu_mphf_serialized_size_buckets.restype = i64; L.sgpu_mphf_serialized_size_buckets.argtypes = [vp, i32, i32]
    L.sgpu_mphf_serialize_buckets.restype = i32; L.sgpu_mphf_serialize_buckets.argtypes = [vp, i32, i32, vp, i64]
    L.sgpu_mphf_lookup.restype = i32; L.sgpu_mphf_lookup.argtypes = [vp, vp, i64, vp]
    L.sgpu_mphf_free.restype = None; L.sgpu_mphf_free.argtypes = [vp]
    L.sgpu_graph_build.restype = i32; L.sgpu_graph_build.argtypes = [vp, vp, vp, vp, vp, i32, pp]
    L.sgpu_graph_build_ex.restype = i32; L.sgpu_graph_build_ex.argtypes = [vp, vp, vp, vp, vp, i32, u64, pp]
    L.sgpu_graph_build_opts.restype = i32; L.sgpu_graph_build_opts.argtypes = [vp, vp, vp, vp, vp, C.POINTER(SgpuGraphOptions), pp]
    L.sgpu_graph_build_streamed.restype = i32; L.sgpu_graph_build_streamed.argtypes = [vp, vp, vp, vp, vp, C.POINTER(SgpuGraphOptions), pp]
    L.sgpu_graph_at_clipper_stats.restype = i32; L.sgpu_graph_at_clipper_stats.argtypes = [vp, vp]
    L.sgpu_graph_tip_clipper_stats.restype = i32; L.sgpu_graph_tip_clipper_stats.argtypes = [vp, vp]
    L.sgpu_graph_masks.restype = i32; L.sgpu_graph_masks.argtypes = [vp, vp, i64]
    L.sgpu_graph_coverage.restype = i32; L.sgpu_graph_coverage.argtypes = [vp, vp, i64]
    L.sgpu_graph_histogram.restype = i64; L.sgpu_graph_histogram.argtypes = [vp, vp, i64]
    L.sgpu_graph_num_unitigs.restype = i64; L.sgpu_graph_num_unitigs.argtypes = [vp]
    L.sgpu_graph_unitig_bases.restype = i64; L.sgpu_graph_unitig_bases.argtypes = [vp]
    L.sgpu_graph_unitigs.restype = i32; L.sgpu_graph_unitigs.argtypes = [vp, vp, vp]
    L.sgpu_graph_gfa.restype = i64; L.sgpu_graph_gfa.argtypes = [vp, C.c_char_p, vp, i64]
    L.sgpu_graph_write_gfa.restype = i32; L.sgpu_graph_write_gfa.argtypes = [vp, C.c_char_p, C.c_char_p]
    L.sgpu_graph_fastg.restype = i64; L.sgpu_graph_fastg.argtypes = [vp, vp, vp, i64]
    L.sgpu_graph_write_fastg.restype = i32; L.sgpu_graph_write_fastg.argtypes = [vp, vp, C.c_char_p]
    L.sgpu_graph_unitigs_fasta.restype = i64; L.sgpu_graph_unitigs_fasta.argtypes = [vp, vp, vp, i64]
    L.sgpu_graph_write_unitigs_fasta.restype = i32; L.sgpu_graph_write_unitigs_fasta.argtypes = [vp, vp, C.c_char_p]
    L.sgpu_graph_format_stats.restype = i32; L.sgpu_graph_format_stats.argtypes = [vp, C.POINTER(SgpuFormatStats)]
    L.sgpu_format_coverage.restype = i32; L.sgpu_format_coverage.argtypes = [vp, i32, vp, vp, i64, vp]
    L.sgpu_graph_free.restype = None; L.sgpu_graph_free.argtypes = [vp]
    L.sgpu_edge_index_build.restype = i32; L.sgpu_edge_index_build.argtypes = [vp, vp, i32, i32, pp]
    L.sgpu_edge_index_k.restype = i32; L.sgpu_edge_index_k.argtypes = [vp]
    L.sgpu_edge_index_size.restype = i64; L.sgpu_edge_index_size.argtypes = [vp]
    L.sgpu_edge_index_serialized_size.restype = i64; L.sgpu_edge_index_serialized_size.argtypes = [vp]
    L.sgpu_edge_index_serialize.restype = i32; L.sgpu_edge_index_serialize.argtypes = [vp, vp, i64]
    L.sgpu_edge_index_values.restype = i32; L.sgpu_edge_index_values.argtypes = [vp, vp, vp, i64]
    L.sgpu_edge_index_lookup.restype = i32; L.sgpu_edge_index_lookup.argtypes = [vp, vp, i64, vp]
    L.sgpu_edge_index_free.restype = None; L.sgpu_edge_index_free.argtypes = [vp]
    L.sgpu_dist_begin.restype = i32; L.sgpu_dist_begin.argtypes = [vp, i32, i32, i32, i32, i32, pp]
    L.sgpu_dist_begin_kpomers.restype = i32; L.sgpu_dist_begin_kpomers.argtypes = [vp, vp, i32, i32, i32, i32, pp]
    L.sgpu_dist_num_partitions.restype = i64; L.sgpu_dist_num_partitions.argtypes = [vp]
    L.sgpu_dist_local_counts.restype = i32; L.sgpu_dist_local_counts.argtypes = [vp, vp]
    L.sgpu_dist_plan.restype = i32; L.sgpu_dist_plan.argtypes = [vp, vp, C.POINTER(u64)]
    L.sgpu_dist_free_bytes.restype = i32; L.sgpu_dist_free_bytes.argtypes = [vp, C.POINTER(u64)]
    L.sgpu_dist_next_pass.restype = i32; L.sgpu_dist_next_pass.argtypes = [vp, u64, C.POINTER(i32)]
    L.sgpu_dist_ipc_handle.restype = i32; L.sgpu_dist_ipc_handle.argtypes = [vp, vp]
    L.sgpu_dist_open_peers.restype = i32; L.sgpu_dist_open_peers.argtypes = [vp, vp]
    L.sgpu_dist_scatter.restype = i32; L.sgpu_dist_scatter.argtypes = [vp, i32]
    L.sgpu_dist_exchange.restype = i32; L.sgpu_dist_exchange.argtypes = [vp, i32]
    L.sgpu_dist_sort.restype = i32; L.sgpu_dist_sort.argtypes = [vp, i32]
    L.sgpu_dist_end.restype = i32; L.sgpu_dist_end.argtypes = [vp, pp]
    L.sgpu_dist_free.restype = None; L.sgpu_dist_free.argtypes = [vp]
    L.sgpu_dist_plan_host.restype = i32; L.sgpu_dist_plan_host.argtypes = [i32, i32, i32, vp, u64, i32, vp, C.POINTER(u64)]
    L.sgpu_dist_cov_begin.restype = i32; L.sgpu_dist_cov_begin.argtypes = [vp, i32, C.c_uint, i32, i32, pp]
    L.sgpu_dist_cov_ipc_handle.restype = i32; L.sgpu_dist_cov_ipc_handle.argtypes = [vp, vp]
    L.sgpu_dist_cov_open_peers.restype = i32; L.sgpu_dist_cov_open_peers.argtypes = [vp, vp]
    L.sgpu_dist_cov_bound.restype = i32; L.sgpu_dist_cov_bound.argtypes = [vp]
    L.sgpu_dist_cov_fill.restype = i32; L.sgpu_dist_cov_fill.argtypes = [vp]
    L.sgpu_dist_cov_filter.restype = i32; L.sgpu_dist_cov_filter.argtypes = [vp, i32, vp, vp]
    L.sgpu_dist_cov_free.restype = None; L.sgpu_dist_cov_free.argtypes = [vp]
    L.sgpu_dist_cov_layout_host.restype = i32; L.sgpu_dist_cov_layout_host.argtypes = [i32, u64, vp, i64, vp, C.POINTER(u64)]
    L.sgpu_dist_ext_begin.restype = i32; L.sgpu_dist_ext_begin.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, pp]
    L.sgpu_dist_ext_local_counts.restype = i32; L.sgpu_dist_ext_local_counts.argtypes = [vp, vp]
    L.sgpu_dist_ext_plan.restype = i32; L.sgpu_dist_ext_plan.argtypes = [vp, vp, C.POINTER(u64)]
    L.sgpu_dist_ext_free_bytes.restype = i32; L.sgpu_dist_ext_free_bytes.argtypes = [vp, C.POINTER(u64)]
    L.sgpu_dist_ext_next_pass.restype = i32; L.sgpu_dist_ext_next_pass.argtypes = [vp, u64, C.POINTER(i32)]
    L.sgpu_dist_ext_ipc_handle.restype = i32; L.sgpu_dist_ext_ipc_handle.argtypes = [vp, vp]
    L.sgpu_dist_ext_open_peers.restype = i32; L.sgpu_dist_ext_open_peers.argtypes = [vp, vp]
    L.sgpu_dist_ext_scatter.restype = i32; L.sgpu_dist_ext_scatter.argtypes = [vp, i32]
    L.sgpu_dist_ext_apply.restype = i32; L.sgpu_dist_ext_apply.argtypes = [vp, i32]
    L.sgpu_dist_ext_masks.restype = i32; L.sgpu_dist_ext_masks.argtypes = [vp, vp, i64]
    L.sgpu_dist_ext_coverage.restype = i32; L.sgpu_dist_ext_coverage.argtypes = [vp, vp, i64]
    L.sgpu_dist_ext_histogram.restype = i64; L.sgpu_dist_ext_histogram.argtypes = [vp, vp, i64]
    L.sgpu_dist_ext_times.restype = i32; L.sgpu_dist_ext_times.argtypes = [vp, vp]
    L.sgpu_dist_ext_free.restype = None; L.sgpu_dist_ext_free.argtypes = [vp]
    L.sgpu_dist_ext_plan_host.restype = i32; L.sgpu_dist_ext_plan_host.argtypes = [i32, i32, vp, vp, u64, i32, vp, C.POINTER(u64)]
    L.sgpu_dist_graph_begin.restype = i32; L.sgpu_dist_graph_begin.argtypes = [vp, vp, vp, vp, vp, u64, pp]
    L.sgpu_dist_graph_begin_opts.restype = i32; L.sgpu_dist_graph_begin_opts.argtypes = [vp, vp, vp, vp, vp, u64, C.POINTER(SgpuGraphOptions), pp]
    for name in ("at_edges_probe", "at_edges_apply", "at_tips_probe", "tip_probe", "isolate", "unlink", "junctions"):
        f = getattr(L, "sgpu_dist_graph_" + name)
        f.restype = i32; f.argtypes = [vp]
    L.sgpu_dist_graph_masks.restype = i32; L.sgpu_dist_graph_masks.argtypes = [vp, vp, i64]
    L.sgpu_dist_graph_clipper_stats.restype = i32; L.sgpu_dist_graph_clipper_stats.argtypes = [vp, vp, vp, vp]
    L.sgpu_dist_graph_clipper_times.restype = i32; L.sgpu_dist_graph_clipper_times.argtypes = [vp, vp]
    L.sgpu_dist_graph_ipc_handle.restype = i32; L.sgpu_dist_graph_ipc_handle.argtypes = [vp, vp]
    L.sgpu_dist_graph_open_peers.restype = i32; L.sgpu_dist_graph_open_peers.argtypes = [vp, vp]
    L.sgpu_dist_graph_unitigs.restype = i32; L.sgpu_dist_graph_unitigs.argtypes = [vp]
    L.sgpu_dist_graph_clear_visited.restype = i32; L.sgpu_dist_graph_clear_visited.argtypes = [vp]
    L.sgpu_dist_graph_loops.restype = i32; L.sgpu_dist_graph_loops.argtypes = [vp]
    L.sgpu_dist_graph_stats.restype = i32; L.sgpu_dist_graph_stats.argtypes = [vp, vp]
    L.sgpu_dist_graph_edges.restype = i32; L.sgpu_dist_graph_edges.argtypes = [vp, vp, vp, vp, vp, vp]
    L.sgpu_dist_graph_bucket_counts.restype = i32; L.sgpu_dist_graph_bucket_counts.argtypes = [vp, vp, vp]
    L.sgpu_dist_graph_times.restype = i32; L.sgpu_dist_graph_times.argtypes = [vp, vp]
    L.sgpu_dist_graph_free.restype = None; L.sgpu_dist_graph_free.argtypes = [vp]
    L.sgpu_dist_edge_index_begin.restype = i32; L.sgpu_dist_edge_index_begin.argtypes = [vp, vp, i32, i32, vp, vp, pp]
    L.sgpu_dist_edge_index_count_begin.restype = i32; L.sgpu_dist_edge_index_count_begin.argtypes = [vp, i32, i32, pp]
    L.sgpu_dist_edge_index_keys.restype = i32; L.sgpu_dist_edge_index_keys.argtypes = [vp, vp, vp, i32]
    for name in ("ipc_handle", "open_peers", "advance", "times"):
        f = getattr(L, "sgpu_dist_edge_index_" + name)
        f.restype = i32; f.argtypes = [vp, vp]
    for name in ("merge", "ranks", "fill"):
        f = getattr(L, "sgpu_dist_edge_index_" + name)
        f.restype = i32; f.argtypes = [vp]
    L.sgpu_dist_edge_index_level_done.restype = i32; L.sgpu_dist_edge_index_level_done.argtypes = [vp, u64, vp]
    L.sgpu_dist_edge_index_values.restype = i32; L.sgpu_dist_edge_index_values.argtypes = [vp, vp, vp, i64]
    L.sgpu_dist_edge_index_k.restype = i32; L.sgpu_dist_edge_index_k.argtypes = [vp]
    L.sgpu_dist_edge_index_size.restype = i64; L.sgpu_dist_edge_index_size.argtypes = [vp]
    L.sgpu_dist_edge_index_slot_range.restype = i32; L.sgpu_dist_edge_index_slot_range.argtypes = [vp, vp, vp]
    L.sgpu_dist_edge_index_serialized_size.restype = i64; L.sgpu_dist_edge_index_serialized_size.argtypes = [vp]
    L.sgpu_dist_edge_index_serialize.restype = i32; L.sgpu_dist_edge_index_serialize.argtypes = [vp, vp, i64]
    L.sgpu_dist_edge_index_lookup.restype = i32; L.sgpu_dist_edge_index_lookup.argtypes = [vp, vp, i64, vp]
    L.sgpu_dist_edge_index_free.restype = None; L.sgpu_dist_edge_index_free.argtypes = [vp]
    L.sgpu_dist_edge_numbers_host.restype = i32; L.sgpu_dist_edge_numbers_host.argtypes = [i32, i32, i32, vp, vp, vp, u64, u64, vp]
    L.sgpu_edge_index_vertex_prefix_host.restype = i64; L.sgpu_edge_index_vertex_prefix_host.argtypes = [vp, vp, i64, i32, vp]
    L.sgpu_dist_slot_range_host.restype = i32; L.sgpu_dist_slot_range_host.argtypes = [u64, i32, i32, vp, vp]
    L.sgpu_graph_from_edges.restype = i32; L.sgpu_graph_from_edges.argtypes = [i32, vp, i64, vp, vp, vp, vp, i64, pp]
    L.sgpu_selftest.restype = i32; L.sgpu_selftest.argtypes = [vp, i32, i32, i32, u64, vp, i64, vp]
    _lib = L
    return L
