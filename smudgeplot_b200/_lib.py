"""ctypes binding of libhetmers_b200.so (include/hetmers_b200.h).  The library is built in-tree by
`make lib` / `__graft_entry__.build()`; if it is missing this module raises -- there is no CPU or
PyTorch fallback for the hetmers path."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HETMERS_LIB") or os.path.join(HERE, "lib", "libhetmers_b200.so")   # (override: tuning builds)
BIN_PATH = os.path.join(HERE, "bin", "hetmers")

SMAX, FMAX = 1000, 500
PLOT_W = FMAX + 1
PLOT_CELLS = (SMAX + 1) * (FMAX + 1)

# every symbol include/hetmers_b200.h declares (tests check the .so exports all of them)
ABI_SYMBOLS = [
    "hm_last_error", "hm_abi_version", "hm_device_count", "hm_device_info",
    "hm_k_unpack_records", "hm_k_build_bucket_index", "hm_k_pass1_degree", "hm_k_pass2_plot",
    "hm_k_min_count", "hm_k_find_keys", "hm_pick_bucket_bits", "hm_k_pass2_extract", "hm_scan_extract", "hm_pass2_scratch_bytes",
    "hm_k_build_filter", "hm_filter_words", "hm_pick_filter_bits",
    "hm_dev_alloc", "hm_dev_free", "hm_ipc_export", "hm_ipc_open", "hm_ipc_close", "hm_p2p_native_atomics",
    "hm_scan_create", "hm_prewarm", "hm_set_io_threads", "hm_scan_destroy", "hm_scan_examine", "hm_scan_condition", "hm_scan_run", "hm_hetmers_host",
    "hm_scan_run_path", "hm_scan_is_symmetric", "hm_symm_plan", "hm_symm_seeds", "hm_k_symm_fingerprint", "hm_k_symm_runscan", "hm_k_symm_runs", "hm_k_symm_resolve",
    "hm_k_symm_extract",
    "hm_symm_status", "hm_symm_align_cut",
    "hm_scan_download", "hm_set_device_budget", "hm_stream_plan", "hm_stream_plan_shards", "hm_scan_residency", "hm_table_open", "hm_table_close", "hm_table_view", "hm_write_smu",
    "hm_rank_scan_create", "hm_rank_scan_create_share", "hm_rank_scan_destroy", "hm_rank_scan_cuts", "hm_rank_scan_pass1", "hm_rank_scan_bloom",
    "hm_rank_scan_prepare", "hm_rank_scan_slices", "hm_rank_scan_route", "hm_rank_scan_answer", "hm_rank_scan_settle",
    "hm_rank_scan_result", "hm_rank_scan_residency",
    "hm_rank_scan_extract_prepare", "hm_rank_scan_extract_slices", "hm_rank_scan_extract_route",
    "hm_rank_scan_extract_settle", "hm_rank_scan_extract_result", "hm_sort_pair_records",
    "hm_condition_range_bytes", "hm_condition_plan", "hm_scan_condition_files",
    "hm_table_write_open", "hm_table_write_buckets", "hm_table_write_append", "hm_table_write_close",
    "hm_table_write_abort", "hm_table_write_place", "hm_table_write_at", "hm_table_write_seal",
    "hm_set_condition_gpus", "hm_scan_condition_host", "hm_table_write_open_host", "hm_table_write_close_host",
    "hm_host_table_free", "hm_scan_create_streamed",
    "hm_k_cond_hist", "hm_k_shard_route_count", "hm_k_shard_route_scatter", "hm_k_shard_settle_bytes",
    "hm_k_shard_settle", "hm_shard_condition_bytes",
    "hm_k_shard_route_count_window", "hm_k_shard_route_scatter_window", "hm_k_cond_pack", "hm_rank_condition_bytes",
    "hm_rank_condition_cut",
    "hm_rank_scan_extract_records", "hm_k_pairs_hist", "hm_k_pairs_route_count", "hm_k_pairs_route_scatter",
    "hm_pairs_sort_scratch_bytes", "hm_k_pairs_sort", "hm_k_pairs_label_bounds", "hm_k_pairs_format", "hm_pairs_bytes",
    "hm_scan_write_pairs", "hm_scan_pairs_hist", "hm_pair_windows",
    "hm_set_list_host_budget", "hm_scan_spill_stats", "hm_spill_plan",
    "hm_rank_scan_set_list_host_budget", "hm_rank_scan_host_lists", "hm_rank_scan_spill_stats", "hm_rank_spill_plan",
]


class HostTable(C.Structure):
    _fields_ = [("kmer", C.c_int32), ("ibyte", C.c_int32), ("nparts", C.c_int32), ("minval", C.c_int32),
                ("nels", C.c_int64), ("index", C.POINTER(C.c_int64)), ("part_nels", C.POINTER(C.c_int64)),
                ("part_rec", C.POINTER(C.c_void_p)), ("part_fd", C.POINTER(C.c_int32)),
                ("part_fd_off", C.POINTER(C.c_int64))]


MAX_SHARDS = 16


class Shards(C.Structure):
    """hm_shards: shard offsets + every owner's full-length incidence array as seen from this GPU"""
    _fields_ = [("n_shards", C.c_int32), ("self_", C.c_int32), ("off", C.c_int64 * (MAX_SHARDS + 1)),
                ("deg", C.c_void_p * MAX_SHARDS), ("scratch", C.c_void_p), ("scratch_bytes", C.c_int64)]


class SymmLayout(C.Structure):
    """hm_symm_layout: work area of the strand-symmetric scan"""
    _fields_ = [("bytes", C.c_int64), ("off_header", C.c_int64), ("off_bloom", C.c_int64), ("seg_words", C.c_int64),
                ("off_cand_key", C.c_int64), ("off_cand_lo", C.c_int64), ("off_cand_meta", C.c_int64),
                ("cand_cap", C.c_int64), ("range", C.c_int64), ("off_runs", C.c_int64), ("runs_cap", C.c_int64),
                ("n_seg", C.c_int32), ("pad", C.c_int32)]


class SymmShards(C.Structure):
    """hm_symm_shards: run-aligned shard cuts + the first key of every shard"""
    _fields_ = [("n_seg", C.c_int32), ("self_", C.c_int32), ("off", C.c_int64 * (MAX_SHARDS + 1)),
                ("first_key", C.c_uint64 * MAX_SHARDS)]


SYMM_ASYMMETRIC, SYMM_OVERFLOW = 1, 2


class StreamLayout(C.Structure):
    """hm_stream_layout: what the streamed scan plans for a table under a device budget"""
    _fields_ = [("budget", C.c_int64), ("chunk", C.c_int64), ("fixed_bytes", C.c_int64), ("chunk_bytes", C.c_int64),
                ("list_bytes", C.c_int64), ("chunk_list_bytes", C.c_int64)]


class SpillStats(C.Structure):
    """hm_spill_stats: what the last streamed run did with its lists (host memory when spilled)"""
    _fields_ = [("spilled", C.c_int32), ("pad", C.c_int32), ("flushes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("host_peak_bytes", C.c_int64), ("partitions", C.c_int64), ("rounds", C.c_int64),
                ("h2d_bytes", C.c_int64), ("slice", C.c_int64), ("part", C.c_int64),
                ("first_key_queries", C.c_int64), ("ms_pass1", C.c_double), ("ms_flush", C.c_double), ("ms_pass2", C.c_double)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "pad"}
        d["spilled"] = bool(d["spilled"])
        return d


class SpillLayout(C.Structure):
    """hm_spill_layout: pass 2's slices and S partitions for lists in host memory"""
    _fields_ = [("room", C.c_int64), ("slice", C.c_int64), ("queries", C.c_int64), ("part", C.c_int64),
                ("part_bits", C.c_int32), ("pad", C.c_int32), ("slice_bytes", C.c_int64), ("part_bytes", C.c_int64)]


SPILL_MIN, SPILL_SORT_Q, SPILL_SORT_FIXED = 1024, 32, 64 << 10
SPILL_MAX_SLICE, SPILL_MAX_PART = 0x3FFFFFF0, 0xFFFFFFEF   # 32-bit query indices; 32-bit partition bucket index

COND_HIST_BITS = 20
COND_MAX_GPUS = 16


class ConditionStats(C.Structure):
    """hm_condition_stats: what hm_scan_condition_files / hm_scan_condition_host did"""
    _fields_ = [("nels_in", C.c_int64), ("nels_out", C.c_int64), ("ranges", C.c_int32), ("passes", C.c_int32),
                ("peak_bytes", C.c_int64), ("bytes_read", C.c_int64), ("bytes_written", C.c_int64),
                ("ms_hist", C.c_double), ("ms_ranges", C.c_double), ("ms_write", C.c_double), ("ms_total", C.c_double),
                ("budget_bytes", C.c_int64), ("gpus", C.c_int32), ("pad", C.c_int32), ("ms_write_max", C.c_double),
                ("gpu_peak_bytes", C.c_int64 * COND_MAX_GPUS)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k not in ("pad", "gpu_peak_bytes")}
        d["gpu_peak_bytes"] = list(self.gpu_peak_bytes)[:max(self.gpus, 1)]
        return d


class ConditionLayout(C.Structure):
    """hm_condition_layout: what hm_condition_plan chooses for a table under a device budget"""
    _fields_ = [("budget", C.c_int64), ("chunk", C.c_int64), ("fixed_bytes", C.c_int64), ("range_room", C.c_int64),
                ("range_cap", C.c_int64), ("range_bytes", C.c_int64), ("n_ranges", C.c_int32), ("hist_bits", C.c_int32)]


BUDGET_RESERVE = 1 << 30
EXTRACT_MIN_BYTES = 2 * PLOT_CELLS + (1 << 16)   # HM_EXTRACT_MIN_BYTES: device room hm_scan_extract's symmetric route needs


class PairRec(C.Structure):
    """hm_pair_rec: one line of extract_kmer_pairs' output"""
    _fields_ = [("key_hi", C.c_uint64), ("key_lo", C.c_uint64), ("smudge", C.c_uint32),
                ("pos", C.c_uint8), ("alt", C.c_uint8), ("pad", C.c_uint16)]


class PairsStats(C.Structure):
    """hm_pairs_stats: what hm_scan_write_pairs did"""
    _fields_ = [("records", C.c_int64), ("passes", C.c_int64), ("windows", C.c_int64), ("room", C.c_int64),
                ("peak_bytes", C.c_int64), ("budget", C.c_int64), ("path", C.c_int32), ("planned", C.c_int32),
                ("ms_hist", C.c_double), ("ms_list", C.c_double), ("ms_sort", C.c_double), ("ms_format", C.c_double),
                ("ms_d2h", C.c_double), ("ms_write", C.c_double), ("ms_writer_busy", C.c_double),
                ("ms_total", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ScanStats(C.Structure):
    _fields_ = [("nels", C.c_int64), ("n_gpus", C.c_int32), ("bucket_bits", C.c_int32),
                ("filter_bits", C.c_int32), ("path", C.c_int32),
                ("ms_h2d_unpack", C.c_double), ("ms_pass1", C.c_double), ("ms_pass2", C.c_double),
                ("ms_scan", C.c_double), ("ms_total", C.c_double), ("kernel_launches", C.c_int64),
                ("ms_alloc", C.c_double), ("ms_records", C.c_double), ("ms_index", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class HetmersError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libhetmers_b200 error {code}: {msg}")
        self.code = code


_lib = None


def lib():
    """Load the shared library once; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `make lib` (or __graft_entry__.build()); "
                          "the hetmers path has no CPU / PyTorch fallback")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    L.hm_last_error.restype = C.c_char_p
    L.hm_device_info.argtypes = [i32, C.c_char_p, i32, C.POINTER(i32), C.POINTER(i64)]
    L.hm_k_unpack_records.argtypes = [vp, i64, i64, vp, i32, i32, vp, vp, vp, vp]
    L.hm_k_build_bucket_index.argtypes = [vp, i64, i32, vp, i32, vp]
    L.hm_k_pass1_degree.argtypes = [vp, vp, vp, i64, vp, i32, i32, vp, i32, i32, i64, i64, vp, vp, C.POINTER(Shards), vp]
    L.hm_dev_alloc.argtypes = [i64, C.POINTER(vp)]
    L.hm_dev_free.argtypes = [vp]
    L.hm_ipc_export.argtypes = [vp, C.c_char_p]
    L.hm_ipc_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.hm_ipc_close.argtypes = [vp]
    L.hm_p2p_native_atomics.argtypes = [i32, i32]
    L.hm_k_build_filter.argtypes = [vp, i64, i32, vp, vp]
    L.hm_filter_words.argtypes = [i32]
    L.hm_filter_words.restype = i64
    L.hm_pick_filter_bits.argtypes = [i64]
    L.hm_k_pass2_plot.argtypes = [vp, vp, vp, i32, i64, i64, vp, C.POINTER(Shards), vp]
    L.hm_k_pass2_extract.argtypes = [vp, vp, vp, vp, vp, i32, i64, i64, vp, vp, i64, vp, C.POINTER(Shards), vp]
    L.hm_k_min_count.argtypes = [vp, i64, i64, vp, vp]
    L.hm_k_find_keys.argtypes = [vp, vp, i64, vp, i32, i32, vp, vp, i64, vp, vp]
    L.hm_pick_bucket_bits.argtypes = [i64]
    L.hm_pass2_scratch_bytes.argtypes = [i64, i32]
    L.hm_pass2_scratch_bytes.restype = i64
    L.hm_symm_plan.argtypes = [i64, i64, i32, i32, C.POINTER(SymmLayout)]
    L.hm_symm_seeds.argtypes = [C.POINTER(C.c_uint64)]
    L.hm_symm_seeds.restype = None
    L.hm_k_symm_fingerprint.argtypes = [vp, vp, vp, i64, i64, i32, C.POINTER(C.c_uint64), vp, vp]
    L.hm_k_symm_runscan.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, i64, i64, vp, C.POINTER(SymmLayout),
                                    C.POINTER(SymmShards), vp]
    L.hm_k_symm_runs.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, i64, i64, vp, C.POINTER(SymmLayout),
                                 C.POINTER(SymmShards), vp]
    L.hm_k_symm_resolve.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, vp, C.POINTER(SymmLayout),
                                    C.POINTER(SymmShards), vp, vp]
    L.hm_k_symm_extract.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, vp, C.POINTER(SymmLayout),
                                    C.POINTER(SymmShards), vp, i64, i64, vp, i64, vp, vp]
    L.hm_symm_status.argtypes = [vp, C.POINTER(SymmLayout), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), vp]
    L.hm_symm_align_cut.argtypes = [vp, i64, i32, i64, C.POINTER(i64)]
    L.hm_scan_create.argtypes = [C.POINTER(HostTable), C.POINTER(i32), i32, C.POINTER(vp)]
    L.hm_scan_create_streamed.argtypes = L.hm_scan_create.argtypes
    L.hm_scan_destroy.argtypes = [vp]
    L.hm_scan_destroy.restype = None
    L.hm_scan_examine.argtypes = [vp, i32, C.POINTER(i32), C.POINTER(i32)]
    L.hm_scan_condition.argtypes = [vp, i32, i32, i32, C.POINTER(i64)]
    L.hm_scan_run.argtypes = [vp, vp, C.POINTER(ScanStats)]
    L.hm_scan_run_path.argtypes = [vp, i32, vp, C.POINTER(ScanStats)]
    L.hm_scan_is_symmetric.argtypes = [vp]
    L.hm_scan_extract.argtypes = [vp, vp, C.POINTER(C.POINTER(PairRec)), C.POINTER(i64)]
    L.hm_hetmers_host.argtypes = [C.POINTER(HostTable), C.POINTER(i32), i32, vp, C.POINTER(ScanStats)]
    L.hm_scan_download.argtypes = [vp, vp, vp, vp, vp]
    L.hm_set_device_budget.argtypes = [i64]
    L.hm_set_device_budget.restype = None
    L.hm_stream_plan.argtypes = [i64, i32, i32, i64, C.POINTER(StreamLayout)]
    L.hm_stream_plan_shards.argtypes = [i64, i32, i32, i64, i32, C.POINTER(StreamLayout)]
    L.hm_scan_residency.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.hm_set_list_host_budget.argtypes = [i64]
    L.hm_set_list_host_budget.restype = None
    L.hm_scan_spill_stats.argtypes = [vp, C.POINTER(SpillStats)]
    L.hm_spill_plan.argtypes = [i64, i64, i32, i64, C.POINTER(SpillLayout)]
    L.hm_rank_scan_set_list_host_budget.argtypes = [vp, i64]
    L.hm_rank_scan_host_lists.argtypes = [vp]
    L.hm_rank_scan_spill_stats.argtypes = [vp, C.POINTER(SpillStats)]
    L.hm_rank_spill_plan.argtypes = [i64, i64, i32, i32, i32, i64, C.POINTER(SpillLayout)]
    u64p, i64p = C.POINTER(C.c_uint64), C.POINTER(i64)
    L.hm_rank_scan_create.argtypes = [C.POINTER(HostTable), i32, i32, i32, u64p, C.POINTER(vp)]
    L.hm_rank_scan_create_share.argtypes = [C.POINTER(HostTable), i64, i64p, u64p, i32, i32, i32, u64p, C.POINTER(vp)]
    L.hm_rank_scan_destroy.argtypes = [vp]
    L.hm_rank_scan_destroy.restype = None
    L.hm_rank_scan_cuts.argtypes = [vp, i64p, u64p]
    L.hm_rank_scan_pass1.argtypes = [vp, u64p]
    L.hm_rank_scan_bloom.argtypes = [vp, C.POINTER(vp), i64p]
    L.hm_rank_scan_prepare.argtypes = [vp, i32, i64p, i64p]
    L.hm_rank_scan_slices.argtypes = [vp, i64, i64p, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.hm_rank_scan_route.argtypes = [vp, i64, i64p]
    L.hm_rank_scan_answer.argtypes = [vp, i64]
    L.hm_rank_scan_settle.argtypes = [vp]
    L.hm_rank_scan_result.argtypes = [vp, C.POINTER(vp), u64p]
    L.hm_rank_scan_residency.argtypes = [vp, i64p, i64p, i64p]
    L.hm_rank_scan_extract_prepare.argtypes = [vp, vp, i64p, i64p]
    L.hm_rank_scan_extract_slices.argtypes = L.hm_rank_scan_slices.argtypes
    L.hm_rank_scan_extract_route.argtypes = [vp, i64, i64p]
    L.hm_rank_scan_extract_settle.argtypes = [vp]
    L.hm_rank_scan_extract_result.argtypes = [vp, C.POINTER(C.POINTER(PairRec)), i64p, u64p]
    L.hm_sort_pair_records.argtypes = [vp, i64]
    L.hm_table_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.hm_table_close.argtypes = [vp]
    L.hm_table_close.restype = None
    L.hm_table_view.argtypes = [vp]
    L.hm_table_view.restype = C.POINTER(HostTable)
    L.hm_write_smu.argtypes = [C.c_char_p, vp]
    L.hm_condition_range_bytes.argtypes = [i64, i32, i32, i32]
    L.hm_condition_range_bytes.restype = i64
    L.hm_condition_plan.argtypes = [i64, i32, i32, i64, i32, vp, i32, vp, C.POINTER(ConditionLayout)]
    L.hm_scan_condition_files.argtypes = [vp, i32, i32, i32, C.c_char_p, C.POINTER(ConditionStats)]
    L.hm_table_write_open.argtypes = [C.c_char_p, i32, i32, i32, i32, i64, C.POINTER(vp)]
    L.hm_table_write_buckets.argtypes = [vp, i64, i64, vp]
    L.hm_table_write_append.argtypes = [vp, vp, i64]
    L.hm_table_write_close.argtypes = [vp]
    L.hm_table_write_abort.argtypes = [vp]
    L.hm_table_write_abort.restype = None
    L.hm_table_write_place.argtypes = [vp, i64, i64, vp, C.POINTER(i64)]
    L.hm_table_write_at.argtypes = [vp, i64, vp, i64]
    L.hm_table_write_seal.argtypes = [vp]
    L.hm_table_write_seal.restype = None
    L.hm_set_condition_gpus.argtypes = [i32]
    L.hm_scan_condition_host.argtypes = [vp, i32, i32, i32, i64, C.POINTER(C.POINTER(HostTable)),
                                         C.POINTER(ConditionStats)]
    L.hm_table_write_open_host.argtypes = [i32, i32, i32, i64, C.POINTER(vp)]
    L.hm_table_write_close_host.argtypes = [vp, C.POINTER(C.POINTER(HostTable))]
    L.hm_host_table_free.argtypes = [C.POINTER(HostTable)]
    L.hm_host_table_free.restype = None
    L.hm_k_cond_hist.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp, vp]
    L.hm_k_shard_route_count.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp, i32, vp, vp, vp]
    L.hm_k_shard_route_scatter.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp, vp, vp, vp, vp, i64, i64, vp, vp, vp]
    L.hm_k_shard_settle_bytes.argtypes = [i32, i64, i64]
    L.hm_k_shard_settle_bytes.restype = i64
    L.hm_k_shard_settle.argtypes = [i32, vp, vp, vp, i64, i64, vp, i64, vp, vp, vp, C.POINTER(i64), vp]
    L.hm_shard_condition_bytes.argtypes = [i32, i32, i32, i64, i64, i64, i64, i64, i32]
    L.hm_shard_condition_bytes.restype = i64
    L.hm_k_shard_route_count_window.argtypes = L.hm_k_shard_route_count.argtypes
    L.hm_k_shard_route_scatter_window.argtypes = L.hm_k_shard_route_scatter.argtypes
    L.hm_k_cond_pack.argtypes = [i32, i32, vp, vp, vp, i64, i64, i64, vp, vp, vp]
    L.hm_rank_condition_bytes.argtypes = [i32, i32, i32, i64, i64, i64, i64, i32]
    L.hm_rank_condition_bytes.restype = i64
    L.hm_rank_condition_cut.argtypes = [i32, i32, i32, i64, i32, i64, vp, i64, vp, C.POINTER(i64)]
    L.hm_rank_scan_extract_records.argtypes = L.hm_rank_scan_extract_result.argtypes
    L.hm_k_pairs_hist.argtypes = [vp, i64, i32, vp, vp]
    L.hm_k_pairs_route_count.argtypes = [vp, i64, i32, vp, i32, vp, vp]
    L.hm_k_pairs_route_scatter.argtypes = [vp, i64, i32, vp, i32, vp, vp, i64, vp, vp]
    L.hm_pairs_sort_scratch_bytes.argtypes = [i64]
    L.hm_pairs_sort_scratch_bytes.restype = i64
    L.hm_k_pairs_sort.argtypes = [vp, vp, i64, vp, i64, C.POINTER(i32), vp]
    L.hm_k_pairs_label_bounds.argtypes = [vp, i64, i32, vp, vp]
    L.hm_k_pairs_format.argtypes = [vp, i64, i32, vp, vp]
    L.hm_pairs_bytes.argtypes = [i32, i64]
    L.hm_pairs_bytes.restype = i64
    L.hm_scan_write_pairs.argtypes = [vp, vp, i32, C.POINTER(C.c_char_p), C.POINTER(PairsStats)]
    L.hm_scan_pairs_hist.argtypes = [vp, vp, vp]
    L.hm_pair_windows.argtypes = [vp, i64, i32, i64, i64p, vp]
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise HetmersError(rc, lib().hm_last_error().decode(errors="replace"))
