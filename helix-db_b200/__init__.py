"""helix-db_b200 — host-side mirror of HelixDB's vector-index read API over the C ABI of libhelix_b200 (CUDA, sm_90a).

The reference's production vector queries funnel through
``ValidatedVectorReadIndex::<D>::{search, search_restricted}``
(crates/db/src/search/vector/read_index.rs:81-101) with ``SearchParams``
(search/vector/mod.rs:411-621), ``RestrictedVectorCandidates`` (restricted.rs:344-389),
``SearchResult`` (result.rs:20-40) and ``HelixDbError`` (crates/db/src/error.rs).  This module
gives the same names, argument meaning and error behaviour on top of ``libhelix_b200.so``
(include/helix_b200.h) through ctypes, so the parity tests read like the reference's own tests.

There is no CPU fallback: if the CUDA library is missing or no device is present, every search raises.
Import it as ``helix_db_b200`` (see the shim at the repository root; the directory name is not a Python
identifier).
"""
from __future__ import annotations

import ctypes as C
import enum
import os
from dataclasses import dataclass
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libhelix_b200.so"
if os.environ.get("HELIX_B200_LIB"):            # an alternate BUILD of the same library (A/B of a compile-time option)
    LIB_PATH = Path(os.environ["HELIX_B200_LIB"]).resolve()

# ---- status codes (include/helix_b200.h) ------------------------------------------------------------------
HX_OK = 0
HX_ERR_INDEX_NOT_FOUND = 1
HX_ERR_INVALID_DIMENSION = 2
HX_ERR_INVALID_VECTOR_COMPONENT = 3
HX_ERR_ZERO_NORM_COSINE = 4
HX_ERR_MAGNITUDE_EXCEEDED = 5
HX_ERR_INVALID_VECTOR_CONFIG = 6
HX_ERR_QUERY = 7
HX_ERR_INVARIANT_VIOLATION = 8
HX_ERR_INVALID_PARAMETER = 9
HX_ERR_CUDA = 10
HX_ERR_OUT_OF_MEMORY = 11
HX_ERR_UNSUPPORTED = 12

_VARIANT = {
    HX_ERR_INDEX_NOT_FOUND: "IndexNotFound",
    HX_ERR_INVALID_DIMENSION: "InvalidDimension",
    HX_ERR_INVALID_VECTOR_COMPONENT: "InvalidVectorComponent",
    HX_ERR_ZERO_NORM_COSINE: "ZeroNormCosineVector",
    HX_ERR_MAGNITUDE_EXCEEDED: "VectorComponentMagnitudeExceeded",
    HX_ERR_INVALID_VECTOR_CONFIG: "InvalidVectorConfig",
    HX_ERR_QUERY: "Query",
    HX_ERR_INVARIANT_VIOLATION: "InvariantViolation",
    HX_ERR_INVALID_PARAMETER: "VectorParameterError",
    HX_ERR_CUDA: "Cuda",
    HX_ERR_OUT_OF_MEMORY: "OutOfMemory",
    HX_ERR_UNSUPPORTED: "Unsupported",
}


class HelixDbError(Exception):
    """Mirror of the HelixDbError variants reachable on this path (crates/db/src/error.rs:379-661)."""

    def __init__(self, code: int, message: str = "", index: int = 0):
        self.code = code
        self.variant = _VARIANT.get(code, f"Status{code}")
        self.index = index
        super().__init__(f"{self.variant}: {message}")


class VectorParameterError(HelixDbError):
    pass


class Metric(enum.IntEnum):
    Euclidean = 0
    Cosine = 1
    Manhattan = 2


class SimHashMode(enum.IntEnum):
    Off = 0
    Adaptive = 1
    Always = 2


class _Config(C.Structure):
    _fields_ = [("dimension", C.c_uint32), ("metric", C.c_int32), ("m", C.c_uint32), ("m0", C.c_uint32),
                ("ef_construction", C.c_uint32), ("device", C.c_int32), ("storage", C.c_uint32),
                ("reserved", C.c_uint32)]


class _Params(C.Structure):
    _fields_ = [("k", C.c_uint32), ("ef", C.c_uint32), ("simhash_mode", C.c_int32), ("pre_sampling_ratio", C.c_float),
                ("collect_stats", C.c_uint32), ("query_dimension", C.c_uint32)]


class SearchStats(C.Structure):
    """Subset of SearchStats (search/vector/mod.rs:668-679) the device path reports."""
    _fields_ = [("expansion_steps", C.c_uint64), ("neighbors_examined", C.c_uint64),
                ("distance_computations", C.c_uint64), ("vectors_loaded", C.c_uint64),
                ("upper_layer_steps", C.c_uint64), ("algorithmic_bytes", C.c_uint64),
                ("kernel_launches", C.c_uint64), ("reserved", C.c_uint64)]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f, _ in self._fields_ if f != "reserved"}


class _SimHashConfig(C.Structure):
    _fields_ = [("simhash_threshold", C.c_uint32), ("sampling_ratio", C.c_float), ("adaptive_enabled", C.c_uint32),
                ("adaptive_failure_prob", C.c_float)]


class _PolicyParams(C.Structure):
    _fields_ = [("bypass_min_frontier", C.c_uint32), ("bypass_window_expansions", C.c_uint32),
                ("bypass_min_filter_rate", C.c_float), ("read_budget_multiplier", C.c_uint32),
                ("sampling_ratio_override", C.c_float), ("failure_prob_override", C.c_float), ("reserved", C.c_uint32 * 2)]


class PolicyStats(C.Structure):
    """The SimHash-related SearchStats counters (search/vector/mod.rs:640-700), summed over the queries of a call."""
    _fields_ = [(n, C.c_uint64) for n in (
        "simhash_filtered", "simhash_examined", "simhash_missing_hash", "simhash_passed_before_sampling",
        "simhash_passed_after_sampling", "simhash_bypass_expansions", "simhash_skipped_candidates",
        "pre_simhash_sample_kept", "pre_simhash_sample_dropped", "simhash_bypass_trigger_budget",
        "simhash_bypass_trigger_low_yield", "rng_draws")]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f, _ in self._fields_}


class _Tuning(C.Structure):
    # hx_tuning (include/helix_b200.h): launch-shape knobs, -1 = built-in default
    _fields_ = [(f, C.c_int32) for f in (
        "ring_warps", "ring_rows", "visited_log2", "visited_pool", "l2_hint", "prefetch_below", "lat_warps", "lat_admit_seq",
        "lat_spec", "phase_prof", "pipeline", "scan_fused", "pol_warps", "pol_min_rows", "pol_cta", "pol_early_sim",
        "build_max_batch")]


class _ServiceConfig(C.Structure):
    _fields_ = [("k", C.c_uint32), ("ef", C.c_uint32), ("capacity", C.c_uint32), ("max_batch", C.c_uint32),
                ("n_streams", C.c_uint32), ("ctas_per_sm", C.c_uint32), ("cta_warps", C.c_uint32),
                ("rows_in_flight", C.c_uint32), ("visited_log2", C.c_uint32), ("min_batch", C.c_uint32),
                ("batch_window_us", C.c_uint32), ("flags", C.c_uint32)]


class ServiceStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("submitted", "completed", "launches", "max_batch_seen", "dispatcher_sleeps",
                                          "completer_wakes")] + \
               [(n, C.c_uint32) for n in ("cta_warps", "rows_in_flight", "visited_cap", "smem_bytes", "ctas_per_sm",
                                          "reserved")]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f, _ in self._fields_ if f != "reserved"}


class FilteredBudgets(C.Structure):
    """FilteredGraphBudgets (restricted.rs:220-260)."""
    _fields_ = [(n, C.c_uint32) for n in ("ef_filtered", "routing_rows", "bridge_rows", "vector_payloads", "sampled_seeds")]


class FilteredStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("vector_payload_requests", "distance_computations", "routing_rows", "bridge_rows",
                                          "bridge_frontier_pushes", "iterations", "kernel_launches", "reserved")]

    def as_dict(self):
        return {f: int(getattr(self, f)) for f, _ in self._fields_ if f != "reserved"}


# every symbol include/helix_b200.h declares (checked by tests/test_abi_surface.py)
ABI_SYMBOLS = [
    "hx_index_create", "hx_index_destroy", "hx_index_load_vectors", "hx_index_generate_vectors",
    "hx_generate_queries", "hx_index_download_vectors", "hx_index_load_graph", "hx_index_set_entry",
    "hx_index_build", "hx_index_graph_info", "hx_index_download_graph", "hx_search", "hx_search_restricted",
    "hx_search_restricted_multi", "hx_restricted_plan", "hx_search_device", "hx_search_restricted_device",
    "hx_map_candidates_device", "hx_merge_topk_device", "hx_search_dense", "hx_last_error", "hx_last_error_index",
    "hx_version", "hx_last_kernel_ms", "hx_index_load_vector_rows", "hx_index_load_neighbor_rows",
    "hx_decode_neighbor_row", "hx_encode_neighbor_row", "hx_index_export_neighbor_row",
    "hx_parse_vector_key", "hx_encode_vector_key", "hx_index_set_simhash_config", "hx_index_load_simhash",
    "hx_index_set_simhash_planes", "hx_index_compute_simhash", "hx_index_download_simhash",
    "hx_order_code_from_simhash_bits", "hx_policy_params_default", "hx_search_ex", "hx_candidates_create",
    "hx_candidates_destroy", "hx_candidates_len", "hx_search_restricted_sets",
    "hx_search_batch", "hx_device_flags", "hx_service_create", "hx_service_destroy", "hx_service_submit",
    "hx_service_poll", "hx_service_wait", "hx_service_search", "hx_service_get_stats",
    "hx_restricted_service_create", "hx_service_submit_restricted", "hx_service_submit_restricted_set",
    "hx_service_search_restricted", "hx_service_search_restricted_set",
    "hx_shard_unique_id", "hx_shard_group_create", "hx_shard_group_destroy", "hx_search_sharded_device",
    "hx_search_sharded", "hx_search_restricted_sharded", "hx_shard_group_last_ms",
    "hx_index_upsert_vectors", "hx_index_set_levels", "hx_index_upsert_neighbor_rows", "hx_index_delete_vectors",
    "hx_index_load_upper_vector_rows", "hx_index_set_version", "hx_index_get_version", "hx_index_build_ex",
    "hx_filtered_budgets", "hx_search_filtered_graph", "hx_index_get_tuning", "hx_index_set_tuning",
    "hx_search_dense_restricted", "hx_search_dense_restricted_set",
    "hx_search_dense_exact", "hx_search_dense_restricted_exact", "hx_search_dense_restricted_exact_set",
    "hx_candidates_make_resident", "hx_candidates_resident_bytes", "hx_search_dense_restricted_set_device",
]

_lib = None


def load_library():
    """dlopen libhelix_b200.so.  Raises (never falls back) when the CUDA extension is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise HelixDbError(HX_ERR_CUDA, f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; "
                                        f"g.build()'` (there is no CPU fallback)")
    L = C.CDLL(str(LIB_PATH))
    vp, sz = C.c_void_p, C.c_size_t
    u64p, u32p, u16p, fp = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint16), C.POINTER(C.c_float)
    L.hx_index_create.restype = C.c_int32
    L.hx_index_create.argtypes = [C.POINTER(_Config), C.POINTER(vp)]
    L.hx_index_destroy.restype = None
    L.hx_index_destroy.argtypes = [vp]
    L.hx_index_get_tuning.restype = C.c_int32
    L.hx_index_get_tuning.argtypes = [vp, C.POINTER(_Tuning)]
    L.hx_index_set_tuning.restype = C.c_int32
    L.hx_index_set_tuning.argtypes = [vp, C.POINTER(_Tuning)]
    L.hx_index_load_vectors.restype = C.c_int32
    L.hx_index_load_vectors.argtypes = [vp, u64p, fp, sz]
    L.hx_index_generate_vectors.restype = C.c_int32
    L.hx_index_generate_vectors.argtypes = [vp, C.c_uint64, sz, C.c_uint64, C.c_uint32, C.c_float, C.c_uint32]
    L.hx_generate_queries.restype = C.c_int32
    L.hx_generate_queries.argtypes = [vp, C.c_uint64, C.c_uint32, C.c_float, C.c_uint64, sz, fp, C.c_uint32]
    L.hx_index_download_vectors.restype = C.c_int32
    L.hx_index_download_vectors.argtypes = [vp, sz, sz, fp, u64p]
    L.hx_index_load_graph.restype = C.c_int32
    L.hx_index_load_graph.argtypes = [vp, C.c_uint16, u64p, u32p, u64p, sz]
    L.hx_index_set_entry.restype = C.c_int32
    L.hx_index_set_entry.argtypes = [vp, C.c_uint64, C.c_uint16]
    L.hx_index_build.restype = C.c_int32
    L.hx_index_build.argtypes = [vp, u16p, C.c_uint64]
    L.hx_index_graph_info.restype = C.c_int32
    L.hx_index_graph_info.argtypes = [vp, u64p, u64p, u16p, u32p, u32p]
    L.hx_index_download_graph.restype = C.c_int32
    L.hx_index_download_graph.argtypes = [vp, u16p, u32p, u32p, u64p, u32p, u16p, u32p, u32p, sz]
    L.hx_search.restype = C.c_int32
    L.hx_search.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, fp, u32p, C.POINTER(SearchStats)]
    L.hx_search_restricted.restype = C.c_int32
    L.hx_search_restricted.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, sz, u64p, fp, u32p,
                                       C.POINTER(SearchStats)]
    L.hx_search_restricted_multi.restype = C.c_int32
    L.hx_search_restricted_multi.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, u64p, u64p, fp, u32p,
                                             C.POINTER(SearchStats)]
    L.hx_restricted_plan.restype = C.c_int32
    L.hx_restricted_plan.argtypes = [C.c_uint64, C.c_uint32]
    L.hx_search_device.restype = C.c_int32
    L.hx_search_device.argtypes = [vp, vp, sz, C.POINTER(_Params), vp, vp, vp, vp, C.POINTER(SearchStats)]
    L.hx_search_restricted_device.restype = C.c_int32
    L.hx_search_restricted_device.argtypes = [vp, vp, sz, C.POINTER(_Params), vp, vp, C.c_uint64, C.c_uint64, vp, vp,
                                              vp, vp]
    L.hx_map_candidates_device.restype = C.c_int32
    L.hx_map_candidates_device.argtypes = [vp, vp, C.c_uint64, vp, vp, vp]
    L.hx_merge_topk_device.restype = C.c_int32
    L.hx_merge_topk_device.argtypes = [C.c_int32, vp, vp, vp, C.c_uint32, sz, C.c_uint32, vp, vp, vp, vp]
    L.hx_search_dense.restype = C.c_int32
    L.hx_search_dense.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, fp, u32p, C.POINTER(SearchStats)]
    L.hx_search_dense_restricted.restype = C.c_int32
    L.hx_search_dense_restricted.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, sz, u64p, fp, u32p,
                                             C.POINTER(SearchStats)]
    L.hx_search_dense_restricted_set.restype = C.c_int32
    L.hx_search_dense_restricted_set.argtypes = [vp, fp, sz, C.POINTER(_Params), vp, u64p, fp, u32p, C.POINTER(SearchStats)]
    L.hx_search_dense_exact.restype = C.c_int32
    L.hx_search_dense_exact.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, fp, u32p, C.POINTER(C.c_uint8), C.POINTER(SearchStats)]
    L.hx_search_dense_restricted_exact.restype = C.c_int32
    L.hx_search_dense_restricted_exact.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, sz, u64p, fp, u32p, C.POINTER(C.c_uint8),
                                                   C.POINTER(SearchStats)]
    L.hx_search_dense_restricted_exact_set.restype = C.c_int32
    L.hx_search_dense_restricted_exact_set.argtypes = [vp, fp, sz, C.POINTER(_Params), vp, u64p, fp, u32p, C.POINTER(C.c_uint8),
                                                       C.POINTER(SearchStats)]
    L.hx_last_error.restype = C.c_char_p
    L.hx_last_error_index.restype = C.c_uint32
    L.hx_version.restype = C.c_char_p
    L.hx_last_kernel_ms.restype = C.c_int32
    L.hx_last_kernel_ms.argtypes = [vp, fp, u32p]
    u8p = C.POINTER(C.c_uint8)
    L.hx_index_load_vector_rows.restype = C.c_int32
    L.hx_index_load_vector_rows.argtypes = [vp, u64p, u8p, sz]
    L.hx_index_load_neighbor_rows.restype = C.c_int32
    L.hx_index_load_neighbor_rows.argtypes = [vp, C.c_uint16, u64p, u8p, u64p, sz]
    L.hx_decode_neighbor_row.restype = C.c_int32
    L.hx_decode_neighbor_row.argtypes = [C.c_uint16, u8p, sz, u64p, sz, C.POINTER(sz), u64p, C.POINTER(C.c_int32)]
    L.hx_encode_neighbor_row.restype = C.c_int32
    L.hx_encode_neighbor_row.argtypes = [C.c_uint16, u64p, sz, u8p, sz, C.POINTER(sz)]
    L.hx_index_export_neighbor_row.restype = C.c_int32
    L.hx_index_export_neighbor_row.argtypes = [vp, C.c_uint16, C.c_uint64, u8p, sz, C.POINTER(sz)]
    L.hx_parse_vector_key.restype = C.c_int32
    L.hx_parse_vector_key.argtypes = [u8p, sz, vp]
    L.hx_encode_vector_key.restype = C.c_int32
    L.hx_encode_vector_key.argtypes = [vp, u8p, sz, C.POINTER(sz)]
    L.hx_index_set_simhash_config.restype = C.c_int32
    L.hx_index_set_simhash_config.argtypes = [vp, C.POINTER(_SimHashConfig)]
    L.hx_index_load_simhash.restype = C.c_int32
    L.hx_index_load_simhash.argtypes = [vp, u64p, u64p, sz]
    L.hx_index_set_simhash_planes.restype = C.c_int32
    L.hx_index_set_simhash_planes.argtypes = [vp, fp]
    L.hx_index_compute_simhash.restype = C.c_int32
    L.hx_index_compute_simhash.argtypes = [vp]
    L.hx_index_download_simhash.restype = C.c_int32
    L.hx_index_download_simhash.argtypes = [vp, sz, sz, u64p]
    L.hx_order_code_from_simhash_bits.restype = C.c_uint64
    L.hx_order_code_from_simhash_bits.argtypes = [C.c_uint64]
    L.hx_policy_params_default.restype = None
    L.hx_policy_params_default.argtypes = [C.POINTER(_PolicyParams)]
    L.hx_candidates_create.restype = C.c_int32
    L.hx_candidates_create.argtypes = [vp, u64p, sz, C.POINTER(vp)]
    L.hx_candidates_destroy.restype = None
    L.hx_candidates_destroy.argtypes = [vp]
    L.hx_candidates_len.restype = C.c_uint64
    L.hx_candidates_len.argtypes = [vp]
    L.hx_candidates_make_resident.restype = C.c_int32
    L.hx_candidates_make_resident.argtypes = [vp, vp]
    L.hx_candidates_resident_bytes.restype = C.c_uint64
    L.hx_candidates_resident_bytes.argtypes = [vp]
    L.hx_search_dense_restricted_set_device.restype = C.c_int32
    L.hx_search_dense_restricted_set_device.argtypes = [vp, vp, sz, C.POINTER(_Params), vp, vp, vp, vp, vp, vp]
    L.hx_search_restricted_sets.restype = C.c_int32
    L.hx_search_restricted_sets.argtypes = [vp, fp, sz, C.POINTER(_Params), C.POINTER(vp), sz, u64p, fp, u32p,
                                            C.POINTER(SearchStats)]
    L.hx_search_ex.restype = C.c_int32
    L.hx_search_ex.argtypes = [vp, fp, sz, C.POINTER(_Params), C.POINTER(_PolicyParams), u64p, u64p, fp, u32p,
                               C.POINTER(SearchStats), C.POINTER(PolicyStats)]
    i32p = C.POINTER(C.c_int32)
    L.hx_search_batch.restype = C.c_int32
    L.hx_search_batch.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, fp, u32p, i32p, C.POINTER(SearchStats)]
    L.hx_device_flags.restype = C.c_int32
    L.hx_device_flags.argtypes = [vp, vp, u32p, i32p]
    L.hx_service_create.restype = C.c_int32
    L.hx_service_create.argtypes = [vp, C.POINTER(_ServiceConfig), C.POINTER(vp)]
    L.hx_service_destroy.restype = None
    L.hx_service_destroy.argtypes = [vp]
    L.hx_service_submit.restype = C.c_int32
    L.hx_service_submit.argtypes = [vp, fp, u64p]
    L.hx_service_poll.restype = C.c_int32
    L.hx_service_poll.argtypes = [vp, C.c_uint64, i32p, u64p, fp, u32p]
    L.hx_service_wait.restype = C.c_int32
    L.hx_service_wait.argtypes = [vp, C.c_uint64, u64p, fp, u32p]
    L.hx_service_search.restype = C.c_int32
    L.hx_service_search.argtypes = [vp, fp, u64p, fp, u32p]
    L.hx_service_get_stats.restype = C.c_int32
    L.hx_service_get_stats.argtypes = [vp, C.POINTER(ServiceStats)]
    L.hx_restricted_service_create.restype = C.c_int32
    L.hx_restricted_service_create.argtypes = [vp, C.POINTER(_ServiceConfig), C.c_uint64, C.POINTER(vp)]
    L.hx_service_submit_restricted.restype = C.c_int32
    L.hx_service_submit_restricted.argtypes = [vp, fp, u64p, sz, u64p]
    L.hx_service_submit_restricted_set.restype = C.c_int32
    L.hx_service_submit_restricted_set.argtypes = [vp, fp, vp, u64p]
    L.hx_service_search_restricted.restype = C.c_int32
    L.hx_service_search_restricted.argtypes = [vp, fp, u64p, sz, u64p, fp, u32p]
    L.hx_service_search_restricted_set.restype = C.c_int32
    L.hx_service_search_restricted_set.argtypes = [vp, fp, vp, u64p, fp, u32p]
    L.hx_filtered_budgets.restype = None
    L.hx_filtered_budgets.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(FilteredBudgets)]
    L.hx_search_filtered_graph.restype = C.c_int32
    L.hx_search_filtered_graph.argtypes = [vp, fp, sz, C.POINTER(_Params), C.POINTER(FilteredBudgets), u64p, sz, u64p, u64p,
                                           fp, u32p, C.POINTER(FilteredStats)]
    L.hx_index_build_ex.restype = C.c_int32
    L.hx_index_build_ex.argtypes = [vp, u16p, C.c_uint64, C.c_int32]
    L.hx_index_upsert_vectors.restype = C.c_int32
    L.hx_index_upsert_vectors.argtypes = [vp, u64p, fp, sz]
    L.hx_index_set_levels.restype = C.c_int32
    L.hx_index_set_levels.argtypes = [vp, u64p, u16p, sz]
    L.hx_index_upsert_neighbor_rows.restype = C.c_int32
    L.hx_index_upsert_neighbor_rows.argtypes = [vp, C.c_uint16, u64p, u32p, u64p, sz]
    L.hx_index_delete_vectors.restype = C.c_int32
    L.hx_index_delete_vectors.argtypes = [vp, u64p, sz]
    L.hx_index_load_upper_vector_rows.restype = C.c_int32
    L.hx_index_load_upper_vector_rows.argtypes = [vp, u64p, u8p, sz]
    L.hx_index_set_version.restype = C.c_int32
    L.hx_index_set_version.argtypes = [vp, C.c_uint64, C.c_uint64]
    L.hx_index_get_version.restype = C.c_int32
    L.hx_index_get_version.argtypes = [vp, u64p, u64p, u64p]
    L.hx_shard_unique_id.restype = C.c_int32
    L.hx_shard_unique_id.argtypes = [u8p, sz]
    L.hx_shard_group_create.restype = C.c_int32
    L.hx_shard_group_create.argtypes = [vp, C.c_uint32, C.c_uint32, u8p, C.POINTER(vp)]
    L.hx_shard_group_destroy.restype = None
    L.hx_shard_group_destroy.argtypes = [vp]
    L.hx_search_sharded_device.restype = C.c_int32
    L.hx_search_sharded_device.argtypes = [vp, C.c_int32, vp, sz, C.POINTER(_Params), C.c_uint32, vp, vp, vp, vp]
    L.hx_search_sharded.restype = C.c_int32
    L.hx_search_sharded.argtypes = [vp, C.c_int32, fp, sz, C.POINTER(_Params), C.c_uint32, u64p, fp, u32p]
    L.hx_search_restricted_sharded.restype = C.c_int32
    L.hx_search_restricted_sharded.argtypes = [vp, fp, sz, C.POINTER(_Params), u64p, sz, u64p, fp, u32p]
    L.hx_shard_group_last_ms.restype = C.c_int32
    L.hx_shard_group_last_ms.argtypes = [vp, fp, fp]
    _lib = L
    return L


def _raise(code: int):
    L = load_library()
    msg = (L.hx_last_error() or b"").decode("utf-8", "replace")
    idx = int(L.hx_last_error_index())
    cls = VectorParameterError if code == HX_ERR_INVALID_PARAMETER else HelixDbError
    raise cls(code, msg, idx)


def _ck(code: int):
    if code != HX_OK:
        _raise(code)


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(C.POINTER(C.c_float))


def _u64(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a, a.ctypes.data_as(C.POINTER(C.c_uint64))


def _u32(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return a, a.ctypes.data_as(C.POINTER(C.c_uint32))


# ---- reference-shaped value types -------------------------------------------------------------------------
class SearchResult:
    """SearchResult{entity_id, score} (search/vector/result.rs:20-40)."""
    __slots__ = ("_id", "_score")

    def __init__(self, entity_id: int, score: float):
        self._id, self._score = int(entity_id), np.float32(score)

    def entity_id(self) -> int:
        return self._id

    def score(self) -> np.float32:
        return self._score

    def __repr__(self):
        return f"SearchResult(entity_id={self._id}, score={float(self._score)!r})"

    def __eq__(self, o):
        return isinstance(o, SearchResult) and self._id == o._id and self._score.tobytes() == o._score.tobytes()


class SearchParams:
    """SearchParams builder (search/vector/mod.rs:480-621).  ``SearchParams.new(k)``: ef = max(k,100),
    SimHashMode.Adaptive.  ``Off`` + pre-sampling 1.0 is the strict-exhaustive specialisation; every other combination runs
    the SimHash filtering / sampling policy kernel (needs the node fingerprints)."""

    def __init__(self, k: int):
        if k <= 0:
            raise VectorParameterError(HX_ERR_INVALID_PARAMETER, "result count must be non-zero")
        self._k = int(k)
        self._ef = max(self._k, 100)
        self._mode = SimHashMode.Adaptive
        self._pre_ratio = None
        self._bypass = (24, 4, 0.12, 3)          # min frontier, window expansions, min filter rate, read budget multiplier
        self._sampling_ratio = None
        self._failure_prob = None
        self.collect_stats = False
        self.query_dimension = 0

    @classmethod
    def new(cls, k: int) -> "SearchParams":
        return cls(k)

    def k(self):
        return self._k

    def ef(self):
        return self._ef

    def with_ef(self, ef: int) -> "SearchParams":
        if ef < self._k:
            raise VectorParameterError(HX_ERR_INVALID_PARAMETER,
                                       f"search beam width must be at least {self._k}, got {ef}")
        self._ef = int(ef)
        return self

    def with_simhash_mode(self, mode: SimHashMode) -> "SearchParams":
        self._mode = SimHashMode(mode)
        return self

    def with_pre_simhash_sampling_ratio(self, ratio: float) -> "SearchParams":
        if not (0.0 <= ratio <= 1.0):
            raise VectorParameterError(HX_ERR_INVALID_PARAMETER, "ratio must be in the unit interval")
        self._pre_ratio = float(ratio)
        return self

    def with_simhash_bypass_tuning(self, min_frontier: int, window_expansions: int, min_filter_rate: float,
                                   read_budget_multiplier: int) -> "SearchParams":   # mod.rs:563-592
        if min_frontier <= 0 or window_expansions <= 0 or read_budget_multiplier <= 0 or not (0.0 <= min_filter_rate <= 1.0):
            raise VectorParameterError(HX_ERR_INVALID_PARAMETER, "invalid SimHash bypass tuning")
        self._bypass = (int(min_frontier), int(window_expansions), float(min_filter_rate), int(read_budget_multiplier))
        return self

    def with_simhash_sampling_ratio(self, ratio: float) -> "SearchParams":             # mod.rs:594-598
        if not (0.0 <= ratio <= 1.0):
            raise VectorParameterError(HX_ERR_INVALID_PARAMETER, "ratio must be in the unit interval")
        self._sampling_ratio = float(ratio)
        return self

    def with_simhash_failure_prob(self, failure_prob: float) -> "SearchParams":        # mod.rs:606-613
        if not (0.0 < failure_prob < 1.0):
            raise VectorParameterError(HX_ERR_INVALID_PARAMETER, "failure probability must be in (0, 1)")
        self._failure_prob = float(failure_prob)
        return self

    @classmethod
    def throughput_profile_floor_92(cls, k: int) -> "SearchParams":                     # mod.rs:615-621
        return (cls(k).with_ef(max(k, 48)).with_simhash_mode(SimHashMode.Adaptive)
                .with_pre_simhash_sampling_ratio(0.20).with_simhash_bypass_tuning(24, 4, 0.12, 3))

    def _policy(self) -> "_PolicyParams":
        p = _PolicyParams()
        p.bypass_min_frontier, p.bypass_window_expansions, p.bypass_min_filter_rate, p.read_budget_multiplier = self._bypass
        p.sampling_ratio_override = -1.0 if self._sampling_ratio is None else self._sampling_ratio
        p.failure_prob_override = -1.0 if self._failure_prob is None else self._failure_prob
        return p

    @classmethod
    def strict(cls, k: int, ef: int | None = None) -> "SearchParams":
        """The reference's strict baseline: Off + pre-sampling 1.0 (mod.rs:518-554)."""
        p = cls(k).with_simhash_mode(SimHashMode.Off).with_pre_simhash_sampling_ratio(1.0)
        return p.with_ef(ef) if ef is not None else p

    def requires_query_simhash(self) -> bool:   # mod.rs:556-561
        return self._mode != SimHashMode.Off or (self._pre_ratio is not None and self._pre_ratio < 1.0)

    def _c(self) -> _Params:
        ratio = -1.0 if self._pre_ratio is None else self._pre_ratio      # negative = no override (Option::None)
        return _Params(self._k, self._ef, int(self._mode), ratio, 1 if self.collect_stats else 0,
                       int(self.query_dimension))


class DeviceCandidates:
    """A candidate set resident on the device (hx_candidates)."""

    def __init__(self, L, h, n, ix=None):
        self.L, self.h, self.n, self.ix = L, h, n, ix

    def __len__(self):
        return int(self.n)

    def make_resident(self):
        """hx_candidates_make_resident: build the set's tensor-core view once (blocking); the dense set entries then skip
        the per-call compaction, gather and view reduction, and search_dense_restricted_set_device accepts the set."""
        _ck(self.L.hx_candidates_make_resident(self.ix, self.h))
        return self

    @property
    def resident_bytes(self):
        """Device memory the resident view holds (0 while the set is not resident)."""
        return int(self.L.hx_candidates_resident_bytes(self.h))

    def close(self):
        if self.h:
            self.L.hx_candidates_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RestrictedVectorCandidates:
    """RestrictedVectorCandidates::from_ids (restricted.rs:356-371): unique ascending ids, at most 1e6."""
    MAX = 1_000_000

    def __init__(self, ids: np.ndarray):
        self.ids = ids

    @classmethod
    def from_ids(cls, ids) -> "RestrictedVectorCandidates":
        a = np.unique(np.asarray(list(ids) if not isinstance(ids, np.ndarray) else ids, dtype=np.uint64))
        if a.size > cls.MAX:
            raise HelixDbError(HX_ERR_QUERY, f"restricted vector search accepts at most {cls.MAX} unique candidates")
        return cls(a)

    def is_empty(self):
        return self.ids.size == 0

    def contains(self, node_id: int) -> bool:
        i = np.searchsorted(self.ids, np.uint64(node_id))
        return bool(i < self.ids.size and self.ids[i] == node_id)

    def __len__(self):
        return int(self.ids.size)


class VectorIndexConfig:
    """VectorIndexConfig::new(name, property, dimension).with_m(..) (defaults config/indexes.rs:374-408)."""

    def __init__(self, name: str, prop: str, dimension: int):
        self.name, self.property, self.dimension = name, prop, int(dimension)
        self.m, self.m0, self.ef_construction = 16, 32, 200

    def with_m(self, m):
        self.m = int(m)
        return self

    def with_m0(self, m0):
        self.m0 = int(m0)
        return self

    def with_ef_construction(self, e):
        self.ef_construction = int(e)
        return self


class VectorIndex:
    """Device-resident stand-in for ``VectorIndex::<D>`` (search/vector/index.rs).

    The reference reads rows through SlateDB; here the rows are mirrored once into HBM
    (``load_vectors`` / ``load_graph`` / ``set_entry`` or ``build``) and then searched."""

    def __init__(self, metric: Metric, config: VectorIndexConfig, device: int = 0, storage: int = 0):
        self.L = load_library()
        self.metric, self.config, self.device = Metric(metric), config, device
        cfg = _Config(config.dimension, int(self.metric), config.m, config.m0, config.ef_construction, device,
                      storage, 0)
        h = C.c_void_p()
        _ck(self.L.hx_index_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self.dim = config.dimension

    def close(self):
        if getattr(self, "h", None):
            self.L.hx_index_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- mirror management ----
    def load_vectors(self, ids, rows):
        ia, ip = _u64(ids)
        ra, rp = _f32(rows)
        if ra.size != ia.size * self.dim:
            raise HelixDbError(HX_ERR_INVALID_DIMENSION, f"expected {ia.size}x{self.dim} floats, got {ra.size}")
        _ck(self.L.hx_index_load_vectors(self.h, ip, rp, ia.size))

    def generate_vectors(self, first_id, n, seed, n_centroids=1024, sigma=0.3, kind=0):
        _ck(self.L.hx_index_generate_vectors(self.h, first_id, n, seed, n_centroids, sigma, kind))

    def generate_queries(self, seed, n, first_query=0, n_centroids=1024, sigma=0.3, kind=0):
        out = np.empty((n, self.dim), dtype=np.float32)
        _ck(self.L.hx_generate_queries(self.h, seed, n_centroids, sigma, first_query, n,
                                       out.ctypes.data_as(C.POINTER(C.c_float)), kind))
        return out

    def download_vectors(self, first_slot, n):
        rows = np.empty((n, self.dim), dtype=np.float32)
        ids = np.empty(n, dtype=np.uint64)
        _ck(self.L.hx_index_download_vectors(self.h, first_slot, n, rows.ctypes.data_as(C.POINTER(C.c_float)),
                                             ids.ctypes.data_as(C.POINTER(C.c_uint64))))
        return ids, rows

    def load_graph(self, layer, node_ids, offsets, neighbors):
        na, np_ = _u64(node_ids)
        oa, op = _u32(offsets)
        nb, nbp = _u64(neighbors)
        _ck(self.L.hx_index_load_graph(self.h, layer, np_, op, nbp, na.size))

    def set_entry(self, entry_point, max_layer):
        _ck(self.L.hx_index_set_entry(self.h, entry_point, max_layer))

    def load_vector_rows(self, ids, rows: bytes):
        """Hydrate from the reference's encoded item rows `[header f32][f32 x dim]` (mod.rs:866-949)."""
        ia, ip = _u64(ids)
        buf = (C.c_uint8 * max(len(rows), 1)).from_buffer_copy(rows if rows else b"\0")
        if len(rows) != ia.size * (4 + 4 * self.dim):
            raise HelixDbError(HX_ERR_INVARIANT_VIOLATION, "item rows must be 4+4*dimension bytes each")
        _ck(self.L.hx_index_load_vector_rows(self.h, ip, buf, ia.size))

    def load_neighbor_rows(self, layer, node_ids, rows):
        """Hydrate one layer from encoded neighbour row values (list of bytes, one per node)."""
        na, np_ = _u64(node_ids)
        blob = b"".join(rows)
        offs = np.zeros(len(rows) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(r) for r in rows])
        buf = (C.c_uint8 * max(len(blob), 1)).from_buffer_copy(blob if blob else b"\0")
        _ck(self.L.hx_index_load_neighbor_rows(self.h, layer, np_, buf, offs.ctypes.data_as(C.POINTER(C.c_uint64)), na.size))

    def export_neighbor_row(self, layer, node_id) -> bytes:
        out = (C.c_uint8 * (8 * 4096 + 8))()
        n = C.c_size_t(0)
        _ck(self.L.hx_index_export_neighbor_row(self.h, layer, node_id, out, len(out), C.byref(n)))
        return bytes(out[:n.value])

    def build(self, levels=None, seed=0, sequential=False):
        """hx_index_build_ex.  sequential=True: one insert_hnsw at a time — the reference's graph for the same insertion
        order and levels (parity runs, small indexes); default: batched concurrent insertion."""
        lp = None
        if levels is not None:
            la = np.ascontiguousarray(levels, dtype=np.uint16)
            lp = la.ctypes.data_as(C.POINTER(C.c_uint16))
        _ck(self.L.hx_index_build_ex(self.h, lp, seed, 1 if sequential else 0))

    def graph_info(self):
        n, e, ml, s0, su = C.c_uint64(0), C.c_uint64(0), C.c_uint16(0), C.c_uint32(0), C.c_uint32(0)
        _ck(self.L.hx_index_graph_info(self.h, C.byref(n), C.byref(e), C.byref(ml), C.byref(s0), C.byref(su)))
        return dict(n=int(n.value), entry_point=int(e.value), max_layer=int(ml.value), layer0_stride=int(s0.value),
                    upper_stride=int(su.value))

    def download_graph(self):
        gi = self.graph_info()
        n, s0, su = gi["n"], gi["layer0_stride"], gi["upper_stride"]
        nup = C.c_uint64(0)
        _ck(self.L.hx_index_download_graph(self.h, None, None, None, C.byref(nup), None, None, None, None, 0))
        rows = int(nup.value)
        levels = np.zeros(max(n, 1), dtype=np.uint16)
        deg0 = np.zeros(max(n, 1), dtype=np.uint32)
        nbr0 = np.zeros(max(n * s0, 1), dtype=np.uint32)
        un = np.zeros(max(rows, 1), dtype=np.uint32)
        ul = np.zeros(max(rows, 1), dtype=np.uint16)
        ud = np.zeros(max(rows, 1), dtype=np.uint32)
        unb = np.zeros(max(rows * su, 1), dtype=np.uint32)
        _ck(self.L.hx_index_download_graph(
            self.h, levels.ctypes.data_as(C.POINTER(C.c_uint16)), deg0.ctypes.data_as(C.POINTER(C.c_uint32)),
            nbr0.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(nup), un.ctypes.data_as(C.POINTER(C.c_uint32)),
            ul.ctypes.data_as(C.POINTER(C.c_uint16)), ud.ctypes.data_as(C.POINTER(C.c_uint32)),
            unb.ctypes.data_as(C.POINTER(C.c_uint32)), rows))
        gi.update(levels=levels[:n], deg0=deg0[:n], nbr0=nbr0[:n * s0], upper_node=un[:rows], upper_layer=ul[:rows],
                  upper_deg=ud[:rows], upper_nbr=unb[:rows * su])
        return gi

    # ---- incremental maintenance: a committed write arrives as row patches + a new version token (SURVEY §8f.2) ----
    def upsert_vectors(self, ids, rows):
        ia, ip = _u64(ids)
        ra, rp = _f32(rows)
        if ra.size != ia.size * self.dim:
            raise HelixDbError(HX_ERR_INVALID_DIMENSION, f"expected {ia.size}x{self.dim} floats, got {ra.size}")
        _ck(self.L.hx_index_upsert_vectors(self.h, ip, rp, ia.size))

    def set_levels(self, ids, levels):
        ia, ip = _u64(ids)
        la = np.ascontiguousarray(levels, dtype=np.uint16)
        _ck(self.L.hx_index_set_levels(self.h, ip, la.ctypes.data_as(C.POINTER(C.c_uint16)), ia.size))

    def upsert_neighbor_rows(self, layer, node_ids, offsets, neighbors):
        na, np_ = _u64(node_ids)
        oa, op = _u32(offsets)
        nb, nbp = _u64(neighbors)
        _ck(self.L.hx_index_upsert_neighbor_rows(self.h, layer, np_, op, nbp, na.size))

    def delete_vectors(self, ids):
        ia, ip = _u64(ids)
        _ck(self.L.hx_index_delete_vectors(self.h, ip, ia.size))

    def load_upper_vector_rows(self, ids, rows: bytes):
        """`[0x13]` hot-lane item rows (`[header f32][f32 x dim]` each)."""
        ia, ip = _u64(ids)
        if len(rows) != ia.size * (4 + 4 * self.dim):
            raise HelixDbError(HX_ERR_INVARIANT_VIOLATION, "item rows must be 4+4*dimension bytes each")
        buf = (C.c_uint8 * max(len(rows), 1)).from_buffer_copy(rows if rows else b"\0")
        _ck(self.L.hx_index_load_upper_vector_rows(self.h, ip, buf, ia.size))

    def tune(self, **knobs):
        """hx_index_set_tuning: launch-shape knobs for experiments / A-B tests (fields of hx_tuning).  The handle starts from
        the environment's values (HX_RING_WARPS, ...); ``tune(x=..)`` overrides fields on top of those, ``tune()`` alone
        returns to them.  Results are bit-identical for every setting."""
        _ck(self.L.hx_index_set_tuning(self.h, None))
        if knobs:
            t = _Tuning()
            _ck(self.L.hx_index_get_tuning(self.h, C.byref(t)))
            for key, val in knobs.items():
                if not hasattr(t, key):
                    raise TypeError(f"unknown tuning knob {key!r}")
                setattr(t, key, int(val))
            _ck(self.L.hx_index_set_tuning(self.h, C.byref(t)))

    def tuning(self) -> dict:
        t = _Tuning()
        _ck(self.L.hx_index_get_tuning(self.h, C.byref(t)))
        return {f: int(getattr(t, f)) for f, _ in _Tuning._fields_}

    def set_version(self, generation: int, visible_seq: int):
        _ck(self.L.hx_index_set_version(self.h, generation, visible_seq))

    def version(self):
        g, v, p = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        _ck(self.L.hx_index_get_version(self.h, C.byref(g), C.byref(v), C.byref(p)))
        return int(g.value), int(v.value), int(p.value)

    # ---- SimHash policy state (production-default mode) ----
    def set_simhash_config(self, threshold=43, sampling_ratio=0.8, adaptive_enabled=True, adaptive_failure_prob=0.1):
        """VectorIndexConfig simhash_threshold / sampling_ratio / adaptive_enabled / adaptive_failure_prob
        (config/indexes.rs:398-406)."""
        cfg = _SimHashConfig(int(threshold), float(sampling_ratio), 1 if adaptive_enabled else 0, float(adaptive_failure_prob))
        _ck(self.L.hx_index_set_simhash_config(self.h, C.byref(cfg)))

    def load_simhash(self, ids, bits):
        """The [0x12] SimHash rows (8 bytes LE each) decoded to u64."""
        ia, ip = _u64(ids)
        ba, bp = _u64(bits)
        _ck(self.L.hx_index_load_simhash(self.h, ip, bp, ia.size))

    def set_simhash_planes(self, planes):
        """SimHasher::hyperplanes(): 64 x dimension f32, plane-major."""
        pa, pp = _f32(planes)
        if pa.size != 64 * self.dim:
            raise HelixDbError(HX_ERR_INVALID_DIMENSION, "hyperplane table must be 64 x dimension")
        _ck(self.L.hx_index_set_simhash_planes(self.h, pp))

    def compute_simhash(self):
        _ck(self.L.hx_index_compute_simhash(self.h))

    def download_simhash(self, first_slot, n):
        out = np.zeros(n, dtype=np.uint64)
        _ck(self.L.hx_index_download_simhash(self.h, first_slot, n, out.ctypes.data_as(C.POINTER(C.c_uint64))))
        return out

    def search_ex(self, queries, params: SearchParams, query_simhash=None, stats=None, policy_stats=None):
        """hx_search_ex: the full SearchParams surface; query fingerprints given or projected from the planes."""
        qa, qp = _f32(queries)
        qd = params.query_dimension or self.dim
        B = qa.size // qd if qa.ndim != 1 or qa.size != qd else 1
        cp = params._c()
        pol = params._policy()
        k = cp.k
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        ps = policy_stats if policy_stats is not None else PolicyStats()
        if query_simhash is not None:
            sa, sp = _u64(query_simhash)
        else:
            sp = None
        _ck(self.L.hx_search_ex(self.h, qp, B, C.byref(cp), C.byref(pol), sp, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                sc.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_uint32)),
                                C.byref(st), C.byref(ps)))
        return ids, sc, cnt

    # ---- search ----
    def _search_raw(self, queries, params: SearchParams, stats=None):
        qa, qp = _f32(queries)
        qd = params.query_dimension or self.dim
        B = qa.size // qd if qa.ndim != 1 or qa.size != qd else 1
        cp = params._c()
        k = cp.k
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search(self.h, qp, B, C.byref(cp), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                             sc.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_uint32)),
                             C.byref(st)))
        return ids, sc, cnt

    def search(self, query, params: SearchParams):
        """VectorIndex::search (index.rs:1578): one query -> Vec<SearchResult> sorted by (score, id)."""
        ids, sc, cnt = self._search_raw(np.asarray(query, dtype=np.float32).reshape(1, -1), params)
        return [SearchResult(ids[0, i], sc[0, i]) for i in range(int(cnt[0]))]

    def search_with_stats(self, query, params: SearchParams):
        params.collect_stats = True
        st = SearchStats()
        ids, sc, cnt = self._search_raw(np.asarray(query, dtype=np.float32).reshape(1, -1), params, st)
        return [SearchResult(ids[0, i], sc[0, i]) for i in range(int(cnt[0]))], st

    def search_batch(self, queries, params: SearchParams, stats=None):
        return self._search_raw(np.asarray(queries, dtype=np.float32), params, stats)

    def search_batch_status(self, queries, params: SearchParams, stats=None):
        """hx_search_batch: one status per query (an invalid query, or one that exhausts a device-side bound, fails alone).
        Returns (ids, scores, counts, status[B])."""
        qa, qp = _f32(queries)
        qd = params.query_dimension or self.dim
        B = qa.size // qd
        cp = params._c()
        k = cp.k
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        status = np.zeros(B, dtype=np.int32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_batch(self.h, qp, B, C.byref(cp), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                   sc.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_uint32)),
                                   status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(st)))
        return ids, sc, cnt, status

    def device_flags(self, stream_ptr=0):
        """hx_device_flags: (flags, status) of the device-buffer calls issued on the stream since the last read."""
        fl, stc = C.c_uint32(0), C.c_int32(0)
        _ck(self.L.hx_device_flags(self.h, stream_ptr, C.byref(fl), C.byref(stc)))
        return int(fl.value), int(stc.value)

    def service(self, k: int, ef: int = 0, **kw) -> "SearchService":
        """A query service on this index: concurrent one-query callers coalesced into shared launches."""
        return SearchService(self, k, ef, **kw)

    def restricted_service(self, k: int, arena_ids: int = 0, **kw) -> "RestrictedSearchService":
        """A restricted query service: concurrent one-query search_restricted callers coalesced into shared scans."""
        return RestrictedSearchService(self, k, arena_ids, **kw)

    def search_restricted(self, query, params: SearchParams, allowed: RestrictedVectorCandidates):
        """VectorIndex::search_restricted (restricted.rs:466-479); exact for every |C| <= 1e6."""
        ids, sc, cnt = self.search_restricted_batch(np.asarray(query, dtype=np.float32).reshape(1, -1), params,
                                                    allowed)
        return [SearchResult(ids[0, i], sc[0, i]) for i in range(int(cnt[0]))]

    def search_restricted_batch(self, queries, params: SearchParams, allowed: RestrictedVectorCandidates, stats=None):
        qa, qp = _f32(queries)
        qd = params.query_dimension or self.dim
        B = qa.size // qd
        cp = params._c()
        k = cp.k
        ca, cpnt = _u64(allowed.ids)
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_restricted(self.h, qp, B, C.byref(cp), cpnt, ca.size,
                                        ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                        sc.ctypes.data_as(C.POINTER(C.c_float)),
                                        cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(st)))
        return ids, sc, cnt

    def search_filtered_graph(self, queries, params: SearchParams, allowed: RestrictedVectorCandidates, query_simhash=None,
                              budgets=None, stats=None):
        """hx_search_filtered_graph: the reference's filter-aware (ACORN) walk, restricted.rs:837-1148 (approximate)."""
        qa, qp = _f32(queries)
        B = qa.size // self.dim
        cp = params._c()
        k = cp.k
        ca, cpnt = _u64(allowed.ids)
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        bp = None
        if budgets is not None:
            bb = FilteredBudgets(*[int(x) for x in budgets])
            bp = C.byref(bb)
        sp = None
        if query_simhash is not None:
            sa, sp = _u64(query_simhash)
        st = stats if stats is not None else FilteredStats()
        _ck(self.L.hx_search_filtered_graph(self.h, qp, B, C.byref(cp), bp, cpnt, ca.size, sp,
                                            ids.ctypes.data_as(C.POINTER(C.c_uint64)), sc.ctypes.data_as(C.POINTER(C.c_float)),
                                            cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(st)))
        return ids, sc, cnt

    def cache_candidates(self, allowed: "RestrictedVectorCandidates") -> "DeviceCandidates":
        """Upload a candidate set once (label bitmap reuse, SURVEY §8d); returns a handle for search_restricted_sets."""
        ca, cp = _u64(allowed.ids)
        h = C.c_void_p()
        _ck(self.L.hx_candidates_create(self.h, cp, ca.size, C.byref(h)))
        return DeviceCandidates(self.L, h, ca.size, self.h)

    def search_restricted_sets(self, queries, params: SearchParams, sets, stats=None):
        """One DeviceCandidates per query, or a single one shared by all queries."""
        qa, qp = _f32(queries)
        B = qa.size // self.dim
        cp = params._c()
        k = cp.k
        sets = list(sets) if isinstance(sets, (list, tuple)) else [sets]
        arr = (C.c_void_p * len(sets))(*[x.h for x in sets])
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_restricted_sets(self.h, qp, B, C.byref(cp), arr, len(sets),
                                             ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                             sc.ctypes.data_as(C.POINTER(C.c_float)),
                                             cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(st)))
        return ids, sc, cnt

    def search_restricted_multi(self, queries, params: SearchParams, cand_ids, cand_offsets, stats=None):
        qa, qp = _f32(queries)
        B = qa.size // self.dim
        cp = params._c()
        k = cp.k
        ca, cpnt = _u64(cand_ids)
        oa, op = _u64(cand_offsets)
        assert oa.size == B + 1
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_restricted_multi(self.h, qp, B, C.byref(cp), cpnt, op,
                                              ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                              sc.ctypes.data_as(C.POINTER(C.c_float)),
                                              cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(st)))
        return ids, sc, cnt

    def search_dense_batch(self, queries, params: SearchParams, stats=None):
        qa, qp = _f32(queries)
        B = qa.size // self.dim
        cp = params._c()
        k = cp.k
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_dense(self.h, qp, B, C.byref(cp), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                   sc.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_uint32)),
                                   C.byref(st)))
        return ids, sc, cnt

    def search_dense_restricted_batch(self, queries, params: SearchParams, allowed: RestrictedVectorCandidates, stats=None):
        """hx_search_dense_restricted: the tensor-core path over one candidate set shared by every query."""
        qa, qp = _f32(queries)
        B = qa.size // (params.query_dimension or self.dim)
        cp = params._c()
        k = cp.k
        ca, cpnt = _u64(allowed.ids)
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_dense_restricted(self.h, qp, B, C.byref(cp), cpnt, ca.size,
                                              ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                              sc.ctypes.data_as(C.POINTER(C.c_float)),
                                              cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(st)))
        return ids, sc, cnt

    def search_dense_restricted_sets(self, queries, params: SearchParams, device_set: "DeviceCandidates", stats=None):
        """hx_search_dense_restricted_set: the same with a device-resident set (cache_candidates)."""
        qa, qp = _f32(queries)
        B = qa.size // self.dim
        cp = params._c()
        k = cp.k
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        st = stats if stats is not None else SearchStats()
        _ck(self.L.hx_search_dense_restricted_set(self.h, qp, B, C.byref(cp), device_set.h,
                                                  ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                  sc.ctypes.data_as(C.POINTER(C.c_float)),
                                                  cnt.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(st)))
        return ids, sc, cnt

    # ---- exact tensor-core search: (ids, scores, counts, how); how per query: 0 certified, 1 rescanned, 2 exact scan ----
    def _dense_exact(self, fn, queries, params: SearchParams, set_args, stats):
        qa, qp = _f32(queries)
        B = qa.size // (params.query_dimension or self.dim)
        cp = params._c()
        k = cp.k
        ids = np.zeros((B, k), dtype=np.uint64)
        sc = np.zeros((B, k), dtype=np.float32)
        cnt = np.zeros(B, dtype=np.uint32)
        how = np.zeros(B, dtype=np.uint8)
        st = stats if stats is not None else SearchStats()
        _ck(fn(self.h, qp, B, C.byref(cp), *set_args, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
               sc.ctypes.data_as(C.POINTER(C.c_float)), cnt.ctypes.data_as(C.POINTER(C.c_uint32)),
               how.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(st)))
        return ids, sc, cnt, how

    def search_dense_exact_batch(self, queries, params: SearchParams, stats=None):
        """hx_search_dense_exact: hx_search_restricted's answer over every live id, through the tensor cores where the
        certificate proves it and the exact scan for the queries it cannot."""
        return self._dense_exact(self.L.hx_search_dense_exact, queries, params, (), stats)

    def search_dense_restricted_exact_batch(self, queries, params: SearchParams, allowed: RestrictedVectorCandidates,
                                            stats=None):
        """hx_search_dense_restricted_exact: the same over one candidate set shared by every query."""
        ca, cpnt = _u64(allowed.ids)
        return self._dense_exact(self.L.hx_search_dense_restricted_exact, queries, params, (cpnt, ca.size), stats)

    def search_dense_restricted_exact_sets(self, queries, params: SearchParams, device_set: "DeviceCandidates", stats=None):
        """hx_search_dense_restricted_exact_set: the same with a device-resident set (cache_candidates)."""
        return self._dense_exact(self.L.hx_search_dense_restricted_exact_set, queries, params, (device_set.h,), stats)

    # ---- device-buffer path (raw pointers, e.g. torch tensors' data_ptr()) ----
    def search_device(self, d_queries_ptr, B, params: SearchParams, d_ids_ptr, d_scores_ptr, d_counts_ptr,
                      stream_ptr=0, stats=None):
        cp = params._c()
        _ck(self.L.hx_search_device(self.h, d_queries_ptr, B, C.byref(cp), d_ids_ptr, d_scores_ptr, d_counts_ptr,
                                    stream_ptr, C.byref(stats) if stats is not None else None))

    def search_restricted_device(self, d_queries_ptr, B, params, d_slots_ptr, d_offsets_ptr, total, max_per_query,
                                 d_ids_ptr, d_scores_ptr, d_counts_ptr, stream_ptr=0):
        cp = params._c()
        _ck(self.L.hx_search_restricted_device(self.h, d_queries_ptr, B, C.byref(cp), d_slots_ptr, d_offsets_ptr,
                                               total, max_per_query, d_ids_ptr, d_scores_ptr, d_counts_ptr,
                                               stream_ptr))

    def search_dense_restricted_set_device(self, d_queries_ptr, B, params: SearchParams, device_set: "DeviceCandidates",
                                           d_ids_ptr, d_scores_ptr, d_counts_ptr, d_how_ptr=None, stream_ptr=0):
        """hx_search_dense_restricted_set_device: the tensor-core path over a resident set (make_resident), enqueued on the
        stream without synchronising.  d_how_ptr (B bytes, optional): 0 certified, 1 not certified (not rescanned), 2 exact
        scan."""
        cp = params._c()
        _ck(self.L.hx_search_dense_restricted_set_device(self.h, d_queries_ptr, B, C.byref(cp), device_set.h, d_ids_ptr,
                                                         d_scores_ptr, d_counts_ptr, d_how_ptr, stream_ptr))

    def map_candidates_device(self, d_ids_ptr, n, d_slots_ptr, stream_ptr=0):
        _ck(self.L.hx_map_candidates_device(self.h, d_ids_ptr, n, d_slots_ptr, None, stream_ptr))

    def last_kernel_ms(self):
        ms, n = C.c_float(0), C.c_uint32(0)
        _ck(self.L.hx_last_kernel_ms(self.h, C.byref(ms), C.byref(n)))
        return float(ms.value), int(n.value)


class SearchService:
    """hx_service: the reference's calling pattern (one query per call from many concurrent tasks, read_index.rs:81-101)
    served by shared launches.  ``search`` blocks; ``submit`` / ``poll`` are the async pair."""

    def __init__(self, index: VectorIndex, k: int, ef: int = 0, capacity: int = 0, max_batch: int = 0, n_streams: int = 0,
                 ctas_per_sm: int = 0, cta_warps: int = 0, rows_in_flight: int = 0, visited_log2: int = 0,
                 min_batch: int = 0, batch_window_us: int = 0, flags: int = 0):
        self.L, self.index, self.k = index.L, index, int(k)
        cfg = _ServiceConfig(int(k), int(ef), capacity, max_batch, n_streams, ctas_per_sm, cta_warps, rows_in_flight,
                             visited_log2, min_batch, batch_window_us, flags)
        h = C.c_void_p()
        _ck(self.L.hx_service_create(index.h, C.byref(cfg), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.hx_service_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def submit(self, query) -> int:
        qa, qp = _f32(query)
        if qa.size != self.index.dim:
            raise HelixDbError(HX_ERR_INVALID_DIMENSION, f"invalid dimension: expected {self.index.dim}, got {qa.size}")
        t = C.c_uint64(0)
        _ck(self.L.hx_service_submit(self.h, qp, C.byref(t)))
        return int(t.value)

    def _out(self):
        return np.zeros(self.k, dtype=np.uint64), np.zeros(self.k, dtype=np.float32), C.c_uint32(0)

    def poll(self, ticket: int):
        """None while the query is running, else the list of SearchResult (raises the query's own error)."""
        ids, sc, cnt = self._out()
        done = C.c_int32(0)
        _ck(self.L.hx_service_poll(self.h, ticket, C.byref(done), ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                   sc.ctypes.data_as(C.POINTER(C.c_float)), C.byref(cnt)))
        if not done.value:
            return None
        return [SearchResult(ids[i], sc[i]) for i in range(int(cnt.value))]

    def wait(self, ticket: int):
        ids, sc, cnt = self._out()
        _ck(self.L.hx_service_wait(self.h, ticket, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                   sc.ctypes.data_as(C.POINTER(C.c_float)), C.byref(cnt)))
        return [SearchResult(ids[i], sc[i]) for i in range(int(cnt.value))]

    def search(self, query):
        qa, qp = _f32(query)
        if qa.size != self.index.dim:
            raise HelixDbError(HX_ERR_INVALID_DIMENSION, f"invalid dimension: expected {self.index.dim}, got {qa.size}")
        ids, sc, cnt = self._out()
        _ck(self.L.hx_service_search(self.h, qp, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                     sc.ctypes.data_as(C.POINTER(C.c_float)), C.byref(cnt)))
        return [SearchResult(ids[i], sc[i]) for i in range(int(cnt.value))]

    def stats(self) -> dict:
        st = ServiceStats()
        _ck(self.L.hx_service_get_stats(self.h, C.byref(st)))
        return st.as_dict()


class RestrictedSearchService(SearchService):
    """hx_restricted_service_create: ValidatedVectorReadIndex::search_restricted's calling pattern (one query and one
    candidate set per call from many concurrent tasks, read_index.rs:92-101) served by shared exact-scan launches.
    ``allowed`` is a RestrictedVectorCandidates (ids copied at submit) or a DeviceCandidates (resident on the device; it
    must stay open until the ticket's results are out).  Answers are bit-identical to search_restricted."""

    def __init__(self, index: VectorIndex, k: int, arena_ids: int = 0, capacity: int = 0, max_batch: int = 0,
                 n_streams: int = 0, min_batch: int = 0, batch_window_us: int = 0, flags: int = 0):
        self.L, self.index, self.k = index.L, index, int(k)
        cfg = _ServiceConfig(int(k), 0, capacity, max_batch, n_streams, 0, 0, 0, 0, min_batch, batch_window_us, flags)
        h = C.c_void_p()
        _ck(self.L.hx_restricted_service_create(index.h, C.byref(cfg), int(arena_ids), C.byref(h)))
        self.h = h

    def _query(self, query):
        qa, qp = _f32(query)
        if qa.size != self.index.dim:
            raise HelixDbError(HX_ERR_INVALID_DIMENSION, f"invalid dimension: expected {self.index.dim}, got {qa.size}")
        return qa, qp

    def submit(self, query, allowed) -> int:
        qa, qp = self._query(query)
        t = C.c_uint64(0)
        if isinstance(allowed, DeviceCandidates):
            _ck(self.L.hx_service_submit_restricted_set(self.h, qp, allowed.h, C.byref(t)))
        else:
            ca, cp = _u64(allowed.ids)
            _ck(self.L.hx_service_submit_restricted(self.h, qp, cp, ca.size, C.byref(t)))
        return int(t.value)

    def search(self, query, allowed):
        qa, qp = self._query(query)
        ids, sc, cnt = self._out()
        op = (ids.ctypes.data_as(C.POINTER(C.c_uint64)), sc.ctypes.data_as(C.POINTER(C.c_float)), C.byref(cnt))
        if isinstance(allowed, DeviceCandidates):
            _ck(self.L.hx_service_search_restricted_set(self.h, qp, allowed.h, *op))
        else:
            ca, cp = _u64(allowed.ids)
            _ck(self.L.hx_service_search_restricted(self.h, qp, cp, ca.size, *op))
        return [SearchResult(ids[i], sc[i]) for i in range(int(cnt.value))]


def merge_topk_device(device, d_all_ids, d_all_scores, d_all_counts, n_shards, B, k, d_out_ids, d_out_scores,
                      d_out_counts, stream_ptr=0):
    _ck(load_library().hx_merge_topk_device(device, d_all_ids, d_all_scores, d_all_counts, n_shards, B, k, d_out_ids,
                                            d_out_scores, d_out_counts, stream_ptr))


def decode_neighbor_row(layer: int, row: bytes):
    """Decode one encoded neighbour row value (values/vectors.rs, values/vectors/neighbors.rs) -> (ids, simhash|None)."""
    L = load_library()
    buf = (C.c_uint8 * max(len(row), 1)).from_buffer_copy(row if row else b"\0")
    cap = max(len(row) // 8 + 1, 1)
    out = np.zeros(cap, dtype=np.uint64)
    cnt, sh, has = C.c_size_t(0), C.c_uint64(0), C.c_int32(0)
    _ck(L.hx_decode_neighbor_row(layer, buf, len(row), out.ctypes.data_as(C.POINTER(C.c_uint64)), cap, C.byref(cnt),
                                 C.byref(sh), C.byref(has)))
    return out[:cnt.value].tolist(), (int(sh.value) if has.value else None)


def encode_neighbor_row(layer: int, ids) -> bytes:
    L = load_library()
    a, p = _u64(ids)
    out = (C.c_uint8 * (8 * a.size + 8))()
    n = C.c_size_t(0)
    _ck(L.hx_encode_neighbor_row(layer, p, a.size, out, len(out), C.byref(n)))
    return bytes(out[:n.value])


class KeyKind(enum.IntEnum):
    """Row families of one vector index (encoding/v1/keys/vectors.rs:23-52)."""
    Other = 0
    Vector = 1
    Layer0Neighbors = 2
    UpperNeighbors = 3
    SimHash = 4
    UpperVector = 5
    Metadata = 6


class _CVectorKey(C.Structure):
    _fields_ = [("kind", C.c_int32), ("layer", C.c_uint16), ("reserved", C.c_uint16), ("index_id", C.c_uint64),
                ("order_code", C.c_uint64), ("node_id", C.c_uint64)]


@dataclass(frozen=True)
class VectorKey:
    kind: KeyKind
    index_id: int
    node_id: int = 0
    layer: int = 0
    order_code: int = 0


def parse_vector_key(key: bytes) -> VectorKey:
    """VectorKey::parse_from_slice (keys/vectors.rs:311-470) for the row families the mirror consumes."""
    L = load_library()
    buf = (C.c_uint8 * max(len(key), 1)).from_buffer_copy(key if key else b"\0")
    out = _CVectorKey()
    _ck(L.hx_parse_vector_key(buf, len(key), C.byref(out)))
    return VectorKey(KeyKind(out.kind), int(out.index_id), int(out.node_id), int(out.layer), int(out.order_code))


def encode_vector_key(key: VectorKey) -> bytes:
    L = load_library()
    ck = _CVectorKey(int(key.kind), key.layer, 0, key.index_id, key.order_code, key.node_id)
    out = (C.c_uint8 * 32)()
    n = C.c_size_t(0)
    _ck(L.hx_encode_vector_key(C.byref(ck), out, len(out), C.byref(n)))
    return bytes(out[:n.value])


def restricted_plan(n_candidates: int, dimension: int) -> str:
    """RestrictedExecutionPlan the reference would choose (restricted.rs:426-453)."""
    return "Exact" if load_library().hx_restricted_plan(n_candidates, dimension) == 0 else "FilteredGraph"


def version() -> str:
    return load_library().hx_version().decode()
