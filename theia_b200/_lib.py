"""ctypes binding of the C ABI declared in include/theia_tad.h.

There is NO CPU fallback: if the CUDA library is missing the import of the engine fails
loudly, and ``tad_init`` fails when no GPU is visible.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libtheia_tad.so")

TAD_NPHASES = 10
PHASE_NAMES = ("h2d", "hist", "scan", "scatter", "exchange", "group", "spill", "detect", "d2h", "sync")
ALGOS = {"EWMA": 0, "ARIMA": 1, "DBSCAN": 2}
STATE_NAMES = ("NEW", "SCHEDULED", "RUNNING", "COMPLETED", "FAILED")
TAD_MEM_HOST, TAD_MEM_DEVICE = 0, 1
TAD_FLAG_EMIT_ALL, TAD_FLAG_PROFILE, TAD_FLAG_SHARE, TAD_FLAG_FIT_BESIDE, TAD_FLAG_LEND = 1, 2, 4, 8, 16
TAD_FLAG_RANK_STREAM = 32
TAD_REDUCE_MAX, TAD_REDUCE_SUM = 0, 1

EXPORTS = ("tad_abi_version", "tad_strerror", "tad_init", "tad_shutdown", "tad_alloc_columns",
           "tad_free_columns", "tad_submit", "tad_poll", "tad_wait", "tad_result", "tad_cancel",
           "tad_release", "tad_get_unique_id", "tad_alloc_ns_columns", "tad_ch_string_index", "tad_ch_parse_ipv4",
           "tad_ch_format_ipv4", "tad_ch_dictionary", "tad_set_memory_budget", "tad_job_memory", "tad_submit_stream",
           "tad_stream_push", "tad_stream_end", "tad_set_host_budget", "tad_job_host_memory",
           "tad_stream_push_text", "tad_job_names", "tad_ch_format_names", "tad_submit_stream_filtered", "tad_job_progress",
           "tad_set_fit_sharing", "tad_job_yields", "tad_submit_stream_filtered_ns", "tad_stream_push_text_ns",
           "tad_job_lent")
TAD_NAME_OPS = {"any": 0, "eq": 1, "nonempty": 2, "icontains": 3}


class TadConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("world_size", C.c_int32), ("rank", C.c_int32), ("flags", C.c_uint32),
                ("nccl_unique_id", C.c_void_p), ("nccl_unique_id_bytes", C.c_size_t)]


class TadColumns(C.Structure):
    _fields_ = [("rows", C.c_uint64), ("capacity", C.c_uint64), ("mem", C.c_int32), ("reserved", C.c_int32),
                ("src_ip", C.c_void_p), ("dst_ip", C.c_void_p), ("src_port", C.c_void_p), ("dst_port", C.c_void_p),
                ("proto", C.c_void_p), ("flow_start", C.c_void_p), ("flow_end", C.c_void_p), ("value", C.c_void_p),
                ("src_ns", C.c_void_p), ("dst_ns", C.c_void_p)]


class TadTextColumn(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("nbytes", C.c_uint64), ("marks", C.c_void_p)]


class TadStreamFilter(C.Structure):
    _fields_ = [("op", C.c_int32 * 2), ("pattern", C.c_void_p * 2), ("pattern_len", C.c_uint32 * 2), ("proto_eq", C.c_int32)]


class TadStreamFilterNs(C.Structure):
    _fields_ = [("rows", TadStreamFilter), ("n_ns_ignore", C.c_uint32), ("ns_ignore_bytes", C.c_void_p),
                ("ns_ignore_offsets", C.c_void_p)]


class TadJobSpec(C.Structure):
    _fields_ = [("algo", C.c_int32), ("reducer", C.c_int32), ("start_time", C.c_uint32), ("end_time", C.c_uint32),
                ("flags", C.c_uint32), ("n_ns_ignore", C.c_uint32), ("ns_ignore", C.c_void_p), ("id", C.c_char * 40),
                ("global_rows", C.c_uint64)]


class TadStatus(C.Structure):
    _fields_ = [("state", C.c_int32), ("completed_stages", C.c_int32), ("total_stages", C.c_int32), ("error", C.c_int32),
                ("err_msg", C.c_char * 256), ("rows_in", C.c_uint64), ("rows_kept", C.c_uint64), ("rows_owned", C.c_uint64),
                ("points", C.c_uint64), ("series", C.c_uint64), ("result_rows", C.c_uint64), ("spill_rows", C.c_uint64),
                ("gpu_launches", C.c_uint64), ("device_ms", C.c_double), ("total_ms", C.c_double),
                ("phase_ms", C.c_double * TAD_NPHASES)]


class TadProgress(C.Structure):
    _fields_ = [("passes_done", C.c_uint32), ("passes", C.c_uint32), ("fits_done", C.c_uint64), ("fits_total", C.c_uint64)]


class TadRows(C.Structure):
    _fields_ = [("rows", C.c_uint64), ("src_ip", C.c_void_p), ("dst_ip", C.c_void_p), ("src_port", C.c_void_p),
                ("dst_port", C.c_void_p), ("proto", C.c_void_p), ("flow_start", C.c_void_p), ("flow_end", C.c_void_p),
                ("stddev", C.c_void_p), ("algo_calc", C.c_void_p), ("throughput", C.c_void_p), ("anomaly", C.c_void_p)]


_lib = None


def load():
    """Load libtheia_tad.so (built in-tree by theia_b200.build).  Raises if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "theia_b200: %s not found -- build it with `python -m theia_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.tad_abi_version.restype = C.c_int
    L.tad_strerror.restype = C.c_char_p
    L.tad_strerror.argtypes = [C.c_int]
    L.tad_init.argtypes = [C.POINTER(TadConfig), C.POINTER(C.c_void_p)]
    L.tad_shutdown.argtypes = [C.c_void_p]
    L.tad_shutdown.restype = None
    L.tad_alloc_columns.argtypes = [C.c_void_p, C.c_uint64, C.c_int32, C.POINTER(TadColumns)]
    L.tad_free_columns.argtypes = [C.c_void_p, C.POINTER(TadColumns)]
    L.tad_alloc_ns_columns.argtypes = [C.c_void_p, C.POINTER(TadColumns)]
    L.tad_submit.argtypes = [C.c_void_p, C.POINTER(TadJobSpec), C.POINTER(TadColumns), C.POINTER(C.c_void_p)]
    L.tad_submit_stream.argtypes = [C.c_void_p, C.POINTER(TadJobSpec), C.c_uint64, C.POINTER(C.c_void_p)]
    L.tad_submit_stream_filtered.argtypes = [C.c_void_p, C.POINTER(TadJobSpec), C.c_uint64, C.POINTER(TadStreamFilter),
                                             C.POINTER(C.c_void_p)]
    L.tad_submit_stream_filtered_ns.argtypes = [C.c_void_p, C.POINTER(TadJobSpec), C.c_uint64, C.POINTER(TadStreamFilterNs),
                                                C.POINTER(C.c_void_p)]
    L.tad_debug_name_match.argtypes = [C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    L.tad_debug_ns_match.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64]
    L.tad_debug_name_hash.restype = C.c_uint64
    L.tad_debug_name_hash.argtypes = [C.c_void_p, C.c_uint32]
    L.tad_debug_text_dict_new.argtypes = [C.c_int, C.c_uint32, C.c_uint64, C.POINTER(C.c_void_p)]
    L.tad_debug_text_dict_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint64,
                                             C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
    L.tad_debug_text_dict_grow.argtypes = [C.c_void_p, C.c_uint32]
    L.tad_debug_text_dict_freeze.argtypes = [C.c_void_p]
    L.tad_debug_text_dict_names.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_void_p,
                                            C.c_void_p, C.c_void_p]
    L.tad_debug_text_dict_free.argtypes = [C.c_void_p]
    L.tad_debug_ns_match_device.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p,
                                            C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64,
                                            C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]
    L.tad_stream_push.argtypes = [C.c_void_p, C.POINTER(TadColumns)]
    L.tad_stream_end.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    L.tad_stream_push_text.argtypes = [C.c_void_p, C.POINTER(TadColumns), C.POINTER(TadTextColumn), C.POINTER(TadTextColumn)]
    L.tad_stream_push_text_ns.argtypes = [C.c_void_p, C.POINTER(TadColumns)] + [C.POINTER(TadTextColumn)] * 4
    L.tad_job_names.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]
    L.tad_poll.argtypes = [C.c_void_p, C.POINTER(TadStatus)]
    L.tad_wait.argtypes = [C.c_void_p, C.c_int64, C.POINTER(TadStatus)]
    L.tad_result.argtypes = [C.c_void_p, C.POINTER(TadRows)]
    L.tad_cancel.argtypes = [C.c_void_p]
    L.tad_release.argtypes = [C.c_void_p]
    L.tad_get_unique_id.argtypes = [C.c_void_p, C.c_size_t]
    L.tad_debug_loopback_id.argtypes = [C.c_int, C.c_void_p, C.c_size_t]
    L.tad_debug_loopback_release.argtypes = [C.c_void_p, C.c_size_t]
    L.tad_job_progress.argtypes = [C.c_void_p, C.POINTER(TadProgress)]
    L.tad_set_memory_budget.argtypes = [C.c_void_p, C.c_uint64]
    L.tad_job_memory.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
    L.tad_set_fit_sharing.argtypes = [C.c_void_p, C.c_uint64]
    L.tad_job_yields.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_double)]
    L.tad_job_lent.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_double)]
    L.tad_set_host_budget.argtypes = [C.c_void_p, C.c_uint64]
    L.tad_job_host_memory.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.tad_ch_string_index.argtypes = [C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)]
    L.tad_ch_parse_ipv4.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    L.tad_ch_format_ipv4.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.tad_ch_format_names.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_size_t,
                                      C.POINTER(C.c_size_t)]
    L.tad_ch_dictionary.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]
    _lib = L
    return L
