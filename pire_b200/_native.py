"""ctypes binding of the C ABI in include/pire_b200.h.

The shared library is built in-tree (``make`` / ``__graft_entry__.build()``) as
pire_b200/libpire_b200.so.  There is no Python or CPU fallback for the scan
path: if the library is missing, importing this module raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpire_b200.so")

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)

RUN_ASYNC_EXCHANGE = 8
COMM_ID_BYTES = 128
RUN_BEGIN = 1
RUN_END = 2
RUN_LINES = 4
VARIANT_AUTO, VARIANT_PLAIN, VARIANT_PRED, VARIANT_PRIV, VARIANT_LOOK, VARIANT_LOOK64, VARIANT_LOOK1 = 0, 1, 2, 3, 4, 5, 6
VARIANT_LOOK_RING1 = 7
VARIANT_SLOTS = 8
VARIANT_NAMES = {VARIANT_PLAIN: "plain", VARIANT_PRED: "pred", VARIANT_PRIV: "priv", VARIANT_LOOK: "look", VARIANT_LOOK64: "look64",
                 VARIANT_LOOK1: "look1", VARIANT_LOOK_RING1: "look_ring1"}

# every symbol include/pire_b200.h declares
SYMBOLS = [
    "pire_gpu_scanner_create", "pire_gpu_scanner_destroy", "pire_gpu_scanner_info",
    "pire_gpu_scanner_set_variant", "pire_gpu_scanner_set_max_hot", "pire_gpu_run_batch",
    "pire_gpu_run_batch_host", "pire_gpu_prefix_batch", "pire_gpu_suffix_batch", "pire_gpu_count_batch", "pire_gpu_scanner_set_count_mode", "pire_gpu_length_order", "pire_gpu_run_batch_ordered", "pire_gpu_split_lines", "pire_gpu_run_lines", "pire_gpu_scanner_tune", "pire_gpu_scanner_autoselect", "pire_gpu_launch_count", "pire_gpu_initial",
    "pire_gpu_next", "pire_gpu_final", "pire_gpu_dead", "pire_gpu_accepted_regexps",
    "pire_gpu_synth_fill_device", "pire_gpu_synth_fill_host", "pire_gpu_synth_mixed_lengths_device",
    "pire_gpu_synth_mixed_lengths_host", "pire_gpu_synth_mixed_fill_device", "pire_gpu_synth_mixed_fill_host",
    "pire_gpu_last_error", "pire_gpu_version",
    "pire_gpu_accept_words", "pire_gpu_accept_sets", "pire_gpu_synth_fill_host_indexed",
    "pire_gpu_shard_bounds", "pire_gpu_sharded_words", "pire_gpu_comm_get_id", "pire_gpu_comm_create",
    "pire_gpu_comm_adopt", "pire_gpu_comm_destroy", "pire_gpu_comm_info", "pire_gpu_comm_wait", "pire_gpu_run_sharded", "pire_gpu_comm_gather_bits",
    "pire_gpu_run_string", "pire_gpu_run_batch_from", "pire_gpu_count_string", "pire_gpu_count_batch_from",
    "pire_gpu_match_ends_string", "pire_gpu_match_ends_batch_from",
    "pire_gpu_match_starts_string", "pire_gpu_match_starts_batch", "pire_gpu_run_pair_batch",
    "pire_gpu_match_ends_lines", "pire_gpu_match_starts_lines",
    "pire_gpu_line_stream_create", "pire_gpu_line_stream_feed", "pire_gpu_line_stream_destroy",
    "pire_gpu_run_pair_lines",
    "pire_gpu_slow_scanner_create", "pire_gpu_slow_scanner_destroy", "pire_gpu_slow_scanner_info", "pire_gpu_slow_run_batch",
    "pire_gpu_slow_initial", "pire_gpu_slow_next", "pire_gpu_slow_final",
]


class Info(C.Structure):
    _fields_ = [("states", C.c_uint32), ("letters", C.c_uint32), ("regexps", C.c_uint32), ("initial", C.c_uint32),
                ("empty", C.c_uint32), ("hot_rows", C.c_uint32), ("variant", C.c_uint32), ("tuned", C.c_uint32),
                ("table_bytes", C.c_uint64), ("shared_bytes", C.c_uint64), ("device", C.c_int32),
                ("reserved", C.c_uint32)]


class SlowInfo(C.Structure):
    _fields_ = [("states", C.c_uint32), ("letters", C.c_uint32), ("regexps", C.c_uint32), ("set_words", C.c_uint32),
                ("start", C.c_uint32), ("empty", C.c_uint32), ("table_bytes", C.c_uint64), ("shared_bytes", C.c_uint64),
                ("device", C.c_int32), ("reserved", C.c_uint32)]


class LineFrame(C.Structure):
    _fields_ = [("d_text", C.c_void_p), ("d_line_offsets", C.c_void_p), ("n_lines", C.c_uint64), ("n_bytes", C.c_uint64),
                ("first_line", C.c_uint64), ("first_byte", C.c_uint64)]


class Synth(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("first_string", C.c_uint64), ("n_strings", C.c_uint64),
                ("string_len", C.c_uint32), ("kind", C.c_uint32), ("plant_every", C.c_uint32),
                ("n_plants", C.c_uint32), ("plants", C.c_char_p), ("plants_bytes", C.c_uint32), ("tail", C.c_uint32)]


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "pire_b200: %s is missing. Build it with `make` (or __graft_entry__.build()); "
            "the scan path is CUDA-only and has no fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    lib.pire_gpu_scanner_create.argtypes = [vp, C.c_size_t, C.c_int, C.POINTER(vp)]
    lib.pire_gpu_scanner_destroy.argtypes = [vp]
    lib.pire_gpu_scanner_destroy.restype = None
    lib.pire_gpu_scanner_info.argtypes = [vp, C.POINTER(Info)]
    lib.pire_gpu_scanner_set_variant.argtypes = [vp, C.c_uint32]
    lib.pire_gpu_scanner_set_max_hot.argtypes = [vp, C.c_uint32]
    lib.pire_gpu_run_batch.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp]
    lib.pire_gpu_run_string.argtypes = [vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp]
    lib.pire_gpu_run_batch_from.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp]
    lib.pire_gpu_run_pair_batch.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.pire_gpu_run_pair_lines.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp, vp, vp]
    lib.pire_gpu_run_batch_host.argtypes = [vp, vp, C.c_uint64, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp]
    lib.pire_gpu_prefix_batch.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, vp, vp]
    lib.pire_gpu_suffix_batch.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, vp, vp]
    lib.pire_gpu_scanner_set_count_mode.argtypes = [vp, C.c_uint32]
    lib.pire_gpu_count_batch.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp]
    lib.pire_gpu_count_string.argtypes = [vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp]
    lib.pire_gpu_count_batch_from.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp]
    lib.pire_gpu_match_ends_string.argtypes = [vp, vp, C.c_uint64, C.c_uint32, vp, C.c_uint64, vp, vp, C.c_uint64, vp, vp, vp, vp]
    lib.pire_gpu_match_ends_batch_from.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp, C.c_uint64, vp,
                                                   vp, vp, vp]
    lib.pire_gpu_match_starts_string.argtypes = [vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint64, vp, vp, vp, vp,
                                                 C.c_uint64, vp, vp, vp]
    lib.pire_gpu_match_starts_batch.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, vp, C.c_uint32, C.c_uint64, vp, vp, vp, vp,
                                                vp, C.c_uint64, vp, vp, vp]
    lib.pire_gpu_match_ends_lines.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, C.c_uint64, vp, vp, vp, vp]
    lib.pire_gpu_match_starts_lines.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint32, C.c_uint64, vp, vp, vp, vp, vp, C.c_uint64,
                                                vp, vp, vp]
    lib.pire_gpu_line_stream_create.argtypes = [C.c_int, C.c_uint64, C.POINTER(vp)]
    lib.pire_gpu_line_stream_feed.argtypes = [vp, vp, C.c_uint64, C.c_int, vp, C.POINTER(C.c_uint64), C.POINTER(LineFrame)]
    lib.pire_gpu_line_stream_destroy.argtypes = [vp]
    lib.pire_gpu_line_stream_destroy.restype = None
    lib.pire_gpu_length_order.argtypes = [vp, C.c_uint64, vp, C.c_int, vp]
    lib.pire_gpu_run_batch_ordered.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, vp]
    lib.pire_gpu_split_lines.argtypes = [vp, C.c_uint64, vp, C.c_uint64, C.POINTER(C.c_uint64), C.c_int, vp]
    lib.pire_gpu_run_lines.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp, vp]
    lib.pire_gpu_scanner_tune.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp]
    lib.pire_gpu_scanner_autoselect.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, C.POINTER(C.c_float)]
    lib.pire_gpu_launch_count.restype = C.c_uint64
    lib.pire_gpu_initial.argtypes = [vp]
    lib.pire_gpu_initial.restype = C.c_uint32
    lib.pire_gpu_next.argtypes = [vp, C.c_uint32, C.c_uint32]
    lib.pire_gpu_next.restype = C.c_uint32
    lib.pire_gpu_final.argtypes = [vp, C.c_uint32]
    lib.pire_gpu_dead.argtypes = [vp, C.c_uint32]
    lib.pire_gpu_accepted_regexps.argtypes = [vp, C.c_uint32, u32p, C.c_size_t]
    lib.pire_gpu_accepted_regexps.restype = C.c_size_t
    lib.pire_gpu_synth_fill_device.argtypes = [C.POINTER(Synth), vp, C.c_int, vp]
    lib.pire_gpu_synth_fill_host.argtypes = [C.POINTER(Synth), vp, C.c_uint64, C.c_uint64]
    lib.pire_gpu_synth_mixed_lengths_device.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, vp, C.c_int, vp]
    lib.pire_gpu_synth_mixed_lengths_host.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, vp]
    lib.pire_gpu_synth_mixed_fill_device.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, vp, vp, C.c_int, vp]
    lib.pire_gpu_synth_mixed_fill_host.argtypes = [C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, vp, vp]
    lib.pire_gpu_last_error.restype = C.c_char_p
    lib.pire_gpu_version.restype = C.c_char_p
    lib.pire_gpu_accept_words.argtypes = [vp]
    lib.pire_gpu_accept_words.restype = C.c_uint32
    lib.pire_gpu_accept_sets.argtypes = [vp, vp, C.c_uint64, vp, vp]
    lib.pire_gpu_synth_fill_host_indexed.argtypes = [C.POINTER(Synth), vp, vp, C.c_uint64]
    lib.pire_gpu_shard_bounds.argtypes = [C.c_uint64, C.c_int, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.pire_gpu_shard_bounds.restype = None
    lib.pire_gpu_sharded_words.argtypes = [C.c_uint64, C.c_int]
    lib.pire_gpu_sharded_words.restype = C.c_uint64
    lib.pire_gpu_comm_get_id.argtypes = [vp]
    lib.pire_gpu_comm_create.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    lib.pire_gpu_comm_adopt.argtypes = [vp, C.c_int, C.POINTER(vp)]
    lib.pire_gpu_comm_destroy.argtypes = [vp]
    lib.pire_gpu_comm_destroy.restype = None
    lib.pire_gpu_comm_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.pire_gpu_comm_wait.argtypes = [vp, vp]
    lib.pire_gpu_comm_gather_bits.argtypes = [vp, C.c_uint64, vp, C.c_uint32, vp]
    lib.pire_gpu_run_sharded.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp]
    lib.pire_gpu_slow_scanner_create.argtypes = [vp, C.c_size_t, C.c_int, C.POINTER(vp)]
    lib.pire_gpu_slow_scanner_destroy.argtypes = [vp]
    lib.pire_gpu_slow_scanner_destroy.restype = None
    lib.pire_gpu_slow_scanner_info.argtypes = [vp, C.POINTER(SlowInfo)]
    lib.pire_gpu_slow_run_batch.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp]
    lib.pire_gpu_slow_initial.argtypes = [vp, vp]
    lib.pire_gpu_slow_next.argtypes = [vp, vp, C.c_uint32, vp]
    lib.pire_gpu_slow_final.argtypes = [vp, vp]
    return lib


lib = _load()


class PireGpuError(RuntimeError):
    """Mirror of Pire::Error (pire/stub/stl.h:213-217) for the C ABI's status codes."""

    def __init__(self, code, where):
        self.code = code
        msg = lib.pire_gpu_last_error()
        super().__init__("%s failed (%d): %s" % (where, code, msg.decode(errors="replace") if msg else ""))


def check(rc, where):
    if rc != 0:
        raise PireGpuError(rc, where)
