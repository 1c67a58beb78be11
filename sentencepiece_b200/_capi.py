"""ctypes binding of include/spm_b200.h (the C-ABI shared library built in-tree).

There is deliberately no fallback: if libspm_b200.so is missing or no H100 is
visible, loading / engine creation raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libspm_b200.so")

# every symbol include/spm_b200.h declares
EXPORTS = [
    "spm_engine_create", "spm_engine_create_from_serialized", "spm_engine_destroy", "spm_engine_set_types",
    "spm_last_error", "spm_encode_ids", "spm_encode_spans", "spm_encode_ids_device", "spm_host_alloc",
    "spm_host_free", "spm_engine_get_info", "spm_engine_set_tuning", "spm_nbest_encode", "spm_set_random_seed",
    "spm_sample_encode_ids", "spm_decode_ids", "spm_engine_set_unk_surface", "spm_calculate_entropy",
    "spm_sample_encode_and_score", "spm_engine_cache_reset", "spm_engine_set_encode_frame", "spm_encode_pieces",
    "spm_nbest_encode_pieces", "spm_sample_encode_pieces", "spm_sample_encode_and_score_pieces",
    "spm_encode_ids_device_padded", "spm_decode_ids_device", "spm_normalize", "spm_encode_offsets",
    "spm_decode_offsets", "spm_encode_offsets_device_padded", "spm_encode_windows_device", "spm_encode_pairs_device",
    "spm_decode_stream_device",
]

# spm_normalize: the n2o entry of a sentence whose reference norm_to_orig is empty
NORM_TO_ORIG_EMPTY = 0xFFFFFFFF

# spm_encode_ids_device_padded flags, and spm_encode_offsets_device_padded's character offsets
PAD_TRUNCATE, PAD_LEFT, OFFSETS_CHARS = 1, 2, 4
# spm_encode_pairs_device: truncation strategies by name, and the overflow flag
PAIR_TRUNCATION = {"none": 0, "longest_first": 1, "only_first": 2, "only_second": 3}
PAIR_OVERFLOW = 8
SPM_ERR_CAPACITY = 4
# spm_decode_stream_state: bytes per row, and the byte and bit of its done flag
STREAM_STATE_BYTES, STREAM_FLAGS_BYTE, STREAM_DONE = 16, 12, 1


class ModelDesc(ctypes.Structure):
    _fields_ = [("model_type", ctypes.c_int32), ("vocab_size", ctypes.c_int32),
                ("piece_bytes", ctypes.c_char_p), ("piece_off", ctypes.c_void_p),
                ("scores", ctypes.c_void_p), ("types", ctypes.c_void_p),
                ("byte_fallback", ctypes.c_uint8), ("treat_whitespace_as_suffix", ctypes.c_uint8),
                ("add_dummy_prefix", ctypes.c_uint8), ("remove_extra_whitespaces", ctypes.c_uint8),
                ("escape_whitespaces", ctypes.c_uint8), ("reserved_", ctypes.c_uint8 * 3),
                ("charsmap", ctypes.c_char_p), ("charsmap_bytes", ctypes.c_size_t)]


class EngineInfo(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int32), ("sm_count", ctypes.c_int32), ("model_type", ctypes.c_int32),
                ("vocab_size", ctypes.c_int32), ("unk_id", ctypes.c_int32), ("min_score", ctypes.c_float),
                ("max_score", ctypes.c_float), ("trie_units", ctypes.c_uint32), ("trie_hot_units", ctypes.c_uint32),
                ("charsmap_units", ctypes.c_uint32), ("last_kernel_launches", ctypes.c_uint64),
                ("last_kernel_ms", ctypes.c_float), ("last_main_kernel_ms", ctypes.c_float),
                ("last_h2d_bytes", ctypes.c_uint64), ("last_d2h_bytes", ctypes.c_uint64),
                ("last_deferred", ctypes.c_uint64), ("last_unk_detour", ctypes.c_uint64)]


_lib = None


def load():
    """Loads libspm_b200.so (raises if it has not been built: run __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: the CUDA engine has not been built "
                           "(python -c 'import __graft_entry__ as g; g.build()'); there is no CPU fallback")
    L = ctypes.CDLL(LIB_PATH)
    vp, cp, sz = ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t
    P = ctypes.POINTER
    L.spm_engine_create.argtypes = [P(ModelDesc), ctypes.c_int, P(vp)]
    L.spm_engine_create_from_serialized.argtypes = [cp, sz, ctypes.c_int, P(vp)]
    L.spm_engine_destroy.argtypes = [vp]
    L.spm_engine_destroy.restype = None
    L.spm_engine_set_types.argtypes = [vp, vp]
    L.spm_engine_cache_reset.argtypes = [vp]
    L.spm_engine_set_encode_frame.argtypes = [vp, vp, ctypes.c_uint32, ctypes.c_int, vp, ctypes.c_uint32]
    L.spm_last_error.argtypes = [vp]
    L.spm_last_error.restype = cp
    L.spm_encode_ids.argtypes = [vp, vp, vp, sz, P(vp), P(vp)]
    L.spm_encode_spans.argtypes = [vp, vp, vp, sz, P(vp), P(vp), P(vp), P(vp), P(vp), P(vp)]
    L.spm_normalize.argtypes = [vp, vp, vp, sz, ctypes.c_int, P(vp), P(vp), P(vp)]
    L.spm_encode_pieces.argtypes = [vp, vp, vp, sz, cp, sz, ctypes.c_int, P(vp), P(vp), P(vp), P(vp), P(vp)]
    L.spm_encode_offsets.argtypes = [vp, vp, vp, sz, ctypes.c_int32, cp, sz, ctypes.c_int] + [P(vp)] * 7
    L.spm_encode_ids_device.argtypes = [vp, vp, vp, sz, ctypes.c_uint64, vp, ctypes.c_uint64, vp,
                                        P(ctypes.c_uint64), vp]
    u32, u64 = ctypes.c_uint32, ctypes.c_uint64
    L.spm_encode_ids_device_padded.argtypes = [vp, vp, vp, sz, u64, vp, u64, u32, ctypes.c_int32, u32, vp, P(u32), vp]
    L.spm_encode_offsets_device_padded.argtypes = [vp, vp, vp, sz, u64, ctypes.c_int32, vp, vp, u64, u32, ctypes.c_int32,
                                                   u32, vp, P(u32), vp]
    L.spm_encode_windows_device.argtypes = [vp, vp, vp, sz, u64, u32, u32, ctypes.c_int32, u32, ctypes.c_int32, vp, vp,
                                            u64, vp, vp, vp, P(u64), vp]
    L.spm_encode_pairs_device.argtypes = [vp, vp, vp, sz, u64, P(ctypes.c_int32), u32, P(ctypes.c_int32), u32,
                                          P(ctypes.c_int32), u32, u32, u32, u32, ctypes.c_int32, u32, vp, vp, vp, u64,
                                          u64, vp, vp, vp, P(u64), P(u32), vp]
    L.spm_decode_ids_device.argtypes = [vp, vp, u32, u64, sz, u32, vp, ctypes.c_int64, P(vp), P(vp), vp]
    L.spm_decode_stream_device.argtypes = [vp, vp, u32, u64, sz, u32, vp, ctypes.c_int64, vp, vp, P(vp), P(vp), vp]
    L.spm_host_alloc.argtypes = [sz]
    L.spm_host_alloc.restype = vp
    L.spm_host_free.argtypes = [vp]
    L.spm_host_free.restype = None
    L.spm_engine_get_info.argtypes = [vp, P(EngineInfo)]
    L.spm_engine_set_tuning.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.spm_nbest_encode.argtypes = [vp, vp, vp, sz, ctypes.c_int, P(vp), P(vp), P(vp), P(vp)]
    L.spm_set_random_seed.argtypes = [vp, ctypes.c_uint32]
    L.spm_sample_encode_ids.argtypes = [vp, vp, vp, sz, ctypes.c_int, ctypes.c_float, P(vp), P(vp)]
    L.spm_decode_ids.argtypes = [vp, vp, vp, sz, P(vp), P(vp)]
    L.spm_decode_offsets.argtypes = [vp, vp, vp, sz, P(vp), P(vp), P(vp)]
    L.spm_engine_set_unk_surface.argtypes = [vp, cp, sz]
    L.spm_calculate_entropy.argtypes = [vp, vp, vp, sz, ctypes.c_float, P(vp)]
    L.spm_sample_encode_and_score.argtypes = [vp, vp, vp, sz, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int,
                                              P(vp), P(vp), P(vp)]
    L.spm_nbest_encode_pieces.argtypes = [vp, vp, vp, sz, ctypes.c_int, cp, sz, ctypes.c_int] + [P(vp)] * 7
    L.spm_sample_encode_pieces.argtypes = [vp, vp, vp, sz, ctypes.c_int, ctypes.c_float, cp, sz, ctypes.c_int] + [P(vp)] * 5
    L.spm_sample_encode_and_score_pieces.argtypes = [vp, vp, vp, sz, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int,
                                                     cp, sz, ctypes.c_int] + [P(vp)] * 6
    _lib = L
    return L
