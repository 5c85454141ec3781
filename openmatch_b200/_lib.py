"""ctypes binding of libopenmatch_b200.so (C ABI declared in include/openmatch_b200.h).

There is no CPU fallback: if the shared library is missing this module raises at import of the symbol
table, and every compute entry point raises RuntimeError when no sm_90 device is present.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OPENMATCH_B200_LIB") or os.path.join(_HERE, "lib", "libopenmatch_b200.so")

OM_F32, OM_BF16, OM_F16, OM_I8 = 0, 1, 2, 3
OM_HOST, OM_DEVICE = 0, 1
OM_ARCH_BERT, OM_ARCH_T5ENC, OM_ARCH_ROBERTA, OM_ARCH_MPNET, OM_ARCH_DISTILBERT = 0, 1, 2, 3, 4
OM_POOL_FIRST, OM_POOL_MEAN = 0, 1
OM_REDUCE_MEAN, OM_REDUCE_SUM = 0, 1


class EncoderDesc(ctypes.Structure):
    _fields_ = [("arch", c_int32), ("layers", c_int32), ("hidden", c_int32), ("heads", c_int32), ("ffn", c_int32),
                ("vocab", c_int32), ("max_pos", c_int32), ("type_vocab", c_int32), ("ln_eps", c_float),
                ("pooling", c_int32), ("has_head", c_int32), ("head_out", c_int32), ("normalize", c_int32),
                ("rel_buckets", c_int32), ("rel_max_distance", c_int32), ("max_batch_tokens", c_int32)]


class SearchFilter(ctypes.Structure):
    """om_search_filter: device pointers (0 = absent) of the allowed-row bitmap and of the exclusion CSR."""
    _fields_ = [("allow_bits", c_void_p), ("allow_words", c_int64), ("exclude_offsets", c_void_p),
                ("exclude_ids", c_void_p)]


# name -> (restype, argtypes); must list every symbol of include/openmatch_b200.h
SIGNATURES = {
    "om_abi_version": (c_int, []),
    "om_last_error": (c_char_p, []),
    "om_device_sm_count": (c_int, []),
    "om_encoder_create": (c_int, [POINTER(EncoderDesc), POINTER(c_void_p)]),
    "om_encoder_set_weight": (c_int, [c_void_p, c_char_p, c_void_p, c_int, POINTER(c_int64), c_int]),
    "om_encoder_finalize": (c_int, [c_void_p]),
    "om_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int64, c_void_p,
                          c_void_p]),
    "om_encode_packed": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int64, c_void_p,
                                 c_void_p]),
    "om_encode_pairs": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int, c_void_p, c_int,
                                c_void_p, c_int, c_void_p, c_int, c_int64, c_void_p]),
    "om_encoder_rep_dim": (c_int, [c_void_p]),
    "om_encoder_destroy": (None, [c_void_p]),
    "om_index_create": (c_int, [c_int, POINTER(c_void_p)]),
    "om_index_create_typed": (c_int, [c_int, c_int, POINTER(c_void_p)]),
    "om_index_create_host": (c_int, [c_int, c_int, c_int64, POINTER(c_void_p)]),
    "om_index_storage": (c_int, [c_void_p]),
    "om_index_reserve_rows": (c_int, [c_void_p, c_int64, POINTER(c_void_p), POINTER(c_int64)]),
    "om_index_add": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p]),
    "om_index_reserve": (c_int, [c_void_p, c_int64, POINTER(c_void_p)]),
    "om_index_commit": (c_int, [c_void_p, c_int64, c_void_p]),
    "om_index_ntotal": (c_int64, [c_void_p]),
    "om_index_dim": (c_int, [c_void_p]),
    "om_index_reset": (c_int, [c_void_p]),
    "om_index_search": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int64,
                                c_void_p]),
    "om_comm_unique_id": (c_int, [c_void_p]),
    "om_comm_init": (c_int, [c_void_p, c_int, c_int, POINTER(c_void_p)]),
    "om_comm_destroy": (None, [c_void_p]),
    "om_index_search_sharded": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                        c_int64, c_void_p]),
    "om_index_search_filtered": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int64,
                                         POINTER(SearchFilter), c_void_p]),
    "om_index_search_sharded_filtered": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                                 c_int, c_int64, POINTER(SearchFilter), c_void_p]),
    "om_index_range_search": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "om_index_range_search_sharded": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                                              c_int64, c_void_p]),
    "om_index_range_search_filtered": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int64,
                                               POINTER(SearchFilter), c_void_p]),
    "om_index_range_search_sharded_filtered": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                                       c_int, c_int64, POINTER(SearchFilter), c_void_p]),
    "om_index_range_results": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "om_index_set_param": (c_int, [c_void_p, c_char_p, c_int64]),
    "om_index_get_stat": (c_int64, [c_void_p, c_char_p]),
    "om_index_destroy": (None, [c_void_p]),
    "om_topk_merge_n": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "om_contrastive_loss_fwd_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_float,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "om_debug_loss_phase_ns": (c_int, [c_void_p]),
}

_lib = None


def load():
    """Loads the shared library once; raises RuntimeError with build instructions if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libopenmatch_b200.so is not built (%s). Run `python -m openmatch_b200.build` (needs nvcc); "
            "openmatch_b200 has no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch
        fn.restype = res
        fn.argtypes = args
    if lib.om_abi_version() != 2:
        raise RuntimeError("libopenmatch_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int) -> int:
    if rc < 0:
        msg = load().om_last_error()
        raise RuntimeError("openmatch_b200: %s (code %d)" % (msg.decode() if msg else "unknown error", rc))
    return rc


def current_stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
