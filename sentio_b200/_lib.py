"""ctypes binding of libsentio_b200.so (C ABI declared in include/sentio_b200.h).

There is deliberately NO fallback: if the shared library is missing or no H100 is visible, importing the engine
raises.  The product never imports oracle/.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
# SENTIO_B200_LIB: load another build of the same sources (A/B measurements of kernel variants, python -m sentio_b200.build --variant)
LIB_PATH = Path(os.environ.get("SENTIO_B200_LIB") or _PKG / "libsentio_b200.so")

c_i64p = C.POINTER(C.c_int64)
c_i32p = C.POINTER(C.c_int32)
c_u16p = C.POINTER(C.c_uint16)
c_f32p = C.POINTER(C.c_float)
c_f64p = C.POINTER(C.c_double)


class SbCeConfig(C.Structure):
    _fields_ = [("vocab_size", C.c_int32), ("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32),
                ("intermediate", C.c_int32), ("max_pos", C.c_int32), ("type_vocab", C.c_int32), ("ln_eps", C.c_float)]


# name -> (restype, argtypes); mirrors include/sentio_b200.h one to one (tests/test_abi.py checks the header too)
SIGNATURES = {
    "sb_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "sb_destroy": (None, [C.c_void_p]),
    "sb_last_error": (C.c_char_p, []),
    "sb_version": (C.c_int, []),
    "sb_num_sms": (C.c_int, [C.c_void_p]),
    "sb_sync": (C.c_int, [C.c_void_p]),
    "sb_host_alloc": (C.c_void_p, [C.c_size_t]),
    "sb_host_free": (None, [C.c_void_p]),
    "sb_stream": (C.c_void_p, [C.c_void_p]),
    "sb_launch_count": (C.c_int64, [C.c_void_p]),
    "sb_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "sb_profile_read": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "sb_dense_load": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64]),
    "sb_dense_load_metric": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64,
                                       C.c_int32]),
    "sb_dense_metric": (C.c_int32, [C.c_void_p, C.c_int]),
    "sb_dense_load_storage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64,
                                        C.c_int32, C.c_int32]),
    "sb_dense_storage": (C.c_int32, [C.c_void_p, C.c_int]),
    "sb_dense_set_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "sb_dense_count": (C.c_int64, [C.c_void_p, C.c_int]),
    "sb_dense_dim": (C.c_int32, [C.c_void_p, C.c_int]),
    "sb_dense_topk": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    "sb_dense_topk_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "sb_dense_fetch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_void_p]),
    "sb_dense_tags_load": (C.c_int, [C.c_void_p, C.c_int, C.c_int32, C.c_void_p, C.c_int64]),
    "sb_dense_topk_filtered": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_dense_topk_filtered_dev": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p]),
    "sb_dense_fallback_count": (C.c_int64, [C.c_void_p]),
    "sb_dense_values_load": (C.c_int, [C.c_void_p, C.c_int, C.c_int32, C.c_void_p, C.c_int64]),
    "sb_dense_values_write": (C.c_int, [C.c_void_p, C.c_int, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]),
    "sb_dense_topk_where": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_dense_recommend": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                     C.c_void_p, C.c_void_p]),
    "sb_dense_groups": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_dense_group_rounds": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "sb_dense_reserve": (C.c_int, [C.c_void_p, C.c_int, C.c_int64]),
    "sb_dense_upsert": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]),
    "sb_dense_tags_write": (C.c_int, [C.c_void_p, C.c_int, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64]),
    "sb_dense_delete": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                  C.POINTER(C.c_int64)]),
    "sb_bm25_load": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                               C.c_int64, C.c_double, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double,
                               C.c_int64]),
    "sb_bm25_count": (C.c_int64, [C.c_void_p]),
    "sb_bm25_topk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                               C.c_void_p]),
    "sb_bm25_topk_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_bm25_scores": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "sb_bm25_tags_load": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]),
    "sb_bm25_topk_filtered": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_bm25_topk_filtered_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                            C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_fuse": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_int32,
                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                          C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_fuse_dev": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_int32,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                              C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_semantic_mmr": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                  C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "sb_ce_load": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(SbCeConfig)]),
    "sb_ce_score": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                              C.c_void_p]),
    "sb_ce_score_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "sb_bm25_build_tokens": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "sb_bm25_build_read": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_bm25_build_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_bm25_build_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_double, C.c_double, C.c_double,
                                       C.c_int64]),
    "sb_enc_load": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(SbCeConfig), C.c_void_p, C.c_void_p, C.c_int32]),
    "sb_enc_dim": (C.c_int32, [C.c_void_p]),
    "sb_enc_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                               C.c_void_p]),
    "sb_enc_embed_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_void_p]),
    "sb_ce_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32]),
    "sb_ce_tokens_load": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64]),
    "sb_rerank_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_ce_gemm_test": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_void_p]),
    "sb_hybrid_topk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                 C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_hybrid_topk_filtered": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_hybrid_rerank_topk": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double,
                                        C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_doc_chars_load": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64]),
    "sb_select_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sb_merge_shards_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None


class SentioB200Error(RuntimeError):
    pass


def load_library(path: os.PathLike | None = None) -> C.CDLL:
    """dlopen the C-ABI library and attach prototypes.  Raises if it has not been built (python -m sentio_b200.build)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = Path(path) if path else LIB_PATH
    if not p.exists():
        raise SentioB200Error(
            f"{p} not found: build it with `python -m sentio_b200.build` (nvcc, sm_90a). "
            "sentio_b200 has no CPU fallback.")
    lib = C.CDLL(str(p))
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == ABI drift; tests/test_abi.py guards it
        fn.restype = restype
        fn.argtypes = argtypes
    if path is None:
        _lib = lib
    return lib


class SentioB200ArgError(SentioB200Error, ValueError):
    """SB_ERR_ARG: the call rejected its input (and changed nothing)."""


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load_library().sb_last_error()
        cls = SentioB200ArgError if rc == -2 else SentioB200Error
        raise cls(f"{what} failed (rc={rc}): {msg.decode('utf-8', 'replace') if msg else '?'}")
