"""ctypes binding of include/easyrag_b200.h.  No CPU fallback: a missing library is an error."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ.get("EASYRAG_B200_LIB", _PKG / "_lib" / "libeasyrag_b200.so"))


class EzrError(RuntimeError):
    pass


class Bm25IndexStruct(C.Structure):
    """``ezr_bm25_index`` (include/easyrag_b200.h)."""
    _fields_ = [
        ("n_docs", C.c_int64),
        ("n_postings", C.c_int64),
        ("vocab", C.c_int32),
        ("score_type", C.c_int32),
        ("range_size", C.c_int32),
        ("n_ranges", C.c_int32),
        ("indptr", C.c_void_p),
        ("post_doc", C.c_void_p),
        ("post_w", C.c_void_p),
        ("range_off", C.c_void_p),
        ("doc_group", C.c_void_p),
        ("monotone", C.c_int32),
        ("pk_scale_log2", C.c_int32),
        ("post_pk", C.c_void_p),
        ("term_max", C.c_void_p),
    ]


F64, F32 = 0, 1
BM25_RANGE = 8192          # overwritten from ezr_bm25_range_size() when the library loads

_p, _i32, _i64, _sz, _dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t, C.c_double
_IX = C.POINTER(Bm25IndexStruct)

# name -> (restype, argtypes); every symbol declared in include/easyrag_b200.h
SIGNATURES = {
    "ezr_version": (C.c_int, []),
    "ezr_last_error": (C.c_char_p, []),
    "ezr_device_check": (C.c_int, []),
    "ezr_bm25_range_size": (C.c_int, []),
    "ezr_bm25_doc_norm": (C.c_int, [_p, _i64, _dbl, _dbl, _dbl, _dbl, _p, _p]),
    "ezr_bm25_weights": (C.c_int, [_p, _p, _p, _i32, _i64, _p, _p, _dbl, _i32, _p, _p]),
    "ezr_bm25_range_index": (C.c_int, [_p, _p, _i32, _i32, _i32, _p, _p]),
    "ezr_bm25_build_block": (C.c_int, []),
    "ezr_bm25_build_workspace": (_sz, [_i64, _i64, _i32]),
    "ezr_bm25_build_count": (C.c_int, [_p, _p, _i64, _i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _i32, _p, _sz,
                                       C.POINTER(C.c_int32), _p]),
    "ezr_bm25_build_fill": (C.c_int, [_p, _i64, _i64, _i32, _p, _p, _p, _p, _sz, _p]),
    "ezr_bm25_shard_count": (C.c_int, [_p, _p, _i32, _i32, _i32, _p, _p, _p, _p]),
    "ezr_bm25_shard_copy": (C.c_int, [_p, _p, _p, _p, _i32, _i32, _p, _p, _p]),
    "ezr_bm25_pack": (C.c_int, [_p, _p, _i64, _i32, _p, C.POINTER(C.c_int32), _p, _p]),
    "ezr_bm25_pack_f32": (C.c_int, [_p, _p, _i64, _i32, _p, C.POINTER(C.c_int32), _p, _p]),
    "ezr_bm25_term_max": (C.c_int, [_p, _p, _i32, _p, _p]),
    "ezr_bm25_set_skipping": (C.c_int, [_i32]),
    "ezr_bm25_set_plan": (C.c_int, [_i32]),
    "ezr_bm25_set_span": (C.c_int, [_i32]),
    "ezr_bm25_cand_capacity": (C.c_int, []),
    "ezr_bm25_topk_workspace": (_sz, [_IX, _i32, _i32]),
    "ezr_bm25_topk": (C.c_int, [_IX, _p, _p, _i32, _i32, _p, _i32, _p, _p, _p, _p, _sz, _p]),
    "ezr_bm25_scores": (C.c_int, [_IX, _p, _p, _i32, _p, _p]),
    "ezr_bm25_extract_caps": (C.c_int, [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "ezr_bm25_extract": (C.c_int, [_p, _p, _p, _i32, _p, _p, _p, _p, _i32, _i32, _i32, _p, _i64, _p, _dbl, _dbl,
                                   _dbl, _dbl, _i32, _p, _p, _p, _p]),
    "ezr_select_rows_workspace": (_sz, [_i32, _i64, _i32, _i32]),
    "ezr_select_rows": (C.c_int, [_p, _i32, _i32, _i64, _i64, _i32, _i32, _p, _p, _i32, _p, _p, _p, _p, _sz, _p]),
    "ezr_merge_topk_workspace": (_sz, [_i32, _i32, _i32, _i32]),
    "ezr_merge_topk": (C.c_int, [_p, _p, _i32, _i32, _i32, _i64, _i32, _p, _p, _p, _p, _sz, _p]),
    "ezr_merge_topk_parts": (C.c_int, [_p, _p, _i32, _i32, _i32, _i64, _i32, _i64, _i32, _p, _p, _p, _p]),
    "ezr_merge_sorted_parts": (C.c_int, [_p, _p, _i32, _i32, _i32, _i64, _i32, _i64, _i32, _p, _p, _p, _i64, _p]),
    "ezr_dense_topk_workspace": (_sz, [_i64, _i32, _i32, _i32]),
    "ezr_dense_topk": (C.c_int, [_p, _i64, _i32, _i64, _p, _i32, _i64, _i32, _p, _p, _i32, _p, _p, _p, _p, _sz, _p]),
    "ezr_normalize_rows": (C.c_int, [_p, _i32, _i64, _i64, _i32, _p, _i64, _p]),
    "ezr_dense_quantize_rows": (C.c_int, [_p, _i64, _i64, _i32, _p, _i64, _p, _p, _p, _p, _p]),
    "ezr_dense_s8_topk_workspace": (_sz, [_i64, _i32, _i32, _i32]),
    "ezr_dense_s8_topk": (C.c_int, [_p, _i64, _i32, _i64, _p, _i32, _i64, _i32, _p, _p, _i32, _p, _p, _p, _p, _i64,
                                    _p, _p, _p, _p, _sz, _p]),
    "ezr_dense_s8_set_capacity": (C.c_int, [_i32]),
    "ezr_dense_cand_topk_workspace": (_sz, [_i64, _i32, _i32, _i32]),
    "ezr_dense_cand_topk": (C.c_int, [_p, _i64, _i32, _i64, _p, _i32, _i64, _i32, _p, _p, _i32, _p, _p, _p, _p, _p,
                                      _sz, _p]),
    "ezr_dense_cand_set_capacity": (C.c_int, [_i32]),
    "ezr_dense_set_kernel": (C.c_int, [_i32]),
    "ezr_dense_last_kernel": (C.c_char_p, []),
    "ezr_dense_wide_workspace": (_sz, [_i64, _i32, _i32, _i32]),
    "ezr_dense_set_stage_cap": (C.c_int, [_i32]),
    "ezr_dense_set_probe": (C.c_int, [_i32]),
    "ezr_rrf_fuse": (C.c_int, [_p, _p, _p, _p, _i32, _i32, _p, _i32, _i32, _i32, _p, _p, _p, _p]),
    "ezr_gemm_bf16": (C.c_int, [_p, _i32, _i32, _i64, _p, _i32, _i64, _p, _p, _i64, _p, _i64, _i32, _p]),
    "ezr_gemm_fp8": (C.c_int, [_p, _p, _i32, _i32, _i64, _p, _p, _i32, _i64, _p, _p, _i64, _p, _i64, _i32, _p]),
    "ezr_quant_rows_fp8": (C.c_int, [_p, _i64, _i32, _i32, _p, _i64, _p, _p]),
    "ezr_quant_weight_fp8": (C.c_int, [_p, _i64, _i32, _i32, _p, _i64, _p, _p]),
    "ezr_rmsnorm_fp8": (C.c_int, [_p, _i64, _p, C.c_float, _i32, _i32, _p, _i64, _p, _i64, _p, _p]),
    "ezr_layernorm_fp8": (C.c_int, [_p, _i64, _p, _p, C.c_float, _i32, _i32, _p, _i64, _p, _i64, _p, _p]),
    "ezr_attn_bidir": (C.c_int, [_p, _i64, _i64, _p, _i32, _i32, _i32, _i32, _i32, C.c_float, _p, _i64, _p]),
    "ezr_attn_causal": (C.c_int, [_p, _i64, _i64, _p, _i32, _i32, _i32, _i32, _i32, C.c_float, _p, _i64, _p]),
    "ezr_attn_set_kernel": (C.c_int, [_i32]),
    "ezr_attn_last_kernel": (C.c_char_p, []),
    "ezr_embed_gather": (C.c_int, [_p, _i32, _p, _i64, _i32, _i32, _p, _i64, _p]),
    "ezr_bert_embed": (C.c_int, [_p, _p, _i32, _p, _p, _p, _p, _p, C.c_float, _i32, _i32, _i32, _p, _p]),
    "ezr_rmsnorm": (C.c_int, [_p, _i64, _p, C.c_float, _i32, _i32, _p, _i64, _p]),
    "ezr_layernorm": (C.c_int, [_p, _i64, _p, _p, C.c_float, _i32, _i32, _p, _i64, _p]),
    "ezr_rope": (C.c_int, [_p, _i64, _p, _p, _p, _i32, _i32, _i32, _i32, _p]),
    "ezr_pool_normalize": (C.c_int, [_p, _i64, _p, _i32, _i32, _i32, _p, C.c_float, _i32, _i32, _p, _p, _p]),
    "ezr_launch_count": (C.c_longlong, []),
    "ezr_profile_enable": (C.c_int, [_i32]),
    "ezr_profile_reset": (C.c_int, []),
    "ezr_profile_read": (C.c_int, [_i32, C.POINTER(C.c_double), C.POINTER(C.c_int32)]),
    "ezr_rerank_pack_plan": (C.c_int, [_p, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _i32, _i32, _i32, _p, _p, _p,
                                       C.POINTER(C.c_int64), _p]),
    "ezr_rerank_pack_fill": (C.c_int, [_p, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _p, _i32, _p, _i32, _i32,
                                       _i32, _p, _p, _p, _p]),
    "ezr_cross_pack_workspace": (_sz, [_i32, _i32]),
    "ezr_cross_pack_plan": (C.c_int, [_p, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _i32, _i32, _p, _p,
                                      C.POINTER(C.c_int64), _p, _sz, _p]),
    "ezr_cross_pack_fill": (C.c_int, [_p, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _i32, _i32, _i32, _i32,
                                      _i32, _i32, _p, _p, _p, _p, _p]),
    "ezr_cross_score_topk": (C.c_int, [_p, _i64, _p, _i32, _i32, _p, _i32, _p, C.c_float, _i32, _i32, _p, _p, _p, _p,
                                       _p]),
    "ezr_cross_pair_scores": (C.c_int, [_p, _i32, _i32, _p, C.c_float, _p, _p]),
    "ezr_cross_order_topk": (C.c_int, [_p, _p, _i32, _i32, _p, _i32, _i32, _p, _p, _p, _p, _p]),
    "ezr_pair_union": (C.c_int, [_p, _p, _i32, _i32, _p, _p, _i32, _i32, _i32, _p, _p, _p, _p, _p]),
    "ezr_cross_order_topk_mapped": (C.c_int, [_p, _p, _i32, _i32, _p, _i32, _p, _i32, _i32, _p, _p, _p, _p, _p]),
    "ezr_bert_embed_typed": (C.c_int, [_p, _p, _p, _i32, _p, _p, _p, _i32, _p, _p, C.c_float, _i32, _i32, _i32, _p,
                                       _p]),
    "ezr_fuse_lists": (C.c_int, [_i32, _i32, _p, _p, _p, _i32, _i32, _p, _i32, _i32, _i32, _p, _p, _p, _p]),
    "ezr_fusion_simple": (C.c_int, [_p, _p, _p, _p, _p, _p, _i32, _i32, _p, _i32, _i32, _p, _p, _p, _p]),
    "ezr_vocab_set_hash_bits": (C.c_int, [_i32]),
    "ezr_vocab_table_bytes": (_sz, [_i64]),
    "ezr_vocab_workspace": (_sz, [_i64, _i64]),
    "ezr_vocab_table_init": (C.c_int, [_p, _i64, _p]),
    "ezr_vocab_table_grow": (C.c_int, [_p, _i64, _p, _i64, _p]),
    "ezr_vocab_insert": (C.c_int, [_p, _i64, _p, _i64, _i64, _i64, _p, _i64, _p, _p, _i64, C.POINTER(C.c_int64), _p,
                                   _p, _p, _sz, _p]),
    "ezr_vocab_lookup": (C.c_int, [_p, _i64, _p, _i64, _i64, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "ezr_vocab_read": (C.c_int, [_p, _p, _i64, _i64, _p, _sz, C.POINTER(C.c_int64), _p]),
}

_lib = None


def register(sigs: dict) -> None:
    """Other modules (encoder) add their entry points before first use."""
    SIGNATURES.update(sigs)
    if _lib is not None:
        _bind(_lib, sigs)


def _bind(lib, sigs):
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)         # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise EzrError(
                f"{LIB_PATH} not found: build the CUDA extension first "
                f"(python -m easyrag_b200.build). easyrag_b200 has no CPU fallback.")
        handle = C.CDLL(str(LIB_PATH))
        _bind(handle, SIGNATURES)
        _lib = handle
        global BM25_RANGE
        BM25_RANGE = int(handle.ezr_bm25_range_size())
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().ezr_last_error().decode("utf-8", "replace")
        raise EzrError(f"{what or 'easyrag_b200'} failed (status {rc}): {msg}")


def ptr(t) -> C.c_void_p:
    """Device (or host) address of a torch tensor, None -> NULL."""
    if t is None:
        return C.c_void_p(0)
    return C.c_void_p(t.data_ptr())


def stream_ptr(stream=None) -> C.c_void_p:
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)


def require_cuda() -> None:
    """Product paths call this: there is no CPU implementation to fall back to."""
    import torch
    if not torch.cuda.is_available():
        raise EzrError("easyrag_b200 needs a CUDA device (sm_90a); no CPU fallback exists")
    check(lib().ezr_device_check(), "ezr_device_check")


PROF_SLOTS = {"bm25_cand": 8, "bm25_rescore": 9,
              "bm25_score": 0, "dense_tc": 1, "dense_simt": 2, "merge": 3, "fuse": 4,
              "enc_gemm": 5, "enc_attn": 6, "enc_other": 7,
              "dense_s8_scan": 10, "dense_s8_rescore": 11, "dense_s8_full": 12, "dense_wide": 13,
              "bm25_bound": 14, "dense_cand_gemm": 15, "dense_cand_bound": 16}


def profile_read(name: str):
    """-> (total milliseconds, launches) recorded for a kernel slot since the last reset."""
    ms, n = C.c_double(0), C.c_int32(0)
    check(lib().ezr_profile_read(PROF_SLOTS[name], C.byref(ms), C.byref(n)), "ezr_profile_read")
    return ms.value, n.value
