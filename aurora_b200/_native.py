"""ctypes binding of libaurora_b200.so (include/aurora_b200.h).

There is no Python / CPU implementation behind these names: if the shared library is
missing or fails to load, importing the engine raises -- loudly, with the build command.
"""

from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("AURORA_B200_LIB") or os.path.join(HERE, "libaurora_b200.so")   # override: A/B kernel builds

ABI_VERSION = 3         # must equal AUR_ABI_VERSION of the library that gets loaded (struct layouts below)
AUR_OK = 0
AUR_ERR_INVALID, AUR_ERR_CUDA, AUR_ERR_NOMEM, AUR_ERR_UNSUPPORTED, AUR_ERR_NO_DEVICE = -1, -2, -3, -4, -5
AUR_BF16, AUR_F32, AUR_I8 = 0, 1, 2
KERNEL_AUTO, KERNEL_SIMT, KERNEL_TC1, KERNEL_TC2, KERNEL_LIST = 0, 1, 2, 3, 4
KERNEL_NAMES = {0: "auto", 1: "simt", 2: "wgmma-cta1", 3: "wgmma-cluster2", 4: "list"}
FILTER_LEAF, FILTER_AND, FILTER_OR = 0, 1, 2   # filter program tokens (AUR_FILTER_*)
FUSION_RANKED, FUSION_RELATIVE_SCORE = 0, 1    # aur_hybrid_search's fusion (AUR_FUSION_*)
TC_QUERY_ROWS = 64   # queries per CTA of the tensor-core kernel (kTcQRows, csrc/internal.h): the debug-score row count

# every symbol include/aurora_b200.h declares (tests check the .so exports all of them)
EXPORTS = [
    "aur_abi_version", "aur_last_error", "aur_device_count", "aur_open", "aur_close", "aur_get_stats",
    "aur_set_option", "aur_sync", "aur_add", "aur_add_dev", "aur_export", "aur_read_rows", "aur_live_bits", "aur_export_rows", "aur_compact", "aur_reserve", "aur_remove", "aur_search", "aur_search_ex", "aur_search_subset", "aur_search_lists", "aur_set_attrs", "aur_search_filtered", "aur_filter_ids", "aur_filter_count", "aur_remove_filtered", "aur_search_dev",
    "aur_merge_topk_dev", "aur_merge_topk_packed_dev", "aur_merge_topk_host", "aur_merge_topk_host_f64", "aur_exchange_create", "aur_exchange_connect", "aur_exchange_close",
    "aur_exchange_status", "aur_search_exchange_dev", "aur_cosine_pairs", "aur_dev_malloc", "aur_dev_free", "aur_memcpy_h2d", "aur_memcpy_d2h",
    "aur_debug_tc_scores", "aur_debug_simt_scores", "aur_debug_list_scores",
    "aur_kw_open", "aur_kw_close", "aur_kw_reserve", "aur_kw_add", "aur_kw_remove", "aur_kw_compact", "aur_kw_get_stats", "aur_kw_set_attrs",
    "aur_kw_search", "aur_kw_search_multi", "aur_kw_reindex", "aur_kw_set_option", "aur_kw_get_index_stats",
    "aur_kw_read_rows", "aur_kw_vocab_open", "aur_kw_vocab_close", "aur_kw_vocab_size", "aur_kw_vocab_read",
    "aur_kw_vocab_set_option", "aur_kw_add_text",
    "aur_hybrid_search", "aur_hybrid_search_multi", "aur_hybrid_search_filtered",
    "aur_encoder_open", "aur_encoder_close", "aur_encoder_load", "aur_encode", "aur_encode_append",
    "aur_encoder_replicate", "aur_encode_append_multi", "aur_encode_texts", "aur_encode_pair_cosines", "aur_encode_append_texts_multi", "aur_encoder_get_stats", "aur_tokenizer_open", "aur_tokenizer_open_mem", "aur_tokenizer_close", "aur_tokenizer_info",
    "aur_tokenize", "aur_tokenize_windows", "aur_encode_text_append", "aur_debug_gemm", "aur_debug_attention", "aur_debug_encoder_hidden",
]


class AurConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("dim", C.c_int32), ("dtype", C.c_int32), ("reserved", C.c_int32),
                ("capacity", C.c_int64)]


class AurStats(C.Structure):
    _fields_ = [("rows", C.c_int64), ("live", C.c_int64), ("capacity", C.c_int64), ("dim", C.c_int32),
                ("dtype", C.c_int32), ("last_kernel", C.c_int32), ("last_launches", C.c_int32),
                ("last_kernel_ms", C.c_float), ("last_total_ms", C.c_float), ("last_finalize_ms", C.c_float),
                ("last_merge_ms", C.c_float), ("last_candidates", C.c_int64), ("last_candidates_max", C.c_int32),
                ("last_tile_n", C.c_int32)]


class AurKwStats(C.Structure):
    _fields_ = [("docs", C.c_int64), ("live", C.c_int64), ("capacity", C.c_int64), ("postings_used", C.c_int64),
                ("postings_allocated", C.c_int64), ("total_len", C.c_int64), ("last_launches", C.c_int32),
                ("last_ms", C.c_float), ("last_terms", C.c_int32), ("last_spilled", C.c_int32)]


class AurKwIndexStats(C.Structure):
    _fields_ = [("indexed_rows", C.c_int64), ("index_postings", C.c_int64), ("index_bytes", C.c_int64),
                ("builds", C.c_int64), ("last_build_ms", C.c_float), ("last_path", C.c_int32),
                ("last_postings", C.c_int64)]


KW_PATH_FORWARD, KW_PATH_INDEX = 1, 2   # AUR_KW_PATH_* bits of AurKwIndexStats.last_path
KW_PATH_AUTO_OPT, KW_PATH_FORWARD_OPT, KW_PATH_INDEX_OPT = 0, 1, 2   # aur_kw_set_option "kw_path" values


class AurEncoderConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32),
                ("inter", C.c_int32), ("vocab", C.c_int32), ("max_pos", C.c_int32), ("type_vocab", C.c_int32),
                ("pool", C.c_int32), ("normalize", C.c_int32), ("max_tokens", C.c_int32), ("max_seqs", C.c_int32),
                ("ln_eps", C.c_float), ("reserved", C.c_int32)]


class AurEncoderStats(C.Structure):
    _fields_ = [("tokens", C.c_int64), ("seqs", C.c_int64), ("launches", C.c_int32), ("total_ms", C.c_float),
                ("gemm_ms", C.c_float), ("attn_ms", C.c_float), ("gemm_flops", C.c_double), ("attn_flops", C.c_double)]


class NativeLibraryMissing(RuntimeError):
    pass


class AuroraError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"aurora_b200 error {code}: {message}")
        self.code = code


_lib = None


def load():
    """Load the CUDA library.  Never falls back to anything else."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryMissing(
            f"{LIB_PATH} not found. Build it with `python -m aurora_b200.build` (needs nvcc, targets sm_90a). "
            "aurora_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    sigs = {
        "aur_abi_version": (C.c_int, []),
        "aur_last_error": (C.c_char_p, []),
        "aur_device_count": (C.c_int, []),
        "aur_open": (C.c_int, [C.POINTER(AurConfig), C.POINTER(vp)]),
        "aur_close": (C.c_int, [vp]),
        "aur_get_stats": (C.c_int, [vp, C.POINTER(AurStats)]),
        "aur_set_option": (C.c_int, [vp, C.c_char_p, i64]),
        "aur_sync": (C.c_int, [vp]),
        "aur_add": (C.c_int, [vp, vp, vp, vp, vp, i64]),
        "aur_add_dev": (C.c_int, [vp, vp, vp, vp, vp, i64, vp]),
        "aur_export": (C.c_int, [vp, vp, vp, vp, vp, vp, i64]),
        "aur_remove": (C.c_int, [vp, vp, i64, C.POINTER(i64)]),
        "aur_compact": (C.c_int, [vp, C.POINTER(i64)]),
        "aur_reserve": (C.c_int, [vp, i64]),
        "aur_read_rows": (C.c_int, [vp, i64, i64, vp, vp]),
        "aur_live_bits": (C.c_int, [vp, vp, vp, i64, C.POINTER(i64), C.POINTER(i64)]),
        "aur_export_rows": (C.c_int, [vp, i64, i64, vp, vp, vp, vp]),
        "aur_search_ex": (C.c_int, [vp, vp, i32, i32, vp, vp, vp, vp, C.POINTER(i64)]),
        "aur_search_subset": (C.c_int, [vp, vp, i32, i32, vp, i64, vp, vp]),
        "aur_search_lists": (C.c_int, [vp, vp, i32, i32, vp, vp, i32, vp, vp, vp, C.POINTER(i64)]),
        "aur_search": (C.c_int, [vp, vp, i32, i32, vp, vp, vp, vp]),
        "aur_set_attrs": (C.c_int, [vp, i32, vp, vp, i64]),
        "aur_search_filtered": (C.c_int, [vp, vp, i32, i32, vp, vp, i32, vp, i64, vp, i64, vp, vp, vp, C.POINTER(i64)]),
        "aur_filter_ids": (C.c_int, [vp, vp, i32, vp, i64, vp, i64, C.POINTER(i64)]),
        "aur_filter_count": (C.c_int, [vp, vp, i32, vp, i64, C.POINTER(i64)]),
        "aur_remove_filtered": (C.c_int, [vp, vp, i32, vp, i64, vp, i64, C.POINTER(i64)]),
        "aur_search_dev": (C.c_int, [vp, vp, i32, i32, vp, vp, vp, vp, vp, vp]),
        "aur_merge_topk_dev": (C.c_int, [i32, vp, vp, i32, i32, i32, vp, vp, vp, vp]),
        "aur_merge_topk_host": (C.c_int, [vp, vp, i32, i32, i32, i32, vp, vp]),
        "aur_merge_topk_host_f64": (C.c_int, [vp, vp, i32, i32, i32, i32, vp, vp]),
        "aur_merge_topk_packed_dev": (C.c_int, [i32, vp, i32, i32, i32, vp, vp, vp, vp]),
        "aur_exchange_create": (C.c_int, [i32, i32, i32, i32, i32, C.POINTER(vp), vp]),
        "aur_exchange_connect": (C.c_int, [vp, vp]),
        "aur_exchange_close": (C.c_int, [vp]),
        "aur_exchange_status": (C.c_int, [vp, C.POINTER(i64), C.POINTER(i32)]),
        "aur_search_exchange_dev": (C.c_int, [vp, vp, vp, i32, i32, vp, vp, vp]),
        "aur_cosine_pairs": (C.c_int, [i32, vp, vp, i64, i32, i32, vp]),
        "aur_dev_malloc": (C.c_int, [i32, C.c_uint64, C.POINTER(vp)]),
        "aur_dev_free": (C.c_int, [i32, vp]),
        "aur_memcpy_h2d": (C.c_int, [i32, vp, vp, C.c_uint64]),
        "aur_memcpy_d2h": (C.c_int, [i32, vp, vp, C.c_uint64]),
        "aur_debug_tc_scores": (C.c_int, [vp, vp, i32, i32, vp, i64, C.POINTER(i32), C.POINTER(i32), vp]),
        "aur_debug_simt_scores": (C.c_int, [vp, vp, i32, vp, vp, vp, i64, C.POINTER(i64)]),
        "aur_debug_list_scores": (C.c_int, [vp, vp, i32, vp, vp, i32, vp, vp, i64, C.POINTER(i64)]),
        "aur_kw_open": (C.c_int, [i32, i64, i64, C.POINTER(vp)]),
        "aur_kw_close": (C.c_int, [vp]),
        "aur_kw_add": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, i64]),
        "aur_kw_remove": (C.c_int, [vp, vp, i64, C.POINTER(i64)]),
        "aur_kw_compact": (C.c_int, [vp, C.POINTER(i64)]),
        "aur_kw_reserve": (C.c_int, [vp, i64]),
        "aur_kw_get_stats": (C.c_int, [vp, C.POINTER(AurKwStats)]),
        "aur_kw_set_attrs": (C.c_int, [vp, i32, vp, vp, i64]),
        "aur_kw_search": (C.c_int, [vp, vp, vp, i32, i32, vp, vp, vp, i64, vp, vp, C.POINTER(i64)]),
        "aur_kw_search_multi": (C.c_int, [vp, i32, vp, vp, i32, i32, vp, vp, vp, i64, vp, vp, vp]),
        "aur_kw_reindex": (C.c_int, [vp]),
        "aur_kw_set_option": (C.c_int, [vp, C.c_char_p, i64]),
        "aur_kw_get_index_stats": (C.c_int, [vp, C.POINTER(AurKwIndexStats)]),
        "aur_kw_read_rows": (C.c_int, [vp, i64, i64, vp, vp, vp, vp, i64, C.POINTER(i64)]),
        "aur_kw_vocab_open": (C.c_int, [i32, C.POINTER(vp)]),
        "aur_kw_vocab_close": (C.c_int, [vp]),
        "aur_kw_vocab_size": (C.c_int, [vp, C.POINTER(i64), C.POINTER(i64)]),
        "aur_kw_vocab_read": (C.c_int, [vp, i64, i64, vp, i64, vp]),
        "aur_kw_vocab_set_option": (C.c_int, [vp, C.c_char_p, i64]),
        "aur_kw_add_text": (C.c_int, [vp, i32, vp, vp, vp, vp, C.c_char_p, vp, i64]),
        "aur_hybrid_search": (C.c_int, [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp]),
        "aur_hybrid_search_multi": (C.c_int, [vp, vp, i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp]),
        "aur_hybrid_search_filtered": (C.c_int, [vp, vp, i32, vp, i32, i32, vp, vp, vp, vp, i32, vp, i64, vp, i64, vp, vp,
                                                 i32, i32, vp, vp, vp, vp]),
        "aur_encoder_open": (C.c_int, [C.POINTER(AurEncoderConfig), C.POINTER(vp)]),
        "aur_encoder_close": (C.c_int, [vp]),
        "aur_encoder_load": (C.c_int, [vp, C.c_char_p, vp, i64]),
        "aur_encode": (C.c_int, [vp, vp, vp, i32, vp, vp]),
        "aur_encode_append": (C.c_int, [vp, vp, vp, vp, i32, vp, vp, vp]),
        "aur_encoder_replicate": (C.c_int, [vp, i32, C.POINTER(vp)]),
        "aur_encode_append_multi": (C.c_int, [vp, vp, i32, vp, vp, i32, vp, vp, vp, i32, i32]),
        "aur_encode_texts": (C.c_int, [vp, vp, vp, i32, vp, i32, vp, vp]),
        "aur_encode_pair_cosines": (C.c_int, [vp, vp, vp, i32, vp, i32, vp, vp, i64, i32, vp, vp]),
        "aur_encode_append_texts_multi": (C.c_int, [vp, vp, i32, vp, vp, i32, vp, i32, vp, vp, vp, i32, i32]),
        "aur_encoder_get_stats": (C.c_int, [vp, C.POINTER(AurEncoderStats)]),
        "aur_tokenizer_open": (C.c_int, [C.c_char_p, i32, C.POINTER(vp)]),
        "aur_tokenizer_open_mem": (C.c_int, [C.c_char_p, i64, i32, C.POINTER(vp)]),
        "aur_tokenizer_close": (C.c_int, [vp]),
        "aur_tokenizer_info": (C.c_int, [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]),
        "aur_tokenize": (C.c_int, [vp, C.c_char_p, vp, i32, i32, vp, i64, vp, i32]),
        "aur_tokenize_windows": (C.c_int, [vp, C.c_char_p, vp, i32, i32, vp, i64, vp, i32, vp, vp, i32]),
        "aur_encode_text_append": (C.c_int, [vp, vp, vp, C.c_char_p, vp, i32, i32, i32, i32, vp, vp, vp, i32]),
        "aur_debug_gemm": (C.c_int, [i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, C.POINTER(C.c_float)]),
        "aur_debug_attention": (C.c_int, [i32, vp, vp, i32, i32, i32, vp, C.POINTER(C.c_float)]),
        "aur_debug_encoder_hidden": (C.c_int, [vp, vp, i64]),
    }
    for name, (res, args) in sigs.items():
        if not hasattr(lib, name) and os.environ.get("AURORA_B200_AB_OLD_ABI"):
            continue
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    if lib.aur_abi_version() != ABI_VERSION and not os.environ.get("AURORA_B200_AB_OLD_ABI"):   # (A/B runs against older builds)
        raise NativeLibraryMissing(f"{LIB_PATH} has ABI version {lib.aur_abi_version()}, this binding needs {ABI_VERSION}: "
                                   "rebuild it with `python -m aurora_b200.build --force`")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != AUR_OK:
        msg = load().aur_last_error()
        raise AuroraError(rc, msg.decode("utf-8", "replace") if msg else "unknown error")
