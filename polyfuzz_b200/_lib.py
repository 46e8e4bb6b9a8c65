"""ctypes binding of libpfz.so (include/pfz.h).  There is no CPU fallback: if the library is
missing or a call fails, a RuntimeError carrying pfz_last_error() is raised."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libpfz.so")
_lib = None

c_i32, c_i64, c_u32, c_f64, c_vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32, ctypes.c_double, ctypes.c_void_p

# name -> argtypes (restype is int unless listed in _RESTYPES); mirrors include/pfz.h one to one
_PROTOS = {
    "pfz_abi_version": [],
    "pfz_last_error": [],
    "pfz_launch_count": [],
    "pfz_device_info": [c_vp, c_vp, c_vp, c_vp],
    "pfz_scan_ws_bytes": [c_i64],
    "pfz_int_alu_probe": [c_i32, c_vp, c_vp, c_vp],
    "pfz_alphabet_mark": [c_vp, c_i64, c_vp, c_vp],
    "pfz_ngram_rows": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_u32, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_df_dense": [c_vp, c_vp, c_vp, c_i32, c_vp, c_vp],
    "pfz_vocab_compact_dense": [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_gather_codes": [c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp],
    "pfz_sort_u64": [c_vp, c_i64, c_vp],
    "pfz_vocab_from_sorted": [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_idf_lookup": [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp],
    "pfz_tfidf_emit": [c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_index_build": [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_spcos_topk": [c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32,
                       c_i64, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp],
    "pfz_topk_merge": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp],
    "pfz_spcos_topk_hash": [c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_i64, c_i32,
                            c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_spcos_block_ws_bytes": [c_i32, c_i64, c_i32, c_i32],
    "pfz_spcos_block_gcnt_offset": [c_i32, c_i64, c_i32, c_i32],
    "pfz_index_pack_q26": [c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_index_pack_q15": [c_vp, c_vp, c_vp, c_i32, c_vp, c_vp],
    "pfz_spcos_topk_block": [c_vp, c_vp, c_vp, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32,
                             c_i64, c_i64, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_lev_pack": [c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_lev_argbest": [c_vp, c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_f64, c_i32, c_i64,
                        c_i32, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp],
    "pfz_lev_merge": [c_vp, c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_fuzz_argbest": [c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_i32, c_vp],
    "pfz_lev_topk": [c_vp, c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_f64, c_i32, c_i64,
                     c_i32, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_dl_argbest": [c_vp, c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_f64, c_i32, c_i64,
                       c_i32, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp],
    "pfz_dl_topk": [c_vp, c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_f64, c_i32, c_i64,
                    c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_fuzz_topk":[c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_i32, c_i32, c_vp],
    "pfz_tok_side": [c_vp, c_vp, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_tok_union": [c_vp, c_vp, c_i32, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_tok_remap": [c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_frame_tail_ws_bytes": [c_i64],
    "pfz_frame_tail_count": [c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp],
    "pfz_frame_tail_copy": [c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_rows_to_bf16": [c_vp, c_i32, c_i64, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp],
    "pfz_dense_cos_topk": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp],
    "pfz_rows_prep_exact": [c_vp, c_i32, c_i64, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_dense_cos_topk_f16": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp],
    "pfz_dense_exact_rescore": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_f64, c_i32, c_i64, c_i64,
                                c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_dense_exact_fallback_ws_bytes": [c_i32, c_i32, c_i32],
    "pfz_dense_exact_fallback": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp],
    "pfz_dense_topn_bound": [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_i32, c_f64, c_vp, c_vp],
    "pfz_dense_cos_cand": [c_vp, c_vp, c_i32, c_i32, c_i32, c_f64, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_dense_cos_cand_f16": [c_vp, c_vp, c_i32, c_i32, c_i32, c_f64, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_dense_topn_exact_rescore": [c_vp, c_vp, c_i32, c_i32, c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp],
    "pfz_dense_topn_select": [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_f64, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp],
}
_RESTYPES = {"pfz_last_error": ctypes.c_char_p, "pfz_scan_ws_bytes": c_i64, "pfz_launch_count": c_i64, "pfz_spcos_block_ws_bytes": c_i64,
             "pfz_spcos_block_gcnt_offset": c_i64,
             "pfz_dense_exact_fallback_ws_bytes": c_i64, "pfz_frame_tail_ws_bytes": c_i64}


def exported_names():
    return list(_PROTOS)


def lib_path():
    return _LIB_PATH


def load():
    """Load libpfz.so; raises RuntimeError if it has not been built (python -m polyfuzz_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(f"{_LIB_PATH} not found: build it with `python -m polyfuzz_b200.build` "
                           "(polyfuzz_b200 has no CPU fallback)")
    lib = ctypes.CDLL(_LIB_PATH)
    for name, args in _PROTOS.items():
        fn = getattr(lib, name)            # AttributeError here == header/library mismatch
        fn.argtypes = args
        fn.restype = _RESTYPES.get(name, ctypes.c_int)
    _lib = lib
    return lib


def call(name, *args):
    """Invoke an int-returning entry point, raising RuntimeError(pfz_last_error()) on failure."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError(f"{name} failed: {lib.pfz_last_error().decode(errors='replace')}")


def launch_count():
    return int(load().pfz_launch_count())
