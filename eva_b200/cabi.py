"""ctypes binding of include/evab200.h (the same stub a reference maintainer
would write, see INTEGRATION.md).  Fails loudly when the CUDA library is
missing; never falls back to a CPU implementation."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libevab200.so")
_lib = None

vp, u64, szt, ci = C.c_void_p, C.c_uint64, C.c_size_t, C.c_int
u64p = C.POINTER(C.c_uint64)

_SIGS = {
    "evab_last_error": (C.c_char_p, []),
    "evab_version": (ci, []),
    "evab_ctx_create": (ci, [u64, u64p, ci, ci, C.POINTER(vp)]),
    "evab_ctx_destroy": (None, [vp]),
    "evab_ctx_N": (u64, [vp]),
    "evab_ctx_k": (ci, [vp]),
    "evab_ctx_device": (ci, [vp]),
    "evab_ctx_sm_count": (ci, [vp]),
    "evab_mem_info": (ci, [vp, C.POINTER(szt), C.POINTER(szt)]),
    "evab_malloc": (ci, [vp, szt, C.POINTER(vp), vp]),
    "evab_free": (ci, [vp, vp, vp]),
    "evab_upload": (ci, [vp, vp, vp, szt, vp]),
    "evab_upload_2d": (ci, [vp, vp, szt, vp, szt, szt, szt, vp]),
    "evab_download": (ci, [vp, vp, vp, szt, vp]),
    "evab_sync": (ci, [vp, vp]),
    "evab_stream_create": (ci, [vp, C.POINTER(vp)]),
    "evab_stream_destroy": (ci, [vp, vp]),
    "evab_event_create": (ci, [vp, C.POINTER(vp)]),
    "evab_event_destroy": (ci, [vp, vp]),
    "evab_event_record": (ci, [vp, vp, vp]),
    "evab_stream_wait_event": (ci, [vp, vp, vp]),
    "evab_graph_begin": (ci, [vp, vp]),
    "evab_graph_end": (ci, [vp, vp, C.POINTER(vp)]),
    "evab_graph_launch": (ci, [vp, vp, vp]),
    "evab_graph_destroy": (ci, [vp, vp]),
    "evab_launch_count": (u64, [vp]),
    "evab_ntt_fwd": (ci, [vp, vp, szt, C.POINTER(ci), ci, vp]),
    "evab_ntt_inv": (ci, [vp, vp, szt, C.POINTER(ci), ci, vp]),
    "evab_rotate_modup_ext_bytes": (szt, [vp, ci]),
    "evab_rotate_modup_work_bytes": (szt, [vp, ci]),
    "evab_hoist_const_bytes": (szt, [vp, ci]),
    "evab_rotate_modup_prepare": (ci, [vp, ci, vp, vp, vp, vp, vp]),
    "evab_rotate_hoist_const": (ci, [vp, ci, u64, vp, vp, vp, vp]),
    "evab_hoist_const_levels_bytes": (szt, [vp]),
    "evab_rotate_hoist_const_levels_work_bytes": (szt, [vp, ci]),
    "evab_rotate_hoist_const_levels": (ci, [vp, ci, u64p, vp, vp, vp, vp]),
    "evab_hoist_indicators_bytes": (szt, [vp, ci]),
    "evab_hoist_indicators": (ci, [vp, ci, u64p, vp, vp]),
    "evab_expand_key_uniform": (ci, [vp, ci, vp, u64p, vp, vp]),
    "evab_expand_cipher_uniform": (ci, [vp, ci, vp, vp, vp, u64p, vp]),
    "evab_gather_ciphers": (ci, [vp, ci, vp, vp, u64p, vp]),
    "evab_compact_work_bytes": (szt, [vp, ci, ci]),
    "evab_compact_ciphers": (ci, [vp, ci, vp, vp, ci, ci, ci, vp, vp]),
    "evab_compact_unpack": (ci, [vp, vp, ci, ci, vp, vp]),
    "evab_compact_finish": (ci, [vp, vp, ci, ci, ci, vp, vp, vp]),
    "evab_rotate_modup_prepared": (ci, [vp, ci, vp, vp, vp, u64, vp, vp, vp, vp]),
    "evab_memset_zero": (ci, [vp, vp, szt, vp]),
    "evab_rotate_modup_scale_c0": (ci, [vp, ci, vp, vp, vp]),
    "evab_rotate_modup_many_work_bytes": (szt, [vp, ci, ci]),
    "evab_rotate_modup_many": (ci, [vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp]),
    "evab_rotate_wsum_work_bytes": (szt, [vp, ci, ci, ci]),
    "evab_rotate_wsum": (ci, [vp, ci, ci, vp, vp, vp, ci, vp, vp, vp, vp, ci, vp, vp, vp, vp]),
    "evab_lazy_rotsum_work_bytes": (szt, [vp, ci, ci]),
    "evab_lazy_rotsum": (ci, [vp, ci, ci, vp, vp, vp, ci, vp, vp, vp, vp, vp, vp]),
    "evab_encode_ext": (ci, [vp, ci, vp, vp, vp, ci, ci, vp, vp, vp]),
    "evab_encode_uniform_ext": (ci, [vp, ci, vp, vp, ci, ci, vp, vp]),
    "evab_decode_work_bytes": (szt, [vp, ci]),
    "evab_decode": (ci, [vp, ci, vp, C.c_double, vp, vp, vp]),
    "evab_set_ntt_cluster": (ci, [ci]),
    "evab_ctx_set_ntt_cluster": (ci, [vp, ci]),
    "evab_ctx_set_ntt_arith": (ci, [vp, ci]),
    "evab_ctx_foldmask": (C.c_uint, [vp]),
    "evab_sum_terms": (ci, [vp, ci, vp, ci, C.POINTER(vp), C.POINTER(ci), C.POINTER(vp), vp]),
    "evab_sum_products": (ci, [vp, ci, vp, ci, C.POINTER(vp), C.POINTER(ci), C.POINTER(vp), C.POINTER(ci), vp]),
    "evab_host_alloc": (ci, [szt, C.POINTER(vp)]),
    "evab_host_free": (ci, [vp]),
    "evab_encode_work_bytes": (szt, [vp, ci]),
    "evab_encode_uniform": (ci, [vp, ci, C.POINTER(C.c_double), C.POINTER(C.c_double), ci, vp, vp]),
    "evab_encode": (ci, [vp, ci, C.POINTER(vp), C.POINTER(C.c_uint32), C.POINTER(C.c_double), ci, vp, vp, vp]),
    "evab_add": (ci, [vp, ci, vp, vp, ci, vp, ci, vp]),
    "evab_sub": (ci, [vp, ci, vp, vp, ci, vp, ci, vp]),
    "evab_add_plain": (ci, [vp, ci, vp, vp, ci, vp, vp]),
    "evab_sub_plain": (ci, [vp, ci, vp, vp, ci, vp, vp]),
    "evab_negate": (ci, [vp, ci, vp, vp, ci, vp]),
    "evab_mul_plain": (ci, [vp, ci, vp, vp, ci, vp, vp]),
    "evab_mul": (ci, [vp, ci, vp, vp, vp, vp]),
    "evab_square": (ci, [vp, ci, vp, vp, vp]),
    "evab_rescale_work_bytes": (szt, [vp, ci]),
    "evab_rescale": (ci, [vp, ci, vp, vp, ci, vp, vp]),
    "evab_copy": (ci, [vp, ci, vp, vp, ci, vp]),
    "evab_set_batch": (ci, [ci, szt, szt]),
    "evab_set_key_bank": (ci, [vp, szt]),
    "evab_set_hoist_inline": (ci, [ci]),
    "evab_set_key_seeded": (ci, [ci]),
    "evab_seeded_key_bytes": (szt, [vp]),
    "evab_set_key_c1_rows": (ci, [vp]),
    "evab_expand_seeded_c1": (ci, [vp, ci, vp, vp, vp]),
    "evab_mod_switch": (ci, [vp, ci, vp, vp, ci, vp]),
    "evab_keyswitch_work_bytes": (szt, [vp, ci]),
    "evab_relinearize": (ci, [vp, ci, vp, vp, vp, vp, vp]),
    "evab_galois_elt_from_step": (u64, [u64, ci]),
    "evab_galois_prepare": (ci, [vp, u64]),
    "evab_rotate": (ci, [vp, ci, vp, vp, u64, vp, vp, vp]),
    "evab_rotate_prepare": (ci, [vp, ci, vp, vp, vp]),
    "evab_rotate_prepared": (ci, [vp, ci, vp, vp, vp, u64, vp, vp, vp]),
}


def exported_symbols():
    return sorted(_SIGS)


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "eva_b200: CUDA library %s is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)" % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib
