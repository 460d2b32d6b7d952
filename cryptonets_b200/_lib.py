"""ctypes binding of libcnhe.so (include/cnhe.h).  There is no CPU fallback: loading fails loudly if the library
has not been built, and every context creation fails if no CUDA device is visible."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libcnhe.so")
_LIB = None

U64P = C.POINTER(C.c_uint64)
DBLP = C.POINTER(C.c_double)
VECP = C.c_void_p
u64, i32, i64, sz = C.c_uint64, C.c_int, C.c_int64, C.c_size_t

# name -> argtypes (all return int unless listed in _RESTYPE)
_SIGS = {
    "cnhe_context_create": [U64P, i32, C.c_uint32, i32, i32, i32, i32, C.POINTER(C.c_void_p)],
    "cnhe_context_create_custom": [U64P, i32, C.c_uint32, U64P, i32, i32, i32, i32, C.POINTER(C.c_void_p)],
    "cnhe_context_destroy": [C.c_void_p],
    "cnhe_context_info": [C.c_void_p, C.POINTER(C.c_uint32)] + [C.POINTER(i32)] * 5,
    "cnhe_context_coeff_moduli": [C.c_void_p, U64P],
    "cnhe_context_plain_moduli": [C.c_void_p, U64P],
    "cnhe_context_bsk_moduli": [C.c_void_p, U64P, C.POINTER(i32)],
    "cnhe_context_product_sum_terms": [C.c_void_p, C.POINTER(i32)],
    "cnhe_context_galois_elts": [C.c_void_p, U64P],
    "cnhe_context_set_option": [C.c_void_p, C.c_char_p, i64],
    "cnhe_context_sync": [C.c_void_p],
    "cnhe_context_stream": [C.c_void_p, i32, U64P],
    "cnhe_context_join_streams": [C.c_void_p],
    "cnhe_context_fork_streams": [C.c_void_p],
    "cnhe_keys_generate": [C.c_void_p, u64],
    "cnhe_keys_save": [C.c_void_p, i32, C.c_void_p, sz, C.POINTER(sz)],
    "cnhe_context_load": [C.c_void_p, sz, i32, C.POINTER(C.c_void_p)],
    "cnhe_keys_save_compact": [C.c_void_p, i32, U64P, i32, C.c_void_p, sz, C.POINTER(sz)],
    "cnhe_context_load_compact": [C.c_void_p, sz, i32, C.POINTER(C.c_void_p)],
    "cnhe_context_add_client_compact": [C.c_void_p, C.c_void_p, sz, C.POINTER(i32)],
    "cnhe_context_remove_client": [C.c_void_p, i32],
    "cnhe_vec_set_key_slot": [VECP, i32],
    "cnhe_vec_key_slot": [VECP, C.POINTER(i32)],
    "cnhe_vecs_rotate": [C.c_void_p, C.POINTER(VECP), i32, i32, C.POINTER(VECP)],
    "cnhe_vecs_stack_batch": [C.c_void_p, C.POINTER(VECP), i32, i32, C.POINTER(VECP)],
    "cnhe_mat_mul_rowmajor_batch": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP), i32, i32, C.POINTER(VECP)],
    "cnhe_mat_dot_rows_batch": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP), i32, u64, C.POINTER(VECP)],
    "cnhe_vecs_duplicate_batch": [C.c_void_p, C.POINTER(VECP), i32, u64, C.POINTER(VECP)],
    "cnhe_vecs_permute_batch": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP), C.POINTER(i32), i32, i32, u64, C.POINTER(VECP)],
    "cnhe_vecs_interleave_batch": [C.c_void_p, C.POINTER(VECP), i32, i32, i32, C.POINTER(VECP)],
    "cnhe_vecs_multiply_plain": [C.c_void_p, C.POINTER(VECP), i32, VECP, C.POINTER(VECP)],
    "cnhe_diag_prepare": [C.c_void_p, C.POINTER(VECP), i32, i32, C.POINTER(C.c_void_p)],
    "cnhe_diag_info": [C.c_void_p, C.POINTER(i32), U64P, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), U64P],
    "cnhe_diag_export": [C.c_void_p, C.c_void_p, i32, i32, U64P, sz, C.POINTER(i32)],
    "cnhe_diag_destroy": [C.c_void_p],
    "cnhe_diag_prepare_ntt": [C.c_void_p, C.POINTER(VECP), i32, i32, u64, C.POINTER(C.c_void_p)],
    "cnhe_diag_ntt_info": [C.c_void_p, C.POINTER(i32), C.POINTER(i32), U64P],
    "cnhe_diag_export_ntt": [C.c_void_p, C.c_void_p, i32, i32, U64P, sz],
    "cnhe_mat_mul_diagonal": [C.c_void_p, C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP)],
    "cnhe_diag_prepare_folded": [C.c_void_p, C.POINTER(VECP), i32, i32, i32, u64, C.POINTER(C.c_void_p)],
    "cnhe_diag_fold_width": [C.c_void_p, C.POINTER(i32)],
    "cnhe_vec_write": [C.c_void_p, VECP, C.c_void_p, sz, C.POINTER(sz)],
    "cnhe_vec_read": [C.c_void_p, C.c_char_p, sz, C.POINTER(VECP), C.POINTER(sz)],
    "cnhe_keys_generate_secure": [C.c_void_p],
    "cnhe_op_counts": [C.c_void_p, U64P, i32, i32],
    "cnhe_op_name": [i32],
    "cnhe_trace_read": [C.c_void_p, C.POINTER(C.c_int32), sz, C.POINTER(sz), i32],
    "cnhe_keys_export": [C.c_void_p, i32, i32, u64, U64P, sz],
    "cnhe_keys_import": [C.c_void_p, i32, i32, u64, U64P, sz],
    "cnhe_keys_set_seed": [C.c_void_p, i32, u64],
    "cnhe_vec_encrypt": [C.c_void_p, DBLP, u64, C.c_double, i32, C.POINTER(VECP)],
    "cnhe_vec_plain": [C.c_void_p, DBLP, u64, C.c_double, i32, C.POINTER(VECP)],
    "cnhe_vec_from_residues": [C.c_void_p, U64P, u64, C.c_double, i32, i32, C.POINTER(VECP)],
    "cnhe_vec_decrypt_residues": [C.c_void_p, VECP, U64P, u64],
    "cnhe_vecs_encrypt": [C.c_void_p, DBLP, i32, u64, C.c_double, C.POINTER(VECP)],
    "cnhe_vec_decrypt": [C.c_void_p, VECP, DBLP, u64],
    "cnhe_vecs_decrypt": [C.c_void_p, C.POINTER(VECP), i32, DBLP, u64],
    "cnhe_vec_copy": [C.c_void_p, VECP, C.POINTER(VECP)],
    "cnhe_vec_destroy": [VECP],
    "cnhe_vecs_destroy": [C.POINTER(VECP), i32],
    "cnhe_vec_meta": [VECP, U64P, DBLP, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), U64P],
    "cnhe_vec_register_scale": [VECP, C.c_double],
    "cnhe_vec_register_dim": [VECP, u64],
    "cnhe_vec_export_raw": [C.c_void_p, VECP, i32, i32, U64P, sz],
    "cnhe_vec_import_raw": [C.c_void_p, U64P, i32, u64, C.c_double, i32, C.POINTER(VECP)],
    "cnhe_vecs_import_raw": [C.c_void_p, U64P, i32, i32, u64, C.c_double, i32, C.POINTER(VECP)],
    "cnhe_vecs_export_raw": [C.c_void_p, C.POINTER(VECP), i32, U64P, sz],
    "cnhe_vecs_export_raw_async": [C.c_void_p, C.POINTER(VECP), i32, U64P, sz, C.POINTER(i32)],
    "cnhe_export_wait": [C.c_void_p, i32],
    "cnhe_vecs_encrypt_compact": [C.c_void_p, DBLP, i32, u64, C.c_double, C.c_void_p, sz, C.POINTER(sz)],
    "cnhe_vecs_import_compact": [C.c_void_p, C.c_void_p, sz, C.POINTER(VECP), i32, C.POINTER(i32)],
    "cnhe_dev_copy": [C.c_void_p, u64, u64, sz],
    "cnhe_prof_enable": [C.c_void_p, i32],
    "cnhe_prof_collect": [C.c_void_p, i32, DBLP, U64P, DBLP],
    "cnhe_vec_device_ptr": [VECP, i32, U64P, C.POINTER(sz)],
    "cnhe_noise_budget": [C.c_void_p, VECP, i32, i32, C.POINTER(i32)],
    "cnhe_vec_add": [C.c_void_p, VECP, VECP, C.POINTER(VECP)],
    "cnhe_vec_sub": [C.c_void_p, VECP, VECP, C.POINTER(VECP)],
    "cnhe_vec_pointwise_multiply": [C.c_void_p, VECP, VECP, C.POINTER(VECP)],
    "cnhe_vec_sum_all_slots": [C.c_void_p, VECP, u64, i32, C.POINTER(VECP)],
    "cnhe_vec_dot_product": [C.c_void_p, VECP, VECP, u64, i32, C.POINTER(VECP)],
    "cnhe_vec_rotate": [C.c_void_p, VECP, i32, C.POINTER(VECP)],
    "cnhe_vec_duplicate": [C.c_void_p, VECP, u64, C.POINTER(VECP)],
    "cnhe_vec_permute": [C.c_void_p, VECP, C.POINTER(VECP), C.POINTER(i32), i32, u64, C.POINTER(VECP)],
    "cnhe_vecs_interleave": [C.c_void_p, C.POINTER(VECP), i32, i32, C.POINTER(VECP)],
    "cnhe_vecs_stack": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP)],
    "cnhe_vecs_generate_sparse_of_array": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP)],
    "cnhe_mat_mul_colmajor_sparse": [C.c_void_p, C.POINTER(VECP), i32, VECP, C.POINTER(VECP)],
    "cnhe_mat_mul_colmajor_sparse_deferred": [C.c_void_p, C.POINTER(VECP), i32, VECP, C.POINTER(VECP)],
    "cnhe_mat_mul_rowmajor": [C.c_void_p, C.POINTER(VECP), i32, VECP, i32, C.POINTER(VECP)],
    "cnhe_mat_mul_rowmajor_shard": [C.c_void_p, C.POINTER(VECP), i32, VECP, i32, i32, i32, C.POINTER(VECP)],
    "cnhe_layer_conv_dense": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(C.c_int32), C.POINTER(VECP), C.POINTER(VECP), i32, i32,
                              C.POINTER(VECP)],
    "cnhe_layer_square": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP)],
    "cnhe_layer_poly2": [C.c_void_p, C.POINTER(VECP), i32, VECP, VECP, VECP, C.POINTER(VECP)],
    "cnhe_layer_poly": [C.c_void_p, C.POINTER(VECP), i32, C.POINTER(VECP), i32, C.POINTER(VECP)],
    "cnhe_layer_activation_conv_dense": [C.c_void_p, C.POINTER(VECP), i32, VECP, VECP, VECP, C.POINTER(C.c_int32), C.POINTER(VECP),
                                         C.POINTER(VECP), i32, i32, C.POINTER(VECP)],
    "cnhe_dev_alloc": [C.c_void_p, sz, U64P],
    "cnhe_dev_free": [C.c_void_p, u64],
    "cnhe_dev_upload": [C.c_void_p, u64, U64P, sz],
    "cnhe_dev_download": [C.c_void_p, U64P, u64, sz],
    "cnhe_raw_ntt": [C.c_void_p, u64, u64, i32, i32, i32, i32],
    "cnhe_raw_multiply": [C.c_void_p, i32, u64, u64, i32, u64],
    "cnhe_raw_relinearize": [C.c_void_p, i32, u64, i32, u64],
    "cnhe_raw_multiply_relin": [C.c_void_p, i32, u64, u64, i32, u64],
    "cnhe_raw_apply_galois": [C.c_void_p, i32, u64, i32, u64, u64],
    "cnhe_raw_rotate_rows": [C.c_void_p, i32, u64, i32, i32, u64],
    "cnhe_raw_behz_lift": [C.c_void_p, u64, i32, u64],
    "cnhe_raw_behz_floor": [C.c_void_p, i32, u64, i32, u64],
    "cnhe_raw_import_products": [C.c_void_p, U64P, i32, u64, C.c_double, i32, C.POINTER(VECP)],
    "cnhe_raw_event_timing": [C.c_void_p, i32],
    "cnhe_raw_elapsed_ms": [C.c_void_p, C.POINTER(C.c_float)],
    "cnhe_kernel_launch_count": [C.c_void_p],
    "cnhe_capture_begin": [C.c_void_p],
    "cnhe_capture_end": [C.c_void_p, C.POINTER(C.c_void_p)],
    "cnhe_capture_abort": [C.c_void_p],
    "cnhe_graph_launch": [C.c_void_p],
    "cnhe_graph_slots": [C.c_void_p, C.POINTER(C.c_int32), i32, C.POINTER(C.c_int32)],
    "cnhe_graph_bind": [C.c_void_p, C.POINTER(C.c_int32), i32],
    "cnhe_graph_info": [C.c_void_p, U64P, U64P],
    "cnhe_graph_destroy": [C.c_void_p],
    "cnhe_vecs_assign": [C.c_void_p, C.POINTER(VECP), C.POINTER(VECP), i32],
    "cnhe_last_error": [],
    "cnhe_version": [],
}
_RESTYPE = {"cnhe_op_name": C.c_char_p, "cnhe_last_error": C.c_char_p, "cnhe_version": C.c_char_p, "cnhe_kernel_launch_count": C.c_uint64}

EXPORTS = sorted(_SIGS)


class CnheError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            raise ImportError(
                "cryptonets_b200/libcnhe.so is missing: build it with `python -m cryptonets_b200.build` "
                "(needs nvcc; there is no CPU fallback)")
        L = C.CDLL(_SO)
        for name, args in _SIGS.items():
            f = getattr(L, name)  # raises AttributeError if the symbol is not exported
            f.argtypes = args
            f.restype = _RESTYPE.get(name, C.c_int)
        _LIB = L
    return _LIB


def check(rc):
    if rc != 0:
        raise CnheError(rc, lib().cnhe_last_error().decode())
