"""ctypes loader for the in-tree C-ABI library (include/dpfhe.h).

There is no CPU fallback: if libdpfhe.so is missing it is built with nvcc, and if that is
impossible the import fails loudly.
"""
import ctypes as C
import os

from . import build as _build

_lib = None

SYMBOLS = {
    # name: (restype, argtypes)
    "dpfhe_last_error": (C.c_char_p, []),
    "dpfhe_version": (C.c_char_p, []),
    "dpfhe_context_create": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "dpfhe_context_destroy": (None, [C.c_void_p]),
    "dpfhe_get_modulus": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64)]),
    "dpfhe_get_psi": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64)]),
    "dpfhe_get_root_powers": (C.c_int, [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]),
    "dpfhe_context_device_bytes": (C.c_size_t, [C.c_void_p]),
    "dpfhe_ntt_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ntt_inv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_poly_mul_pointwise": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_poly_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_tensor": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_keyswitch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_mul_relin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_mul_plain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_mul_plain_acc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_rotate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_rotate_hoisted": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_mul_plain_inner": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_mod_switch_down": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_keyswitch_hybrid": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_ct_mul_relin_hybrid": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_rotate_hybrid": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_grouped_digits": (C.c_int, [C.c_void_p, C.c_uint, C.POINTER(C.c_uint)]),
    "dpfhe_keyswitch_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_ct_mul_relin_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_rotate_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_rotate_hoisted_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64,
                                               C.c_void_p]),
    "dpfhe_mod_down_special": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_mod_down_special_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_ct_mul_relin_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_rotate_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_ct_mul_relin_hybrid_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_rotate_hybrid_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_mod_switch_down_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_ckks_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]),
    "dpfhe_ckks_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]),
    "dpfhe_ckks_encode_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double]),
    "dpfhe_ckks_decode_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double]),
    "dpfhe_bgv_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_bgv_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_bgv_encode_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_bgv_decode_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_random_seed": (C.c_int, [C.c_char_p]),
    "dpfhe_secret_keygen": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]),
    "dpfhe_relin_keygen": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]),
    "dpfhe_galois_keygen": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]),
    "dpfhe_encrypt": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_decrypt": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_secret_keygen_host": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p]),
    "dpfhe_relin_keygen_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_char_p, C.c_void_p]),
    "dpfhe_galois_keygen_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_void_p]),
    "dpfhe_encrypt_host": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_decrypt_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t]),
    "dpfhe_public_keygen": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]),
    "dpfhe_encrypt_public": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_public_keygen_host": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_void_p]),
    "dpfhe_encrypt_public_host": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_fill_uniform": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ntt_fwd_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_ntt_inv_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_ct_mul_relin_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_ct_mul_plain_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_rotate_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_context_trim": (C.c_int, [C.c_void_p]),
    "dpfhe_context_device": (C.c_int, [C.c_void_p]),
    "dpfhe_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "dpfhe_synchronize": (C.c_int, [C.c_void_p]),
    "dpfhe_galois_element": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]),
    "dpfhe_rotate_steps": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_host_alloc_near": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_size_t, C.POINTER(C.c_int)]),
    "dpfhe_device_numa_node": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "dpfhe_bind_thread_near": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "dpfhe_device_alloc": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_size_t]),
    "dpfhe_device_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dpfhe_ipc_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_char_p]),
    "dpfhe_ipc_open": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "dpfhe_ipc_close": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dpfhe_multi_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p)]),
    "dpfhe_multi_destroy": (None, [C.c_void_p]),
    "dpfhe_multi_device_count": (C.c_int, [C.c_void_p]),
    "dpfhe_multi_context": (C.c_void_p, [C.c_void_p, C.c_int]),
    "dpfhe_multi_shard": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "dpfhe_multi_ct_mul_relin_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_multi_ct_mul_relin_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_multi_rotate_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_multi_ct_mul_relin_gather": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p, C.c_int, C.c_size_t]),
    "dpfhe_linear_create": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "dpfhe_linear_create_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_uint64,
                                              C.POINTER(C.c_void_p)]),
    "dpfhe_linear_destroy": (None, [C.c_void_p]),
    "dpfhe_linear_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_linear_apply_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_ct_lincomb": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_add_plain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_add_plain_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_polyeval_create_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_void_p)]),
    "dpfhe_polyeval_result_limbs": (C.c_uint, [C.c_void_p]),
    "dpfhe_polyeval_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_polyeval_apply_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_polyeval_destroy": (None, [C.c_void_p]),
    "dpfhe_polyeval_create_ckks": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_double, C.c_double, C.c_void_p, C.POINTER(C.c_void_p)]),
    "dpfhe_polyeval_result_scale": (C.c_double, [C.c_void_p]),
    "dpfhe_rotate_sum_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64,
                                           C.c_void_p]),
    "dpfhe_rotate_sum_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                C.c_uint64]),
    "dpfhe_ct_dot_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64,
                                       C.c_void_p]),
    "dpfhe_ct_dot_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                            C.c_uint64]),
    "dpfhe_ct_mul_relin_rescale_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64,
                                                     C.c_void_p]),
    "dpfhe_ct_mul_relin_rescale_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                          C.c_uint64]),
    "dpfhe_ct_dot_rescale_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                               C.c_uint64, C.c_void_p]),
    "dpfhe_ct_dot_rescale_grouped_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                    C.c_uint64]),
    "dpfhe_ct_mul_relin_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                   C.c_uint64, C.c_void_p]),
    "dpfhe_ct_mul_relin_rescale_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                           C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_ct_dot_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_ct_dot_rescale_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_rotate_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t,
                                             C.c_uint64, C.c_void_p]),
    "dpfhe_rotate_sum_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_rotate_hoisted_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_linear_create_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p,
                                                    C.c_uint64, C.POINTER(C.c_void_p)]),
    "dpfhe_slotsum_create_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64,
                                                     C.POINTER(C.c_void_p)]),
    "dpfhe_ct_mul_relin_rescale_grouped_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                                C.c_size_t, C.c_uint64]),
    "dpfhe_ct_dot_rescale_grouped_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                          C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_slotsum_steps": (C.c_int, [C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t)]),
    "dpfhe_slotsum_create_grouped": (C.c_int, [C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]),
    "dpfhe_slotsum_apply": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_slotsum_apply_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_slotsum_destroy": (None, [C.c_void_p]),
    "dpfhe_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_size_t]),
    "dpfhe_host_free": (C.c_int, [C.c_void_p]),
    "dpfhe_launch_count": (C.c_uint64, [C.c_void_p]),
    "dpfhe_debug_phase_cycles": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dpfhe_describe": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
}


# the entry points of include/dpfhe_level.h (DESIGN.md section 2.22), which dpfhe.h includes
LEVEL_SYMBOLS = {
    "dpfhe_ckks_encode_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]),
    "dpfhe_ckks_decode_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double, C.c_void_p]),
    "dpfhe_ckks_encode_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double]),
    "dpfhe_ckks_decode_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double]),
    "dpfhe_bgv_encode_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_bgv_decode_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_bgv_encode_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_bgv_decode_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]),
    "dpfhe_encrypt_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_encrypt_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_encrypt_public_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_encrypt_public_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t]),
    "dpfhe_decrypt_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_decrypt_level_host": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.c_size_t]),
    "dpfhe_ct_add_plain_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_mul_plain_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_ct_lincomb_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "dpfhe_mod_switch_down_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p]),
    "dpfhe_polyeval_create_grouped_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_uint64, C.c_void_p, C.c_size_t, C.c_void_p,
                                                      C.POINTER(C.c_void_p)]),
    "dpfhe_polyeval_create_ckks_level": (C.c_int, [C.c_void_p, C.c_uint, C.c_uint, C.c_void_p, C.c_size_t, C.c_double, C.c_double, C.c_void_p,
                                                   C.POINTER(C.c_void_p)]),
}

# the entry points of include/dpfhe_seeded.h (DESIGN.md section 2.23), which dpfhe.h includes
_V, _U, _U64, _SZ = C.c_void_p, C.c_uint, C.c_uint64, C.c_size_t
SEEDED_SYMBOLS = {
    "dpfhe_seeded_public_seed": (C.c_int, [_V, _V]),
    "dpfhe_encrypt_seeded": (C.c_int, [_V, _U64, _V, _V, _U64, _V, _V, _SZ, _V]),
    "dpfhe_encrypt_seeded_host": (C.c_int, [_V, _U64, _V, _V, _U64, _V, _V, _SZ]),
    "dpfhe_encrypt_seeded_level": (C.c_int, [_V, _U, _U64, _V, _V, _U64, _V, _V, _SZ, _V]),
    "dpfhe_encrypt_seeded_level_host": (C.c_int, [_V, _U, _U64, _V, _V, _U64, _V, _V, _SZ]),
    "dpfhe_expand_ciphertexts": (C.c_int, [_V, _V, _U64, _V, _V, _SZ, _V]),
    "dpfhe_expand_ciphertexts_level": (C.c_int, [_V, _U, _V, _U64, _V, _V, _SZ, _V]),
    "dpfhe_upload_seeded_ciphertexts": (C.c_int, [_V, _V, _U64, _V, _V, _SZ]),
    "dpfhe_upload_seeded_ciphertexts_level": (C.c_int, [_V, _U, _V, _U64, _V, _V, _SZ]),
    "dpfhe_relin_keygen_seeded": (C.c_int, [_V, _U, _U64, _V, _V, _V, _V]),
    "dpfhe_relin_keygen_seeded_host": (C.c_int, [_V, _U, _U64, _V, _V, _V]),
    "dpfhe_galois_keygen_seeded": (C.c_int, [_V, _U, _U64, _V, _SZ, _V, _V, _V, _V]),
    "dpfhe_galois_keygen_seeded_host": (C.c_int, [_V, _U, _U64, _V, _SZ, _V, _V, _V]),
    "dpfhe_expand_switch_keys": (C.c_int, [_V, _U, _V, _SZ, _V, _V, _V, _V]),
    "dpfhe_upload_seeded_switch_keys": (C.c_int, [_V, _U, _V, _SZ, _V, _V, _V]),
    "dpfhe_expand_switch_keys_host": (C.c_int, [_V, _U, _V, _SZ, _V, _V, _V]),
}

# the entry points of include/dpfhe_compact.h (DESIGN.md section 2.24), which dpfhe.h includes
COMPACT_SYMBOLS = {
    "dpfhe_compact_ciphertexts": (C.c_int, [_V, _U, _U, _U64, _V, _V, _SZ, _V]),
    "dpfhe_download_compact_ciphertexts": (C.c_int, [_V, _U, _U, _U64, _V, _V, _SZ]),
    "dpfhe_decrypt_compact": (C.c_int, [_V, _U, _U64, _V, _V, _V, _SZ, _V]),
    "dpfhe_decrypt_compact_host": (C.c_int, [_V, _U, _U64, _V, _V, _V, _SZ]),
}


class dpfhe_params(C.Structure):
    _fields_ = [("log_n", C.c_uint32), ("n_limbs", C.c_uint32), ("moduli", C.POINTER(C.c_uint64))]


def so_path():
    return _build.SO


def load():
    global _lib
    if _lib is not None:
        return _lib
    path = _build.SO
    if not os.path.exists(path):
        _build.build()          # raises if nvcc is unavailable: no fallback
    lib = C.CDLL(path)
    for name, (res, args) in list(SYMBOLS.items()) + list(LEVEL_SYMBOLS.items()) + list(SEEDED_SYMBOLS.items()) + list(COMPACT_SYMBOLS.items()):
        fn = getattr(lib, name)   # AttributeError if the library does not export what include/dpfhe.h (with its included headers) declares
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
