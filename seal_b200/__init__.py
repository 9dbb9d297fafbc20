"""seal_b200 -- Python (ctypes) binding of libseal_b200.so, the H100 (sm_90a) drop-in for the RNS-polynomial hot
path of microsoft/SEAL (NTT/INTT, CKKS/BFV/BGV multiply, relinearize, rotate, rescale) and the operations around it
(plaintext operations, wire format, BatchEncoder, Decryptor -- SURVEY 8f).

The product is the C-ABI library (include/seal_b200.h) and, for C++ users, the header-only shims
(include/seal_b200/{evaluator,batchencoder,decryptor}.hpp).  This module exists for tests and bench.py: it mirrors the reference's operator
names (Evaluator.multiply / relinearize / rescale_to_next / rotate_rows / apply_galois / transform_to_ntt ...)
on raw uint64 slabs laid out like seal::Ciphertext::data().  There is no CPU fallback: importing works anywhere, but
creating a Context raises unless the CUDA library is built and an H100 is present.
"""
import ctypes as C
import os

import numpy as np

BFV, CKKS, BGV = 1, 2, 3
# step modes of add_many (SB200_FOLD_*): add or sub, optionally ORed with FOLD_SCALED
FOLD_ADD, FOLD_SUB, FOLD_SCALED = 0, 1, 2
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libseal_b200.so")
_u64p = C.POINTER(C.c_uint64)
_lib = None

_STATUS = {-1: ValueError, -2: RuntimeError, -3: IndexError, -4: RuntimeError, -5: MemoryError, -6: ValueError}

# every symbol include/seal_b200.h declares (checked by tests/test_host_logic.py)
SYMBOLS = [
    "sb200_last_error", "sb200_context_create", "sb200_context_destroy", "sb200_coeff_modulus_create",
    "sb200_get_ntt_tables", "sb200_get_base_bsk", "sb200_galois_elt_from_step", "sb200_launch_count",
    "sb200_device_bytes", "sb200_context_set_limit", "sb200_device_malloc", "sb200_device_free", "sb200_host_malloc", "sb200_host_free", "sb200_memcpy_h2d", "sb200_memcpy_d2h", "sb200_memcpy_d2d", "sb200_memcpy_d2d_2d", "sb200_stream_synchronize", "sb200_upload_rows", "sb200_download_rows", "sb200_rescale_to_next_sized", "sb200_mod_switch_to_next_sized", "sb200_relinearize_sized", "sb200_rescale_to_next_sized_host", "sb200_mod_switch_to_next_sized_host", "sb200_relinearize_sized_host", "sb200_device_numa_node", "sb200_device_index", "sb200_keyswitch_chunk", "sb200_profile_enable", "sb200_profile_reset", "sb200_profile_read", "sb200_profile_read_work", "sb200_selftest_rate", "sb200_profile_read_work32", "sb200_selftest_ksint_info", "sb200_selftest_ksint_forward", "sb200_selftest_ksint_inverse", "sb200_selftest_ksint_product",
    "sb200_kswitch_key_create", "sb200_kswitch_key_load", "sb200_kswitch_keys_load", "sb200_kswitch_key_device_bytes",
    "sb200_kswitch_key_destroy", "sb200_ntt_forward",
    "sb200_ntt_inverse", "sb200_multiply", "sb200_multiply_sized", "sb200_square", "sb200_add", "sb200_sub", "sb200_negate", "sb200_multiply_plain", "sb200_batch_encode", "sb200_batch_decode", "sb200_plain_to_ntt", "sb200_multiply_plain_coeff", "sb200_add_plain_coeff", "sb200_relinearize", "sb200_multiply_relinearize", "sb200_rescale_to_next",
    "sb200_mod_switch_to_next", "sb200_apply_galois", "sb200_ntt_forward_host", "sb200_ntt_inverse_host",
    "sb200_multiply_host", "sb200_multiply_sized_host", "sb200_square_host", "sb200_add_host", "sb200_sub_host", "sb200_negate_host", "sb200_multiply_plain_host", "sb200_batch_encode_host", "sb200_batch_decode_host", "sb200_plain_to_ntt_host", "sb200_multiply_plain_coeff_host", "sb200_add_plain_coeff_host",
    "sb200_multiply_plain_n", "sb200_multiply_plain_coeff_n", "sb200_add_plain_coeff_n", "sb200_add_plain_ntt", "sb200_multiply_plain_n_host",
    "sb200_multiply_plain_coeff_n_host", "sb200_add_plain_coeff_n_host", "sb200_add_plain_ntt_host",
    "sb200_add_many", "sb200_add_many_host", "sb200_multiply_plain_sum", "sb200_multiply_plain_sum_host", "sb200_multiply_sum", "sb200_multiply_sum_host", "sb200_relinearize_host", "sb200_multiply_relinearize_host", "sb200_rescale_to_next_host",
    "sb200_mod_switch_to_next_host", "sb200_apply_galois_host", "sb200_apply_galois_add", "sb200_apply_galois_add_host",
    "sb200_rotate_sum", "sb200_rotate_sum_host", "sb200_apply_galois_multiply_plain_add", "sb200_apply_galois_multiply_plain_add_host",
    "sb200_diagonal_sum", "sb200_diagonal_sum_host", "sb200_get_parms_id", "sb200_ciphertext_inspect",
    "sb200_ciphertext_save_size", "sb200_ciphertext_load", "sb200_ciphertext_save", "sb200_secret_key_create",
    "sb200_secret_key_destroy", "sb200_decrypt", "sb200_decrypt_host", "sb200_invariant_noise_budget", "sb200_invariant_noise_budget_host", "sb200_encrypt_zero_symmetric", "sb200_public_key_create", "sb200_public_key_destroy", "sb200_encrypt_zero_asymmetric", "sb200_encrypt_zero_symmetric_prng", "sb200_encrypt_zero_asymmetric_prng", "sb200_encrypt_symmetric", "sb200_encrypt_asymmetric", "sb200_kswitch_key_generate", "sb200_public_key_generate", "sb200_ciphertext_save_seeded_size", "sb200_ciphertext_save_seeded",
    "sb200_public_key_generate_seeded", "sb200_kswitch_keys_save_seeded_size", "sb200_kswitch_keys_generate_seeded", "sb200_ckks_encode", "sb200_ckks_decode", "sb200_ckks_encode_host", "sb200_ckks_decode_host",
    "sb200_ckks_encode_scalar", "sb200_ckks_encode_scalar_host",
    "sb200_group_create", "sb200_group_destroy", "sb200_group_size", "sb200_group_context", "sb200_group_slice",
    "sb200_group_kswitch_key_create", "sb200_group_kswitch_key_destroy", "sb200_group_multiply_relinearize_host",
    "sb200_group_relinearize_host", "sb200_group_apply_galois_host", "sb200_group_multiply_host", "sb200_group_rescale_to_next_host",
    "sb200_group_mod_switch_to_next_host", "sb200_group_ntt_forward_host", "sb200_group_ntt_inverse_host",
]


class CtInfo(C.Structure):
    """sb200_ct_info: the metadata of one serialized seal::Ciphertext (include/seal_b200.h)"""
    _fields_ = [("parms_id", C.c_uint64 * 4), ("size", C.c_uint64), ("poly_modulus_degree", C.c_uint64),
                ("coeff_modulus_size", C.c_uint64), ("correction_factor", C.c_uint64), ("scale", C.c_double),
                ("is_ntt_form", C.c_int32), ("seeded", C.c_int32), ("data_offset", C.c_uint64), ("data_words", C.c_uint64),
                ("stream_bytes", C.c_uint64), ("seed_offset", C.c_uint64), ("compr_mode", C.c_uint64)]


def lib():
    """Load libseal_b200.so (fails loudly if the CUDA extension has not been built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp, sz, u64, i32, u32 = C.c_void_p, C.c_size_t, C.c_uint64, C.c_int, C.c_uint32
        L.sb200_last_error.restype = C.c_char_p
        L.sb200_context_create.argtypes = [i32, sz, _u64p, sz, u64, i32, C.POINTER(vp)]
        L.sb200_context_destroy.argtypes = [vp]
        L.sb200_coeff_modulus_create.argtypes = [sz, C.POINTER(i32), sz, _u64p]
        L.sb200_get_ntt_tables.argtypes = [vp, sz, _u64p, _u64p, _u64p, _u64p, _u64p]
        L.sb200_get_base_bsk.argtypes = [vp, sz, _u64p, sz, C.POINTER(sz)]
        L.sb200_galois_elt_from_step.restype = u32
        L.sb200_galois_elt_from_step.argtypes = [vp, i32]
        L.sb200_launch_count.restype = C.c_ulonglong
        L.sb200_launch_count.argtypes = [vp]
        L.sb200_device_bytes.restype = sz
        L.sb200_device_bytes.argtypes = [vp]
        L.sb200_context_set_limit.argtypes = [vp, i32, sz]
        L.sb200_keyswitch_chunk.restype = sz
        L.sb200_keyswitch_chunk.argtypes = [vp, sz, sz, i32]
        L.sb200_device_numa_node.argtypes = [vp]
        L.sb200_device_index.argtypes = [vp]
        L.sb200_profile_enable.argtypes = [vp, i32]
        L.sb200_profile_reset.argtypes = [vp]
        L.sb200_profile_read.argtypes = [vp, sz, C.c_char_p, sz, C.POINTER(C.c_double), C.POINTER(C.c_ulonglong),
                                         C.POINTER(C.c_double)]
        L.sb200_profile_read_work.argtypes = [vp, sz, C.c_char_p, sz, C.POINTER(C.c_double), C.POINTER(C.c_ulonglong),
                                              C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.sb200_selftest_rate.argtypes = [vp, i32, C.POINTER(C.c_double)]
        L.sb200_profile_read_work32.argtypes = [vp, sz, C.c_char_p, sz, C.POINTER(C.c_double), C.POINTER(C.c_ulonglong),
                                                C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                                C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.sb200_selftest_ksint_info.argtypes = [vp, C.POINTER(i32), C.POINTER(u32)]
        L.sb200_selftest_ksint_forward.argtypes = [vp, _u64p, sz, C.POINTER(u32)]
        L.sb200_selftest_ksint_inverse.argtypes = [vp, C.POINTER(u32), sz]
        L.sb200_selftest_ksint_product.argtypes = [vp, C.POINTER(u32), C.POINTER(u32), sz, sz, C.POINTER(u32), i32, C.POINTER(i32)]
        L.sb200_kswitch_key_create.argtypes = [vp, _u64p, sz, C.POINTER(vp)]
        L.sb200_kswitch_key_destroy.argtypes = [vp]
        L.sb200_kswitch_key_load.argtypes = [vp, C.c_char_p, sz, sz, C.POINTER(vp)]
        L.sb200_kswitch_keys_load.argtypes = [vp, C.c_char_p, sz, C.POINTER(sz), sz, C.POINTER(vp), C.POINTER(sz), C.POINTER(sz)]
        L.sb200_kswitch_key_device_bytes.restype = sz
        L.sb200_kswitch_key_device_bytes.argtypes = [vp]
        L.sb200_ntt_forward.argtypes = [vp, sz, sz, sz, vp, vp]
        L.sb200_ntt_inverse.argtypes = [vp, sz, sz, sz, vp, vp]
        L.sb200_multiply.argtypes = [vp, sz, sz, vp, vp, vp, vp]
        L.sb200_square.argtypes = [vp, sz, sz, vp, vp, vp]
        L.sb200_multiply_sized.argtypes = [vp, sz, sz, sz, sz, vp, vp, vp, vp]
        L.sb200_multiply_sized_host.argtypes = [vp, sz, sz, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_add.argtypes = [vp, sz, sz, sz, vp, vp, vp, vp]
        L.sb200_sub.argtypes = [vp, sz, sz, sz, vp, vp, vp, vp]
        L.sb200_negate.argtypes = [vp, sz, sz, sz, vp, vp, vp]
        L.sb200_multiply_plain.argtypes = [vp, sz, sz, sz, vp, vp, vp, vp]
        L.sb200_multiply_plain_host.argtypes = [vp, sz, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_batch_encode.argtypes = [vp, sz, vp, vp, vp]
        L.sb200_batch_decode.argtypes = [vp, sz, vp, vp, vp]
        L.sb200_batch_encode_host.argtypes = [vp, sz, _u64p, _u64p]
        L.sb200_batch_decode_host.argtypes = [vp, sz, _u64p, _u64p]
        L.sb200_plain_to_ntt.argtypes = [vp, sz, sz, vp, vp, vp]
        L.sb200_multiply_plain_coeff.argtypes = [vp, sz, sz, sz, i32, vp, vp, vp, vp]
        L.sb200_add_plain_coeff.argtypes = [vp, sz, sz, sz, i32, vp, vp, _u64p, vp, vp]
        L.sb200_plain_to_ntt_host.argtypes = [vp, sz, sz, _u64p, _u64p]
        L.sb200_multiply_plain_coeff_host.argtypes = [vp, sz, sz, sz, i32, _u64p, _u64p, _u64p]
        L.sb200_add_plain_coeff_host.argtypes = [vp, sz, sz, sz, i32, _u64p, _u64p, _u64p, _u64p]
        L.sb200_multiply_plain_n.argtypes = [vp, sz, sz, sz, sz, vp, vp, vp, vp]
        L.sb200_multiply_plain_coeff_n.argtypes = [vp, sz, sz, sz, sz, i32, vp, vp, vp, vp]
        L.sb200_add_plain_coeff_n.argtypes = [vp, sz, sz, sz, sz, i32, vp, vp, _u64p, vp, vp]
        L.sb200_add_plain_ntt.argtypes = [vp, sz, sz, sz, sz, i32, vp, vp, vp, vp]
        L.sb200_multiply_plain_n_host.argtypes = [vp, sz, sz, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_multiply_plain_coeff_n_host.argtypes = [vp, sz, sz, sz, sz, i32, _u64p, _u64p, _u64p]
        L.sb200_add_plain_coeff_n_host.argtypes = [vp, sz, sz, sz, sz, i32, _u64p, _u64p, _u64p, _u64p]
        L.sb200_add_plain_ntt_host.argtypes = [vp, sz, sz, sz, sz, i32, _u64p, _u64p, _u64p]
        L.sb200_square_host.argtypes = [vp, sz, sz, _u64p, _u64p]
        L.sb200_add_host.argtypes = [vp, sz, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_add_many.argtypes = [vp, sz, sz, sz, C.POINTER(sz), C.POINTER(vp), C.POINTER(i32), _u64p, vp, vp]
        L.sb200_add_many_host.argtypes = [vp, sz, sz, sz, C.POINTER(sz), C.POINTER(vp), C.POINTER(i32), _u64p, _u64p]
        L.sb200_multiply_plain_sum.argtypes = [vp, sz, sz, sz, sz, C.POINTER(sz), C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), i32, i32,
                                               C.POINTER(i32), _u64p, C.POINTER(vp), vp]
        L.sb200_multiply_plain_sum_host.argtypes = [vp, sz, sz, sz, sz, C.POINTER(sz), C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), i32, i32,
                                                    C.POINTER(i32), _u64p, C.POINTER(vp)]
        L.sb200_multiply_sum.argtypes = [vp, sz, sz, sz, sz, C.POINTER(vp), C.POINTER(vp), C.POINTER(i32), _u64p, C.POINTER(vp), vp]
        L.sb200_multiply_sum_host.argtypes = [vp, sz, sz, sz, sz, C.POINTER(vp), C.POINTER(vp), C.POINTER(i32), _u64p, C.POINTER(vp)]
        L.sb200_sub_host.argtypes = [vp, sz, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_negate_host.argtypes = [vp, sz, sz, sz, _u64p, _u64p]
        L.sb200_relinearize.argtypes = [vp, sz, sz, vp, vp, vp, vp]
        L.sb200_multiply_relinearize.argtypes = [vp, sz, sz, vp, vp, vp, vp, vp]
        L.sb200_rescale_to_next.argtypes = [vp, sz, sz, vp, vp, vp]
        L.sb200_mod_switch_to_next.argtypes = [vp, sz, sz, vp, vp, vp]
        L.sb200_rescale_to_next_sized.argtypes = [vp, sz, sz, sz, vp, vp, vp]
        L.sb200_mod_switch_to_next_sized.argtypes = [vp, sz, sz, sz, vp, vp, vp]
        L.sb200_apply_galois.argtypes = [vp, sz, sz, vp, u32, vp, vp, vp]
        L.sb200_ntt_forward_host.argtypes = [vp, sz, sz, sz, _u64p]
        L.sb200_ntt_inverse_host.argtypes = [vp, sz, sz, sz, _u64p]
        L.sb200_multiply_host.argtypes = [vp, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_relinearize_host.argtypes = [vp, sz, sz, _u64p, vp, _u64p]
        L.sb200_multiply_relinearize_host.argtypes = [vp, sz, sz, _u64p, _u64p, vp, _u64p]
        L.sb200_rescale_to_next_host.argtypes = [vp, sz, sz, _u64p, _u64p]
        L.sb200_mod_switch_to_next_host.argtypes = [vp, sz, sz, _u64p, _u64p]
        L.sb200_apply_galois_host.argtypes = [vp, sz, sz, _u64p, u32, vp, _u64p]
        L.sb200_apply_galois_add.argtypes = [vp, sz, sz, vp, u32, vp, vp, vp, vp]
        L.sb200_apply_galois_add_host.argtypes = [vp, sz, sz, _u64p, u32, vp, _u64p, _u64p]
        L.sb200_rotate_sum.argtypes = [vp, sz, sz, vp, sz, C.POINTER(u32), C.POINTER(vp), vp, vp]
        L.sb200_rotate_sum_host.argtypes = [vp, sz, sz, _u64p, sz, C.POINTER(u32), C.POINTER(vp), _u64p]
        L.sb200_apply_galois_multiply_plain_add.argtypes = [vp, sz, sz, vp, u32, vp, sz, vp, vp, vp, vp]
        L.sb200_apply_galois_multiply_plain_add_host.argtypes = [vp, sz, sz, _u64p, u32, vp, sz, _u64p, _u64p, _u64p]
        L.sb200_diagonal_sum.argtypes = [vp, sz, sz, vp, sz, C.POINTER(u32), C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.c_int, vp, vp]
        L.sb200_diagonal_sum_host.argtypes = [vp, sz, sz, _u64p, sz, C.POINTER(u32), C.POINTER(vp), C.POINTER(sz), C.POINTER(vp), C.c_int, _u64p]
        L.sb200_rescale_to_next_sized_host.argtypes = [vp, sz, sz, sz, _u64p, _u64p]
        L.sb200_mod_switch_to_next_sized_host.argtypes = [vp, sz, sz, sz, _u64p, _u64p]
        L.sb200_relinearize_sized_host.argtypes = [vp, sz, sz, sz, _u64p, vp, _u64p]
        L.sb200_get_parms_id.argtypes = [vp, sz, _u64p]
        L.sb200_ciphertext_inspect.argtypes = [C.c_char_p, sz, C.POINTER(CtInfo)]
        L.sb200_ciphertext_save_size.restype = sz
        L.sb200_ciphertext_save_size.argtypes = [vp, sz, sz]
        L.sb200_ciphertext_load.argtypes = [vp, sz, C.POINTER(C.c_char_p), C.POINTER(sz), sz, sz, i32, vp, C.POINTER(CtInfo), vp]
        L.sb200_ciphertext_save.argtypes = [vp, sz, sz, sz, vp, C.POINTER(CtInfo), C.POINTER(vp), sz, vp]
        L.sb200_secret_key_create.argtypes = [vp, _u64p, C.POINTER(vp)]
        L.sb200_secret_key_destroy.argtypes = [vp]
        L.sb200_decrypt.argtypes = [vp, vp, sz, sz, sz, vp, _u64p, vp, vp]
        L.sb200_ckks_encode.argtypes = [vp, sz, sz, vp, sz, i32, C.c_double, vp, vp]
        L.sb200_ckks_decode.argtypes = [vp, sz, sz, vp, C.c_double, vp, vp]
        L.sb200_ckks_encode_host.argtypes = [vp, sz, sz, vp, sz, i32, C.c_double, _u64p]
        L.sb200_ckks_decode_host.argtypes = [vp, sz, sz, _u64p, C.c_double, vp]
        L.sb200_ckks_encode_scalar.argtypes = [vp, sz, sz, i32, vp, C.c_double, vp, vp]
        L.sb200_ckks_encode_scalar_host.argtypes = [vp, sz, sz, i32, vp, C.c_double, _u64p]
        L.sb200_public_key_create.argtypes = [vp, _u64p, C.POINTER(vp)]
        L.sb200_public_key_destroy.argtypes = [vp]
        L.sb200_encrypt_zero_asymmetric.argtypes = [vp, vp, sz, sz, _u64p, vp, vp]
        L.sb200_encrypt_zero_symmetric.argtypes = [vp, vp, sz, sz, _u64p, i32, vp, _u64p, vp]
        L.sb200_encrypt_zero_asymmetric_prng.argtypes = [vp, vp, sz, sz, i32, _u64p, vp, vp]
        L.sb200_encrypt_zero_symmetric_prng.argtypes = [vp, vp, sz, sz, i32, i32, _u64p, i32, vp, _u64p, vp]
        L.sb200_encrypt_symmetric.argtypes = [vp, vp, sz, sz, vp, i32, i32, _u64p, i32, vp, _u64p, vp]
        L.sb200_encrypt_asymmetric.argtypes = [vp, vp, sz, sz, vp, i32, _u64p, vp, vp]
        L.sb200_decrypt_host.argtypes = [vp, vp, sz, sz, sz, _u64p, _u64p, _u64p]
        L.sb200_kswitch_key_generate.argtypes = [vp, vp, u32, i32, i32, _u64p, _u64p, C.POINTER(vp)]
        L.sb200_public_key_generate.argtypes = [vp, vp, i32, i32, _u64p, _u64p, C.POINTER(vp)]
        L.sb200_ciphertext_save_seeded_size.restype = sz
        L.sb200_ciphertext_save_seeded_size.argtypes = [vp, sz]
        L.sb200_ciphertext_save_seeded.argtypes = [vp, sz, sz, vp, C.POINTER(CtInfo), _u64p, i32, C.POINTER(vp), sz, vp]
        L.sb200_public_key_generate_seeded.argtypes = [vp, vp, i32, i32, _u64p, vp, sz, C.POINTER(vp)]
        L.sb200_kswitch_keys_save_seeded_size.restype = sz
        L.sb200_kswitch_keys_save_seeded_size.argtypes = [vp, C.POINTER(u32), sz]
        L.sb200_kswitch_keys_generate_seeded.argtypes = [vp, vp, C.POINTER(u32), sz, i32, i32, _u64p, vp, sz]
        L.sb200_invariant_noise_budget.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp]
        L.sb200_invariant_noise_budget_host.argtypes = [vp, vp, sz, sz, sz, _u64p, C.POINTER(i32)]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise _STATUS.get(rc, RuntimeError)(f"seal_b200 error {rc}: {lib().sb200_last_error().decode()}")


def ciphertext_inspect(stream):
    """metadata of one Ciphertext::save(compr_mode_type::none) stream (pure host, no context needed)"""
    info = CtInfo()
    _check(lib().sb200_ciphertext_inspect(stream, len(stream), C.byref(info)))
    return info


def _hp(a):
    assert isinstance(a, np.ndarray) and a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"], "need C-contiguous uint64"
    return a.ctypes.data_as(_u64p)


def _rotate_sum_args(galois_elts, keys):
    """the element and key-handle arrays of a rotate_sum call (a None key stays a NULL entry)"""
    assert len(galois_elts) == len(keys), "one key per Galois element"
    m = len(galois_elts)
    c_elts = (C.c_uint32 * max(m, 1))(*[int(e) for e in galois_elts])
    c_keys = (C.c_void_p * max(m, 1))(*[None if k is None else k.h for k in keys])
    return c_elts, c_keys


def _dp(t):
    """device pointer of a torch int64/uint64 CUDA tensor (or a raw int)"""
    if isinstance(t, int):
        return C.c_void_p(t)
    assert t.is_cuda and t.is_contiguous() and t.element_size() == 8
    return C.c_void_p(t.data_ptr())


def coeff_modulus_create(n, bits):
    """CoeffModulus::Create (modulus.cpp:144-184)"""
    out = np.zeros(len(bits), dtype=np.uint64)
    b = (C.c_int * len(bits))(*bits)
    _check(lib().sb200_coeff_modulus_create(n, b, len(bits), _hp(out)))
    return [int(x) for x in out]


class KSwitchKey:
    """Device copy of one KSwitchKeys::data()[index] entry ([digit][2][k][n])."""

    def __init__(self, ctx, host_key, stream_index=None):
        self.ctx = ctx
        if stream_index is not None:
            # host_key is a serialized RelinKeys / GaloisKeys object (KSwitchKeys::save, compr_mode none)
            h = C.c_void_p()
            _check(lib().sb200_kswitch_key_load(ctx.h, host_key, len(host_key), stream_index, C.byref(h)))
            self.h = h
            return
        host_key = np.ascontiguousarray(host_key, dtype=np.uint64)
        assert host_key.ndim == 4 and host_key.shape[1] == 2 and host_key.shape[2] == ctx.k and host_key.shape[3] == ctx.n
        self.ctx = ctx
        h = C.c_void_p()
        _check(lib().sb200_kswitch_key_create(ctx.h, _hp(host_key), host_key.shape[0], C.byref(h)))
        self.h = h

    @classmethod
    def wrap(cls, ctx, handle):
        """take ownership of a key handle the library made (sb200_kswitch_key_generate)"""
        self = cls.__new__(cls)
        self.ctx, self.h = ctx, handle
        return self

    @property
    def device_bytes(self):
        """bytes the key holds on the device: its words plus the integer key-switching path's copy"""
        return lib().sb200_kswitch_key_device_bytes(self.h)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                lib().sb200_kswitch_key_destroy(self.h)
                self.h = None
        except Exception:
            pass


class PublicKey:
    """Encryptor state: the public key ([2][k][n], NTT form at the key level) on the device."""

    def __init__(self, ctx, host_key):
        host_key = np.ascontiguousarray(host_key, dtype=np.uint64)
        assert host_key.shape == (2, ctx.k, ctx.n)
        self.ctx = ctx
        h = C.c_void_p()
        _check(lib().sb200_public_key_create(ctx.h, _hp(host_key), C.byref(h)))
        self.h = h

    @classmethod
    def wrap(cls, ctx, handle):
        """take ownership of a key handle the library made (sb200_public_key_generate)"""
        self = cls.__new__(cls)
        self.ctx, self.h = ctx, handle
        return self

    def __del__(self):
        try:
            if getattr(self, "h", None):
                lib().sb200_public_key_destroy(self.h)
                self.h = None
        except Exception:
            pass


class SecretKey:
    """Decryptor state: the secret key ([k][n], NTT form at the key level) and its powers on the device."""

    def __init__(self, ctx, host_key):
        host_key = np.ascontiguousarray(host_key, dtype=np.uint64)
        assert host_key.shape == (ctx.k, ctx.n)
        self.ctx = ctx
        h = C.c_void_p()
        _check(lib().sb200_secret_key_create(ctx.h, _hp(host_key), C.byref(h)))
        self.h = h

    def __del__(self):
        try:
            if getattr(self, "h", None):
                lib().sb200_secret_key_destroy(self.h)
                self.h = None
        except Exception:
            pass


class Context:
    """SEALContext(parms, true, sec_level none) + Evaluator for the hot path, on one H100.

    Host-array methods (numpy in / numpy out) go through the *_host C-ABI entry points; the d_* methods take torch
    CUDA int64 tensors (device-resident slabs) and are stream-ordered on the current torch stream.
    """

    def __init__(self, scheme, n, moduli, plain_modulus=0, device=0):
        self.scheme, self.n, self.moduli, self.k, self.t = scheme, n, [int(m) for m in moduli], len(moduli), plain_modulus
        self.device = device
        m = np.array(self.moduli, dtype=np.uint64)
        h = C.c_void_p()
        _check(lib().sb200_context_create(scheme, n, _hp(m), self.k, plain_modulus, device, C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            lib().sb200_context_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- tables ----
    def ntt_tables(self, i):
        n = self.n
        root, inv_n = C.c_uint64(0), C.c_uint64(0)
        rp, rq, irp = (np.zeros(n, dtype=np.uint64) for _ in range(3))
        _check(lib().sb200_get_ntt_tables(self.h, i, C.byref(root), _hp(rp), _hp(rq), _hp(irp), C.byref(inv_n)))
        return root.value, rp, rq, irp, inv_n.value

    def base_bsk(self, L):
        out = np.zeros(self.k + 4, dtype=np.uint64)
        cnt = C.c_size_t(0)
        _check(lib().sb200_get_base_bsk(self.h, L, _hp(out), len(out), C.byref(cnt)))
        return [int(x) for x in out[: cnt.value]]

    def galois_elt_from_step(self, step):
        return int(lib().sb200_galois_elt_from_step(self.h, step))

    @property
    def launch_count(self):
        return int(lib().sb200_launch_count(self.h))

    @property
    def device_bytes(self):
        return int(lib().sb200_device_bytes(self.h))

    LIMIT_SCRATCH_BYTES, LIMIT_KS_CHUNK, LIMIT_HOST_STAGE_BYTES, LIMIT_KS_ALGORITHM = 0, 1, 2, 3

    def set_limit(self, which, value):
        """sb200_context_set_limit: how a batch is cut into device chunks (results never depend on it)"""
        _check(lib().sb200_context_set_limit(self.h, which, value))

    def keyswitch_chunk(self, L, batch, fused=True):
        return int(lib().sb200_keyswitch_chunk(self.h, L, batch, 1 if fused else 0))

    def profile(self, on=True):
        _check(lib().sb200_profile_enable(self.h, 1 if on else 0))
        _check(lib().sb200_profile_reset(self.h))

    def profile_read(self):
        """[(kernel name, total device ms, launches, algorithmic bytes)] since the last profile()/reset"""
        out, i = [], 0
        name = C.create_string_buffer(128)
        ms, n, by = C.c_double(0), C.c_ulonglong(0), C.c_double(0)
        while lib().sb200_profile_read(self.h, i, name, 128, C.byref(ms), C.byref(n), C.byref(by)) == 0:
            out.append((name.value.decode(), ms.value, n.value, by.value))
            i += 1
        return out

    def profile_read_work(self):
        """[(kernel name, total device ms, launches, algorithmic bytes, butterflies, multiply-accumulates)]"""
        out, i = [], 0
        name = C.create_string_buffer(128)
        ms, n, by, bf, mc = C.c_double(0), C.c_ulonglong(0), C.c_double(0), C.c_double(0), C.c_double(0)
        while lib().sb200_profile_read_work(self.h, i, name, 128, C.byref(ms), C.byref(n), C.byref(by), C.byref(bf), C.byref(mc)) == 0:
            out.append((name.value.decode(), ms.value, n.value, by.value, bf.value, mc.value))
            i += 1
        return out

    def profile_read_work32(self):
        """profile_read_work + (32-bit butterflies, 32x32->64 multiply-accumulates) of the integer key-switching path"""
        out, i = [], 0
        name = C.create_string_buffer(128)
        ms, n, by, bf, mc, b32, m32 = C.c_double(0), C.c_ulonglong(0), C.c_double(0), C.c_double(0), C.c_double(0), C.c_double(0), C.c_double(0)
        while lib().sb200_profile_read_work32(self.h, i, name, 128, C.byref(ms), C.byref(n), C.byref(by), C.byref(bf), C.byref(mc),
                                              C.byref(b32), C.byref(m32)) == 0:
            out.append((name.value.decode(), ms.value, n.value, by.value, bf.value, mc.value, b32.value, m32.value))
            i += 1
        return out

    def ksint_primes(self):
        """auxiliary primes of the integer key-switching path ([] when it is not available: n < 4096)"""
        cnt, pr = C.c_int(0), (C.c_uint32 * 8)()
        _check(lib().sb200_selftest_ksint_info(self.h, C.byref(cnt), pr))
        return [int(pr[i]) for i in range(cnt.value)]

    def ksint_forward(self, rows64):
        """rows [R][n] uint64 -> [S][R][n] uint32: residues modulo the auxiliary primes, transformed (bit-reversed order)"""
        rows64 = np.ascontiguousarray(rows64, dtype=np.uint64)
        S = len(self.ksint_primes())
        out = np.empty((S,) + rows64.shape, dtype=np.uint32)
        _check(lib().sb200_selftest_ksint_forward(self.h, rows64.ctypes.data_as(C.POINTER(C.c_uint64)), rows64.shape[0],
                                                  out.ctypes.data_as(C.POINTER(C.c_uint32))))
        return out

    def ksint_inverse(self, data32):
        """[R][S][n] uint32 (values < 2p) -> inverse transforms, not scaled by n^-1, values in [0, 2p)"""
        data32 = np.ascontiguousarray(data32, dtype=np.uint32).copy()
        _check(lib().sb200_selftest_ksint_inverse(self.h, data32.ctypes.data_as(C.POINTER(C.c_uint32)), data32.shape[0]))
        return data32

    def ksint_product(self, dh, key32, kernel):
        """the product step alone: dh [S][L][B][n], key32 [S][L][2][L+1][n] uint32 (canonical residues) -> (Acc [B][2][L+1][S][n]
        with values in [0, 2p), the kernel that ran: 0 register tile, 1 key tile, 2 tensor cores); kernel 0 = the integer-pipe
        kernels, 1 = the INT8 tensor-core kernel where the shape allows it (L <= 32, B >= 16)"""
        dh = np.ascontiguousarray(dh, dtype=np.uint32)
        key32 = np.ascontiguousarray(key32, dtype=np.uint32)
        S, L, B, n = dh.shape
        assert key32.shape == (S, L, 2, L + 1, n)
        out = np.empty((B, 2, L + 1, S, n), dtype=np.uint32)
        ran = C.c_int(-1)
        _check(lib().sb200_selftest_ksint_product(self.h, dh.ctypes.data_as(C.POINTER(C.c_uint32)),
                                                  key32.ctypes.data_as(C.POINTER(C.c_uint32)), L, B,
                                                  out.ctypes.data_as(C.POINTER(C.c_uint32)), kernel, C.byref(ran)))
        return out, ran.value

    def selftest_rate(self, kind):
        """warp-level butterflies (kind 0, 1, 2) / key multiply-accumulates (kind 3) per second, registers only"""
        v = C.c_double(0)
        _check(lib().sb200_selftest_rate(self.h, kind, C.byref(v)))
        return v.value

    def load_key(self, host_key):
        return KSwitchKey(self, host_key)

    def load_key_stream(self, stream, index=0):
        """KSwitchKeys::load of data()[index] from a serialized RelinKeys (index 0) / GaloisKeys ((elt - 1) // 2) object"""
        return KSwitchKey(self, stream, stream_index=index)

    # ---- host-buffer API: a is [batch][size][L][n] (or [size][L][n] for a single ciphertext) ----
    @staticmethod
    def _batched(a, ndim_single=3):
        a = np.ascontiguousarray(a, dtype=np.uint64)
        single = a.ndim == ndim_single
        return (a[None] if single else a), single

    def transform_to_ntt(self, a):
        a, single = self._batched(a)
        d = a.copy()
        _check(lib().sb200_ntt_forward_host(self.h, d.shape[2], d.shape[1], d.shape[0], _hp(d)))
        return d[0] if single else d

    def transform_from_ntt(self, a):
        a, single = self._batched(a)
        d = a.copy()
        _check(lib().sb200_ntt_inverse_host(self.h, d.shape[2], d.shape[1], d.shape[0], _hp(d)))
        return d[0] if single else d

    def multiply(self, a, b):
        a, single = self._batched(a)
        b, _ = self._batched(b)
        B, sa, L, n = a.shape
        sb_ = b.shape[1]
        if (sa, sb_) != (2, 2):  # general-size branch of Evaluator::multiply
            out = np.zeros((B, sa + sb_ - 1, L, n), dtype=np.uint64)
            _check(lib().sb200_multiply_sized_host(self.h, L, sa, sb_, B, _hp(a), _hp(b), _hp(out)))
            return out[0] if single else out
        out = np.zeros((B, 3, L, n), dtype=np.uint64)
        _check(lib().sb200_multiply_host(self.h, L, B, _hp(a), _hp(b), _hp(out)))
        return out[0] if single else out

    def square(self, a):
        a, single = self._batched(a)
        B, _, L, n = a.shape
        out = np.zeros((B, 3, L, n), dtype=np.uint64)
        _check(lib().sb200_square_host(self.h, L, B, _hp(a), _hp(out)))
        return out[0] if single else out

    def _linear(self, fn, a, b=None):
        a, single = self._batched(a)
        B, size, L, n = a.shape
        out = np.zeros_like(a)
        if b is None:
            _check(fn(self.h, L, size, B, _hp(a), _hp(out)))
        else:
            b, _ = self._batched(b)
            assert b.shape == a.shape
            _check(fn(self.h, L, size, B, _hp(a), _hp(b), _hp(out)))
        return out[0] if single else out

    def add(self, a, b):
        return self._linear(lib().sb200_add_host, a, b)

    def sub(self, a, b):
        return self._linear(lib().sb200_sub_host, a, b)

    def negate(self, a):
        return self._linear(lib().sb200_negate_host, a)

    @staticmethod
    def _fold_args(sizes, modes, factors):
        """ctypes arrays of sb200_add_many: sizes [count], modes [count - 1] or None, factors [count - 1][2] or None"""
        count = len(sizes)
        c_sizes = (C.c_size_t * max(count, 1))(*sizes)
        c_modes = None if modes is None else (C.c_int * max(count - 1, 1))(*[int(m) for m in modes])
        f = None if factors is None else np.ascontiguousarray(factors, dtype=np.uint64).reshape(-1)
        return c_sizes, c_modes, f

    def add_many(self, operands, modes=None, factors=None):
        """Evaluator.add_many generalised (sb200_add_many): operands [B][size_j][L][n] (sizes may differ) folded left in one pass;
        modes[j - 1] is step j's FOLD_* mode (None: every step adds), factors[j - 1] = (e1_j, e2_j) the scalars of a scaled step.
        Returns [B][max size_j][L][n]."""
        ops = [self._batched(a)[0] for a in operands]
        single = len(operands) > 0 and np.asarray(operands[0]).ndim == 3
        B, _, L, n = ops[0].shape if ops else (0, 0, 0, 0)
        sizes = [a.shape[1] for a in ops]
        c_sizes, c_modes, f = self._fold_args(sizes, modes, factors)
        out = np.zeros((B, max(sizes) if sizes else 0, L, n), dtype=np.uint64)
        ptrs = (C.c_void_p * max(len(ops), 1))(*[a.ctypes.data for a in ops])
        _check(lib().sb200_add_many_host(self.h, L, B, len(ops), c_sizes, ptrs, c_modes, None if f is None else _hp(f), _hp(out)))
        return out[0] if single else out

    def multiply_plain_sum(self, cts, plains, modes=None, factors=None, ct_is_ntt=True, plain_is_ntt=True):
        """sb200_multiply_plain_sum_host: cts = K arrays [B][size_i][L][n], plains = M K arrays, plains[j K + i] [count][L][n] (NTT
        form) or [count][n] (coefficient form), count 1 (shared) or B; modes / factors as in add_many.  Returns M arrays
        [B][max size_i][L][n]: output j = add_many over i of multiply_plain(cts[i], plains[j K + i])."""
        cts = [np.ascontiguousarray(a, dtype=np.uint64) for a in cts]
        plains = [np.ascontiguousarray(p, dtype=np.uint64) for p in plains]
        K = len(cts)
        M = len(plains) // K if K else 0
        B, _, L, n = cts[0].shape if cts else (0, 0, 0, 0)
        sizes = [a.shape[1] for a in cts]
        c_sizes, c_modes, f = self._fold_args(sizes, modes, factors)
        outs = [np.zeros((B, max(sizes) if sizes else 0, L, n), dtype=np.uint64) for _ in range(M)]
        counts = (C.c_size_t * max(len(plains), 1))(*[p.shape[0] for p in plains])
        p_cts = (C.c_void_p * max(K, 1))(*[a.ctypes.data for a in cts])
        p_plains = (C.c_void_p * max(len(plains), 1))(*[p.ctypes.data for p in plains])
        p_outs = (C.c_void_p * max(M, 1))(*[o.ctypes.data for o in outs])
        _check(lib().sb200_multiply_plain_sum_host(self.h, L, B, K, M, c_sizes, p_cts, counts, p_plains, int(ct_is_ntt), int(plain_is_ntt),
                                                   c_modes, None if f is None else _hp(f), p_outs))
        return outs

    def multiply_sum(self, lhs, rhs, modes=None, factors=None):
        """sb200_multiply_sum_host: lhs = M K arrays and rhs = K arrays, each [B][2][L][n]; modes / factors as in add_many.  Returns
        M arrays [B][3][L][n]: output j = add_many over i of multiply(lhs[j K + i], rhs[i])."""
        lhs = [np.ascontiguousarray(a, dtype=np.uint64) for a in lhs]
        rhs = [np.ascontiguousarray(a, dtype=np.uint64) for a in rhs]
        K = len(rhs)
        M = len(lhs) // K if K else 0
        B, _, L, n = rhs[0].shape if rhs else (0, 0, 0, 0)
        _, c_modes, f = self._fold_args([3] * K, modes, factors)
        outs = [np.zeros((B, 3, L, n), dtype=np.uint64) for _ in range(M)]
        p_lhs = (C.c_void_p * max(len(lhs), 1))(*[a.ctypes.data for a in lhs])
        p_rhs = (C.c_void_p * max(K, 1))(*[a.ctypes.data for a in rhs])
        p_outs = (C.c_void_p * max(M, 1))(*[o.ctypes.data for o in outs])
        _check(lib().sb200_multiply_sum_host(self.h, L, B, K, M, p_lhs, p_rhs, c_modes, None if f is None else _hp(f), p_outs))
        return outs

    def multiply_plain(self, a, plain):
        """Evaluator.multiply_plain, NTT-form ciphertext [B][size][L][n] x NTT-form plaintexts [B][L][n]"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        plain = np.ascontiguousarray(plain).reshape(B, L, n)
        out = np.zeros_like(a)
        _check(lib().sb200_multiply_plain_host(self.h, L, size, B, _hp(a), _hp(plain), _hp(out)))
        return out[0] if single else out

    def batch_encode(self, values):
        """BatchEncoder.encode: [B][n] matrix slots (< t) -> coefficient-form plaintexts [B][n]"""
        v = np.ascontiguousarray(values, dtype=np.uint64)
        single = v.ndim == 1
        v = v[None] if single else v
        out = np.zeros_like(v)
        _check(lib().sb200_batch_encode_host(self.h, v.shape[0], _hp(v), _hp(out)))
        return out[0] if single else out

    def batch_decode(self, plain):
        """BatchEncoder.decode: coefficient-form plaintexts [B][n] -> matrix slots [B][n]"""
        p = np.ascontiguousarray(plain, dtype=np.uint64)
        single = p.ndim == 1
        p = p[None] if single else p
        out = np.zeros_like(p)
        _check(lib().sb200_batch_decode_host(self.h, p.shape[0], _hp(p), _hp(out)))
        return out[0] if single else out

    def ckks_encode(self, values, L, scale):
        """CKKSEncoder.encode: values [B][count] (or [count]) complex128 / float64 -> plaintexts [B][L][n] (NTT form)"""
        v = np.asarray(values)
        is_complex = np.iscomplexobj(v)
        v = np.ascontiguousarray(v, dtype=np.complex128 if is_complex else np.float64)
        single = v.ndim == 1
        v2 = v[None] if single else v
        B, count = v2.shape
        out = np.zeros((B, L, self.n), dtype=np.uint64)
        _check(lib().sb200_ckks_encode_host(self.h, L, B, v2.ctypes.data if count else None, count, int(is_complex), float(scale), _hp(out)))
        return out[0] if single else out

    def ckks_decode(self, plain, scale):
        """CKKSEncoder.decode: plaintexts [B][L][n] (or [L][n]) -> [B][n/2] complex128"""
        p = np.ascontiguousarray(plain, dtype=np.uint64)
        single = p.ndim == 2
        p2 = p[None] if single else p
        B, L, n = p2.shape
        out = np.zeros((B, n // 2), dtype=np.complex128)
        _check(lib().sb200_ckks_decode_host(self.h, L, B, _hp(p2), float(scale), out.ctypes.data))
        return out[0] if single else out

    def d_ckks_encode(self, values, plain, L, batch, count, is_complex, scale):
        _check(lib().sb200_ckks_encode(self.h, L, batch, _dp(values), count, int(is_complex), float(scale), _dp(plain), self._stream()))

    CKKS_SCALAR_REAL, CKKS_SCALAR_COMPLEX, CKKS_SCALAR_INT64 = 0, 1, 2

    def ckks_encode_scalar(self, values, L, scale=1.0):
        """CKKSEncoder.encode of one scalar per plaintext: values [B] (or a scalar) float64 / complex128 / int64, the kind taken from
        the dtype (scale is ignored for int64) -> plaintexts [B][L][n] (or [L][n]), NTT form"""
        v = np.asarray(values)
        if v.dtype == np.float64:
            kind = self.CKKS_SCALAR_REAL
        elif v.dtype == np.complex128:
            kind = self.CKKS_SCALAR_COMPLEX
        elif v.dtype == np.int64:
            kind = self.CKKS_SCALAR_INT64
        else:
            raise TypeError(f"ckks_encode_scalar takes float64, complex128 or int64 values, not {v.dtype}")
        single = v.ndim == 0
        v = np.ascontiguousarray(v.reshape(-1))
        B = v.shape[0]
        out = np.zeros((B, L, self.n), dtype=np.uint64)
        _check(lib().sb200_ckks_encode_scalar_host(self.h, L, B, kind, v.ctypes.data, float(scale), _hp(out)))
        return out[0] if single else out

    def d_ckks_encode_scalar(self, values, plain, L, batch, kind, scale):
        _check(lib().sb200_ckks_encode_scalar(self.h, L, batch, int(kind), _dp(values), float(scale), _dp(plain), self._stream()))

    def d_ckks_decode(self, plain, values, L, batch, scale):
        _check(lib().sb200_ckks_decode(self.h, L, batch, _dp(plain), float(scale), _dp(values), self._stream()))

    def d_invariant_noise_budget(self, ct, sk, budgets, L, size, batch):
        """invariant_noise_budget of the device slab ct [batch][size][L][n] into the int32 CUDA tensor budgets [batch], on the
        current stream"""
        assert budgets.is_cuda and budgets.is_contiguous() and budgets.element_size() == 4
        _check(lib().sb200_invariant_noise_budget(self.h, sk.h, L, size, batch, _dp(ct), C.c_void_p(budgets.data_ptr()), self._stream()))

    def load_secret_key(self, host_key):
        return SecretKey(self, host_key)

    def decrypt(self, a, sk, correction_factors=None):
        """Decryptor.decrypt: [B][size][L][n] -> CKKS [B][L][n] (NTT-form plaintexts), BFV / BGV [B][n] (coefficients mod t)"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        out = np.zeros((B, L, n) if self.scheme == CKKS else (B, n), dtype=np.uint64)
        cf = None if correction_factors is None else _hp(np.ascontiguousarray(correction_factors, dtype=np.uint64).reshape(B))
        _check(lib().sb200_decrypt_host(self.h, sk.h, L, size, B, _hp(a), cf, _hp(out)))
        return out[0] if single else out

    def invariant_noise_budget(self, a, sk):
        """Decryptor.invariant_noise_budget of BFV (coefficient form) / BGV (NTT form) ciphertexts [B][size][L][n] (or one
        [size][L][n], B = 1) -> int32 [B]"""
        a, _ = self._batched(a)
        B, size, L, n = a.shape
        out = np.zeros(B, dtype=np.int32)
        _check(lib().sb200_invariant_noise_budget_host(self.h, sk.h, L, size, B, _hp(a), out.ctypes.data_as(C.POINTER(C.c_int))))
        return out

    def plain_to_ntt(self, plain, L):
        """Evaluator.transform_to_ntt(Plaintext, parms_id of the level with L primes): [B][n] words < t -> [B][L][n]"""
        plain = np.ascontiguousarray(plain, dtype=np.uint64)
        single = plain.ndim == 1
        p = plain[None] if single else plain
        out = np.zeros((p.shape[0], L, self.n), dtype=np.uint64)
        _check(lib().sb200_plain_to_ntt_host(self.h, L, p.shape[0], _hp(p), _hp(out)))
        return out[0] if single else out

    def multiply_plain_coeff(self, a, plain, ct_is_ntt):
        """Evaluator.multiply_plain with coefficient-form plaintexts [B][n]"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        plain = np.ascontiguousarray(plain, dtype=np.uint64).reshape(B, n)
        out = np.zeros_like(a)
        _check(lib().sb200_multiply_plain_coeff_host(self.h, L, size, B, int(ct_is_ntt), _hp(a), _hp(plain), _hp(out)))
        return out[0] if single else out

    def add_plain_coeff(self, a, plain, subtract=False, correction_factors=None):
        """Evaluator.add_plain / sub_plain with coefficient-form plaintexts [B][n] (BFV, BGV)"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        plain = np.ascontiguousarray(plain, dtype=np.uint64).reshape(B, n)
        out = np.zeros_like(a)
        cf = None if correction_factors is None else _hp(np.ascontiguousarray(correction_factors, dtype=np.uint64).reshape(B))
        _check(lib().sb200_add_plain_coeff_host(self.h, L, size, B, int(subtract), _hp(a), _hp(plain), cf, _hp(out)))
        return out[0] if single else out

    # ---- plaintext operations with one plaintext per ciphertext ([B] leading axis) or one for the whole batch (no batch axis) ----
    def _plains(self, plain, B, shape):
        """plaintexts as (plain_count, contiguous uint64 array): [B] + shape, or shape alone (one plaintext for the batch)"""
        p = np.ascontiguousarray(plain, dtype=np.uint64)
        count = 1 if p.shape == tuple(shape) else B
        assert p.shape in (tuple(shape), (B,) + tuple(shape)), (p.shape, shape)
        return count, p

    def multiply_plain_n(self, a, plain):
        """Evaluator.multiply_plain, NTT-form ciphertexts [B][size][L][n] x NTT-form plaintexts [B][L][n] or one [L][n]"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        count, p = self._plains(plain, B, (L, n))
        out = np.zeros_like(a)
        _check(lib().sb200_multiply_plain_n_host(self.h, L, size, B, count, _hp(a), _hp(p), _hp(out)))
        return out[0] if single else out

    def multiply_plain_coeff_n(self, a, plain, ct_is_ntt):
        """Evaluator.multiply_plain with coefficient-form plaintexts [B][n] or one [n]"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        count, p = self._plains(plain, B, (n,))
        out = np.zeros_like(a)
        _check(lib().sb200_multiply_plain_coeff_n_host(self.h, L, size, B, count, int(ct_is_ntt), _hp(a), _hp(p), _hp(out)))
        return out[0] if single else out

    def add_plain_coeff_n(self, a, plain, subtract=False, correction_factors=None):
        """Evaluator.add_plain / sub_plain with coefficient-form plaintexts [B][n] or one [n] (BFV, BGV); correction_factors: one
        per plaintext"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        count, p = self._plains(plain, B, (n,))
        out = np.zeros_like(a)
        cf = None if correction_factors is None else _hp(np.ascontiguousarray(correction_factors, dtype=np.uint64).reshape(count))
        _check(lib().sb200_add_plain_coeff_n_host(self.h, L, size, B, count, int(subtract), _hp(a), _hp(p), cf, _hp(out)))
        return out[0] if single else out

    def add_plain_ntt(self, a, plain, subtract=False):
        """CKKS Evaluator.add_plain / sub_plain: c_0 +/- NTT-form plaintexts [B][L][n] or one [L][n]"""
        a, single = self._batched(a)
        B, size, L, n = a.shape
        count, p = self._plains(plain, B, (L, n))
        out = np.zeros_like(a)
        _check(lib().sb200_add_plain_ntt_host(self.h, L, size, B, count, int(subtract), _hp(a), _hp(p), _hp(out)))
        return out[0] if single else out

    def relinearize(self, c3, key):
        c3, single = self._batched(c3)
        B, _, L, n = c3.shape
        out = np.zeros((B, 2, L, n), dtype=np.uint64)
        _check(lib().sb200_relinearize_host(self.h, L, B, _hp(c3), key.h, _hp(out)))
        return out[0] if single else out

    def multiply_relinearize(self, a, b, key):
        a, single = self._batched(a)
        b, _ = self._batched(b)
        B, _, L, n = a.shape
        out = np.zeros((B, 2, L, n), dtype=np.uint64)
        _check(lib().sb200_multiply_relinearize_host(self.h, L, B, _hp(a), _hp(b), key.h, _hp(out)))
        return out[0] if single else out

    def rescale_to_next(self, a):
        a, single = self._batched(a)
        B, size, L, n = a.shape
        out = np.zeros((B, size, max(L - 1, 0), n), dtype=np.uint64)
        _check(lib().sb200_rescale_to_next_sized_host(self.h, L, size, B, _hp(a), _hp(out)))
        return out[0] if single else out

    def mod_switch_to_next(self, a):
        a, single = self._batched(a)
        B, size, L, n = a.shape
        out = np.zeros((B, size, max(L - 1, 0), n), dtype=np.uint64)
        _check(lib().sb200_mod_switch_to_next_sized_host(self.h, L, size, B, _hp(a), _hp(out)))
        return out[0] if single else out

    def relinearize_step(self, c, key):
        """one step of relinearize_internal's loop on size >= 3 ciphertexts: (c0, c1) += switch_key(c_last); size unchanged"""
        c, single = self._batched(c)
        B, size, L, n = c.shape
        out = np.zeros_like(c)
        _check(lib().sb200_relinearize_sized_host(self.h, L, size, B, _hp(c), key.h, _hp(out)))
        return out[0] if single else out

    def apply_galois(self, a, galois_elt, key):
        a, single = self._batched(a)
        B, _, L, n = a.shape
        out = np.zeros((B, 2, L, n), dtype=np.uint64)
        _check(lib().sb200_apply_galois_host(self.h, L, B, _hp(a), galois_elt, key.h, _hp(out)))
        return out[0] if single else out

    def apply_galois_add(self, a, galois_elt, key, b, out=None):
        """sb200_apply_galois_add_host: b + apply_galois(a), a and b [B][2][L][n]; out (may be b) or a fresh array"""
        a, single = self._batched(a)
        b, _ = self._batched(b)
        B, _, L, n = a.shape
        if out is None:
            out = np.zeros((B, 2, L, n), dtype=np.uint64)
        _check(lib().sb200_apply_galois_add_host(self.h, L, B, _hp(a), galois_elt, None if key is None else key.h, _hp(b), _hp(out)))
        return out[0] if single else out

    def apply_galois_multiply_plain_add(self, a, galois_elt, key, plain, b, out=None):
        """sb200_apply_galois_multiply_plain_add_host: b + plain * apply_galois(a), a and b [B][2][L][n], plain [count][L][n] (NTT
        form, count 1 or B); out (may be b) or a fresh array"""
        a, single = self._batched(a)
        b, _ = self._batched(b)
        plain = np.ascontiguousarray(plain, dtype=np.uint64)
        if plain.ndim == 2:
            plain = plain[None]
        B, _, L, n = a.shape
        if out is None:
            out = np.zeros((B, 2, L, n), dtype=np.uint64)
        _check(lib().sb200_apply_galois_multiply_plain_add_host(self.h, L, B, _hp(a), galois_elt, None if key is None else key.h,
                                                                plain.shape[0], _hp(plain), _hp(b), _hp(out)))
        return out[0] if single else out

    def diagonal_sum(self, a, galois_elts, keys, plains, plain_is_ntt=True):
        """sb200_diagonal_sum_host: sum_i plains[i] * apply_galois(a, galois_elts[i]) with keys[i] (element 1: no rotation, its key may
        be None); a [B][2][L][n], plains[i] [count_i][L][n] (NTT form) or [count_i][n] (coefficient form), count_i 1 or B"""
        a, single = self._batched(a)
        B, _, L, n = a.shape
        plains = [np.ascontiguousarray(p, dtype=np.uint64) for p in plains]
        out = np.zeros((B, 2, L, n), dtype=np.uint64)
        c_elts, c_keys = _rotate_sum_args(galois_elts, keys)
        m = len(plains)
        counts = (C.c_size_t * max(m, 1))(*[p.shape[0] for p in plains])
        p_plains = (C.c_void_p * max(m, 1))(*[p.ctypes.data for p in plains])
        _check(lib().sb200_diagonal_sum_host(self.h, L, B, _hp(a), len(galois_elts), c_elts, c_keys, counts, p_plains, int(plain_is_ntt),
                                             _hp(out)))
        return out[0] if single else out

    def rotate_sum(self, a, galois_elts, keys):
        """sb200_rotate_sum_host: y_0 = a, y_{j+1} = y_j + apply_galois(y_j, galois_elts[j]) with keys[j]; returns y_steps"""
        a, single = self._batched(a)
        B, _, L, n = a.shape
        out = np.zeros((B, 2, L, n), dtype=np.uint64)
        c_elts, c_keys = _rotate_sum_args(galois_elts, keys)
        _check(lib().sb200_rotate_sum_host(self.h, L, B, _hp(a), len(galois_elts), c_elts, c_keys, _hp(out)))
        return out[0] if single else out

    def rotate(self, a, step, key):
        """rotate_rows (BFV) / rotate_vector (CKKS) by `step` with the Galois key of that step's element"""
        return self.apply_galois(a, self.galois_elt_from_step(step), key)

    # ---- device-resident API (torch CUDA tensors, current stream) ----
    @staticmethod
    def _stream():
        import torch

        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def d_ntt_forward(self, t, L, size, batch):
        _check(lib().sb200_ntt_forward(self.h, L, size, batch, _dp(t), self._stream()))

    def d_ntt_inverse(self, t, L, size, batch):
        _check(lib().sb200_ntt_inverse(self.h, L, size, batch, _dp(t), self._stream()))

    def d_multiply(self, a, b, out3, L, batch):
        _check(lib().sb200_multiply(self.h, L, batch, _dp(a), _dp(b), _dp(out3), self._stream()))

    def d_multiply_plain(self, a, plain, out, L, size, batch):
        _check(lib().sb200_multiply_plain(self.h, L, size, batch, _dp(a), _dp(plain), _dp(out), self._stream()))

    def d_multiply_plain_n(self, a, plain, out, L, size, batch, plain_count):
        _check(lib().sb200_multiply_plain_n(self.h, L, size, batch, plain_count, _dp(a), _dp(plain), _dp(out), self._stream()))

    def d_multiply_plain_coeff_n(self, a, plain, out, L, size, batch, plain_count, ct_is_ntt):
        _check(lib().sb200_multiply_plain_coeff_n(self.h, L, size, batch, plain_count, int(ct_is_ntt), _dp(a), _dp(plain), _dp(out),
                                                  self._stream()))

    def d_add_plain_coeff_n(self, a, plain, out, L, size, batch, plain_count, subtract=False, correction_factors=None):
        cf = None if correction_factors is None else np.ascontiguousarray(correction_factors, dtype=np.uint64).reshape(plain_count)
        _check(lib().sb200_add_plain_coeff_n(self.h, L, size, batch, plain_count, int(subtract), _dp(a), _dp(plain),
                                             None if cf is None else _hp(cf), _dp(out), self._stream()))

    def d_add_plain_ntt(self, a, plain, out, L, size, batch, plain_count, subtract=False):
        _check(lib().sb200_add_plain_ntt(self.h, L, size, batch, plain_count, int(subtract), _dp(a), _dp(plain), _dp(out), self._stream()))

    def d_add_many(self, operands, out, L, batch, sizes, modes=None, factors=None):
        """sb200_add_many on device tensors: operands [batch][sizes[j]][L][n] (tensors or raw device pointers), out
        [batch][max sizes][L][n]; modes / factors as in add_many"""
        c_sizes, c_modes, f = self._fold_args(sizes, modes, factors)
        ptrs = (C.c_void_p * max(len(operands), 1))(*[_dp(t).value for t in operands])
        _check(lib().sb200_add_many(self.h, L, batch, len(operands), c_sizes, ptrs, c_modes, None if f is None else _hp(f), _dp(out),
                                    self._stream()))

    def d_multiply_plain_sum(self, cts, plains, outs, L, batch, sizes, plain_counts, ct_is_ntt=True, plain_is_ntt=True, modes=None,
                             factors=None):
        """sb200_multiply_plain_sum on device tensors (or raw device pointers): cts [K] of [batch][sizes[i]][L][n], plains [M K] with
        plain_counts [M K], outs [M] of [batch][max sizes][L][n]; modes / factors as in add_many"""
        c_sizes, c_modes, f = self._fold_args(sizes, modes, factors)
        counts = (C.c_size_t * max(len(plain_counts), 1))(*plain_counts)
        p_cts = (C.c_void_p * max(len(cts), 1))(*[_dp(t).value for t in cts])
        p_plains = (C.c_void_p * max(len(plains), 1))(*[_dp(t).value for t in plains])
        p_outs = (C.c_void_p * max(len(outs), 1))(*[_dp(t).value for t in outs])
        _check(lib().sb200_multiply_plain_sum(self.h, L, batch, len(cts), len(outs), c_sizes, p_cts, counts, p_plains, int(ct_is_ntt),
                                              int(plain_is_ntt), c_modes, None if f is None else _hp(f), p_outs, self._stream()))

    def d_multiply_sum(self, lhs, rhs, outs, L, batch, modes=None, factors=None):
        """sb200_multiply_sum on device tensors (or raw device pointers): lhs [M K] and rhs [K] of [batch][2][L][n], outs [M] of
        [batch][3][L][n]; modes / factors as in add_many"""
        _, c_modes, f = self._fold_args([3] * len(rhs), modes, factors)
        p_lhs = (C.c_void_p * max(len(lhs), 1))(*[_dp(t).value for t in lhs])
        p_rhs = (C.c_void_p * max(len(rhs), 1))(*[_dp(t).value for t in rhs])
        p_outs = (C.c_void_p * max(len(outs), 1))(*[_dp(t).value for t in outs])
        _check(lib().sb200_multiply_sum(self.h, L, batch, len(rhs), len(outs), p_lhs, p_rhs, c_modes, None if f is None else _hp(f), p_outs,
                                        self._stream()))

    def d_multiply_sized(self, a, b, out, L, size_a, size_b, batch):
        _check(lib().sb200_multiply_sized(self.h, L, size_a, size_b, batch, _dp(a), _dp(b), _dp(out), self._stream()))

    def parms_id(self, L):
        """EncryptionParameters::parms_id() of the level with L primes (L = k: the key level)"""
        out = (C.c_uint64 * 4)()
        _check(lib().sb200_get_parms_id(self.h, L, out))
        return tuple(out)

    def d_load_ciphertexts(self, streams, out, L, size, validate=True):
        """Ciphertext::load (or unsafe_load) of serialized ciphertexts straight into the device slab `out`"""
        B = len(streams)
        arr = (C.c_char_p * B)(*streams)
        lens = (C.c_size_t * B)(*[len(s) for s in streams])
        infos = (CtInfo * B)()
        _check(lib().sb200_ciphertext_load(self.h, B, arr, lens, L, size, 1 if validate else 0, _dp(out), infos, self._stream()))
        return list(infos)

    def d_save_ciphertexts(self, t, L, size, batch, is_ntt_form, scale=1.0, correction_factor=1):
        """Ciphertext::save(compr_mode_type::none) of a device slab [batch][size][L][n] -> list of bytes"""
        cap = lib().sb200_ciphertext_save_size(self.h, L, size)
        bufs = [C.create_string_buffer(cap) for _ in range(batch)]
        outs = (C.c_void_p * batch)(*[C.addressof(b) for b in bufs])
        meta = (CtInfo * batch)()
        for m in meta:
            m.is_ntt_form, m.scale, m.correction_factor = int(is_ntt_form), scale, correction_factor
        _check(lib().sb200_ciphertext_save(self.h, batch, L, size, _dp(t), meta, outs, cap, self._stream()))
        return [b.raw for b in bufs]

    def d_save_ciphertexts_seeded(self, t, L, batch, public_seeds, prng, is_ntt_form, scale=1.0, correction_factor=1):
        """Serializable<Ciphertext>::save(compr_mode_type::none) of a device slab [batch][2][L][n] of seeded symmetric encryptions
        (made with save_seed; public_seeds [batch][8] as they returned them, prng = their ciphertext_prng) -> list of bytes: c_0 and
        the seed of c_1 per ciphertext"""
        seeds = np.ascontiguousarray(public_seeds, dtype=np.uint64).reshape(batch, 8)
        cap = lib().sb200_ciphertext_save_seeded_size(self.h, L)
        bufs = [C.create_string_buffer(cap) for _ in range(batch)]
        outs = (C.c_void_p * batch)(*[C.addressof(b) for b in bufs])
        meta = (CtInfo * batch)()
        for m in meta:
            m.is_ntt_form, m.scale, m.correction_factor = int(is_ntt_form), scale, correction_factor
        _check(lib().sb200_ciphertext_save_seeded(self.h, batch, L, _dp(t), meta, _hp(seeds), prng, outs, cap, self._stream()))
        return [b.raw for b in bufs]

    def load_public_key(self, host_key):
        return PublicKey(self, host_key)

    def d_encrypt_zero_asymmetric(self, pk, out2, L, batch, seeds=None, prng=1):
        """Encryptor(public key).encrypt_zero for a batch into the device slab out2 [batch][2][L][n]; seeds [batch][8] words (None =
        fresh from the OS entropy source) of PRNGs of type prng (SEAL's prng_type: 1 = blake2xb, 2 = shake256)"""
        seeds = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64).reshape(batch, 8)
        _check(lib().sb200_encrypt_zero_asymmetric_prng(self.h, pk.h, L, batch, prng, None if seeds is None else _hp(seeds), _dp(out2),
                                                        self._stream()))

    def d_encrypt_zero_symmetric(self, sk, out2, L, batch, bootstrap_seeds=None, save_seed=False, want_public_seeds=False,
                                 bootstrap_prng=1, ciphertext_prng=1):
        """Encryptor.encrypt_zero_symmetric for a batch into the device slab out2 [batch][2][L][n]; bootstrap_seeds [batch][8] words
        (None = fresh from the OS entropy source); returns the public seeds [batch][8] when asked for (the seeded wire form).
        bootstrap_prng = prng_type of the bootstrap PRNGs (the parameters' random generator), ciphertext_prng = the one c_1 is expanded
        with (the reference's default factory); 1 = blake2xb, 2 = shake256"""
        seeds = None if bootstrap_seeds is None else np.ascontiguousarray(bootstrap_seeds, dtype=np.uint64).reshape(batch, 8)
        pub = np.zeros((batch, 8), dtype=np.uint64) if want_public_seeds else None
        _check(lib().sb200_encrypt_zero_symmetric_prng(self.h, sk.h, L, batch, bootstrap_prng, ciphertext_prng,
                                                       None if seeds is None else _hp(seeds), int(save_seed), _dp(out2),
                                                       None if pub is None else _hp(pub), self._stream()))
        return pub

    def d_encrypt_symmetric(self, sk, plain, out2, L, batch, bootstrap_seeds=None, save_seed=False, want_public_seeds=False,
                            bootstrap_prng=1, ciphertext_prng=1):
        """Encryptor.encrypt_symmetric of the device plaintexts `plain` (CKKS: [batch][L][n] NTT form; BFV / BGV: [batch][n] words < t
        at the first level) into the device slab out2 [batch][2][L][n]; seeds, PRNG types and the returned public seeds as for
        d_encrypt_zero_symmetric"""
        seeds = None if bootstrap_seeds is None else np.ascontiguousarray(bootstrap_seeds, dtype=np.uint64).reshape(batch, 8)
        pub = np.zeros((batch, 8), dtype=np.uint64) if want_public_seeds else None
        _check(lib().sb200_encrypt_symmetric(self.h, sk.h, L, batch, _dp(plain), bootstrap_prng, ciphertext_prng,
                                             None if seeds is None else _hp(seeds), int(save_seed), _dp(out2),
                                             None if pub is None else _hp(pub), self._stream()))
        return pub

    def d_encrypt_asymmetric(self, pk, plain, out2, L, batch, seeds=None, prng=1):
        """Encryptor(public key).encrypt of the device plaintexts `plain` (layout as d_encrypt_symmetric) into the device slab out2
        [batch][2][L][n]; seeds as for d_encrypt_zero_asymmetric"""
        seeds = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64).reshape(batch, 8)
        _check(lib().sb200_encrypt_asymmetric(self.h, pk.h, L, batch, _dp(plain), prng, None if seeds is None else _hp(seeds), _dp(out2),
                                              self._stream()))

    def _encrypt_host(self, plain, L):
        """host plaintexts -> (device copy, device output slab, batch, level, single) for the host encryption forms"""
        import torch

        p = np.ascontiguousarray(plain, dtype=np.uint64)
        single = p.ndim == (2 if self.scheme == CKKS else 1)
        p = p[None] if single else p
        if L is None:
            L = p.shape[1] if self.scheme == CKKS else max(self.k - 1, 1)
        d_plain = torch.from_numpy(p.view(np.int64)).cuda()
        out = torch.empty((p.shape[0], 2, L, self.n), dtype=torch.int64, device="cuda")
        return d_plain, out, p.shape[0], L, single

    def encrypt_symmetric(self, sk, plain, bootstrap_seeds=None, save_seed=False, want_public_seeds=False, bootstrap_prng=1,
                          ciphertext_prng=1, L=None):
        """d_encrypt_symmetric on host arrays: plaintexts [B][L][n] (CKKS) / [B][n] (BFV, BGV), or one without the batch axis ->
        ciphertexts [B][2][L][n] (and the public seeds [B][8] when asked for)"""
        d_plain, out, B, L, single = self._encrypt_host(plain, L)
        pub = self.d_encrypt_symmetric(sk, d_plain, out, L, B, bootstrap_seeds, save_seed, want_public_seeds, bootstrap_prng, ciphertext_prng)
        ct = out.cpu().numpy().view(np.uint64)
        ct = ct[0] if single else ct
        return (ct, pub) if want_public_seeds else ct

    def encrypt_asymmetric(self, pk, plain, seeds=None, prng=1, L=None):
        """d_encrypt_asymmetric on host arrays (layouts as encrypt_symmetric)"""
        d_plain, out, B, L, single = self._encrypt_host(plain, L)
        self.d_encrypt_asymmetric(pk, d_plain, out, L, B, seeds, prng)
        ct = out.cpu().numpy().view(np.uint64)
        return ct[0] if single else ct

    # ---- KeyGenerator(context, secret_key) ----
    def generate_kswitch_key(self, sk, galois_elt=0, seeds=None, bootstrap_prng=1, ciphertext_prng=1, host=True, device=True):
        """KeyGenerator.create_relin_keys (galois_elt 0) / the Galois key of one element for the secret key sk, generated on the
        device; seeds [k-1][8] bootstrap seeds, one per digit (None = fresh from the OS entropy source).  Returns (host words
        [k-1][2][k][n] or None, KSwitchKey or None)"""
        digits = self.k - 1
        seeds = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64).reshape(max(digits, 1), 8)
        words = np.zeros((digits, 2, self.k, self.n), dtype=np.uint64) if host else None
        h = C.c_void_p()
        _check(lib().sb200_kswitch_key_generate(self.h, sk.h, galois_elt, bootstrap_prng, ciphertext_prng,
                                                None if seeds is None else _hp(seeds), None if words is None else _hp(words),
                                                C.byref(h) if device else None))
        return words, (KSwitchKey.wrap(self, h) if device else None)

    def generate_public_key(self, sk, seed=None, bootstrap_prng=1, ciphertext_prng=1, host=True, device=True):
        """KeyGenerator.create_public_key for the secret key sk on the device; seed [8] (None = fresh).  Returns (host words
        [2][k][n] or None, PublicKey or None)"""
        seed = None if seed is None else np.ascontiguousarray(seed, dtype=np.uint64).reshape(8)
        words = np.zeros((2, self.k, self.n), dtype=np.uint64) if host else None
        h = C.c_void_p()
        _check(lib().sb200_public_key_generate(self.h, sk.h, bootstrap_prng, ciphertext_prng, None if seed is None else _hp(seed),
                                               None if words is None else _hp(words), C.byref(h) if device else None))
        return words, (PublicKey.wrap(self, h) if device else None)

    def generate_public_key_seeded(self, sk, seed=None, bootstrap_prng=1, ciphertext_prng=1, device=False):
        """KeyGenerator.create_public_key() as its Serializable<PublicKey> saves it (compr_mode none), generated on the device; seed
        [8] (None = fresh).  Returns (bytes, PublicKey or None)"""
        seed = None if seed is None else np.ascontiguousarray(seed, dtype=np.uint64).reshape(8)
        cap = lib().sb200_ciphertext_save_seeded_size(self.h, self.k)
        buf = C.create_string_buffer(cap)
        h = C.c_void_p()
        _check(lib().sb200_public_key_generate_seeded(self.h, sk.h, bootstrap_prng, ciphertext_prng, None if seed is None else _hp(seed),
                                                      C.addressof(buf), cap, C.byref(h) if device else None))
        return buf.raw, (PublicKey.wrap(self, h) if device else None)

    def kswitch_keys_seeded_size(self, galois_elts):
        e = (C.c_uint32 * max(len(galois_elts), 1))(*galois_elts)
        return lib().sb200_kswitch_keys_save_seeded_size(self.h, e, len(galois_elts))

    def generate_kswitch_keys_seeded(self, sk, galois_elts, seeds=None, bootstrap_prng=1, ciphertext_prng=1, capacity=None):
        """KeyGenerator.create_relin_keys() (galois_elts [0]) / create_galois_keys(galois_elts) as their Serializable saves them
        (compr_mode none), generated on the device; seeds [distinct elements][k-1][8] in draw order (None = fresh) -> bytes"""
        galois_elts = [int(x) for x in galois_elts]
        e = (C.c_uint32 * max(len(galois_elts), 1))(*galois_elts)
        size = lib().sb200_kswitch_keys_save_seeded_size(self.h, e, len(galois_elts))
        cap = size if capacity is None else capacity
        buf = C.create_string_buffer(max(cap, 1))
        seeds = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64)
        _check(lib().sb200_kswitch_keys_generate_seeded(self.h, sk.h, e, len(galois_elts), bootstrap_prng, ciphertext_prng,
                                                        None if seeds is None else _hp(seeds), C.addressof(buf), cap))
        return buf.raw[:size]

    def load_kswitch_keys(self, stream, indices=None, capacity=None):
        """KSwitchKeys::load of the entries `indices` of a RelinKeys / GaloisKeys stream (none, zlib or seeded) in one pass; None =
        every non-empty slot, at most `capacity` of them (default n, the slot count of a GaloisKeys object).  Returns a list of
        KSwitchKey, each with its slot in `.slot`"""
        if indices is None:
            cap = self.n if capacity is None else capacity
            idx = None
        else:
            cap = len(indices)
            idx = (C.c_size_t * max(cap, 1))(*[int(i) for i in indices])
        out = (C.c_void_p * max(cap, 1))()
        slots = (C.c_size_t * max(cap, 1))()
        got = C.c_size_t(0)
        _check(lib().sb200_kswitch_keys_load(self.h, stream, len(stream), idx, cap, out, slots, C.byref(got)))
        keys = []
        for i in range(got.value):
            key = KSwitchKey.wrap(self, C.c_void_p(out[i]))
            key.slot = slots[i]
            keys.append(key)
        return keys

    def d_relinearize(self, in3, key, out2, L, batch):
        _check(lib().sb200_relinearize(self.h, L, batch, _dp(in3), key.h, _dp(out2), self._stream()))

    def d_multiply_relinearize(self, a, b, key, out2, L, batch):
        _check(lib().sb200_multiply_relinearize(self.h, L, batch, _dp(a), _dp(b), key.h, _dp(out2), self._stream()))

    def d_rescale_to_next(self, in2, out2, L, batch):
        _check(lib().sb200_rescale_to_next(self.h, L, batch, _dp(in2), _dp(out2), self._stream()))

    def d_mod_switch_to_next(self, in2, out2, L, batch):
        _check(lib().sb200_mod_switch_to_next(self.h, L, batch, _dp(in2), _dp(out2), self._stream()))

    def d_rescale_to_next_sized(self, a, out, L, size, batch):
        """rescale_to_next of ciphertexts of `size` polynomials: [batch][size][L][n] -> [batch][size][L-1][n]"""
        _check(lib().sb200_rescale_to_next_sized(self.h, L, size, batch, _dp(a), _dp(out), self._stream()))

    def d_mod_switch_to_next_sized(self, a, out, L, size, batch):
        """mod_switch_to_next of ciphertexts of `size` polynomials: [batch][size][L][n] -> [batch][size][L-1][n]"""
        _check(lib().sb200_mod_switch_to_next_sized(self.h, L, size, batch, _dp(a), _dp(out), self._stream()))

    def d_apply_galois(self, in2, galois_elt, key, out2, L, batch):
        _check(lib().sb200_apply_galois(self.h, L, batch, _dp(in2), galois_elt, key.h, _dp(out2), self._stream()))

    def d_apply_galois_add(self, in2, galois_elt, key, addend2, out2, L, batch):
        """sb200_apply_galois_add: out2 = addend2 + apply_galois(in2); out2 may be addend2, addend2 may be in2"""
        _check(lib().sb200_apply_galois_add(self.h, L, batch, _dp(in2), galois_elt, None if key is None else key.h,
                                            None if addend2 is None else _dp(addend2), _dp(out2), self._stream()))

    def d_apply_galois_multiply_plain_add(self, in2, galois_elt, key, plain, plain_count, addend2, out2, L, batch):
        """sb200_apply_galois_multiply_plain_add: out2 = addend2 + plain * apply_galois(in2), plain_count (1 or batch) NTT-form
        plaintexts [L][n]; out2 may be addend2, addend2 may be in2"""
        _check(lib().sb200_apply_galois_multiply_plain_add(self.h, L, batch, _dp(in2), galois_elt, None if key is None else key.h, plain_count,
                                                           None if plain is None else _dp(plain), None if addend2 is None else _dp(addend2),
                                                           _dp(out2), self._stream()))

    def d_diagonal_sum(self, in2, galois_elts, keys, plains, plain_counts, out2, L, batch, plain_is_ntt=True):
        """sb200_diagonal_sum: out2 = sum_i plains[i] * apply_galois(in2, galois_elts[i]) with keys[i] (element 1: no rotation, key may
        be None); plains[i] holds plain_counts[i] (1 or batch) plaintexts, NTT form [L][n] or coefficient form [n]"""
        c_elts, c_keys = _rotate_sum_args(galois_elts, keys)
        m = len(plains)
        counts = (C.c_size_t * max(m, 1))(*plain_counts)
        p_plains = (C.c_void_p * max(m, 1))(*[None if p is None else _dp(p).value for p in plains])
        _check(lib().sb200_diagonal_sum(self.h, L, batch, _dp(in2), len(galois_elts), c_elts, c_keys, counts, p_plains, int(plain_is_ntt),
                                        _dp(out2), self._stream()))

    def d_rotate_sum(self, in2, galois_elts, keys, out2, L, batch):
        """sb200_rotate_sum: the chain y_{j+1} = y_j + apply_galois(y_j, galois_elts[j]) from in2, y_steps to out2 (may be in2)"""
        c_elts, c_keys = _rotate_sum_args(galois_elts, keys)
        _check(lib().sb200_rotate_sum(self.h, L, batch, _dp(in2), len(galois_elts), c_elts, c_keys, _dp(out2), self._stream()))
