"""ctypes binding of libcosnarks_gpu.so (the C ABI declared in include/cosnarks_gpu.h).

This is the Python stand-in for the Rust `extern "C"` shim a co-snarks maintainer would write
(INTEGRATION.md); tests and bench.py drive the library through it.  There is no CPU fallback: if
the shared library is missing, `load()` raises, and without a CUDA device `Context()` raises with
the library's error message.
"""
import ctypes as C
import os

import numpy as np

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")  # see csrc/cs_api.cu: read when the CUDA context is created

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libcosnarks_gpu.so")

CS_BN254, CS_BLS12_381 = 0, 1
CS_G1, CS_G2 = 0, 1
CS_PLAIN, CS_REP3 = 0, 1
R3B_ADD, R3B_SUB, R3B_ADD_PUBLIC, R3B_SUB_PUBLIC, R3B_PUBLIC_SUB, R3B_MUL_PUBLIC, R3B_NEG, R3B_PROMOTE = range(8)
CS_PART_A, CS_PART_B1, CS_PART_B2, CS_PART_L, CS_PART_H, CS_PART_ALL = 1, 2, 4, 8, 16, 31

u64p = C.POINTER(C.c_uint64)
u32p = C.POINTER(C.c_uint32)


class CsError(RuntimeError):
    pass


class Rep3Prf(C.Structure):
    _fields_ = [("seed1", C.c_uint8 * 32), ("word_pos1", C.c_uint64), ("seed2", C.c_uint8 * 32),
                ("word_pos2", C.c_uint64), ("rounds", C.c_uint)]


ARITH_POLY_NAMES = ("w_l", "w_r", "w_o", "w_4", "w_l_shift", "w_4_shift", "q_m", "q_l", "q_r", "q_o", "q_4", "q_c", "q_arith")


class HonkArithPolys(C.Structure):  # cs_honk_arith_polys: device pointers
    _fields_ = [(n, C.c_void_p) for n in ARITH_POLY_NAMES]


class KeyDesc(C.Structure):
    _fields_ = [
        ("curve", C.c_int),
        ("num_constraints", C.c_size_t), ("num_instance_variables", C.c_size_t), ("num_witness_variables", C.c_size_t),
        ("a_row_ptr", u32p), ("a_col", u32p), ("a_coeff", u64p), ("a_nnz", C.c_size_t),
        ("b_row_ptr", u32p), ("b_col", u32p), ("b_coeff", u64p), ("b_nnz", C.c_size_t),
        ("alpha_g1", u64p), ("beta_g1", u64p), ("beta_g2", u64p), ("delta_g1", u64p), ("delta_g2", u64p),
        ("a_query", u64p), ("a_query_len", C.c_size_t),
        ("b_g1_query", u64p), ("b_g1_query_len", C.c_size_t),
        ("b_g2_query", u64p), ("b_g2_query_len", C.c_size_t),
        ("l_query", u64p), ("l_query_len", C.c_size_t),
        ("h_query", u64p), ("h_query_len", C.c_size_t),
        ("window_bits", C.c_int),
        ("c_row_ptr", u32p), ("c_col", u32p), ("c_coeff", u64p), ("c_nnz", C.c_size_t),
    ]


class PlonkKeyDesc(C.Structure):
    _fields_ = [
        ("curve", C.c_int),
        ("n_vars", C.c_uint32), ("n_public", C.c_uint32), ("domain_size", C.c_uint32), ("n_additions", C.c_uint32),
        ("n_constraints", C.c_uint32),
        ("k1_mont", u64p), ("k2_mont", u64p), ("vk_points", u64p),
        ("additions_ids", u32p), ("additions_factors", u64p),
        ("map_a", u32p), ("map_b", u32p), ("map_c", u32p),
        ("q_coeffs", u64p * 5), ("q_evals", u64p * 5), ("s_coeffs", u64p * 3), ("s_evals", u64p * 3),
        ("lagrange_evals", u64p), ("p_tau", u64p), ("n_p_tau", C.c_size_t),
    ]


NET_SEND_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t)
NET_RECV_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t)


class NetCallbacks(C.Structure):
    _fields_ = [("user", C.c_void_p), ("send", NET_SEND_FN), ("recv", NET_RECV_FN)]


# name -> (restype, argtypes); every symbol include/cosnarks_gpu.h declares
SIGNATURES = {
    "cs_rep3_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_rep3_batch_open_send": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "cs_rep3_batch_open_finish": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_honk_commit_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_uint, C.c_void_p]),
    "cs_fr_inv": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p]),
    "cs_shamir_state_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]),
    "cs_shamir_state_fork": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    "cs_shamir_state_pairs": (C.c_size_t, [C.c_void_p]),
    "cs_shamir_state_rand": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_shamir_state_free": (None, [C.c_void_p]),
    "cs_shamir_open_lagrange": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "cs_shamir_degree_reduce_many": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "cs_shamir_degree_reduce_point": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_shamir_open_half_point": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "cs_shamir_double_sharings": (C.c_int, [C.c_void_p] * 3 + [C.c_size_t, C.c_void_p, C.c_void_p]),
    "cs_groth16_shamir_prove": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 6),
    "cs_groth16_prove_with_shamir_bridge": (C.c_int, [C.c_void_p] * 10),
    "cs_share_rep3_device": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_fr_rand_device": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64, C.c_void_p, C.c_size_t]),
    "cs_rep3_witness_read": (C.c_int, [C.c_char_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                       C.POINTER(C.c_size_t), C.POINTER(C.c_int)]),
    "cs_rep3_replicate_additive": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "cs_net_from_callbacks": (C.c_int, [C.c_int, C.c_int, C.POINTER(NetCallbacks), C.POINTER(C.c_void_p)]),
    "cs_net_peer_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "cs_net_peer_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "cs_net_peer_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "cs_net_peer_connect_local": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "cs_net_send": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "cs_net_recv": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "cs_net_sendrecv": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t]),
    "cs_net_bytes_sent": (C.c_uint64, [C.c_void_p]),
    "cs_net_free": (None, [C.c_void_p]),
    "cs_rep3_state_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "cs_rep3_state_from_seeds": (C.c_int, [C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.POINTER(C.c_void_p)]),
    "cs_rep3_state_fork": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "cs_rep3_state_prf": (C.c_int, [C.c_void_p, C.POINTER(Rep3Prf)]),
    "cs_rep3_state_advance": (C.c_int, [C.c_void_p, C.c_uint64]),
    "cs_rep3_state_rand": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "cs_rep3_state_free": (None, [C.c_void_p]),
    "cs_os_random": (C.c_int, [C.c_void_p, C.c_size_t]),
    "cs_groth16_rep3_prove": (C.c_int, [C.c_void_p] * 12),
    "cs_groth16_rep3_prove_main": (C.c_int, [C.c_void_p] * 13),
    "cs_groth16_rep3_prove_helper": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 5),
    "cs_last_error": (C.c_char_p, []),
    "cs_version": (C.c_char_p, []),
    "cs_ctx_create": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "cs_ctx_destroy": (None, [C.c_void_p]),
    "cs_ctx_synchronize": (C.c_int, [C.c_void_p]),
    "cs_ctx_launch_count": (C.c_uint64, [C.c_void_p]),
    "cs_dev_alloc": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    "cs_dev_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "cs_host_alloc_pinned": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "cs_host_free_pinned": (C.c_int, [C.c_void_p]),
    "cs_memcpy_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_memcpy_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_bases_upload": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "cs_bases_free": (None, [C.c_void_p]),
    "cs_bases_len": (C.c_size_t, [C.c_void_p]),
    "cs_bases_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_size_t)]),
    "cs_ctx_set_table_budget": (C.c_int, [C.c_void_p, C.c_size_t]),
    "cs_groth16_pk_table_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint), C.POINTER(C.c_size_t)]),
    "cs_msm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.POINTER(C.c_int)]),
    "cs_msm_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.POINTER(C.c_int)]),
    "cs_msm_rep3_shares": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    "cs_msm_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "cs_msm_stage_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "cs_msm_timeline_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "cs_sumcheck_gate_separator": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_uint, C.c_void_p]),
    "cs_sumcheck_fold": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_size_t, C.c_void_p]),
    "cs_sumcheck_arith_round": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_fixed_base_mul": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "cs_domain_create": (C.c_int, [C.c_void_p, C.c_int, C.c_uint, C.c_void_p, C.POINTER(C.c_void_p)]),
    "cs_domain_free": (None, [C.c_void_p]),
    "cs_domain_size": (C.c_size_t, [C.c_void_p]),
    "cs_ifft_in_to_out": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]),
    "cs_fft_out_to_in": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]),
    "cs_fft": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]),
    "cs_ifft": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]),
    "cs_eval_poly": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_uint, C.c_void_p, C.c_void_p]),
    "cs_bit_reverse": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_uint, C.c_uint]),
    "cs_ifft_in_to_out_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]),
    "cs_fft_out_to_in_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint]),
    "cs_vec_mul": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_vec_add": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_vec_sub": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_vec_scale_table": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint]),
    "cs_rep3_local_mul_vec": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_vec_lincomb": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.c_void_p, C.c_uint, C.c_size_t, C.c_void_p]),
    "cs_rep3_masks_device": (C.c_int, [C.c_void_p, C.c_int, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.c_uint, C.c_size_t, C.c_void_p]),
    "cs_rep3_mul_vec_reshare": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(Rep3Prf), C.c_void_p, C.c_void_p]),
    "cs_rep3_set_b": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "cs_ipc_export": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_ipc_open": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "cs_ipc_close": (C.c_int, [C.c_void_p, C.c_void_p]),
    "cs_plonk_pk_create": (C.c_int, [C.c_void_p, C.POINTER(PlonkKeyDesc), C.POINTER(C.c_void_p)]),
    "cs_bases_from_crs_file": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "cs_plonk_pk_free": (None, [C.c_void_p]),
    "cs_plonk_pk_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_void_p]),
    "cs_plonk_pk_from_zkey": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]),
    "cs_plonk_prove_plain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "cs_keccak256": (C.c_int, [C.c_char_p, C.c_size_t, C.c_void_p]),
    "cs_plonk_rep3_create": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "cs_plonk_rep3_free": (None, [C.c_void_p]),
    "cs_plonk_rep3_arena": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.POINTER(C.c_uint)]),
    "cs_plonk_rep3_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "cs_plonk_rep3_io": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]),
    "cs_plonk_rep3_round1": (C.c_int, [C.c_void_p, C.POINTER(Rep3Prf), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                       C.c_void_p, C.c_void_p]),
    "cs_plonk_rep3_step": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "cs_plonk_rep3_prf_words": (C.c_uint64, [C.c_void_p]),
    "cs_plonk_rep3_connect_io": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_plonk_shamir_create": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "cs_plonk_shamir_free": (None, [C.c_void_p]),
    "cs_plonk_shamir_prove": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t] + [C.c_void_p] * 4),
    "cs_plonk_shamir_pairs": (C.c_size_t, [C.c_void_p]),
    "cs_plonk_shamir_pair_ms": (C.c_double, [C.c_void_p]),
    "cs_plonk_shamir_device_bytes": (C.c_size_t, [C.c_void_p]),
    "cs_plonk_rep3_prove": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    "cs_chacha_keystream": (C.c_int, [C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint, C.c_uint, C.c_void_p]),
    "cs_rep3_to_shamir": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_groth16_pk_create": (C.c_int, [C.c_void_p, C.POINTER(KeyDesc), C.POINTER(C.c_void_p)]),
    "cs_groth16_pk_from_zkey": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]),
    "cs_wtns_read": (C.c_int, [C.c_char_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "cs_groth16_pk_free": (None, [C.c_void_p]),
    "cs_groth16_domain_size": (C.c_size_t, [C.c_void_p]),
    "cs_groth16_pk_curve": (C.c_int, [C.c_void_p]),
    "cs_plonk_pk_curve": (C.c_int, [C.c_void_p]),
    "cs_groth16_witness_map": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_groth16_witness_map_libsnark": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_groth16_prove_plain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_groth16_prove_plain_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_groth16_prove_plain_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                               C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_groth16_rep3_local_parts": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint] + [C.c_void_p] * 11),
    "cs_groth16_rep3_local_prf": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint] + [C.c_void_p] * 12),
    "cs_groth16_shamir_local": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 9),
    "cs_groth16_rep3_local": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 11),
    "cs_point_scalar_mul": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_point_add": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_point_neg": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "cs_fr_to_mont": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_fr_from_mont": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_fq_to_mont": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_fq_from_mont": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]),
    "cs_fr_mul": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_fr_add": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_fr_sub": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "cs_groth16_roots_of_unity": (C.c_int, [C.c_int, C.c_uint, C.c_void_p, C.c_void_p]),
}

_LIBS = {}


def load(path=None, strict=True):
    """Load the shared library and attach signatures.  Raises if it is missing -- build it with
    `python -c "import __graft_entry__ as g; g.build()"` (nvcc, sm_90a)."""
    path = os.path.abspath(path or DEFAULT_LIB)
    if path in _LIBS:
        return _LIBS[path]
    if not os.path.exists(path):
        raise CsError("%s not found: the CUDA extension is not built (no CPU fallback exists)" % path)
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        if not strict and not hasattr(lib, name):
            continue
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _LIBS[path] = lib
    return lib


# ------------------------------------------------------------------------------------------ data helpers
def limbs_of(curve, field):
    """64-bit limbs of a field element: field in {'fr', 'fq'}."""
    if field == "fr":
        return 4
    return 4 if curve == CS_BN254 else 6


def ints_to_limbs(vals, nlimbs):
    """list of python ints -> np.uint64 array [len, nlimbs], little-endian limbs."""
    vals = list(vals)
    raw = b"".join(int(v).to_bytes(8 * nlimbs, "little") for v in vals)
    return np.frombuffer(raw, dtype=np.uint64).reshape(len(vals), nlimbs).copy()


def limbs_to_ints(arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint64)
    nl = arr.shape[-1]
    flat = arr.reshape(-1, nl)
    raw = flat.tobytes()
    return [int.from_bytes(raw[i * 8 * nl:(i + 1) * 8 * nl], "little") for i in range(flat.shape[0])]


def to_mont_ints(vals, p, nlimbs):
    R = 1 << (64 * nlimbs)
    return [int(v) * R % p for v in vals]


def from_mont_ints(vals, p, nlimbs):
    Rinv = pow(1 << (64 * nlimbs), -1, p)
    return [int(v) * Rinv % p for v in vals]


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(a)  # raw device / host address


class Context:
    """cs_ctx wrapper.  `stream` may be a raw cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream)."""

    def __init__(self, device=0, stream=None, lib_path=None):
        self.lib = load(lib_path)
        h = C.c_void_p()
        self._check(self.lib.cs_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h)))
        self.h = h
        self.device = device

    def _check(self, rc):
        if rc != 0:
            raise CsError("cosnarks_gpu error %d: %s" % (rc, self.lib.cs_last_error().decode()))

    def close(self):
        if getattr(self, "h", None):
            self.lib.cs_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def synchronize(self):
        self._check(self.lib.cs_ctx_synchronize(self.h))

    def launch_count(self):
        return int(self.lib.cs_ctx_launch_count(self.h))

    def set_table_budget(self, nbytes):
        """Cap the device bytes of base sets and keys created from now on (cs_ctx_set_table_budget); 0 = automatic."""
        self._check(self.lib.cs_ctx_set_table_budget(self.h, int(nbytes)))

    # ---- device memory
    def alloc(self, nbytes):
        p = C.c_void_p()
        self._check(self.lib.cs_dev_alloc(self.h, nbytes, C.byref(p)))
        return p.value

    def free(self, dptr):
        self._check(self.lib.cs_dev_free(self.h, C.c_void_p(dptr)))

    def h2d(self, dptr, arr):
        arr = np.ascontiguousarray(arr)
        self._check(self.lib.cs_memcpy_h2d(self.h, C.c_void_p(dptr), _ptr(arr), arr.nbytes))

    def d2h(self, dptr, shape, dtype=np.uint64):
        out = np.empty(shape, dtype=dtype)
        self._check(self.lib.cs_memcpy_d2h(self.h, _ptr(out), C.c_void_p(dptr), out.nbytes))
        return out

    def to_device(self, arr):
        arr = np.ascontiguousarray(arr)
        d = self.alloc(arr.nbytes)
        self.h2d(d, arr)
        return d

    # ---- MSM
    def bases_upload(self, curve, group, points_mont, window_bits=0):
        points_mont = np.ascontiguousarray(points_mont, dtype=np.uint64)
        h = C.c_void_p()
        self._check(self.lib.cs_bases_upload(self.h, curve, group, _ptr(points_mont), points_mont.shape[0],
                                             window_bits, C.byref(h)))
        return Bases(self, h, curve, group)

    def bases_from_crs_file(self, path, n, offset=0, window_bits=0):
        """Ignition CRS file (bn254_g1.dat layout) -> device base set (cs_bases_from_crs_file)."""
        h = C.c_void_p()
        self._check(self.lib.cs_bases_from_crs_file(self.h, str(path).encode(), offset, n, window_bits, C.byref(h)))
        return Bases(self, h, CS_BN254, CS_G1)

    def msm(self, bases, scalars, offset=0, n=None, montgomery=True, device=False):
        plimbs = limbs_of(bases.curve, "fq") * (2 if bases.group == CS_G1 else 4)
        out = np.zeros(plimbs, dtype=np.uint64)
        inf = C.c_int(0)
        if device:
            assert n is not None
            self._check(self.lib.cs_msm_device(self.h, bases.h, offset, C.c_void_p(scalars), n, int(montgomery),
                                               _ptr(out), C.byref(inf)))
        else:
            scalars = np.ascontiguousarray(scalars, dtype=np.uint64)
            if n is None:
                n = scalars.shape[0]
            self._check(self.lib.cs_msm(self.h, bases.h, offset, _ptr(scalars) if n else None, n, int(montgomery),
                                        _ptr(out), C.byref(inf)))
        return out, bool(inf.value)

    def msm_rep3_shares(self, bases, shares, offset=0):
        shares = np.ascontiguousarray(shares, dtype=np.uint64)
        n = shares.shape[0]
        plimbs = limbs_of(bases.curve, "fq") * (2 if bases.group == CS_G1 else 4)
        oa, ob = np.zeros(plimbs, dtype=np.uint64), np.zeros(plimbs, dtype=np.uint64)
        self._check(self.lib.cs_msm_rep3_shares(self.h, bases.h, offset, _ptr(shares) if n else None, n, _ptr(oa), _ptr(ob)))
        return oa, ob

    def msm_profile(self, enable=True):
        self._check(self.lib.cs_msm_profile(self.h, int(enable)))

    def msm_stage_ms(self):
        arr = (C.c_float * 5)()
        self._check(self.lib.cs_msm_stage_ms(self.h, arr))
        return [float(x) for x in arr]

    def msm_timeline_ms(self):
        """[5 workspaces][6 stage boundaries] in ms after the last fork (Groth16: A, B1, B2, L, H); -1 = no event."""
        arr = (C.c_float * 30)()
        self._check(self.lib.cs_msm_timeline_ms(self.h, arr))
        return [[float(arr[w * 6 + i]) for i in range(6)] for w in range(5)]

    def fixed_base_mul(self, curve, group, base_mont, scalars, montgomery=True):
        scalars = np.ascontiguousarray(scalars, dtype=np.uint64)
        base_mont = np.ascontiguousarray(base_mont, dtype=np.uint64)
        n = scalars.shape[0]
        out = np.zeros((n, base_mont.size), dtype=np.uint64)
        self._check(self.lib.cs_fixed_base_mul(self.h, curve, group, _ptr(base_mont), _ptr(scalars), n,
                                               int(montgomery), _ptr(out)))
        return out

    # ---- NTT
    def domain(self, curve, log_n, group_gen_mont=None):
        h = C.c_void_p()
        g = None if group_gen_mont is None else np.ascontiguousarray(group_gen_mont, dtype=np.uint64)
        self._check(self.lib.cs_domain_create(self.h, curve, log_n, _ptr(g), C.byref(h)))
        return Domain(self, h, curve, log_n)

    def vec_lincomb(self, curve, d_inputs, weights_mont, n, d_out):
        k = len(d_inputs)
        arr = (C.c_void_p * k)(*[C.c_void_p(p) for p in d_inputs])
        w = np.ascontiguousarray(weights_mont, dtype=np.uint64)
        self._check(self.lib.cs_vec_lincomb(self.h, curve, arr, _ptr(w), k, n, C.c_void_p(d_out)))

    def rep3_masks_device(self, curve, seed1, pos1, seed2, pos2, n, d_out, rounds=12):
        self._check(self.lib.cs_rep3_masks_device(self.h, curve, bytes(seed1), pos1, bytes(seed2), pos2, rounds, n,
                                                  C.c_void_p(d_out)))

    def rep3_mul_vec_reshare(self, curve, d_a, d_b, n, prf_args, d_out, d_next_out=None):
        """mul_vec = local_mul_vec + reshare_vec as one kernel (arithmetic.rs:132-160); asynchronous."""
        prf = None
        if prf_args is not None:
            s1, p1, s2, p2, rounds = prf_args
            prf = Rep3Prf((C.c_uint8 * 32)(*bytes(s1)), p1, (C.c_uint8 * 32)(*bytes(s2)), p2, rounds)
        self._check(self.lib.cs_rep3_mul_vec_reshare(self.h, curve, C.c_void_p(d_a), C.c_void_p(d_b), n,
                                                     C.byref(prf) if prf is not None else None, C.c_void_p(d_out),
                                                     C.c_void_p(d_next_out) if d_next_out else None))

    def rep3_set_b(self, curve, d_recv, n, d_out):
        self._check(self.lib.cs_rep3_set_b(self.h, curve, C.c_void_p(d_recv), n, C.c_void_p(d_out)))

    def rep3_batch(self, curve, op, party, d_x, d_y, d_out, n):
        """Batched VM opcode on device share vectors (cs_rep3_batch; op = R3B_*)."""
        self._check(self.lib.cs_rep3_batch(self.h, curve, op, party, _ptr(d_x), _ptr(d_y), _ptr(d_out), n))

    def honk_commit_batch(self, crs, kind, d_polys, lens):
        """CoUtils::commit for up to 4 polynomials at once -> [k (x2 for Rep3), point limbs] affine Montgomery."""
        k = len(d_polys)
        per = 2 if kind == CS_REP3 else 1
        pl = limbs_of(crs.curve, "fq") * (2 if crs.group == CS_G1 else 4)
        out = np.zeros((k * per, pl), dtype=np.uint64)
        ptrs = (C.c_void_p * k)(*[C.c_void_p(p) for p in d_polys])
        ln = (C.c_size_t * k)(*lens)
        self._check(self.lib.cs_honk_commit_batch(self.h, crs.h, kind, ptrs, ln, k, _ptr(out)))
        return out

    # ---- UltraHonk sumcheck kernels (csrc/cs_sumcheck.cuh)
    def sumcheck_gate_separator(self, curve, betas_mont, d_out):
        b = np.ascontiguousarray(betas_mont, dtype=np.uint64).reshape(-1, 4)
        self._check(self.lib.cs_sumcheck_gate_separator(self.h, curve, _ptr(b) if b.shape[0] else None, b.shape[0], _ptr(d_out)))

    def sumcheck_fold(self, curve, d_in, d_out, shared, length, challenge_mont):
        k = len(d_in)
        pin = (C.c_void_p * k)(*[C.c_void_p(p) for p in d_in])
        pout = (C.c_void_p * k)(*[C.c_void_p(p) for p in d_out])
        u = np.ascontiguousarray(challenge_mont, dtype=np.uint64).reshape(4)
        self._check(self.lib.cs_sumcheck_fold(self.h, curve, pin, pout, k, int(shared), length, _ptr(u)))

    def sumcheck_arith_round(self, curve, kind, party, d_polys, round_size, d_beta_products, periodicity, prf=None):
        """d_polys: name -> device pointer (ARITH_POLY_NAMES).  -> (r0 [6, 4], r1 [5, 4] plain or [5, 2, 4] Rep3)"""
        st = HonkArithPolys(*[C.c_void_p(d_polys[n]) for n in ARITH_POLY_NAMES])
        r0 = np.zeros((6, 4), dtype=np.uint64)
        r1 = np.zeros((5, 2, 4) if kind == CS_REP3 else (5, 4), dtype=np.uint64)
        self._check(self.lib.cs_sumcheck_arith_round(self.h, curve, kind, party, C.byref(st), round_size, _ptr(d_beta_products),
                                                     periodicity, C.byref(prf) if prf is not None else None, _ptr(r0), _ptr(r1)))
        return r0, r1

    def ipc_export(self, d_ptr):
        h = np.zeros(64, dtype=np.uint8)
        self._check(self.lib.cs_ipc_export(self.h, C.c_void_p(d_ptr), _ptr(h)))
        return h

    def ipc_open(self, handle64):
        out = C.c_void_p()
        h = np.ascontiguousarray(handle64, dtype=np.uint8)
        self._check(self.lib.cs_ipc_open(self.h, _ptr(h), C.byref(out)))
        return out.value

    def ipc_close(self, peer_ptr):
        self._check(self.lib.cs_ipc_close(self.h, C.c_void_p(peer_ptr)))

    def chacha_keystream(self, key, first_block, rounds, nblocks):
        out = np.zeros(nblocks * 16, dtype=np.uint32)
        self._check(self.lib.cs_chacha_keystream(self.h, bytes(key), first_block, rounds, nblocks, _ptr(out)))
        return out

    def eval_poly(self, curve, d_coeffs, n, point_mont, batch=1):
        out = np.zeros((batch, 4), dtype=np.uint64)
        self._check(self.lib.cs_eval_poly(self.h, curve, C.c_void_p(d_coeffs), n, batch,
                                          _ptr(np.ascontiguousarray(point_mont, dtype=np.uint64)), _ptr(out)))
        return out

    def roots_of_unity(self, curve, power):
        gen = np.zeros(4, dtype=np.uint64)
        shift = np.zeros(4, dtype=np.uint64)
        self._check(self.lib.cs_groth16_roots_of_unity(curve, power, _ptr(gen), _ptr(shift)))
        return gen, shift


class Bases:
    def __init__(self, ctx, h, curve, group):
        self.ctx, self.h, self.curve, self.group = ctx, h, curve, group

    def __len__(self):
        return int(self.ctx.lib.cs_bases_len(self.h))

    def info(self):
        """-> dict(window_bits, windows, table_rows, device_bytes) (cs_bases_info)"""
        c, w, t, nb = C.c_uint(), C.c_uint(), C.c_uint(), C.c_size_t()
        self.ctx._check(self.ctx.lib.cs_bases_info(self.h, C.byref(c), C.byref(w), C.byref(t), C.byref(nb)))
        return {"window_bits": c.value, "windows": w.value, "table_rows": t.value, "device_bytes": nb.value}

    def free(self):
        if self.h:
            self.ctx.lib.cs_bases_free(self.h)
            self.h = None


class Domain:
    def __init__(self, ctx, h, curve, log_n):
        self.ctx, self.h, self.curve, self.log_n = ctx, h, curve, log_n

    def size(self):
        return int(self.ctx.lib.cs_domain_size(self.h))

    def ifft_in_to_out(self, data, batch=1):
        """data: np.uint64 host array (transformed in place via the host wrapper) or a raw device address."""
        if isinstance(data, np.ndarray):
            self.ctx._check(self.ctx.lib.cs_ifft_in_to_out_host(self.ctx.h, self.h, _ptr(data), batch))
        else:
            self.ctx._check(self.ctx.lib.cs_ifft_in_to_out(self.ctx.h, self.h, C.c_void_p(data), batch))
        return data

    def fft_out_to_in(self, data, batch=1):
        if isinstance(data, np.ndarray):
            self.ctx._check(self.ctx.lib.cs_fft_out_to_in_host(self.ctx.h, self.h, _ptr(data), batch))
        else:
            self.ctx._check(self.ctx.lib.cs_fft_out_to_in(self.ctx.h, self.h, C.c_void_p(data), batch))
        return data

    def fft(self, d_data, batch=1):
        """natural in -> natural out on a device buffer (co-plonk's domain.fft)."""
        self.ctx._check(self.ctx.lib.cs_fft(self.ctx.h, self.h, C.c_void_p(d_data), batch))

    def ifft(self, d_data, batch=1):
        self.ctx._check(self.ctx.lib.cs_ifft(self.ctx.h, self.h, C.c_void_p(d_data), batch))

    def free(self):
        if self.h:
            self.ctx.lib.cs_domain_free(self.h)
            self.h = None


# ------------------------------------------------------------------------------------------ Groth16
class PlonkKey:
    """Device-resident Plonk proving key (cs_plonk_pk) = circom_types::plonk::Zkey as the prover reads it."""

    def __init__(self, ctx, curve, key):
        """key: dict with n_vars, n_public, domain_size, n_additions, n_constraints (ints) and Montgomery-form
        numpy arrays k1, k2 [4], vk_points [8, 2*fq], additions_ids [na, 2] u32, additions_factors [na, 2, 4],
        map_a/b/c u32, q_coeffs/q_evals (5 arrays each), s_coeffs/s_evals (3 each), lagrange_evals
        [max(1, n_public) * 4n, 4], p_tau [m, 2*fq]."""
        self.ctx, self.curve = ctx, curve
        d = PlonkKeyDesc()
        d.curve = curve
        for k in ("n_vars", "n_public", "domain_size", "n_additions", "n_constraints"):
            setattr(d, k, int(key[k]))
        keep = []

        def arr(x, dt):
            a = np.ascontiguousarray(x, dtype=dt)
            keep.append(a)
            return a.ctypes.data_as(u64p if dt == np.uint64 else u32p)
        d.k1_mont, d.k2_mont = arr(key["k1"], np.uint64), arr(key["k2"], np.uint64)
        d.vk_points = arr(key["vk_points"], np.uint64)
        d.additions_ids = arr(key["additions_ids"], np.uint32)
        d.additions_factors = arr(key["additions_factors"], np.uint64)
        for k in ("map_a", "map_b", "map_c"):
            setattr(d, k, arr(key[k], np.uint32))
        for i in range(5):
            d.q_coeffs[i] = arr(key["q_coeffs"][i], np.uint64)
            d.q_evals[i] = arr(key["q_evals"][i], np.uint64)
        for i in range(3):
            d.s_coeffs[i] = arr(key["s_coeffs"][i], np.uint64)
            d.s_evals[i] = arr(key["s_evals"][i], np.uint64)
        d.lagrange_evals = arr(key["lagrange_evals"], np.uint64)
        pt = np.ascontiguousarray(key["p_tau"], dtype=np.uint64)
        keep.append(pt)
        d.p_tau = pt.ctypes.data_as(u64p)
        d.n_p_tau = pt.shape[0]
        h = C.c_void_p()
        ctx._check(ctx.lib.cs_plonk_pk_create(ctx.h, C.byref(d), C.byref(h)))
        self.h = h
        self.fq = limbs_of(curve, "fq")
        del keep

    @classmethod
    def from_zkey(cls, ctx, path, curve=None):
        """snarkjs Plonk .zkey -> device-resident key (cs_plonk_pk_from_zkey); the curve is the one the zkey
        declares, `curve` only asserts it."""
        self = cls.__new__(cls)
        self.ctx = ctx
        h, npub, nwit = C.c_void_p(), C.c_size_t(), C.c_size_t()
        ctx._check(ctx.lib.cs_plonk_pk_from_zkey(ctx.h, str(path).encode(), C.byref(h), C.byref(npub), C.byref(nwit)))
        self.h, self.n_public, self.n_witness = h, npub.value, nwit.value
        self.curve = int(ctx.lib.cs_plonk_pk_curve(h))
        if curve is not None and curve != self.curve:
            ctx.lib.cs_plonk_pk_free(h)
            raise CsError("%s is a curve-%d key, curve %d was requested" % (path, self.curve, curve))
        self.fq = limbs_of(self.curve, "fq")
        return self

    def info(self):
        """-> (n_public, n_witness, domain_size, vk_points [8, 2*fq])."""
        a, b, c = C.c_size_t(), C.c_size_t(), C.c_size_t()
        vk = np.zeros((8, 2 * self.fq), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_plonk_pk_info(self.h, C.byref(a), C.byref(b), C.byref(c), _ptr(vk)))
        return a.value, b.value, c.value, vk

    def prove_plain(self, public_inputs, witness, blinders_mont):
        """Plonk::plain_prove -> (points [9, 2*fq] A B C Z T1 T2 T3 Wxi Wxiw, evals [6, 4] a b c s1 s2 zw), Montgomery."""
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
        wit = np.ascontiguousarray(witness, dtype=np.uint64).reshape(-1, 4)
        bl = np.ascontiguousarray(blinders_mont, dtype=np.uint64).reshape(-1, 4)
        assert bl.shape[0] == 11
        pts = np.zeros((9, 2 * self.fq), dtype=np.uint64)
        evs = np.zeros((6, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_plonk_prove_plain(self.ctx.h, self.h, _ptr(pub), pub.shape[0], _ptr(wit), wit.shape[0],
                                                          _ptr(bl), _ptr(pts), _ptr(evs)))
        return pts, evs

    def free(self):
        if self.h:
            self.ctx.lib.cs_plonk_pk_free(self.h)
            self.h = None


# cs_plonk_rep3_step ids (include/cosnarks_gpu.h)
(R3_ROUND2_A, R3_ROUND2_B, R3_ROUND2_C, R3_ROUND2_D, R3_ROUND2_E, R3_ROUND2_F, R3_ROUND2_G, R3_ROUND3_A, R3_ROUND3_B,
 R3_ROUND4, R3_ROUND5) = range(1, 12)


class PlonkRep3Session:
    """One party's state of a Rep3 co-Plonk proof (cs_plonk_rep3)."""

    def __init__(self, ctx, pk, party):
        self.ctx, self.pk, self.party = ctx, pk, party
        h = C.c_void_p()
        ctx._check(ctx.lib.cs_plonk_rep3_create(ctx.h, pk.h, party, C.byref(h)))
        self.h = h
        p, sb, ns = C.c_void_p(), C.c_size_t(), C.c_uint()
        ctx._check(ctx.lib.cs_plonk_rep3_arena(self.h, C.byref(p), C.byref(sb), C.byref(ns)))
        self.arena, self.slot_bytes, self.n_slots = p.value, sb.value, ns.value
        o, i = C.c_void_p(), C.c_void_p()
        ctx._check(ctx.lib.cs_plonk_rep3_io(self.h, C.byref(o), C.byref(i)))
        self.d_out, self.d_in = o.value, i.value  # additive outputs / opened inputs of the masked vectors

    def connect(self, d_next_arena):
        self.ctx._check(self.ctx.lib.cs_plonk_rep3_connect(self.h, C.c_void_p(d_next_arena) if d_next_arena else None))

    def round1(self, prf_args, public_inputs, witness_shares, blinder_shares):
        s1, p1, s2, p2, rounds = prf_args
        prf = Rep3Prf((C.c_uint8 * 32)(*bytes(s1)), p1, (C.c_uint8 * 32)(*bytes(s2)), p2, rounds)
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
        wit = np.ascontiguousarray(witness_shares, dtype=np.uint64).reshape(-1, 8)
        bl = np.ascontiguousarray(blinder_shares, dtype=np.uint64).reshape(-1, 8)
        assert bl.shape[0] == 11
        pts = np.zeros((3, 2 * self.pk.fq), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_plonk_rep3_round1(self.h, C.byref(prf), _ptr(pub), pub.shape[0], _ptr(wit), wit.shape[0],
                                                          _ptr(bl), _ptr(pts)))
        return pts

    def step(self, step, h_in=None, out_shape=None):
        a = None if h_in is None else np.ascontiguousarray(h_in, dtype=np.uint64)
        out = None if out_shape is None else np.zeros(out_shape, dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_plonk_rep3_step(self.h, step, _ptr(a), _ptr(out)))
        return out

    def prf_words(self):
        return int(self.ctx.lib.cs_plonk_rep3_prf_words(self.h))

    def connect_io(self, d_prev_out, d_next_out):
        """The two peers' additive-out vectors: n-sized openings then read peer HBM instead of crossing the net."""
        self.ctx._check(self.ctx.lib.cs_plonk_rep3_connect_io(self.h, C.c_void_p(d_prev_out) if d_prev_out else None,
                                                              C.c_void_p(d_next_out) if d_next_out else None))

    def prove(self, net, state, public_inputs, witness_shares, blinder_shares=None):
        """Rep3CoPlonk::prove for this party, entirely inside the library (cs_plonk_rep3_prove).
        -> (points [9, 2 fq]: A B C Z T1 T2 T3 Wxi Wxiw, evals [6, 4]: a b c s1 s2 zw)"""
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
        wit = np.ascontiguousarray(witness_shares, dtype=np.uint64).reshape(-1, 8)
        bl = None
        if blinder_shares is not None:
            bl = np.ascontiguousarray(blinder_shares, dtype=np.uint64).reshape(-1, 8)
            assert bl.shape[0] == 11
        pts = np.zeros((9, 2 * self.pk.fq), dtype=np.uint64)
        evs = np.zeros((6, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_plonk_rep3_prove(self.h, net.h, state.h, _ptr(pub), pub.shape[0], _ptr(wit) if wit.shape[0] else None,
                                                         wit.shape[0], _ptr(bl), _ptr(pts), _ptr(evs)))
        return pts, evs

    def free(self):
        if self.h:
            self.ctx.lib.cs_plonk_rep3_free(self.h)
            self.h = None


class PlonkShamirSession:
    """One party's Shamir(n, t) co-Plonk prover (cs_plonk_shamir): ShamirCoPlonk::prove inside the library."""

    def __init__(self, ctx, pk, num_parties, threshold, party):
        self.ctx, self.pk, self.party = ctx, pk, party
        h = C.c_void_p()
        ctx._check(ctx.lib.cs_plonk_shamir_create(ctx.h, pk.h, num_parties, threshold, party, C.byref(h)))
        self.h = h

    def prove(self, net, public_inputs, witness_shares, blinder_shares=None):
        """-> (points [9, 2 fq]: A B C Z T1 T2 T3 Wxi Wxiw, evals [6, 4]: a b c s1 s2 zw, this party's 11 blinder
        shares [11, 4]); witness / blinder shares are degree-t Shamir shares (Montgomery), blinders drawn if None."""
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64).reshape(-1, 4)
        wit = np.ascontiguousarray(witness_shares, dtype=np.uint64).reshape(-1, 4)
        bl = None
        if blinder_shares is not None:
            bl = np.ascontiguousarray(blinder_shares, dtype=np.uint64).reshape(-1, 4)
            assert bl.shape[0] == 11
        pts = np.zeros((9, 2 * self.pk.fq), dtype=np.uint64)
        evs = np.zeros((6, 4), dtype=np.uint64)
        bout = np.zeros((11, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_plonk_shamir_prove(self.h, net.h, _ptr(pub), pub.shape[0], _ptr(wit) if wit.shape[0] else None,
                                                           wit.shape[0], _ptr(bl), _ptr(pts), _ptr(evs), _ptr(bout)))
        return pts, evs, bout

    def pairs(self):
        """double sharings the last proof consumed (58 domain_size + 2, + 11 when the blinders were drawn)"""
        return int(self.ctx.lib.cs_plonk_shamir_pairs(self.h))

    def pair_ms(self):
        return float(self.ctx.lib.cs_plonk_shamir_pair_ms(self.h))

    def device_bytes(self):
        """device memory this party's session and Shamir state hold (its high-water mark after a proof)"""
        return int(self.ctx.lib.cs_plonk_shamir_device_bytes(self.h))

    def free(self):
        if self.h:
            self.ctx.lib.cs_plonk_shamir_free(self.h)
            self.h = None


def keccak256(lib, data):
    out = np.zeros(32, dtype=np.uint8)
    rc = lib.cs_keccak256(bytes(data), len(data), _ptr(out))
    assert rc == 0
    return bytes(out)


class Groth16Key:
    """Device-resident proving key + constraint matrices (cs_groth16_pk).

    `arrays` keeps the numpy buffers the descriptor points at alive until the upload is done."""

    def __init__(self, ctx, curve, matrices_csr, points, window_bits=0):
        """matrices_csr: dict(num_constraints, num_instance_variables, num_witness_variables,
        a=(row_ptr u32, col u32, coeff u64[nnz,4] Montgomery), b=(...));
        points: dict of np.uint64 arrays in Montgomery form: alpha_g1, beta_g1, beta_g2, delta_g1, delta_g2,
        a_query, b_g1_query, b_g2_query, l_query, h_query."""
        self.ctx, self.curve = ctx, curve
        d = KeyDesc()
        d.curve = curve
        d.num_constraints = matrices_csr["num_constraints"]
        d.num_instance_variables = matrices_csr["num_instance_variables"]
        d.num_witness_variables = matrices_csr["num_witness_variables"]
        keep = []
        for name in ("a", "b", "c"):
            if name not in matrices_csr:
                continue
            rp, col, coeff = matrices_csr[name]
            rp = np.ascontiguousarray(rp, dtype=np.uint32)
            col = np.ascontiguousarray(col, dtype=np.uint32)
            coeff = np.ascontiguousarray(coeff, dtype=np.uint64)
            keep += [rp, col, coeff]
            setattr(d, name + "_row_ptr", rp.ctypes.data_as(u32p))
            setattr(d, name + "_col", col.ctypes.data_as(u32p))
            setattr(d, name + "_coeff", coeff.ctypes.data_as(u64p))
            setattr(d, name + "_nnz", col.shape[0])
        for name in ("alpha_g1", "beta_g1", "beta_g2", "delta_g1", "delta_g2"):
            arr = np.ascontiguousarray(points[name], dtype=np.uint64)
            keep.append(arr)
            setattr(d, name, arr.ctypes.data_as(u64p))
        for name in ("a_query", "b_g1_query", "b_g2_query", "l_query", "h_query"):
            arr = np.ascontiguousarray(points[name], dtype=np.uint64)
            keep.append(arr)
            setattr(d, name, arr.ctypes.data_as(u64p))
            setattr(d, name + "_len", arr.shape[0])
        d.window_bits = window_bits
        h = C.c_void_p()
        ctx._check(ctx.lib.cs_groth16_pk_create(ctx.h, C.byref(d), C.byref(h)))
        self.h = h
        self.ni = d.num_instance_variables
        self.nw = d.num_witness_variables
        self.fq = limbs_of(curve, "fq")
        del keep

    def table_info(self):
        """-> (table rows, table device bytes) of the key's MSM tables (cs_groth16_pk_table_info)"""
        rows, nb = C.c_uint(), C.c_size_t()
        self.ctx._check(self.ctx.lib.cs_groth16_pk_table_info(self.h, C.byref(rows), C.byref(nb)))
        return rows.value, nb.value

    @classmethod
    def from_zkey(cls, ctx, path, curve=None, window_bits=0):
        """Groth16ZKey::from_reader + upload in one step (cs_groth16_pk_from_zkey).  The curve is the one the
        zkey declares (its base-field modulus); passing `curve` only asserts it."""
        self = cls.__new__(cls)
        self.ctx = ctx
        h = C.c_void_p()
        npub = C.c_size_t(0)
        ctx._check(ctx.lib.cs_groth16_pk_from_zkey(ctx.h, os.fsencode(path), window_bits, C.byref(h), C.byref(npub)))
        self.h = h
        self.curve = int(ctx.lib.cs_groth16_pk_curve(h))
        if curve is not None and curve != self.curve:
            ctx.lib.cs_groth16_pk_free(h)
            raise CsError("%s is a curve-%d key, curve %d was requested" % (path, self.curve, curve))
        self.ni = npub.value + 1
        self.nw = None
        self.fq = limbs_of(self.curve, "fq")
        return self

    def domain_size(self):
        return int(self.ctx.lib.cs_groth16_domain_size(self.h))

    def witness_map(self, public_inputs, witness, kind=CS_PLAIN, party=0, mask1=None, mask2=None):
        n = self.domain_size()
        out = np.zeros((n, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_witness_map(
            self.ctx.h, self.h, kind, party, _ptr(np.ascontiguousarray(public_inputs, dtype=np.uint64)),
            _ptr(np.ascontiguousarray(witness, dtype=np.uint64)), _ptr(mask1), _ptr(mask2), _ptr(out)))
        return out

    def witness_map_libsnark(self, public_inputs, witness, kind=CS_PLAIN, party=0, mask=None):
        n = self.domain_size()
        out = np.zeros((n, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_witness_map_libsnark(
            self.ctx.h, self.h, kind, party, _ptr(np.ascontiguousarray(public_inputs, dtype=np.uint64)),
            _ptr(np.ascontiguousarray(witness, dtype=np.uint64)), _ptr(mask), _ptr(out)))
        return out

    def prove_plain(self, public_inputs, witness, r_mont, s_mont):
        """-> (A, B, C) affine Montgomery limb arrays."""
        a = np.zeros(2 * self.fq, dtype=np.uint64)
        b = np.zeros(4 * self.fq, dtype=np.uint64)
        c = np.zeros(2 * self.fq, dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_prove_plain(
            self.ctx.h, self.h, _ptr(public_inputs), _ptr(witness), _ptr(r_mont), _ptr(s_mont),
            _ptr(a), _ptr(b), _ptr(c)))
        return a, b, c

    def prove_plain_batch(self, public_inputs, witness=None, r_mont=None, s_mont=None, d_witness=None):
        """K plain proofs in one call (cs_groth16_prove_plain_batch).  public_inputs: uint64 [K, ni, 4]; witness:
        uint64 [K, nw, 4] on the host, or d_witness: a device pointer to the same layout; r_mont, s_mont: [K, 4].
        -> (A [K, 2 fq], B [K, 4 fq], C [K, 2 fq]) affine Montgomery limb arrays; row j equals prove_plain's
        result for proof j."""
        pub = np.ascontiguousarray(public_inputs, dtype=np.uint64)
        K = pub.shape[0]
        ni = pub.shape[1] if pub.ndim > 1 else 0
        wit = None if witness is None else np.ascontiguousarray(witness, dtype=np.uint64)
        nw = wit.shape[1] if wit is not None and wit.ndim > 1 else (self.nw or 0)
        r = np.ascontiguousarray(r_mont, dtype=np.uint64)
        s = np.ascontiguousarray(s_mont, dtype=np.uint64)
        if r.size != 4 * K or s.size != 4 * K:
            raise CsError("prove_plain_batch: need one r and one s per proof")
        a = np.zeros((K, 2 * self.fq), dtype=np.uint64)
        b = np.zeros((K, 4 * self.fq), dtype=np.uint64)
        c = np.zeros((K, 2 * self.fq), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_prove_plain_batch(
            self.ctx.h, self.h, K, _ptr(pub), ni, _ptr(wit) if wit is not None and wit.size else None,
            C.c_void_p(d_witness) if d_witness else None, nw, _ptr(r), _ptr(s), _ptr(a), _ptr(b), _ptr(c)))
        return a, b, c

    def prove_plain_device(self, public_inputs, d_witness, r_mont, s_mont):
        a = np.zeros(2 * self.fq, dtype=np.uint64)
        b = np.zeros(4 * self.fq, dtype=np.uint64)
        c = np.zeros(2 * self.fq, dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_prove_plain_device(
            self.ctx.h, self.h, _ptr(public_inputs), C.c_void_p(d_witness), _ptr(r_mont), _ptr(s_mont),
            _ptr(a), _ptr(b), _ptr(c)))
        return a, b, c

    def rep3_local(self, party, public_inputs, witness_shares, mask1, mask2, r_share, s_share, parts=31, prf=None):
        """-> (g_a, g1_b, g2_b, l_acc, h_acc) affine Montgomery half shares.  parts: CS_PART_* bitmask.
        prf = (seed1, pos1, seed2, pos2[, rounds]) draws the two mask vectors on the device instead."""
        g1 = lambda: np.zeros(2 * self.fq, dtype=np.uint64)
        ga, gb1, gb2, l, h = g1(), g1(), np.zeros(4 * self.fq, dtype=np.uint64), g1(), g1()
        p = None
        if prf is not None:
            p = Rep3Prf()
            p.seed1[:] = list(bytes(prf[0]))
            p.word_pos1 = prf[1]
            p.seed2[:] = list(bytes(prf[2]))
            p.word_pos2 = prf[3]
            p.rounds = prf[4] if len(prf) > 4 else 12
        self.ctx._check(self.ctx.lib.cs_groth16_rep3_local_prf(
            self.ctx.h, self.h, party, parts, _ptr(public_inputs), _ptr(witness_shares), _ptr(mask1), _ptr(mask2),
            C.byref(p) if p is not None else None, _ptr(r_share), _ptr(s_share), _ptr(ga), _ptr(gb1), _ptr(gb2),
            _ptr(l), _ptr(h)))
        return ga, gb1, gb2, l, h

    def rep3_prove(self, net0, net1, state, public_inputs, witness_shares=None, d_witness_shares=None, pair=None,
                   want_rs=False):
        """Rep3CoGroth16::prove for this party inside the library (cs_groth16_rep3_prove[_main]).
        -> (A, B, C[, rs]) affine Montgomery; rs = [r.a, r.b, s.a, s.b]."""
        a = np.zeros(2 * self.fq, dtype=np.uint64)
        b = np.zeros(4 * self.fq, dtype=np.uint64)
        c = np.zeros(2 * self.fq, dtype=np.uint64)
        rs = np.zeros((4, 4), dtype=np.uint64)
        dw = C.c_void_p(d_witness_shares) if d_witness_shares else None
        if pair is None:
            rc = self.ctx.lib.cs_groth16_rep3_prove(self.ctx.h, self.h, net0.h, net1.h, state.h, _ptr(public_inputs),
                                                    _ptr(witness_shares), dw, _ptr(a), _ptr(b), _ptr(c), _ptr(rs))
        else:
            rc = self.ctx.lib.cs_groth16_rep3_prove_main(self.ctx.h, self.h, net0.h, net1.h, pair.h, state.h,
                                                         _ptr(public_inputs), _ptr(witness_shares), dw, _ptr(a), _ptr(b),
                                                         _ptr(c), _ptr(rs))
        self.ctx._check(rc)
        return (a, b, c, rs) if want_rs else (a, b, c)

    def rep3_prove_helper(self, party, pair, state, public_inputs, witness_shares=None, d_witness_shares=None):
        dw = C.c_void_p(d_witness_shares) if d_witness_shares else None
        self.ctx._check(self.ctx.lib.cs_groth16_rep3_prove_helper(self.ctx.h, self.h, party, pair.h, state.h,
                                                                  _ptr(public_inputs), _ptr(witness_shares), dw))

    def shamir_prove(self, net0, net1, num_parties, threshold, public_inputs, witness_shares):
        """ShamirCoGroth16::prove inside the library -> (A, B, C, [r_share, s_share])."""
        a = np.zeros(2 * self.fq, dtype=np.uint64)
        b = np.zeros(4 * self.fq, dtype=np.uint64)
        c = np.zeros(2 * self.fq, dtype=np.uint64)
        rs = np.zeros((2, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_shamir_prove(self.ctx.h, self.h, net0.h, net1.h, num_parties, threshold,
                                                             _ptr(public_inputs), _ptr(witness_shares), _ptr(a), _ptr(b),
                                                             _ptr(c), _ptr(rs)))
        return a, b, c, rs

    def prove_with_shamir_bridge(self, net0, net1, public_inputs, witness_rep3_shares):
        """CoGroth16::prove_with_shamir_bridge: Rep3 witness shares in, Shamir(t = 1) prover."""
        a = np.zeros(2 * self.fq, dtype=np.uint64)
        b = np.zeros(4 * self.fq, dtype=np.uint64)
        c = np.zeros(2 * self.fq, dtype=np.uint64)
        rs = np.zeros((2, 4), dtype=np.uint64)
        self.ctx._check(self.ctx.lib.cs_groth16_prove_with_shamir_bridge(self.ctx.h, self.h, net0.h, net1.h, _ptr(public_inputs),
                                                                         _ptr(witness_rep3_shares), _ptr(a), _ptr(b), _ptr(c),
                                                                         _ptr(rs)))
        return a, b, c, rs

    def shamir_local(self, public_inputs, witness_shares, r_share, s_share):
        g1 = lambda: np.zeros(2 * self.fq, dtype=np.uint64)
        ga, gb1, gb2, l, h = g1(), g1(), np.zeros(4 * self.fq, dtype=np.uint64), g1(), g1()
        self.ctx._check(self.ctx.lib.cs_groth16_shamir_local(
            self.ctx.h, self.h, _ptr(public_inputs), _ptr(witness_shares), _ptr(r_share), _ptr(s_share),
            _ptr(ga), _ptr(gb1), _ptr(gb2), _ptr(l), _ptr(h)))
        return ga, gb1, gb2, l, h

    def free(self):
        if self.h:
            self.ctx.lib.cs_groth16_pk_free(self.h)
            self.h = None


class Net:
    """cs_net: one n-party mesh (mpc_net::Network).  Build with Net.peer (mailboxes in GPU memory, CUDA IPC /
    NVLink) or Net.callbacks (any Python transport: send(to, bytes), recv(frm, nbytes) -> bytes)."""

    def __init__(self, lib, h, id, n, keep=None):
        self.lib, self.h, self.id, self.n, self._keep = lib, h, id, n, keep

    @classmethod
    def callbacks(cls, lib, id, n, send, recv):
        def _send(_u, to, data, nbytes):
            try:
                send(to, C.string_at(data, nbytes))
                return 0
            except Exception:  # noqa: BLE001 -- must not unwind through the C frame
                import traceback
                traceback.print_exc()
                return -1

        def _recv(_u, frm, data, nbytes):
            try:
                b = recv(frm, nbytes)
                if len(b) != nbytes:
                    return -2
                C.memmove(data, b, nbytes)
                return 0
            except Exception:  # noqa: BLE001
                import traceback
                traceback.print_exc()
                return -1
        cb = NetCallbacks(None, NET_SEND_FN(_send), NET_RECV_FN(_recv))
        h = C.c_void_p()
        if lib.cs_net_from_callbacks(id, n, C.byref(cb), C.byref(h)):
            raise CsError(lib.cs_last_error().decode())
        return cls(lib, h, id, n, keep=cb)

    @classmethod
    def peer(cls, ctx, id, n):
        h = C.c_void_p()
        ctx._check(ctx.lib.cs_net_peer_create(ctx.h, id, n, C.byref(h)))
        return cls(ctx.lib, h, id, n)

    def _check(self, rc):
        if rc:
            raise CsError(self.lib.cs_last_error().decode())

    def handle(self):
        out = np.zeros(64, dtype=np.uint8)
        self._check(self.lib.cs_net_peer_handle(self.h, _ptr(out)))
        return out

    def connect(self, handles):
        """handles: [n][64] uint8, indexed by party id (other processes' cs_net_peer_handle)."""
        arr = np.ascontiguousarray(handles, dtype=np.uint8).reshape(self.n, 64)
        self._check(self.lib.cs_net_peer_connect(self.h, _ptr(arr)))

    def connect_local(self, nets):
        """nets: the n Net objects living in this process, indexed by party id."""
        arr = (C.c_void_p * self.n)(*[x.h if x is not None else None for x in nets])
        self._check(self.lib.cs_net_peer_connect_local(self.h, arr))

    def send(self, to, data):
        b = bytes(data)
        self._check(self.lib.cs_net_send(self.h, to, b, len(b)))

    def recv(self, frm, nbytes):
        buf = C.create_string_buffer(nbytes)
        self._check(self.lib.cs_net_recv(self.h, frm, buf, nbytes))
        return buf.raw

    def sendrecv(self, to, data, frm, nbytes):
        """Both directions advance together: safe for exchanges larger than the mailbox credit window."""
        b = bytes(data)
        buf = C.create_string_buffer(nbytes)
        self._check(self.lib.cs_net_sendrecv(self.h, to, b, len(b), frm, buf, nbytes))
        return buf.raw

    @property
    def bytes_sent(self):
        return int(self.lib.cs_net_bytes_sent(self.h))

    def free(self):
        if self.h:
            self.lib.cs_net_free(self.h)
            self.h = None


def connect_peer_nets_over_dist(nets, group=None, device="cpu"):
    """Exchange the CUDA IPC handles of per-process peer nets over torch.distributed (bootstrap only) and
    connect them.  `nets`: this process's Net objects (e.g. [net0, net1]), same order on every rank of the group."""
    import torch
    import torch.distributed as dist
    n = dist.get_world_size(group)
    for net in nets:
        t = torch.from_numpy(net.handle().copy()).to(device)
        outs = [torch.empty_like(t) for _ in range(n)]
        dist.all_gather(outs, t, group=group)
        net.connect(np.stack([o.cpu().numpy() for o in outs]))
    dist.barrier(group=group)


class Rep3StateC:
    """cs_rep3_state: Rep3State's correlated randomness inside the library (two ChaCha12 streams)."""

    def __init__(self, lib, h, id):
        self.lib, self.h, self.id = lib, h, id

    @classmethod
    def create(cls, net):
        """Rep3State::new: OS-entropy seed, exchanged with net.reshare (rep3.rs:55-75)."""
        h = C.c_void_p()
        if net.lib.cs_rep3_state_create(net.h, C.byref(h)):
            raise CsError(net.lib.cs_last_error().decode())
        return cls(net.lib, h, net.id)

    @classmethod
    def from_seeds(cls, lib, party, own32, prev32, pos_own=0, pos_prev=0):
        h = C.c_void_p()
        if lib.cs_rep3_state_from_seeds(party, bytes(own32), pos_own, bytes(prev32), pos_prev, C.byref(h)):
            raise CsError(lib.cs_last_error().decode())
        return cls(lib, h, party)

    def prf(self):
        p = Rep3Prf()
        if self.lib.cs_rep3_state_prf(self.h, C.byref(p)):
            raise CsError(self.lib.cs_last_error().decode())
        return bytes(p.seed1), int(p.word_pos1), bytes(p.seed2), int(p.word_pos2), int(p.rounds)

    def clone(self):
        s1, p1, s2, p2, _ = self.prf()
        return Rep3StateC.from_seeds(self.lib, self.id, s1, s2, p1, p2)

    def free(self):
        if self.h:
            self.lib.cs_rep3_state_free(self.h)
            self.h = None


def os_random(lib, nbytes):
    out = np.zeros(nbytes, dtype=np.uint8)
    if lib.cs_os_random(_ptr(out), nbytes):
        raise CsError(lib.cs_last_error().decode())
    return out.tobytes()


def read_rep3_witness(lib, path, curve=CS_BN254):
    """CompressedRep3SharedWitness share file (co-circom split-witness output) -> (public [np, 4], shares, kind):
    kind CS_REP3: shares [nw, 8] (a || b, Montgomery); kind CS_PLAIN: additive half shares [nw, 4]."""
    npub, nwit, kind = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
    if lib.cs_rep3_witness_read(os.fsencode(path), curve, None, 0, None, 0, C.byref(npub), C.byref(nwit), C.byref(kind)):
        raise CsError(lib.cs_last_error().decode())
    per = 2 if kind.value == CS_REP3 else 1
    pub = np.zeros((npub.value, 4), dtype=np.uint64)
    sh = np.zeros((nwit.value, 4 * per), dtype=np.uint64)
    if lib.cs_rep3_witness_read(os.fsencode(path), curve, _ptr(pub), npub.value, _ptr(sh), nwit.value * per,
                                C.byref(npub), C.byref(nwit), C.byref(kind)):
        raise CsError(lib.cs_last_error().decode())
    return pub, sh, kind.value


def read_wtns(lib, path, curve=CS_BN254):
    """witness.wtns -> np.uint64 [nVars, 4] Montgomery (Witness::from_reader)."""
    n = C.c_size_t(0)
    if lib.cs_wtns_read(os.fsencode(path), curve, None, 0, C.byref(n)):
        raise CsError(lib.cs_last_error().decode())
    out = np.zeros((n.value, 4), dtype=np.uint64)
    if lib.cs_wtns_read(os.fsencode(path), curve, _ptr(out), n.value, C.byref(n)):
        raise CsError(lib.cs_last_error().decode())
    return out


# host-side single-point helpers (run on the host inside the library; no context needed)
def point_scalar_mul(lib, curve, group, p, s_mont):
    out = np.zeros_like(p)
    rc = lib.cs_point_scalar_mul(curve, group, _ptr(np.ascontiguousarray(p)), _ptr(np.ascontiguousarray(s_mont)), _ptr(out))
    if rc:
        raise CsError(lib.cs_last_error().decode())
    return out


def point_add(lib, curve, group, p, q):
    out = np.zeros_like(p)
    rc = lib.cs_point_add(curve, group, _ptr(np.ascontiguousarray(p)), _ptr(np.ascontiguousarray(q)), _ptr(out))
    if rc:
        raise CsError(lib.cs_last_error().decode())
    return out


def point_neg(lib, curve, group, p):
    out = np.zeros_like(p)
    rc = lib.cs_point_neg(curve, group, _ptr(np.ascontiguousarray(p)), _ptr(out))
    if rc:
        raise CsError(lib.cs_last_error().decode())
    return out
