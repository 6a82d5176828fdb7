"""ctypes binding of the C-ABI library (include/sbi_b200.h).

The product path has NO CPU fallback: if the shared library is missing or no sm_90 device
is present, calls raise.  PyTorch is used only for device memory and streams; every kernel is
launched through `call`, with raw device pointers, on torch's current stream of the device its
tensors live on.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SBI_B200_LIB") or os.path.join(_HERE, "lib", "libsbi_b200.so")

SBI_NSF_LAYER_STRIDE = 64
SBI_NSF_MAX_BLOCKS = 8
# layer-table field indices (mirror include/sbi_b200.h)
L_NID, L_NTR, L_W0, L_B0, L_WF, L_BF = 0, 1, 2, 3, 4, 5
L_LU_LOWER, L_LU_UPPER, L_LU_DIAG, L_LU_BIAS, L_FEAT, L_HAS_LU, L_BC0, L_BLK0 = 6, 7, 8, 9, 10, 11, 12, 16


class NsfModel(C.Structure):
    _fields_ = [
        ("D", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("NB", C.c_int32),
        ("KB", C.c_int32), ("T", C.c_int32),
        ("Dp", C.c_int32), ("Cp", C.c_int32), ("IDp", C.c_int32), ("Hp", C.c_int32),
        ("PR", C.c_int32), ("TRmax", C.c_int32), ("nf_chunk", C.c_int32),
        ("rpc0", C.c_int32), ("rpc1", C.c_int32), ("rpc2", C.c_int32),
        ("wcap", C.c_int32), ("nbuf", C.c_int32), ("n_params", C.c_int32),
        ("tail_bound", C.c_float), ("inv_sqrt_h", C.c_float), ("min_bw", C.c_float),
        ("min_bh", C.c_float), ("min_d", C.c_float), ("edge_raw", C.c_float),
        ("head", C.c_int32), ("M", C.c_int32), ("cond_mlp", C.c_int32), ("mog_eps", C.c_float),
        ("ld_zscore", C.c_float),
        ("d_params", C.c_void_p), ("d_layer_tab", C.c_void_p), ("d_feat_tab", C.c_void_p),
        ("d_stats", C.c_void_p),
    ]


SBI_NSF_TC_STRIDE = 192
SBI_NSF_TC_MAX_STAGES = 46


class NsfTc(C.Structure):
    _fields_ = [
        ("n_words", C.c_int32), ("stage_cap", C.c_int32),
        ("d_src", C.c_void_p), ("d_tab", C.c_void_p), ("d_tcw", C.c_void_p),
    ]


class MafModel(C.Structure):
    _fields_ = [
        ("D", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("NB", C.c_int32), ("T", C.c_int32),
        ("Dp", C.c_int32), ("Cp", C.c_int32), ("Hp", C.c_int32), ("OUTp", C.c_int32),
        ("rpc0", C.c_int32), ("rpc1", C.c_int32), ("rpcf", C.c_int32),
        ("wcap", C.c_int32), ("nbuf", C.c_int32), ("n_params", C.c_int32),
        ("scale_softplus", C.c_int32),
        ("head", C.c_int32), ("KB", C.c_int32), ("OUTM", C.c_int32),
        ("tail_bound", C.c_float), ("min_w", C.c_float), ("min_h", C.c_float), ("min_d", C.c_float),
        ("isq", C.c_float),
        ("ld_zscore", C.c_float),
        ("d_params", C.c_void_p), ("d_layer_tab", C.c_void_p), ("d_perm_tab", C.c_void_p),
        ("d_stats", C.c_void_p),
    ]


SBI_MAF_LAYER_STRIDE = 32
M_W0, M_B0, M_WC, M_BC, M_WF, M_BF, M_PERM, M_BLK0 = 0, 1, 2, 3, 4, 5, 6, 8


class RatioModel(C.Structure):
    _fields_ = [
        ("Dt", C.c_int32), ("Dx", C.c_int32), ("H", C.c_int32), ("NB", C.c_int32),
        ("Dtp", C.c_int32), ("Dxp", C.c_int32), ("Hp", C.c_int32),
        ("rpc0", C.c_int32), ("rpc1", C.c_int32),
        ("wcap", C.c_int32), ("nbuf", C.c_int32), ("n_params", C.c_int32),
        ("d_params", C.c_void_p), ("d_tab", C.c_void_p), ("d_stats", C.c_void_p),
    ]


class Pairs(C.Structure):
    _fields_ = [
        ("d_theta", C.c_void_p), ("d_x", C.c_void_p), ("d_theta_index", C.c_void_p),
        ("d_x_index", C.c_void_p), ("R", C.c_int64), ("x_shared", C.c_int32),
    ]


R_W0, R_B0, R_WF, R_BF, R_BLK0 = 0, 1, 2, 3, 4


class RatioMlpModel(C.Structure):
    _fields_ = [
        ("Dt", C.c_int32), ("Dx", C.c_int32), ("H", C.c_int32), ("NL", C.c_int32),
        ("Dtp", C.c_int32), ("Dxp", C.c_int32), ("Hp", C.c_int32),
        ("norm", C.c_int32), ("ln_eps", C.c_float),
        ("rpc0", C.c_int32), ("rpc1", C.c_int32),
        ("wcap", C.c_int32), ("nbuf", C.c_int32), ("n_params", C.c_int32),
        ("d_params", C.c_void_p), ("d_tab", C.c_void_p), ("d_stats", C.c_void_p),
    ]


RM_W0, RM_B0, RM_G0, RM_BE0, RM_WF, RM_BF = 0, 1, 2, 3, 8, 9
RM_NORM_NONE, RM_NORM_LAYER = 0, 1


class FmModel(C.Structure):
    _fields_ = [
        ("D", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("NL", C.c_int32), ("TE", C.c_int32),
        ("Dp", C.c_int32), ("Cp", C.c_int32), ("Hp", C.c_int32), ("TEp", C.c_int32),
        ("rpc_i", C.c_int32), ("rpc_c", C.c_int32), ("rpc_m", C.c_int32), ("rpc_t", C.c_int32),
        ("rpc_h", C.c_int32), ("rpc_o", C.c_int32),
        ("wcap", C.c_int32), ("nbuf", C.c_int32), ("n_params", C.c_int32),
        ("noise_scale", C.c_float), ("ln_eps", C.c_float), ("raw", C.c_int32), ("pad_", C.c_int32),
        ("d_params", C.c_void_p), ("d_tab", C.c_void_p), ("d_stats", C.c_void_p),
    ]


F_WI, F_BI, F_WC, F_BC, F_WM, F_BM, F_WT, F_BT, F_WO, F_BO, F_LAYER0 = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 12


class SliceChains(C.Structure):
    _fields_ = [
        ("C", C.c_int32), ("D", C.c_int32), ("num_samples", C.c_int32), ("tuning", C.c_int32),
        ("max_width", C.c_double), ("seed", C.c_uint64),
        ("d_x", C.c_void_p), ("d_width", C.c_void_p), ("d_order", C.c_void_p), ("d_istate", C.c_void_p),
        ("d_fstate", C.c_void_p), ("d_rng", C.c_void_p), ("d_samples", C.c_void_p),
    ]


SBI_HMC_NV0, SBI_HMC_NI, SBI_HMC_NF0 = 11, 14, 10
SBI_HMC_MAX_TREE_DEPTH = 30
SBI_HMC_MAX_WINDOWS = 64
SBI_HMC_TRACE_SCALARS = 5
SBI_HMC_NUTS, SBI_HMC_HMC = 0, 1


class HmcChains(C.Structure):
    _fields_ = [
        ("C", C.c_int32), ("D", C.c_int32), ("algo", C.c_int32), ("max_tree_depth", C.c_int32),
        ("warmup", C.c_int32), ("num_samples", C.c_int32), ("adapt_step_size", C.c_int32),
        ("adapt_mass_matrix", C.c_int32), ("n_windows", C.c_int32), ("win_end", C.c_int32 * SBI_HMC_MAX_WINDOWS),
        ("step_size", C.c_double), ("target_accept", C.c_double), ("trajectory_length", C.c_double),
        ("d_z", C.c_void_p), ("d_vec", C.c_void_p), ("d_istate", C.c_void_p), ("d_fstate", C.c_void_p),
        ("d_normal", C.c_void_p), ("d_uniform", C.c_void_p), ("d_logp", C.c_void_p), ("d_grad", C.c_void_p),
        ("d_params", C.c_void_p), ("d_samples", C.c_void_p), ("d_trace", C.c_void_p),
    ]


class Rows(C.Structure):
    _fields_ = [
        ("d_input", C.c_void_p), ("d_cond", C.c_void_p), ("d_index", C.c_void_p),
        ("R", C.c_int64), ("cond_shared", C.c_int32),
    ]


class TrainWs(C.Structure):
    _fields_ = [
        ("d_input", C.c_void_p), ("d_cond", C.c_void_p), ("d_logp", C.c_void_p),
        ("d_gpart", C.c_void_p), ("d_grad", C.c_void_p), ("d_state", C.c_void_p),
        ("d_step", C.c_void_p), ("d_mask", C.c_void_p), ("d_loss_acc", C.c_void_p),
        ("cap_rows", C.c_int64), ("d_sumsq", C.c_void_p),
        ("tc_pack", C.c_void_p), ("tc_fwd", C.c_void_p), ("tc_bwd", C.c_void_p),
        ("d_save", C.c_void_p), ("save_bytes", C.c_int64),
    ]


SBI_LC2ST_MAX_HIDDEN = 4
SBI_LC2ST_MAX_F = 64
SBI_LC2ST_MAX_WIDTH = 256


SBI_MMD_MAX_ROWS = 65536
SBI_MMD_MAX_SETS = 65536


class Lc2stNet(C.Structure):
    _fields_ = [("F", C.c_int32), ("L", C.c_int32), ("H", C.c_int32 * SBI_LC2ST_MAX_HIDDEN), ("P", C.c_int32)]


class Lc2stOpt(C.Structure):
    _fields_ = [
        ("max_iter", C.c_int32), ("n_iter_no_change", C.c_int32), ("early_stopping", C.c_int32),
        ("shuffle", C.c_int32), ("batch_size", C.c_int32),
        ("beta1", C.c_float), ("beta2", C.c_float), ("one_minus_beta1", C.c_float), ("one_minus_beta2", C.c_float),
        ("eps", C.c_float), ("alpha", C.c_float),
        ("lr_d", C.c_double), ("beta1_d", C.c_double), ("beta2_d", C.c_double), ("tol", C.c_double),
    ]


class Lc2stJob(C.Structure):
    _fields_ = [("row0", C.c_int64), ("n_train", C.c_int32), ("n_val", C.c_int32), ("order0", C.c_int64),
                ("key", C.c_uint64)]


class PeerCtx(C.Structure):
    _fields_ = [("h_peer_ptrs", C.c_void_p), ("world", C.c_int), ("rank", C.c_int), ("d_grad_local", C.c_void_p)]


class _Stream(C.c_void_p):
    """The trailing `void* stream` of an entry point that launches kernels (filled in by `call`)."""


_EXPORTS = {
    "sbi_b200_abi_version": (C.c_int, []),
    "sbi_b200_device_ok": (C.c_int, []),
    "sbi_b200_nsf_logprob": (C.c_int, [C.POINTER(NsfModel), C.POINTER(Rows), C.c_void_p,
                                       C.c_void_p, _Stream]),
    "sbi_b200_nsf_vjp_parts": (C.c_int, [C.c_int64]),
    "sbi_b200_nsf_vjp_save_bytes": (C.c_int64, [C.POINTER(NsfModel), C.c_int64]),
    "sbi_b200_nsf_vjp": (C.c_int, [C.POINTER(NsfModel), C.POINTER(Rows), C.c_void_p, C.c_float,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int64, _Stream]),
    "sbi_b200_nsf_inverse": (C.c_int, [C.POINTER(NsfModel), C.POINTER(Rows), C.c_void_p,
                                       C.c_void_p, _Stream]),
    "sbi_b200_nsf_tc_supported": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc)]),
    "sbi_b200_nsf_tc_pack": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), _Stream]),
    "sbi_b200_nsf_logprob_tc": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), C.POINTER(Rows),
                                          C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_nsf_inverse_tc": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), C.POINTER(Rows),
                                          C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_nsf_vjp_tc_supported": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), C.POINTER(NsfTc)]),
    "sbi_b200_nsf_vjp_tc_parts": (C.c_int, [C.c_int64]),
    "sbi_b200_nsf_vjp_tc_save_bytes": (C.c_int64, [C.POINTER(NsfModel), C.c_int64]),
    "sbi_b200_nsf_vjp_tc": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), C.POINTER(NsfTc), C.POINTER(Rows),
                                      C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int64, _Stream]),
    "sbi_b200_nsf_vjp_tc_cond": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), C.POINTER(NsfTc), C.POINTER(Rows),
                                           C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_int64, _Stream]),
    "sbi_b200_maf_logprob": (C.c_int, [C.POINTER(MafModel), C.POINTER(Rows), C.c_void_p,
                                       C.c_void_p, _Stream]),
    "sbi_b200_maf_vjp_parts": (C.c_int, [C.c_int64]),
    "sbi_b200_maf_vjp": (C.c_int, [C.POINTER(MafModel), C.POINTER(Rows), C.c_void_p, C.c_float,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   _Stream]),
    "sbi_b200_maf_inverse": (C.c_int, [C.POINTER(MafModel), C.POINTER(Rows), C.c_void_p,
                                       C.c_void_p, _Stream]),
    "sbi_b200_ratio_forward": (C.c_int, [C.POINTER(RatioModel), C.POINTER(Pairs), C.c_void_p, _Stream]),
    "sbi_b200_ratio_tc_supported": (C.c_int, [C.POINTER(RatioModel), C.POINTER(NsfTc)]),
    "sbi_b200_ratio_tc_pack": (C.c_int, [C.POINTER(RatioModel), C.POINTER(NsfTc), _Stream]),
    "sbi_b200_ratio_forward_tc": (C.c_int, [C.POINTER(RatioModel), C.POINTER(NsfTc), C.POINTER(Pairs),
                                            C.c_void_p, _Stream]),
    "sbi_b200_ratio_vjp_parts": (C.c_int, [C.c_int64]),
    "sbi_b200_ratio_vjp": (C.c_int, [C.POINTER(RatioModel), C.POINTER(Pairs), C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_ratio_vjp_inputs": (C.c_int, [C.POINTER(RatioModel), C.POINTER(Pairs), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_pair_rows_sum": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                         _Stream]),
    "sbi_b200_ratio_mlp_forward": (C.c_int, [C.POINTER(RatioMlpModel), C.POINTER(Pairs), C.c_void_p, _Stream]),
    "sbi_b200_ratio_mlp_vjp_parts": (C.c_int, [C.c_int64]),
    "sbi_b200_ratio_mlp_vjp": (C.c_int, [C.POINTER(RatioMlpModel), C.POINTER(Pairs), C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_fm_net_vjp": (C.c_int, [C.POINTER(FmModel), C.POINTER(Rows), C.c_void_p, C.c_void_p, C.c_void_p,
                                      _Stream]),
    "sbi_b200_fm_plan": (C.c_int, [C.POINTER(FmModel), C.c_int32, C.POINTER(C.c_int32)]),
    "sbi_b200_fm_forward_div": (C.c_int, [C.POINTER(FmModel), C.POINTER(Rows), C.c_void_p, C.c_int32, C.c_void_p,
                                          C.c_void_p, _Stream]),
    "sbi_b200_made_sample": (C.c_int, [C.POINTER(NsfModel), C.POINTER(Rows), C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_sde_em_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                       C.c_float, C.c_float, C.c_float, _Stream]),
    "sbi_b200_reject_scratch_ints": (C.c_int64, [C.c_int64]),
    "sbi_b200_reject_compact": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                          _Stream]),
    "sbi_b200_sir_scratch_ints": (C.c_int64, [C.c_int64]),
    "sbi_b200_sir_select": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                      C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_void_p, _Stream]),
    "sbi_b200_mmd_ws_bytes": (C.c_int64, [C.c_int32]),
    "sbi_b200_mmd": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                               C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                               _Stream]),
    "sbi_b200_rbf_matrix": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_double,
                                      C.c_void_p, _Stream]),
    "sbi_b200_lc2st_plan":(C.c_int, [C.POINTER(Lc2stNet), C.POINTER(C.c_int32)]),
    "sbi_b200_lc2st_ws_floats": (C.c_int64, [C.POINTER(Lc2stNet), C.c_int32]),
    "sbi_b200_lc2st_train": (C.c_int, [C.POINTER(Lc2stNet), C.POINTER(Lc2stOpt), C.c_void_p, C.c_int32,
                                       C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, _Stream]),
    "sbi_b200_lc2st_eval_chunks": (C.c_int, [C.POINTER(Lc2stNet), C.c_int64]),
    "sbi_b200_lc2st_eval": (C.c_int, [C.POINTER(Lc2stNet), C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_ode_red_size": (C.c_int, [C.c_int64]),
    "sbi_b200_ode_stage": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                     _Stream]),
    "sbi_b200_ode_error_commit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                            _Stream]),
    "sbi_b200_fm_forward": (C.c_int, [C.POINTER(FmModel), C.POINTER(Rows), C.c_void_p, C.c_int32, C.c_void_p,
                                      _Stream]),
    "sbi_b200_fm_vjp_parts": (C.c_int, [C.c_int64]),
    "sbi_b200_fm_loss_vjp": (C.c_int, [C.POINTER(FmModel), C.POINTER(Rows), C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_fm_loss_vjp_cond": (C.c_int, [C.POINTER(FmModel), C.POINTER(Rows), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            _Stream]),
    "sbi_b200_slice_init": (C.c_int, [C.POINTER(SliceChains), C.c_void_p, _Stream]),
    "sbi_b200_slice_step": (C.c_int, [C.POINTER(SliceChains), C.c_void_p, C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_hmc_init": (C.c_int, [C.POINTER(HmcChains), _Stream]),
    "sbi_b200_hmc_step": (C.c_int, [C.POINTER(HmcChains), C.c_void_p, _Stream]),
    "sbi_b200_reduce_partials": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p,
                                           _Stream]),
    "sbi_b200_nll_stats": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, _Stream]),
    "sbi_b200_sumsq_blocks": (C.c_int, [C.c_int64]),
    "sbi_b200_reduce_partials_norm": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                                C.c_void_p, _Stream]),
    "sbi_b200_adam_clip_step_norm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_float,
                                               C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_int,
                                               _Stream]),
    "sbi_b200_adam_clip_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_float,
                                          C.c_float, C.c_float, C.c_float, _Stream]),
    "sbi_b200_nsf_train_step_host": (C.c_int, [C.POINTER(NsfModel), C.POINTER(TrainWs), C.c_void_p,
                                               C.c_void_p, C.c_int64, C.c_float, C.c_float,
                                               C.c_float, C.c_float, C.c_float, C.c_void_p,
                                               _Stream]),
    "sbi_b200_pipe_create": (C.c_void_p, []),
    "sbi_b200_pipe_destroy": (None, [C.c_void_p]),
    "sbi_b200_nsf_train_step_host_async": (C.c_int, [C.POINTER(NsfModel), C.POINTER(TrainWs), C.c_void_p,
                                                     C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float,
                                                     C.c_float, C.c_float, C.c_float, C.c_void_p, _Stream]),
    "sbi_b200_pipe_drain": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sbi_b200_nsf_train_step_host_async_dp": (C.c_int, [C.POINTER(NsfModel), C.POINTER(TrainWs), C.c_void_p,
                                                        C.POINTER(PeerCtx), C.c_void_p, C.c_void_p, C.c_int64,
                                                        C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                                        C.c_void_p, _Stream]),
    "sbi_b200_nsf_logprob_host": (C.c_int, [C.POINTER(NsfModel), C.POINTER(TrainWs), C.c_void_p,
                                            C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                            _Stream]),
    "sbi_b200_peer_bytes": (C.c_int64, [C.c_int64]),
    "sbi_b200_peer_blocks": (C.c_int, [C.c_int64]),
    "sbi_b200_peer_alloc": (C.c_void_p, [C.c_int64]),
    "sbi_b200_peer_free": (C.c_int, [C.c_void_p]),
    "sbi_b200_peer_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sbi_b200_peer_import": (C.c_void_p, [C.c_void_p]),
    "sbi_b200_peer_close": (C.c_int, [C.c_void_p]),
    "sbi_b200_peer_sum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, _Stream]),
    "sbi_b200_peer_error": (C.c_int, [C.c_void_p, C.c_int64]),
    "sbi_b200_nsf_logprob_host_tc": (C.c_int, [C.POINTER(NsfModel), C.POINTER(NsfTc), C.POINTER(TrainWs),
                                               C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                               _Stream]),
}

_lib = None
# `call`'s names: the entry points whose last parameter is the stream, without the `sbi_b200_` prefix
_LAUNCH = {name[len("sbi_b200_"):]: name for name, (_, args) in _EXPORTS.items() if args and args[-1] is _Stream}


def exported_symbols():
    """Names every entry point declared in include/sbi_b200.h."""
    return list(_EXPORTS)


def load():
    """dlopen the library and bind prototypes (no GPU needed for this)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m sbi_b200.build` "
                "(there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _EXPORTS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        if lib.sbi_b200_abi_version() != 1:
            raise RuntimeError("libsbi_b200.so ABI version mismatch")
        _lib = lib
    return _lib


SBI_EINVAL, SBI_ESMEM = -1, -2


class SbiB200Error(RuntimeError):
    """A failed entry point; `rc` is its status (SBI_ESMEM or a CUDA error), None for a check made on the host."""

    def __init__(self, msg: str, rc: Optional[int] = None):
        super().__init__(msg)
        self.rc = rc


def check(rc: int, what: str):
    if rc == 0:
        return
    if rc == SBI_EINVAL:
        raise ValueError(f"{what}: invalid argument (SBI_EINVAL)")
    if rc == SBI_ESMEM:
        raise SbiB200Error(f"{what}: model does not fit the shared-memory budget (SBI_ESMEM)", rc)
    raise SbiB200Error(f"{what}: CUDA error {rc}", rc)


def call(name: str, *args, device=None):
    """Launch `sbi_b200_<name>` on torch's current stream of the device its tensor arguments live on (`device`
    when it has none, e.g. a struct-only call), and raise on a failed status.  Tensors are passed as their data
    pointers; None, numbers, ctypes structs (by reference where the prototype takes a pointer) and arrays as they
    are.  The C side makes that device current for the launch (csrc/device.cuh), so the current device does not
    matter.  Raises before anything launches for a CPU tensor or for tensors on two devices."""
    sym = _LAUNCH.get(name)
    if sym is None:
        raise ValueError(f"sbi_b200_{name} launches no kernel (its last parameter is not the stream): "
                         "call it on `load()`")
    dev = -1
    if device is not None:
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError(f"sbi_b200: {name} was asked to run on {device}; the kernels only run on a CUDA "
                               "(sm_90a) device and there is no CPU fallback")
        dev = torch.cuda.current_device() if device.index is None else device.index
    argv = []
    for a in args:
        if isinstance(a, torch.Tensor):
            if not a.is_cuda:
                require_cuda(a, f"a tensor argument of {name}")
            d = a.get_device()
            if dev < 0:
                dev = d
            elif d != dev:
                raise ValueError(f"{name}: arguments on cuda:{dev} and cuda:{d}; one launch works on one device")
            a = a.data_ptr()
        argv.append(a)
    if dev < 0:
        raise ValueError(f"{name}: no tensor argument to take the device from; pass device=")
    rc = getattr(_lib or load(), sym)(*argv, torch.cuda.current_stream(dev).cuda_stream)
    if rc:
        check(rc, name)


def stream_ptr(device=None) -> int:
    """torch's current stream on `device` (default: the current device), for raw calls outside `call`."""
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(
            f"sbi_b200: `{name}` lives on {t.device}; the kernels only run on a CUDA (sm_90a) "
            "device and there is no CPU fallback")
    return t


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def rows(inp: torch.Tensor, cond: torch.Tensor, index: Optional[torch.Tensor] = None, n: Optional[int] = None,
         shared: bool = False) -> Rows:
    """`Rows` over the tensors: input rows `inp` and condition rows `cond` (`cond[0]` for every row when `shared`),
    gathered through the optional int64 row `index`; n rows, by default as many as `index`, else `inp` has.
    The struct keeps the tensors alive."""
    if n is None:
        n = (inp if index is None else index).shape[0]
    r = Rows(inp.data_ptr(), cond.data_ptr(), None if index is None else index.data_ptr(), n, 1 if shared else 0)
    r._keep = (inp, cond, index)
    return r


def pairs(theta: torch.Tensor, x: torch.Tensor, ti: Optional[torch.Tensor] = None, xi: Optional[torch.Tensor] = None,
          n: Optional[int] = None, x_shared: bool = False) -> Pairs:
    """`Pairs` (theta[ti[r]], x[xi[r]]) over the tensors (row r of each without its index, `x[0]` for every pair
    when `x_shared`); n pairs, by default as many as `ti`, else `theta` has.  The struct keeps the tensors alive."""
    if n is None:
        n = (theta if ti is None else ti).shape[0]
    p = Pairs(theta.data_ptr(), x.data_ptr(), None if ti is None else ti.data_ptr(),
              None if xi is None else xi.data_ptr(), n, 1 if x_shared else 0)
    p._keep = (theta, x, ti, xi)
    return p


def reduce_partials(gpart: torch.Tensor, n_part: int, n_params: int) -> torch.Tensor:
    """The sum of the first `n_part` partial-gradient slabs of `gpart`, as a fresh (n_params,) tensor."""
    g = torch.empty(n_params, dtype=torch.float32, device=gpart.device)
    call("reduce_partials", gpart, n_part, n_params, g)
    return g
