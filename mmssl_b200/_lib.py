"""ctypes binding of libmmssl_b200.so (the C ABI declared in include/mmssl_b200.h).

This is the "reference-side binding" of the drop-in: the reference is Python, so the FFI a
maintainer would add is this ctypes stub.  The library is the ONLY compute back-end: if it is
missing, or the device is not an H100, loading fails loudly -- there is no CPU / eager fallback.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmmssl_b200.so")

c_i64, c_i32, c_f32, c_vp = C.c_int64, C.c_int, C.c_float, C.c_void_p


class CsrDesc(C.Structure):
    """mmssl_csr_t"""
    _fields_ = [("rowptr", c_vp), ("colidx", c_vp), ("vals", c_vp),
                ("n_rows", c_i64), ("n_cols", c_i64), ("nnz", c_i64),
                ("items", c_vp), ("n_items", c_i64), ("split_table", c_vp), ("counters", c_vp),
                ("segs_cap", c_i64)]


class GemmProblem(C.Structure):
    """mmssl_gemm_problem_t"""
    _fields_ = [("a_hi", c_vp), ("a_lo", c_vp), ("lda", c_i64), ("b_hi", c_vp), ("b_lo", c_vp), ("ldb", c_i64),
                ("m", c_i64), ("n", c_i64), ("k", c_i64), ("partial", c_vp), ("split_k", C.c_int32), ("reserved", C.c_int32)]


class SpmmRhs(C.Structure):
    """mmssl_spmm_rhs_t"""
    _fields_ = [("x", c_vp), ("ldx", c_i64), ("y", c_vp), ("ldy", c_i64), ("c", c_vp), ("ldc", c_i64),
                ("ysaved", c_vp), ("ldysaved", c_i64), ("s", c_vp), ("lds", c_i64), ("sbase", c_vp), ("ldsbase", c_i64),
                ("y_mode", C.c_int32), ("n_peers", C.c_int32), ("y_peers", c_vp * 8)]


_SIGS = {
    "mmssl_abi_version": (C.c_int, []),
    "mmssl_last_error": (C.c_char_p, []),
    "mmssl_device_check": (C.c_int, []),
    "mmssl_embed_width_supported": (C.c_int, [c_i32]),
    "mmssl_csr_workspace_bytes": (c_i64, [c_i64, c_i64]),
    "mmssl_csr_from_coo": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "mmssl_csr_row_normalize": (C.c_int, [c_vp, c_i64, c_vp, c_vp]),
    "mmssl_spmm_plan_items_cap": (c_i64, [c_i64, c_i64]),
    "mmssl_spmm_plan_splits_cap": (c_i64, [c_i64]),
    "mmssl_spmm_plan_segs_cap": (c_i64, [c_i64]),
    "mmssl_spmm_plan_workspace_bytes": (c_i64, [c_i64]),
    "mmssl_spmm_plan": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp]),
    "mmssl_spmm_csr_f32": (C.c_int, [C.POINTER(CsrDesc), c_i32, c_i32, C.POINTER(SpmmRhs), c_i32, c_f32, c_i32, c_vp,
                                     c_i64, c_i32, c_vp]),
    "mmssl_spmm_hot_f32": (C.c_int, [C.POINTER(CsrDesc), c_vp, c_vp, c_i32, c_i32, c_i32, C.POINTER(SpmmRhs), c_i32, c_f32, c_i32,
                                     c_vp, c_i64, c_vp]),
    "mmssl_spmm_bulk_plan_splits_cap": (c_i64, [c_i64]),
    "mmssl_spmm_bulk_plan_segs_cap": (c_i64, [c_i64]),
    "mmssl_spmm_bulk_plan_buckets_cap": (c_i64, [c_i64, c_i64]),
    "mmssl_spmm_bulk_plan_workspace_bytes": (c_i64, [c_i64]),
    "mmssl_spmm_bulk_plan": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp]),
    "mmssl_spmm_bulk_f32": (C.c_int, [C.POINTER(CsrDesc), c_vp, c_i64, c_i32, c_i32, C.POINTER(SpmmRhs), c_i32, c_f32, c_i32, c_vp,
                                      c_i64, c_i32, c_vp]),
    "mmssl_reduce_rows_epilogue": (C.c_int, [c_i64, c_i32, c_i32, C.POINTER(SpmmRhs), c_i32, c_f32, c_i32, c_i32, c_vp]),
    "mmssl_sgemm": (C.c_int, [c_i32, c_i32, c_i64, c_i64, c_i64, c_f32, c_vp, c_i64, c_vp, c_i64, c_f32, c_vp, c_i64,
                              c_i32, c_vp]),
    "mmssl_id_fuse_fwd": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_f32, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "mmssl_id_fuse_bwd": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_i64, c_vp]),
    "mmssl_wsum": (C.c_int, [c_vp, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "mmssl_id_fuse2_blocks": (C.c_int, [c_i64]),
    "mmssl_id_fuse2_fwd": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_f32, c_vp, c_vp, c_i64, c_i64, c_i32, c_f32, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "mmssl_id_fuse2_bwd": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_f32, c_vp, c_i64, c_i32, c_f32, c_vp, c_i64,
                                     c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp]),
    "mmssl_dwcat_reduce": (C.c_int, [c_vp, c_i32, c_vp, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "mmssl_combine_fwd": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_f32, c_f32, c_vp, c_i64,
                                    c_vp, c_i64, c_vp]),
    "mmssl_combine_partials": (c_i64, [c_i64, c_i32]),
    "mmssl_combine_bwd": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i64, c_i32,
                                    c_f32, c_f32, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "mmssl_softmax_bwd": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_f32, c_vp, c_i64, c_vp]),
    "mmssl_axpby": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_f32, c_vp, c_f32, c_vp, c_i64, c_vp]),
    "mmssl_mul_mask": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp]),
    "mmssl_sumsq_blocks": (c_i64, [c_i64, c_i32]),
    "mmssl_sumsq": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_vp, c_vp]),
    "mmssl_bpr_blocks": (c_i64, [c_i64, c_i32]),
    "mmssl_bpr": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, c_f32, c_vp,
                            c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "mmssl_infonce_prepare": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_infonce_stats_floats": (c_i64, [c_i64]),
    "mmssl_infonce_loss_blocks": (c_i64, [c_i64]),
    "mmssl_infonce_stats": (C.c_int, [c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_infonce_grad": (C.c_int, [c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_infonce_tc_supported": (C.c_int, [c_i64, c_i32]),
    "mmssl_infonce_tc_workspace_bytes": (c_i64, [c_i64, c_i32]),
    "mmssl_infonce_stats_tc": (C.c_int, [c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "mmssl_infonce_forward_tc": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                           c_vp, c_i64, c_vp]),
    "mmssl_infonce_grad_tc": (C.c_int, [c_vp, c_vp, c_i64, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp]),
    "mmssl_infonce_scatter": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "mmssl_loss_assemble": (C.c_int, [c_vp, c_i64, c_i64, c_f32, c_vp, c_i64, c_vp, c_i64, c_f32, c_vp, c_i64, c_vp,
                                      c_i64, c_i64, c_f32, c_vp, c_vp]),
    "mmssl_step_tick": (C.c_int, [c_vp, c_vp]),
    "mmssl_adamw": (C.c_int, [c_i32, C.POINTER(c_vp), C.POINTER(c_vp), C.POINTER(c_vp), C.POINTER(c_vp),
                              C.POINTER(c_i64), c_vp, c_f32, c_f32, c_f32, c_f32, c_f32, c_vp]),
    "mmssl_dp_fused_adamw": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_f32, c_i32, c_f32, c_f32, c_f32, c_f32, c_f32, c_vp]),
    "mmssl_dp_fused_adamw_dev": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_f32, c_vp, c_f32, c_f32, c_f32, c_f32, c_f32, c_vp]),
    "mmssl_sampler_init": (C.c_int, [c_vp, c_i64, c_vp]),
    "mmssl_sample_triples": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i32, C.c_uint64, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_sampler_workspace_bytes": (c_i64, [c_i64, c_i32]),
    "mmssl_sample_triples_multi": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i32, C.c_uint64, c_vp, c_i32, c_vp, c_i64, c_vp, c_vp, c_vp,
                                             c_vp]),
    "mmssl_eval_rank": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, C.POINTER(c_i32), c_i32,
                                  c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_eval_full_stage": (C.c_int, []),
    "mmssl_eval_rank_full": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, C.POINTER(c_i32),
                                       c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_eval_wide_workspace_bytes": (c_i64, [c_i64, c_i32, c_i64, c_i32]),
    "mmssl_eval_rank_wide": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, C.POINTER(c_i32),
                                       c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_eval_reduce": (C.c_int, [c_vp, c_i64, c_i32, c_vp, c_vp]),
    "mmssl_gan_bn_fwd": (C.c_int, [c_vp] * 7 + [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_bn_bwd": (C.c_int, [c_vp] * 5 + [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_gp_rev_bn": (C.c_int, [c_vp] * 6 + [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_bn_fwd_rev": (C.c_int, [c_vp] * 7 + [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_colsum": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_vp]),
    "mmssl_gan_head_fwd": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "mmssl_gan_head_bwd": (C.c_int, [c_vp, c_f32, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_gp_rows": (C.c_int, [c_vp, c_i64, c_i64, c_f32, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_gp_head_rev": (C.c_int, [c_vp] * 5 + [c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "mmssl_gan_usim_finish": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "mmssl_gan_usim_bwd_pre": (C.c_int, [c_vp] * 6 + [c_i64, c_i64, c_vp, c_vp]),
    "mmssl_gan_real_rows": (C.c_int, [c_vp] * 5 + [c_i64, c_i64, c_f32, c_f32, c_f32, c_vp, c_vp]),
    "mmssl_gan_interpolate": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp]),
    "mmssl_gan_add_scaled": (C.c_int, [c_vp, c_vp, c_f32, c_i64, c_vp]),
    "mmssl_gan_gather_rows": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i32, c_vp, c_vp]),
    "mmssl_gan_scatter_add_rows": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i32, c_vp, c_vp]),
    "mmssl_gather_owned": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp]),
    "mmssl_scatter_add_owned": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_i32, c_vp, c_i64, c_vp]),
    "mmssl_publish_rows": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_vp, c_i64, c_i32, c_i32, C.POINTER(c_vp), c_vp]),
    "mmssl_mc_allreduce_sum": (C.c_int, [c_vp, c_vp, c_i64, c_vp]),
    "mmssl_topk_rows": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i32, c_vp, c_vp]),
    "mmssl_pair_append": (C.c_int, [c_vp, c_i64, c_vp, c_i32, c_vp, c_vp, c_vp]),
    "mmssl_degree_values": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "mmssl_split_bf16": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp]),
    "mmssl_split_bf16_t": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp]),
    "mmssl_split_bf16_t_colsum": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "mmssl_gemm_bf16x3_workspace_floats": (c_i64, [c_i64, c_i64, c_i64, C.POINTER(c_i32)]),
    "mmssl_gemm_bf16x3": (C.c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_i32, c_vp, c_vp]),
    "mmssl_gemm_bf16x3_group_plan": (c_i64, [c_i32, C.POINTER(c_i64), c_i32, C.POINTER(c_i32), C.POINTER(c_i64), c_vp, c_i64]),
    "mmssl_gemm_bf16x3_group": (C.c_int, [c_i32, C.POINTER(GemmProblem), c_i32, c_vp]),
    "mmssl_gemm_bf16x3_wide": (C.c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_f32, c_i32, c_vp, c_i64, c_vp]),
    "mmssl_gemm_wide_set_chunk": (C.c_int, [c_i32]),
    "mmssl_spmm_pipe_set_blocks": (C.c_int, [c_i32]),
    "mmssl_spmm_plan_set_cuts": (C.c_int, [c_i32, c_i32, c_i32, c_i32]),
    "mmssl_proj_epilogue": (C.c_int, [c_vp, c_i32, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "mmssl_wgrad_epilogue": (C.c_int, [c_vp, c_i32, c_i64, c_i64, c_vp, c_i64, c_i32, c_vp]),
    "mmssl_colsum": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp, c_i32, c_vp]),
}

_lib = None

# kernels launched by one call of each entry point (for bench.py's gpu_launches claim)
# (mmssl_sample_triples_multi: an approximate count -- 8 select passes + compaction + draw + CUB's radix sort, whose
# launch count depends on the batch and the key width; 1 when the batch exceeds the eligible users)
KERNELS_PER_CALL = {
    "mmssl_csr_from_coo": 6, "mmssl_csr_row_normalize": 1, "mmssl_spmm_plan": 8, "mmssl_spmm_csr_f32": 1, "mmssl_spmm_hot_f32": 1, "mmssl_spmm_bulk_plan": 9, "mmssl_spmm_bulk_f32": 1, "mmssl_reduce_rows_epilogue": 1, "mmssl_sgemm": 1,
    "mmssl_id_fuse_fwd": 1, "mmssl_id_fuse_bwd": 1, "mmssl_wsum": 1, "mmssl_id_fuse2_fwd": 1, "mmssl_id_fuse2_bwd": 1,
    "mmssl_dwcat_reduce": 1, "mmssl_combine_fwd": 1, "mmssl_combine_bwd": 1, "mmssl_softmax_bwd": 1,
    "mmssl_axpby": 1, "mmssl_mul_mask": 1, "mmssl_sumsq": 1, "mmssl_bpr": 1, "mmssl_infonce_prepare": 1,
    "mmssl_infonce_stats": 2, "mmssl_infonce_grad": 1, "mmssl_infonce_scatter": 1, "mmssl_infonce_stats_tc": 4, "mmssl_infonce_forward_tc": 3, "mmssl_infonce_grad_tc": 1, "mmssl_loss_assemble": 1,
    "mmssl_step_tick": 1, "mmssl_dp_fused_adamw": 1, "mmssl_dp_fused_adamw_dev": 1, "mmssl_sampler_init": 1, "mmssl_sample_triples": 1, "mmssl_sample_triples_multi": 20, "mmssl_adamw": 1, "mmssl_split_bf16": 1, "mmssl_split_bf16_t": 1, "mmssl_split_bf16_t_colsum": 1, "mmssl_gemm_bf16x3": 1, "mmssl_gemm_bf16x3_group": 1, "mmssl_gemm_bf16x3_wide": 1,
    "mmssl_proj_epilogue": 1, "mmssl_wgrad_epilogue": 1, "mmssl_colsum": 1,
    "mmssl_eval_rank": 1, "mmssl_eval_rank_full": 1, "mmssl_eval_rank_wide": 1, "mmssl_eval_reduce": 1,
    "mmssl_gan_bn_fwd": 1, "mmssl_gan_bn_bwd": 1, "mmssl_gan_gp_rev_bn": 1, "mmssl_gan_bn_fwd_rev": 1, "mmssl_gan_colsum": 1,
    "mmssl_gan_head_fwd": 2, "mmssl_gan_head_bwd": 1, "mmssl_gan_gp_rows": 2, "mmssl_gan_gp_head_rev": 2, "mmssl_gan_usim_finish": 1,
    "mmssl_gan_usim_bwd_pre": 1, "mmssl_gan_real_rows": 1, "mmssl_gan_interpolate": 1, "mmssl_gan_add_scaled": 1,
    "mmssl_gan_gather_rows": 1, "mmssl_gan_scatter_add_rows": 1,
    "mmssl_topk_rows": 1, "mmssl_pair_append": 1, "mmssl_degree_values": 2, "mmssl_gather_owned": 1, "mmssl_scatter_add_owned": 1, "mmssl_publish_rows": 1, "mmssl_mc_allreduce_sum": 1,
}
launch_count = 0
call_log = None   # set to a list to record (name) of every kernel-launching call


class _Counted:
    __slots__ = ("fn", "name", "k")

    def __init__(self, fn, name, k):
        self.fn, self.name, self.k = fn, name, k

    def __call__(self, *a):
        global launch_count
        launch_count += self.k
        if call_log is not None:
            call_log.append(self.name)
        return self.fn(*a)


class MmsslLibraryError(RuntimeError):
    pass


def load(require_device: bool = False) -> C.CDLL:
    """Load the shared library (once).  Raises if it has not been built -- no fallback path exists."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MmsslLibraryError(
                f"{LIB_PATH} is missing: build it with `python -m mmssl_b200.build` (nvcc, sm_90a). "
                "mmssl_b200 has no CPU or eager-PyTorch fallback.")
        lib = C.CDLL(LIB_PATH)
        missing = []
        for name, (res, args) in _SIGS.items():
            try:
                fn = getattr(lib, name)
            except AttributeError:
                missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args
            if name in KERNELS_PER_CALL:
                setattr(lib, name, _Counted(fn, name, KERNELS_PER_CALL[name]))
        if missing:
            raise MmsslLibraryError(f"{LIB_PATH} does not export: {missing}")
        if lib.mmssl_abi_version() != 1:
            raise MmsslLibraryError("ABI version mismatch between _lib.py and libmmssl_b200.so")
        _lib = lib
    if require_device:
        if not torch.cuda.is_available():
            raise MmsslLibraryError("mmssl_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        check(_lib.mmssl_device_check())
    return _lib


def exported_symbols():
    return list(_SIGS.keys())


def check(rc: int) -> None:
    if rc != 0:
        msg = _lib.mmssl_last_error().decode() if _lib is not None else "?"
        raise MmsslLibraryError(f"libmmssl_b200 call failed (rc={rc}): {msg}")


def ptr(t) -> c_vp:
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return c_vp(0)
    return c_vp(t.data_ptr())


def stream() -> c_vp:
    return c_vp(torch.cuda.current_stream().cuda_stream)
