"""ctypes binding of librqb200.so (C ABI declared in include/rqb200.h).

The shared library is built in-tree by ``build()`` (nvcc, sm_90a only) and loaded with ctypes -- no torch
extension machinery, no torch types in any signature.  There is NO fallback: if the library is missing or a
call fails, the product path raises.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Optional

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "librqb200.so")
SOURCES = ["api.cu", "rq_simt.cu", "dense.cu", "rq_tc.cu", "rq_tcx.cu", "gemm_tc.cu", "sid.cu", "t5dec.cu", "t5enc.cu", "t5enc_tc.cu",
           "t5rank.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]

_lib: Optional[ctypes.CDLL] = None

c_f32p = ctypes.POINTER(ctypes.c_float)
c_vp = ctypes.c_void_p
c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_f32 = ctypes.c_float
c_size = ctypes.c_size_t

# name -> (restype, argtypes); pointers are passed as integers (c_void_p)
_SIGNATURES = {
    "rqb200_version": (c_int, []),
    "rqb200_last_error": (ctypes.c_char_p, []),
    "rqb200_device_info": (c_int, [c_vp, c_vp, c_vp]),
    "rqb200_rq_workspace_bytes": (c_size, [c_int, c_int, c_int]),
    "rqb200_rq_forward": (c_int, [c_int, c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, c_f32,
                                  c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_size, c_vp]),
    "rqb200_rq_forward_from_ids": (c_int, [c_int, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32, c_vp, c_vp, c_vp,
                                           c_vp, c_vp, c_vp]),
    "rqb200_rq_backward": (c_int, [c_int, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_f32,
                                   c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp, c_i64,
                                   c_vp, c_vp, c_vp]),
    "rqb200_tokenize_tc_state_bytes": (c_size, [c_int, c_int, c_int]),
    "rqb200_tokenize_tc_supported": (c_int, [c_int, c_int, c_int]),
    "rqb200_tokenize_tc_ring_stages": (c_int, [c_int, c_int, c_int]),
    "rqb200_tokenize_tc_prepare": (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_size, c_vp]),
    "rqb200_tokenize_tc_run": (c_int, [c_vp, c_i64, c_int, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_kmeans_assign_accumulate": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                                c_vp, c_size, c_vp]),
    "rqb200_kmeans_finalize": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_vp, c_vp]),
    "rqb200_sgemm": (c_int, [c_int, c_int, c_int, c_int, c_int, c_f32, c_vp, c_i64, c_vp, c_i64, c_f32,
                             c_vp, c_i64, c_int, c_vp, c_i64, c_vp]),
    "rqb200_row_sqnorm": (c_int, [c_vp, c_int, c_int, c_vp, c_vp]),
    "rqb200_dist_finish": (c_int, [c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "rqb200_gumbel_softmax_fwd": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_f32, c_vp]),
    "rqb200_gumbel_row_finish": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_f32, c_vp, c_vp]),
    "rqb200_gumbel_bwd_ge": (c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_gumbel_bwd_softmax": (c_int, [c_vp, c_vp, c_int, c_int, c_f32, c_vp, c_vp, c_vp]),
    "rqb200_gumbel_bwd_gx": (c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_f32, c_int, c_int, c_vp]),
    "rqb200_gumbel_bwd_gc": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_l2norm_fwd": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_f32, c_vp]),
    "rqb200_l2norm_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_f32, c_vp]),
    "rqb200_sid_histogram": (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "rqb200_sid_dedup_workspace_bytes": (c_size, [c_int, c_int, c_int]),
    "rqb200_sid_dedup_rank": (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_size, c_vp]),
    "rqb200_sid_gather": (c_int, [c_vp, c_i64, c_int, c_vp, c_i64, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_sid_trie_workspace_bytes": (c_size, [c_i64, c_int, c_int]),
    "rqb200_sid_trie_scratch_bytes": (c_size, [c_i64, c_int, c_int]),
    "rqb200_sid_trie_build": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_size, c_vp, c_size, c_vp]),
    "rqb200_sid_trie_check": (c_int, [c_vp, c_i64, c_i64, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_sid_trie_beam_select": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                            c_vp, c_vp, c_vp]),
    "rqb200_sid_trie_sample_select": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int,
                                              c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_sid_trie_beam_topk": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                          c_vp, c_vp, c_vp]),
    "rqb200_sid_trie_sample_select_excluding": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                        c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                        c_int, c_int, c_vp]),
    "rqb200_sid_trie_beam_topk_excluding": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                                    c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_including": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                        c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                        c_int, c_int, c_vp]),
    "rqb200_sid_trie_beam_topk_including": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                                    c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_beam_topk_capped": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                                 c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_capped": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                     c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int,
                                                     c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_warped_capped": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                                            c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32,
                                                            c_f32, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_beam_topk_wide": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp,
                                               c_vp, c_vp, c_vp, c_int, c_vp]),
    "rqb200_sid_trie_beam_topk_wide_excluding": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp,
                                                         c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_beam_topk_wide_including": (c_int, [c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp,
                                                         c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_wide_workspace_bytes": (c_size, [c_int, c_int, c_int]),
    "rqb200_sid_trie_sample_select_wide": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int,
                                                   c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_size, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_wide_excluding": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                             c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_size,
                                                             c_int, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_wide_including": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                             c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_size,
                                                             c_int, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_warped": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                     c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32, c_f32, c_vp]),
    "rqb200_sid_trie_sample_select_warped_excluding": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                                               c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32,
                                                               c_f32, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_warped_including": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                                               c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_f32,
                                                               c_f32, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_warped_wide": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int,
                                                          c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_size,
                                                          c_int, c_f32, c_f32, c_vp]),
    "rqb200_sid_trie_sample_select_warped_wide_excluding": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int,
                                                                    c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                                    c_vp, c_vp, c_size, c_int, c_f32, c_f32, c_vp, c_vp, c_vp,
                                                                    c_int, c_int, c_vp]),
    "rqb200_sid_trie_sample_select_warped_wide_including": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int,
                                                                    c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                                    c_vp, c_vp, c_size, c_int, c_f32, c_f32, c_vp, c_vp, c_vp,
                                                                    c_int, c_int, c_vp]),
    "rqb200_sid_items_workspace_bytes": (c_size, [c_i64, c_int, c_int]),
    "rqb200_sid_items_build": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_size, c_vp]),
    "rqb200_sid_items_lookup": (c_int, [c_vp, c_vp, c_i64, c_i64, c_int, c_vp, c_vp]),
    "rqb200_sid_items_retrieve": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_sid_items_retrieve_excluding": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                    c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_exclusion_build": (c_int, [c_vp, c_int, c_int, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                           c_vp]),
    "rqb200_sid_items_retrieve_including": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                    c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_inclusion_build": (c_int, [c_vp, c_int, c_int, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                           c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_sid_topk_rank_hist": (c_int, [c_vp, c_i64, c_vp, c_i64, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "rqb200_sid_rank_hist": (c_int, [c_vp, c_int, c_i64, c_vp, c_vp]),
    "rqb200_sid_trie_counts": (c_int, [c_vp, c_vp, c_vp]),
    "rqb200_sid_trie_level": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_sid_items_offsets": (c_int, [c_i64, c_int, c_int, ctypes.POINTER(c_size), ctypes.POINTER(c_size)]),
    "rqb200_t5rank_cross_attention": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_i64,
                                              c_vp]),
    "rqb200_t5rank_cross_attention_tc": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_i64,
                                                 c_vp]),
    "rqb200_t5rank_children": (c_int, [c_vp, c_i64, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp]),
    "rqb200_t5rank_select": (c_int, [c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5rank_select_excluding": (c_int, [c_vp, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                               c_vp, c_int, c_int, c_vp]),
    "rqb200_t5score_trie_build": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5rank_cross_attention_ragged": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_i64, c_vp]),
    "rqb200_t5exact_frontier": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5exact_frontier_excluding": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_t5exact_frontier_including": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_t5exact_select": (c_int, [c_vp, c_vp, c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_t5exact_select_excluding": (c_int, [c_vp, c_vp, c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_t5exact_select_including": (c_int, [c_vp, c_vp, c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_t5dec_cross_attention": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, c_vp, c_i64,
                                             c_vp]),
    "rqb200_t5dec_self_attention": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                            c_vp, c_i64, c_vp]),
    "rqb200_t5dec_add_norm": (c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_int, c_int, c_f32, c_vp, c_vp]),
    "rqb200_t5enc_offsets": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_t5enc_assemble": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_int, c_int, c_int,
                                      c_int, c_vp, c_vp, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5enc_assemble_capacity": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_int, c_int,
                                               c_int, c_int, c_vp, c_vp, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5enc_attention": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_i64, c_vp]),
    "rqb200_t5enc_scatter": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_vp]),
    "rqb200_t5enc_attention_train": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_f32, c_vp, c_i64,
                                             c_vp, c_vp]),
    "rqb200_t5enc_attention_backward_tiles": (c_int, [c_int]),
    "rqb200_t5enc_attention_backward": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int,
                                                c_int, c_vp, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "rqb200_t5enc_attention_tc": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_i64, c_vp]),
    "rqb200_t5enc_attention_tc_train": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_f32, c_vp, c_i64,
                                                c_vp, c_vp]),
    "rqb200_t5enc_attention_tc_backward_tiles": (c_int, [c_int]),
    "rqb200_t5enc_attention_tc_backward": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_int,
                                                   c_int, c_int, c_vp, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "rqb200_t5enc_dropout_keep":(c_int, [c_vp, c_f32, c_int, c_int, c_int, c_vp, c_vp]),
    "rqb200_t5enc_add_norm_fwd": (c_int, [c_vp, c_vp, c_i64, c_vp, c_int, c_int, c_f32, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5enc_add_norm_bwd_parts": (c_int, [c_int]),
    "rqb200_t5enc_add_norm_bwd": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_t5dec_self_attention_train": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_vp, c_f32, c_vp, c_i64, c_vp, c_vp]),
    "rqb200_t5dec_self_attention_backward": (c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_int, c_vp,
                                                     c_f32, c_vp, c_i64, c_vp, c_vp]),
    "rqb200_t5dec_cross_attention_train": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int,
                                                   c_vp, c_f32, c_vp, c_i64, c_vp, c_vp]),
    "rqb200_t5dec_cross_attention_backward": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp,
                                                      c_vp, c_int, c_int, c_int, c_int, c_vp, c_f32, c_vp, c_i64, c_vp, c_vp, c_i64,
                                                      c_vp]),
    "rqb200_bf16_image_bytes":(c_size, [c_int, c_int]),
    "rqb200_f32_to_bf16_image": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_vp]),
    "rqb200_gemm_bf16": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_i64, c_vp]),
    "rqb200_split_image_bytes": (c_size, [c_int, c_int]),
    "rqb200_f32_to_split_image": (c_int, [c_vp, c_i64, c_int, c_int, c_int, c_vp, c_vp]),
    "rqb200_gemm_split": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "rqb200_gemm_split_k_slices": (c_int, [c_int, c_int, c_int]),
    "rqb200_f32_to_split_image_counted": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp]),
    "rqb200_gemm_split_counted": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp]),
    "rqb200_t5dec_self_attention_counted": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_int, c_int,
                                                    c_int, c_vp, c_i64, c_vp]),
    "rqb200_t5dec_add_norm_counted": (c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_int, c_vp, c_int, c_f32, c_vp,
                                              c_vp]),
    "rqb200_t5rank_cross_attention_ragged_counted": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_vp, c_int, c_vp,
                                                             c_i64, c_vp]),
    "rqb200_t5rank_children_counted": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp]),
    "rqb200_t5exact_frontier_capacity": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp] + [c_vp] * 10 + [c_int] * 3 + [c_vp] * 3 + [c_vp]),
    "rqb200_t5exact_frontier_capacity_excluding": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp] + [c_vp] * 10 + [c_int] * 3 + [c_vp] * 3 + [c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_t5exact_frontier_capacity_including": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_vp] + [c_vp] * 10 + [c_int] * 3 + [c_vp] * 3 + [c_vp, c_vp, c_vp, c_int, c_int, c_vp]),
    "rqb200_gemm_split_k": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_i64, c_vp]),
}


class Rqb200Error(RuntimeError):
    pass


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu into librqb200.so for sm_90a (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB_PATH] + srcs
    if verbose:
        print(" ".join(cmd))
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise Rqb200Error(f"nvcc failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


def load() -> ctypes.CDLL:
    """Load librqb200.so; raises (never falls back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Rqb200Error(
            f"{LIB_PATH} not found: the CUDA extension is required (there is no CPU/PyTorch fallback). "
            "Build it with `python -c 'import __graft_entry__ as g; g.build()'`.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().rqb200_last_error().decode("utf-8", "replace")
        raise Rqb200Error(f"librqb200 {what} failed (code {rc}): {msg}")
