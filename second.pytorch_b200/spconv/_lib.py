"""ctypes binding of libb2second.so (include/b2second.h).

The product path has NO fallback: if the CUDA library is missing or a call fails, this raises.
Memory is owned by torch tensors; raw device pointers and the current CUDA stream are passed down.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2S_LIB", os.path.join(_HERE, "..", "csrc", "libb2second.so"))

_lib = None

c_void_p, c_int, c_float, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
_I3 = ctypes.c_int * 3
_F3 = ctypes.c_float * 3
_F6 = ctypes.c_float * 6

# name -> (restype, argtypes); mirrors include/b2second.h exactly (checked by tests/test_abi.py)
SIGNATURES = {
    "b2s_version": (c_int, []),
    "b2s_last_error": (ctypes.c_char_p, []),
    "b2s_transform_sweep": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p]),
    "b2s_crop_workspace_bytes": (c_size_t, [c_int]),
    "b2s_crop_convex": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_size_t,
                                c_void_p, c_void_p]),
    "b2s_voxelize_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b2s_voxelize_hash_capacity": (c_int, [c_int]),
    "b2s_voxelize": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_hash_build": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2s_rulebook_subm": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                  c_void_p, c_void_p, c_void_p]),
    "b2s_rulebook_conv_workspace_bytes": (c_size_t, [c_int, c_void_p]),
    "b2s_rulebook_conv": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                  c_size_t, c_void_p, c_void_p, c_void_p]),
    "b2s_rulebook_subm_ranked": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                         c_void_p, c_void_p, c_void_p]),
    "b2s_rulebook_pairs": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2s_sparse_conv": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                c_int, c_void_p, c_int, c_void_p]),
    "b2s_to_bev": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                           c_void_p]),
    "b2s_pfn": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                        c_void_p, c_int, c_float, c_float, c_float, c_float, c_void_p, c_void_p]),
    "b2s_pfn_ex": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                           c_void_p, c_int, c_float, c_float, c_float, c_float, c_int, c_void_p, c_void_p]),
    "b2s_crop_nhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2s_crop_nhwc_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                 c_void_p]),
    "b2s_decode_filter": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_int, c_void_p, c_void_p]),
    "b2s_sparse_conv_tc_supported": (c_int, [c_int, c_int]),
    "b2s_sparse_conv_tc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                   c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2s_sparse_tile_plan": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                     c_void_p]),
    "b2s_sparse_conv_tc_plan": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                        c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                        c_int, c_int, c_void_p, c_void_p]),
    "b2s_sparse_conv_tc_plan_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                           c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                           c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2s_sparse_conv_tc_plan_ex2": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                            c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                            c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2s_split_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b2s_split_f16_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "b2s_merge_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b2s_split_f16_autoscale": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                        c_void_p]),
    "b2s_split_f16_autoscale_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                           c_int, c_void_p]),
    "b2s_rulebook_transpose": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "b2s_sparse_conv_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b2s_sparse_conv_wgrad": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                      c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2s_sparse_conv_wgrad_tc_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b2s_sparse_conv_wgrad_tc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                         c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_size_t, c_void_p]),
    "b2s_sparse_conv_wgrad_tc_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                            c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_size_t, c_int, c_void_p]),
    "b2s_pfn_train_workspace_bytes": (c_size_t, [c_int]),
    "b2s_pfn_train_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_int, c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_float,
                                      c_float, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_pfn_train_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                       c_float, c_float, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2s_bn_relu_train_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b2s_bn_relu_train_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_float, c_float, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2s_bn_relu_train_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t,
                                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2s_from_bev":(c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                             c_void_p]),
    "b2s_to_bev_tc": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                              c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2s_to_bev_tc_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                 c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2s_to_bev_tc_ex2": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                  c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "b2s_rpn_strip_bands": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    "b2s_rpn_bg_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p]),
    "b2s_rpn_block_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p]),
    "b2s_rpn_strip_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_void_p]),
    "b2s_conv2d_tc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                              c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2s_conv2d_tc_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                 c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                 c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p]),
    "b2s_conv2d_tc_ex2": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                  c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2s_conv2d_tc_ex3": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                  c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                  c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2s_rpn_tail_tc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2s_rpn_tail_tc_ex": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2s_rpn_tail_tc_ex2": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                    c_void_p]),
    "b2s_decode_filter_strided": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, ctypes.c_longlong,
                                          ctypes.c_longlong, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                          c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2s_decode_filter_segments": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                           c_void_p]),
    "b2s_decode_filter_multiclass": (c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_longlong, ctypes.c_longlong,
                                             ctypes.c_longlong, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                             c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2s_anchor_area_mask_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b2s_anchor_area_mask": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_float, c_void_p,
                                     c_size_t, c_void_p, c_void_p]),
    "b2s_concat_class_detections": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p,
                                            c_void_p]),
    "b2s_nms_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b2s_nms": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                        c_int, c_float, c_int, c_float, c_float, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                        c_size_t, c_void_p]),
    "b2s_vfe_mean": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2s_rotate_iou_eval": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2s_rbbox_overlap_host": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_void_p, c_int]),
    "b2s_nms_aligned_host": (c_int, [c_void_p, c_int, c_float, c_float, c_int, c_void_p, c_int]),
    "b2s_nms_rotated_host": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_float, c_void_p, c_int]),
    "b2s_kitti_convert": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p]),
    "b2s_kitti_overlaps": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int,
                                   ctypes.c_double, c_void_p, c_void_p]),
    "b2s_kitti_eval_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "b2s_kitti_eval": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                               c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2s_assign_targets_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b2s_assign_targets": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int,
                                   c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_augment_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b2s_augment": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                            c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                            c_void_p, c_void_p]),
    "b2s_augment_draws": (c_int, [ctypes.c_uint64, c_void_p, ctypes.c_uint64, c_int, c_void_p, c_int, c_void_p, c_int,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2s_db_sample_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b2s_db_sample": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                              c_void_p, c_void_p]),
    "b2s_detection_loss_workspace_bytes": (c_size_t, [c_int, c_int]),
    "b2s_detection_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                   c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_detection_loss_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p,
                                            c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p]),
    "b2s_optim_workspace_bytes": (c_size_t, [c_int]),
    "b2s_optim_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_train_metrics_workspace_bytes": (c_size_t, [c_int, c_int]),
    "b2s_train_metrics": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_train_metrics_count": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                        c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "b2s_train_metrics_finish": (c_int, [c_void_p, c_void_p, ctypes.c_float, c_void_p, c_void_p, c_void_p]),
    "b2s_pack_sparse_weights": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                        c_void_p]),
    "b2s_pack_sparse_weights_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                           c_int, c_void_p]),
    "b2s_split_halo_f16_autoscale_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_int, c_void_p]),
    "b2s_pack_conv2d_weights_ex": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "b2s_conv2d_wgrad_tc_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "b2s_split_halo_f16_autoscale": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p]),
    "b2s_pack_conv2d_weights": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2s_conv2d_wgrad_tc_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "b2s_conv2d_wgrad_tc": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
}

class AugmentDrawParams(ctypes.Structure):
    """b2s_augment_draw_params (include/b2second.h): the settings of b2s_augment_draws, passed by host pointer."""
    _fields_ = [("loc_std", ctypes.c_double * 3), ("rot_noise", ctypes.c_double * 2),
                ("rotation", ctypes.c_double * 2), ("scaling", ctypes.c_double * 2),
                ("translate_std", ctypes.c_double * 3), ("object_noise", c_int), ("random_flip_x", c_int),
                ("random_flip_y", c_int)]


OPTIM_CHUNK = 4096       # B2S_OPTIM_CHUNK
OPTIM_HYPER_COLS = 5     # B2S_OPTIM_HYPER_COLS


class LossParams(ctypes.Structure):
    """b2s_loss_params (include/b2second.h): the settings of b2s_detection_loss, passed by host pointer."""
    _fields_ = [("alpha", ctypes.c_float), ("gamma", ctypes.c_float), ("sigma", ctypes.c_float),
                ("code_weight", ctypes.c_float * 7), ("pos_cls_weight", ctypes.c_float),
                ("neg_cls_weight", ctypes.c_float), ("loc_weight", ctypes.c_float), ("cls_weight", ctypes.c_float),
                ("dir_weight", ctypes.c_float), ("sin_factor", ctypes.c_float), ("dir_offset", ctypes.c_float),
                ("num_dir_bins", c_int)]


class OptimParams(ctypes.Structure):
    """b2s_optim_params (include/b2second.h): the settings of b2s_optim_step, passed by host pointer."""
    _fields_ = [("weight_decay", ctypes.c_double), ("beta2", ctypes.c_double), ("eps", ctypes.c_double),
                ("max_norm", ctypes.c_double), ("total_step", ctypes.c_longlong), ("decoupled", c_int),
                ("zero_grad", c_int)]


METRICS_MAX_THRESHOLDS = 16   # B2S_METRICS_MAX_THRESHOLDS
METRICS_MAX_CODE = 8          # B2S_METRICS_MAX_CODE
METRICS_RECORD_HEAD = 19      # B2S_METRICS_RECORD_HEAD; the B2S_METRICS_REC_* slots in order:
METRICS_REC = ("rpn_acc", "cls_loss", "cls_loss_rt", "loc_loss", "loc_loss_rt", "cls_pos_rt", "cls_neg_rt", "dir_rt",
               "num_pos", "num_neg", "num_anchors")
METRICS_REC_LOC_ELEM = 11     # B2S_METRICS_REC_LOC_ELEM
METRICS_COUNT_HEAD = 20       # B2S_METRICS_COUNT_HEAD; the B2S_METRICS_CNT_* slots in order:
METRICS_CNT = ("frames", "correct", "cared", "pos", "num_pos", "num_neg", "num_anchors", "cls_loss", "loc_loss",
               "cls_pos", "cls_neg", "dir")
METRICS_CNT_LOC_ELEM = 12     # B2S_METRICS_CNT_LOC_ELEM


class MetricsParams(ctypes.Structure):
    """b2s_metrics_params (include/b2second.h): the settings of b2s_train_metrics, passed by host pointer."""
    _fields_ = [("num_thresholds", c_int), ("thresholds", ctypes.c_float * METRICS_MAX_THRESHOLDS),
                ("acc_threshold", ctypes.c_float)]


class MetricsBuffers(ctypes.Structure):
    """b2s_metrics_buffers (include/b2second.h): device pointers of the reference's running metric buffers."""
    _fields_ = [(n, c_void_p) for n in ("acc_total", "acc_count", "prec_total", "prec_count", "rec_total", "rec_count",
                                        "cls_total", "cls_count", "loc_total", "loc_count")]


class HeadSegment(ctypes.Structure):
    """b2s_head_segment (include/b2second.h): one head map of b2s_decode_filter_segments."""
    _fields_ = [("box", c_void_p), ("cls", c_void_p), ("dir", c_void_p), ("box_batch_stride", ctypes.c_longlong),
                ("cls_batch_stride", ctypes.c_longlong), ("dir_batch_stride", ctypes.c_longlong), ("ch_stride", c_int),
                ("pix_stride", c_int), ("a_loc", c_int), ("H", c_int), ("W", c_int), ("anchor_base", c_int)]


def head_segments(segs):
    """list of dicts with HeadSegment's field names (pointers as ints or None) -> ctypes array for the call."""
    arr = (HeadSegment * len(segs))()
    for i, d in enumerate(segs):
        for k, v in d.items():
            setattr(arr[i], k, v)
    return arr


def load():
    """dlopen libb2second.so and declare every entry point.  Raises if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.path.abspath(LIB_PATH)
    if not os.path.exists(path):
        raise ImportError(
            "libb2second.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C second.pytorch_b200/csrc`).  There is no CPU fallback on the product path." % path)
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.b2s_version() < 214:
        raise ImportError("libb2second.so is too old")
    _lib = lib
    return lib


def check(rc, what):
    if rc < 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, load().b2s_last_error().decode()))
    return rc


def ptr(t):
    """device (or host) pointer of a tensor / None."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def i3(v):
    return _I3(*[int(x) for x in v])


def f3(v):
    return _F3(*[float(x) for x in v])


def f6(v):
    return _F6(*[float(x) for x in v])


def require_cuda(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError("%s must be a CUDA tensor: the b2second spconv backend has no CPU path" % name)


STATUS_BITS = {1: "voxel overflow (more voxels than max_voxels; extra voxels dropped as upstream does)",
               2: "row overflow (strided conv produced more rows than the buffer capacity)",
               4: "hash table full", 8: "candidate overflow (more score survivors than cand_cap)",
               16: "an activation left the fp16 range (|x| > 65504) on the tensor-core path",
               32: "bad frame offsets (that frame was treated as having no ground truth), a bad point permutation, a "
                   "candidate outside the database or a training label outside [-1, num_class]",
               64: "a frame holds more ground truths than the augmentation's per-frame cap (no object noise there)",
               128: "a frame's ground truths plus database candidates exceed the sampler's per-frame cap (no samples "
                    "there)",
               256: "the gradient norm of an optimizer step was inf or NaN (the step was applied, as torch applies it)"}


def status_message(word):
    return "; ".join(msg for bit, msg in STATUS_BITS.items() if word & bit)
