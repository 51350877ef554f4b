"""ctypes binding of the package's native libraries, one `Library` record each in `LIBRARIES`: its file, the ctypes
signatures of its entry points (a dict that mirrors its header under include/ one to one), that header, the namespace
of its kernels, and whether it links against libdva_b200.so.  The linked libraries find libdva_b200.so next to them
through rpath $ORIGIN and share its error string and launch counter, so last_error() and launch_count() cover them
all; entry(name) finds an entry point in whichever library declares it.  Adding a library means adding a record, a
header and a signatures dict here, and the library's sources to the list of linked libraries in csrc/Makefile.

There is NO fallback: if a shared library is missing or a call fails, a RuntimeError is
raised.  PyTorch is used above this layer only for device memory and streams.
"""
import ctypes
import dataclasses
import functools
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# DVA_B200_LIB: developer knob to load a tuning variant of the same library (bench sweeps)
LIB_PATH = os.environ.get("DVA_B200_LIB") or os.path.join(_HERE, "libdva_b200.so")
CSRC_DIR = os.path.join(_HERE, "csrc")

DVA_OK, DVA_EINVAL, DVA_EALIGN, DVA_EUNSUPPORTED = 0, -1, -2, -3
DVA_F32, DVA_BF16, DVA_F16 = 0, 1, 2
REDUCE_CODES = {"sum": 0, "add": 0, "mean": 1, "max": 2, "min": 3}
DTYPE_CODES = {torch.float32: DVA_F32, torch.bfloat16: DVA_BF16, torch.float16: DVA_F16}

_vp, _i64, _i32, _f32, _f64, _sz = (ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float,
                                    ctypes.c_double, ctypes.c_size_t)

# name -> (restype, argtypes); mirrors include/dva_b200.h one to one
SIGNATURES = {
    "dva_abi_version": (_i32, []),
    "dva_last_error": (ctypes.c_char_p, []),
    "dva_launch_count": (_i64, []),
    "dva_segment_csr_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp]),
    "dva_segment_csr_bwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp]),
    "dva_gather_csr": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp]),
    "dva_segment_softmax_csr_fwd": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _f32, _i32, _i32, _vp]),
    "dva_segment_softmax_csr_bwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp]),
    "dva_view_attention_fwd": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                      _i64, _i64, _i64, _i64, _i64, _i32, _f32, _i32, _vp]),
    "dva_view_attention_set_path": (_i32, [_i32]),
    "dva_view_attention_bwd_workspace_bytes": (_sz, [_i64]),
    "dva_view_attention_bwd": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                      _vp, _vp, _i32, _i64, _i64, _i64, _i64, _i64, _i32, _i32,
                                      _vp, _sz, _vp]),
    "dva_qk_scores_fwd": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _f32, _vp]),
    "dva_qk_scores_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _f32, _vp]),
    "dva_heuristic_pool_fwd": (_i32, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _i64, _i64, _i64, _i32,
                                      _i32, _vp]),
    "dva_gather_pool_fwd": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                   _i64, _i64, _i32, _i32, _vp]),
    "dva_gather_pool_bwd": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                   _i64, _i64, _i32, _i32, _vp]),
    "dva_interp_pool_fwd": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                   _i64, _i64, _i64, _i64, _i32, _i32, _vp]),
    "dva_interp_pool_bwd": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                   _i64, _i64, _i64, _i64, _i32, _i32, _vp]),
    "dva_gather_pool_bwd_det_workspace_bytes": (_sz, [_i64, _i64, _i64, _i64]),
    "dva_gather_pool_bwd_det": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                       _i64, _i64, _i32, _i32, _vp, _sz, _vp]),
    "dva_interp_pool_bwd_det_workspace_bytes": (_sz, [_i64, _i64, _i64, _i64]),
    "dva_interp_pool_bwd_det": (_i32, [_vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                       _i64, _i64, _i64, _i64, _i32, _i32, _vp, _sz, _vp]),
    "dva_transpose_last2": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _vp]),
    "dva_knn_cell_ids": (_i32, [_vp, _vp, _i64, _f32, _f32, _f32, _f32, _i32, _i32, _i32, _vp]),
    "dva_knn_grid": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _f32, _f32, _f32, _f32, _i32, _i32, _i32,
                            _vp, _vp, _vp]),
    "dva_knn_query": (_i32, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _i32, _f32, _f32, _f32, _f32, _i32,
                             _i32, _i32, _vp, _vp, _vp]),
    "dva_neighborhood_features": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _f64, _i32, _i32, _vp,
                                         _i64, _i64, _vp]),
    "dva_scatter_add_rows": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp]),
    "dva_scatter_add_rows_det_workspace_bytes": (_sz, [_i64, _i64]),
    "dva_scatter_add_rows_det": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _sz, _vp]),
    "dva_mapping_build_workspace_bytes": (_sz, [_i64, _i64]),
    "dva_mapping_build": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                 _vp, _vp, _sz, _vp]),
    "dva_view_cat_sorting": (_i32, [_vp, _vp, _i64, _i64, _vp, _vp, _vp]),
    "dva_linear_gemm_skinny": (_i32, [_i64, _i64, _i64, _i32]),
    "dva_linear_gemm_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32]),
    "dva_linear_gemm": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp, _sz, _vp]),
    "dva_linear_bnstats_supported": (_i32, [_i64, _i64, _i64]),
    "dva_linear_bnstats_workspace_bytes": (_sz, [_i64, _i64]),
    "dva_linear_bnstats_fwd": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _f32, _f32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dva_bn_workspace_bytes": (_sz, [_i64, _i64]),
    "dva_bn_act_fwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _f32, _f32, _i32, _i32,
                              _vp, _sz, _vp]),
    "dva_bn_act_bwd": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _f32, _i32, _i32, _vp, _sz,
                              _vp]),
    "dva_mlp_layer_bwd_supported": (_i32, [_i64, _i64, _i64]),
    "dva_mlp_layer_bwd_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "dva_mlp_layer_bwd": (_i32, [_vp] * 11 + [_i64, _i64, _i64, _f32, _vp, _sz, _vp]),
    "dva_zbuffer_splat": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64,
                                 _i32, _vp]),
    "dva_splat_boxes": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _f64, _f64, _f64,
                               _i32, _f64, _f64, _vp]),
    "dva_splat_boxes_from_width": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _vp]),
    "dva_project_equirectangular": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64,
                                           _i64, _f32, _f32, _vp]),
    "dva_project_camera": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _f32,
                                  _f32, _vp]),
    "dva_mapping_image_stats": (_i32, [_vp, _vp, _vp, _i32, _i64, _i64, _i64, _vp, _vp, _vp, _vp]),
    "dva_center_roll": (_i32, [_vp, _i64, _i32, _i64, _vp, _vp]),
    "dva_image_remap": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _i32, _vp]),
    "dva_coverage_index_workspace_bytes": (_sz, [_i64, _i64, _i64]),
    "dva_coverage_index": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _sz, _vp]),
    "dva_coverage_pick": (_i32, [_i64, _i64, _i64, _i64, _vp, _vp, _vp, _sz, _vp]),
    "dva_resample_u8": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _i64, _i64, _vp, _vp, _i64, _i32, _vp,
                                _vp, _i64, _i32, _vp, _vp]),
    "dva_nonstatic_mask": (_i32, [_vp, _i64, _i64, _i64, _i64, _vp, _vp]),
    "dva_color_jitter_u8_workspace_bytes": (_sz, [_i64]),
    "dva_color_jitter_u8": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _f32, _f32, _f32, _f32, _f32, _f32,
                                   _vp, _sz, _vp]),
    "dva_image_to_float": (_i32, [_vp, _i32, _vp, _i64, _i64, _i64, _i64, _i32] + [_f32] * 8 + [_vp]),
    "dva_csr_nll_fwd_workspace_bytes": (_sz, [_i64]),
    "dva_csr_nll_fwd": (_i32, [_vp, _i32, _vp, _vp, _i64, _i64, _i32, _i64, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dva_csr_nll_bwd": (_i32, [_vp, _i32, _vp, _vp, _i64, _i64, _i32, _i64, _vp, _vp, _vp, _vp, _vp]),
    "dva_csr_nll_weighted_fwd_workspace_bytes": (_sz, [_i64]),
    "dva_csr_nll_weighted_fwd": (_i32, [_vp, _i32, _vp, _vp, _i64, _i64, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _sz,
                                        _vp]),
    "dva_csr_nll_weighted_bwd": (_i32, [_vp, _i32, _vp, _vp, _i64, _i64, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dva_lovasz_keys": (_i32, [_vp, _i32, _i32, _vp, _i64, _i32, _i64, _vp, _vp]),
    "dva_lovasz_fwd_workspace_bytes": (_sz, [_i64, _i32]),
    "dva_lovasz_fwd": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dva_lovasz_bwd": (_i32, [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp]),
    "dva_csr_pointers_from_sorted":(_i32, [_vp, _vp, _i64, _i64, _vp]),
    "dva_csr_select_values": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _vp]),
}

# name -> (restype, argtypes); mirrors include/dva_eval.h one to one
EVAL_SIGNATURES = {
    "dva_eval_confusion_scores": (_i32, [_vp, _i32, _vp, _vp, _i64, _i32, _i64, _i32, _vp, _vp, _vp]),
    "dva_eval_confusion_pred": (_i32, [_vp, _vp, _i64, _i32, _i64, _i32, _vp, _vp, _vp]),
    "dva_eval_vote": (_i32, [_vp, _i32, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "dva_eval_nn_vote": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp, _i64, _vp, _vp, _i64, _i32, _vp, _i64, _i32, _vp,
                                _vp, _vp, _vp]),
}
# status bits of the evaluation kernels (include/dva_eval.h)
DVA_EVAL_BAD_LABEL, DVA_EVAL_BAD_PRED, DVA_EVAL_BAD_ID = 1, 2, 4

# name -> (restype, argtypes); mirrors include/dva_conv2d.h one to one
CONV_SIGNATURES = {
    "dva_conv2d_weight_prep": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "dva_conv2d_weight_prep_bwd": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "dva_conv2d_fwd_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32]),
    "dva_conv2d_fwd": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _sz,
                              _vp]),
    "dva_conv2d_dgrad": (_i32, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _i32, _vp, _vp, _vp]),
    "dva_conv2d_wgrad_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32, _i32]),
    "dva_conv2d_wgrad": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "dva_conv2d_gn_apply": (_i32, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _vp, _vp,
                                   _vp, _vp, _vp]),
    "dva_conv2d_gn_bwd_workspace_bytes": (_sz, [_i64, _i64, _i32, _i32]),
    "dva_conv2d_gn_bwd": (_i32, [_vp, _vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _vp, _sz,
                                 _vp]),
}
# convolution kinds (include/dva_conv2d.h)
DVA_CONV_3X3_REFLECT, DVA_CONV_2X2_S2, DVA_CONV_1X1 = 0, 1, 2

# name -> (restype, argtypes); mirrors include/dva_unet.h one to one
UNET_SIGNATURES = {
    "dva_unet_weight_prep": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "dva_unet_weight_prep_bwd": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "dva_unet_fwd_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32, _i32]),
    "dva_unet_fwd": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _sz,
                            _vp]),
    "dva_unet_dgrad": (_i32, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _i32, _vp, _vp, _vp]),
    "dva_unet_wgrad_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32, _i32]),
    "dva_unet_wgrad": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "dva_unet_act": (_i32, [_vp, _i64, _f32, _vp, _vp]),
    "dva_unet_act_bwd": (_i32, [_vp, _vp, _i64, _f32, _vp, _vp]),
}
# transposed convolution kinds (include/dva_unet.h)
DVA_UNET_UP_2X2, DVA_UNET_T_3X3 = 0, 1

# name -> (restype, argtypes); mirrors include/dva_resnet.h one to one
RESNET_SIGNATURES = {
    "dva_resnet_weight_prep": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "dva_resnet_fwd_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32]),
    "dva_resnet_conv_bn_fwd": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _f32, _f32, _vp,
                                      _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dva_resnet_conv_dgrad": (_i32, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "dva_resnet_wgrad_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32]),
    "dva_resnet_conv_wgrad": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _sz, _vp]),
    "dva_resnet_bn_apply": (_i32, [_vp, _i64, _i32] + [_vp] * 11 + [_vp]),
    "dva_resnet_bn_bwd_workspace_bytes": (_sz, [_i64, _i32]),
    "dva_resnet_bn_bwd": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dva_resnet_conv_bn_fwd_sums": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp,
                                           _sz, _vp]),
    "dva_resnet_bn_sync_stats": (_i32, [_vp, _i32, _i64, _f32, _f32, _vp, _vp, _vp, _vp, _vp]),
    "dva_resnet_bn_bwd_sums": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "dva_resnet_bn_sync_bwd": (_i32, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "dva_resnet_maxpool": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _vp, _vp]),
    "dva_resnet_maxpool_bwd": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _vp, _vp]),
    "dva_resnet_maxpool_pad": (_i32, [_vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp, _vp]),
    "dva_resnet_maxpool_pad_bwd": (_i32, [_vp, _vp, _i64, _i64, _i64, _i32, _i32, _vp, _vp]),
    "dva_resnet_resize": (_i32, [_vp, _i64, _i64, _i64, _i32, _i64, _i64, _f32, _f32, _vp, _i64, _i64, _vp]),
    "dva_resnet_resize_bwd": (_i32, [_vp, _i64, _i64, _i64, _i64, _i64, _i32, _i64, _i64, _f32, _f32, _vp, _vp]),
}


@dataclasses.dataclass(frozen=True, eq=False)
class Library:
    """One shared library of the package (see the module docstring)."""
    file: str
    signatures: dict
    header: str
    namespace: str
    linked: bool = True

    @property
    def path(self):
        """The package's copy of a linked library; LIB_PATH (DVA_B200_LIB if set) for libdva_b200.so."""
        return os.path.join(_HERE, self.file) if self.linked else LIB_PATH


B200 = Library("libdva_b200.so", SIGNATURES, "dva_b200.h", "dva::", linked=False)
EVAL = Library("libdva_eval.so", EVAL_SIGNATURES, "dva_eval.h", "dva_eval::")
CONV = Library("libdva_conv2d.so", CONV_SIGNATURES, "dva_conv2d.h", "dva_conv2d::")
UNET = Library("libdva_unet.so", UNET_SIGNATURES, "dva_unet.h", "dva_unet::")
RESNET = Library("libdva_resnet.so", RESNET_SIGNATURES, "dva_resnet.h", "dva_resnet::")
LIBRARIES = (B200, EVAL, CONV, UNET, RESNET)

EVAL_LIB_PATH, CONV_LIB_PATH, UNET_LIB_PATH, RESNET_LIB_PATH = EVAL.path, CONV.path, UNET.path, RESNET.path

_LIBRARY_OF_ENTRY = {name: rec for rec in LIBRARIES for name in rec.signatures}
if len(_LIBRARY_OF_ENTRY) != sum(len(rec.signatures) for rec in LIBRARIES):
    raise RuntimeError("an entry point is declared by two libraries")
_loaded = {}      # file -> ctypes.CDLL, each library loaded once per process


def build(verbose=False):
    """Compile the libraries for sm_90a (nvcc cross-compiles without a GPU)."""
    out = subprocess.run(["make", "-C", CSRC_DIR, "-j8"], capture_output=True, text=True)
    if verbose or out.returncode != 0:
        print(out.stdout[-4000:])
        print(out.stderr[-4000:])
    if out.returncode != 0:
        raise RuntimeError("building libdva_b200.so failed")
    return LIB_PATH


def load_library(rec):
    """Load `rec` (once) and declare its entry points' signatures; a linked library loads libdva_b200.so first.
    Raises if it has not been built -- no CPU fallback."""
    lib = _loaded.get(rec.file)
    if lib is not None:
        return lib
    if rec.linked:
        in_tree = os.path.join(_HERE, B200.file)
        if os.path.realpath(LIB_PATH) != os.path.realpath(in_tree):
            # the library would load a second libdva_b200.so, whose error string and launch counter last_error()
            # and launch_count() do not read
            raise RuntimeError(f"{rec.file} links against {in_tree}; it cannot run beside the variant "
                               f"DVA_B200_LIB={LIB_PATH}")
        load_library(B200)
    if not os.path.exists(rec.path):
        raise RuntimeError(
            f"{rec.path} not found: build it with `python -c 'import __graft_entry__ as g; "
            f"g.build()'` (or `make -C deepviewagg_b200/csrc`). deepviewagg_b200 has no CPU "
            f"fallback.")
    lib = ctypes.CDLL(rec.path)
    for name, (res, args) in rec.signatures.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if not rec.linked and lib.dva_abi_version() != 1:
        raise RuntimeError("libdva_b200.so ABI version mismatch")
    _loaded[rec.file] = lib
    return lib


load = functools.partial(load_library, B200)
load_eval = functools.partial(load_library, EVAL)
load_conv = functools.partial(load_library, CONV)
load_unet = functools.partial(load_library, UNET)
load_resnet = functools.partial(load_library, RESNET)


def entry(name):
    """The entry point `name`, from whichever library declares it."""
    return getattr(load_library(_LIBRARY_OF_ENTRY.get(name, B200)), name)


def last_error():
    return load().dva_last_error().decode()


def launch_count():
    return int(load().dva_launch_count())


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {last_error()}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def launch(name, device, *args):
    """Run the entry point `name` on `device`'s current stream, raising like check().

    Every entry point that launches work takes its stream last; it is appended here.  Tensors are
    passed as their device pointer and None as NULL.  `args` holds every tensor, temporaries made in
    the caller's argument list included, until the call returns: a temporary freed before the call
    would hand its block to the next one, and two arguments would alias."""
    fn = entry(name)
    with torch.cuda.device(device):
        check(fn(*[ptr(a) if isinstance(a, torch.Tensor) else a for a in args], stream_ptr()), name)


def workspace(nbytes, device):
    """Scratch buffer of at least `nbytes` bytes, passed on as (ws, ws.numel()).  Never empty, so its
    pointer is never NULL, which most entry points reject even when they need no scratch."""
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "deepviewagg_b200 operators run on CUDA tensors only (sm_90a kernels, no CPU "
                "fallback); got a tensor on " + str(t.device))


def dtype_code(t):
    try:
        return DTYPE_CODES[t.dtype]
    except KeyError:
        raise TypeError(f"unsupported feature dtype {t.dtype}; expected float32/bfloat16/float16")
