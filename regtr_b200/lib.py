"""ctypes binding of libregtr_b200.so (the C ABI declared in include/regtr_b200.h).

The product path has NO fallback: if the CUDA library is missing or a call fails,
`RegtrLibError` is raised.  torch is imported first so that its libcudart is the one in the process
(the library links the CUDA runtime only -- no cuBLAS or other compute library).
"""
from __future__ import annotations

import ctypes
import os
import re

import torch  # noqa: F401  (loads libcudart first)

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libregtr_b200.so')
HEADER = os.path.join(os.path.dirname(HERE), 'include', 'regtr_b200.h')


class RegtrLibError(RuntimeError):
    pass


_c = ctypes
_P = _c.c_void_p
_I = _c.c_int
_F = _c.c_float
_Z = _c.c_size_t

# name -> (restype, argtypes); mirrors include/regtr_b200.h one to one
SIGNATURES = {
    'regtr_version': (_I, []),
    'regtr_build_info': (_c.c_char_p, []),
    'regtr_grid_subsample_ws_bytes': (_Z, [_I, _I]),
    'regtr_grid_subsample_state_bytes': (_Z, [_I]),
    'regtr_grid_subsample': (_I, [_P, _P, _I, _I, _F, _P, _I, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_grid_subsample_sorted_ws_bytes': (_Z, [_I]),
    'regtr_grid_subsample_sorted': (_I, [_P, _P, _I, _I, _F, _P, _I, _P, _P, _P, _Z, _P]),
    'regtr_cellgrid_bytes': (_Z, [_I]),
    'regtr_cellgrid_ws_bytes': (_Z, [_I]),
    'regtr_cellgrid_state_bytes': (_Z, [_I]),
    'regtr_cellgrid_build': (_I, [_P, _P, _I, _I, _F, _P, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_ball_query': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _P, _P]),
    'regtr_kpconv_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_kpconv_fwd_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'regtr_kpconv_fwd': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _I, _I, _I, _F, _P, _P, _Z, _P]),
    'regtr_kpconv_aggregate': (_I, [_P, _P, _P, _P, _P, _I, _I, _P, _P, _I, _I, _F, _P, _P, _I, _P]),
    'regtr_max_pool': (_I, [_P, _P, _I, _I, _P, _I, _I, _P, _P]),
    'regtr_instnorm_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_instnorm_counter_bytes': (_Z, [_I, _I]),
    'regtr_instnorm_act': (_I, [_P, _P, _I, _I, _I, _F, _P, _F, _P, _P, _P, _Z, _P, _P]),
    'regtr_instnorm_apply': (_I, [_P, _P, _I, _I, _I, _P, _P, _F, _P, _P, _P]),
    'regtr_instnorm_part_bytes': (_Z, [_I, _I]),
    'regtr_gemm_tf32x3_instats': (_I, [_P, _I, _P, _P, _I, _P, _I, _I, _I, _I, _P, _P, _I, _F, _P, _P, _P, _Z, _P]),
    'regtr_split_tf32': (_I, [_P, _c.c_longlong, _P, _P, _P]),
    'regtr_gemm_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_gemm_tf32x3': (_I, [_P, _I, _P, _P, _I, _P, _I, _P, _P, _I, _I, _I, _I, _P, _I, _P, _Z, _P]),
    'regtr_pos_embed_sine': (_I, [_P, _I, _P, _I, _I, _F, _P, _P]),
    'regtr_layernorm_pos': (_I, [_P, _P, _P, _P, _P, _I, _P, _P, _I, _F, _P, _P, _P, _P, _P]),
    'regtr_attention_plan': (_I, [_P, _I, _P, _P]),
    'regtr_corr_decode_fwd': (_I, [_P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    'regtr_mha_varlen_fwd': (_I, [_P, _I, _P, _I, _P, _I, _P, _I, _P, _P, _P, _P, _P, _I, _I, _P, _I, _I, _I, _F,
                                  _P, _P]),
    'regtr_gemm_tf32x3_qkv_bf16': (_I, [_P, _I, _P, _P, _I, _P, _I, _I, _I, _I, _P, _I, _P, _I, _P, _P]),
    'regtr_mha_bf16_tc_fwd': (_I, [_P, _I, _P, _I, _I, _P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P]),
    'regtr_gemm_tf32x3_qkv_split': (_I, [_P, _I, _P, _P, _I, _P, _I, _I, _I, _I, _F, _P, _I, _P, _I, _P, _P]),
    'regtr_mha_tf32_tc_fwd': (_I, [_P, _I, _P, _I, _I, _P, _I, _P, _P, _P, _P, _I, _I, _P, _I, _I, _I, _P]),
    'regtr_mha_probs_avg': (_I, [_P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P]),
    'regtr_mha_varlen_bwd_ws_bytes': (_Z, [_I, _I]),
    'regtr_mha_varlen_bwd': (_I, [_P, _I, _P, _I, _P, _I, _P, _I, _P, _I, _P, _P, _I, _P, _I, _P, _I,
                                  _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P, _P, _Z, _P]),
    'regtr_layernorm_bwd_ws_bytes': (_Z, [_I, _I]),
    'regtr_layernorm_bwd': (_I, [_P, _P, _P, _P, _P, _I, _P, _I, _F, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'regtr_relu_bwd': (_I, [_P, _P, _c.c_longlong, _F, _P, _P]),
    'regtr_linear_wgrad_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_linear_wgrad': (_I, [_P, _I, _P, _I, _I, _I, _I, _P, _P, _P, _Z, _P]),
    'regtr_neighbor_csr_ws_bytes': (_Z, [_I]),
    'regtr_neighbor_csr': (_I, [_P, _I, _I, _I, _P, _P, _P, _Z, _P]),
    'regtr_kpconv_bwd_input_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_kpconv_bwd_input': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P, _Z, _P]),
    'regtr_max_pool_bwd_ws_bytes': (_Z, [_I, _I]),
    'regtr_max_pool_bwd': (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _Z, _P]),
    'regtr_instnorm_bwd_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_instnorm_bwd': (_I, [_P, _P, _P, _P, _I, _I, _I, _F, _F, _P, _P, _P, _Z, _P]),
    'regtr_grad_norm_ws_bytes': (_Z, [_I]),
    'regtr_grad_norm': (_I, [_P, _I, _I, _F, _P, _P, _Z, _P]),
    'regtr_grad_scale': (_I, [_P, _I, _I, _P, _P]),
    'regtr_bucket_copy': (_I, [_P, _I, _I, _P, _I, _P]),
    'regtr_adam_step': (_I, [_P, _I, _I, _P]),
    'regtr_split_refresh': (_I, [_P, _I, _I, _P]),
    'regtr_kabsch_fwd': (_I, [_P, _P, _P, _P, _I, _P, _P]),
    'regtr_pose_from_corr': (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _P]),
    'regtr_overlap_coord_bound': (_c.c_double, [_c.c_double, _F]),
    'regtr_overlap_ws_bytes': (_Z, [_I]),
    'regtr_overlap_state_bytes': (_Z, [_I]),
    'regtr_overlap_nn': (_I, [_P, _P, _I, _I, _P, _c.c_double, _F, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_registration_fit': (_I, [_P, _P, _I, _I, _P, _c.c_double, _P, _P, _P, _P]),
    'regtr_registration_information': (_I, [_P, _P, _I, _I, _P, _c.c_double, _P, _P, _P, _P]),
    'regtr_transform_clouds': (_I, [_P, _P, _I, _I, _P, _P, _P]),
    'regtr_pose_graph_ws_bytes': (_Z, [_I, _I, _I, _c.c_longlong]),
    'regtr_pose_graph_optimize': (_I, [_P, _P, _I, _I, _I, _I, _c.c_longlong, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                       _P, _Z, _P]),
    'regtr_icp_ws_bytes': (_Z, [_I, _I]),
    'regtr_icp_state_bytes': (_Z, [_I]),
    'regtr_icp': (_I, [_P, _P, _I, _I, _P, _c.c_double, _F, _I, _c.c_double, _c.c_double, _P, _P, _P, _P, _P, _P,
                       _P, _Z, _P, _Z, _P]),
    'regtr_ransac_ws_bytes': (_Z, [_I, _I, _I, _I, _I]),
    'regtr_ransac': (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _I, _c.c_double, _F, _P, _P, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_fgr_ws_bytes': (_Z, [_I, _I, _I]),
    'regtr_fgr': (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _I, _P, _P, _P, _P, _Z, _P]),
    'regtr_estimate_normals_ws_bytes': (_Z, [_I]),
    'regtr_estimate_normals_state_bytes': (_Z, [_I]),
    'regtr_estimate_normals': (_I, [_P, _P, _I, _I, _c.c_double, _F, _I, _P, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_color_gradients_ws_bytes': (_Z, [_I]),
    'regtr_color_gradients_state_bytes': (_Z, [_I]),
    'regtr_color_gradients': (_I, [_P, _P, _P, _P, _I, _I, _c.c_double, _F, _I, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_fpfh_ws_bytes': (_Z, [_I, _I]),
    'regtr_fpfh_state_bytes': (_Z, [_I]),
    'regtr_fpfh': (_I, [_P, _P, _P, _I, _I, _c.c_double, _F, _I, _P, _P, _P, _P, _Z, _P, _Z, _P]),
    'regtr_feature_match_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'regtr_feature_match': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _Z, _P]),
    'regtr_train_augment_ws_bytes': (_Z, [_I, _I]),
    'regtr_train_augment_state_bytes': (_Z, [_I]),
    'regtr_train_augment': (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _c.c_ulonglong, _c.c_ulonglong, _I, _c.c_double,
                                 _I, _P, _I, _P, _P, _P, _P, _I, _P, _P, _Z, _P, _Z, _P]),
    'regtr_meter_update': (_I, [_P, _P]),
    'regtr_pose_errors': (_I, [_P, _P]),
    'regtr_modelnet_augment': (_I, [_P, _I, _P]),
    'regtr_overlap_pyramid': (_I, [_P, _P]),
    'regtr_sym_weight': (_I, [_P, _P, _P, _P]),
    'regtr_sym_weight_bwd': (_I, [_P, _P, _P]),
    'regtr_loss_ws_bytes': (_Z, [_I, _I]),
    'regtr_loss_pointwise': (_I, [_P, _P, _P]),
    'regtr_loss_pointwise_bwd': (_I, [_P, _P]),
    'regtr_infonce_match': (_I, [_P, _P]),
    'regtr_infonce_fwd': (_I, [_P, _P]),
    'regtr_infonce_bwd': (_I, [_P, _P, _P]),
    'regtr_loss_finalize': (_I, [_P, _P, _P]),
    'regtr_loss_norms': (_I, [_P, _P, _P]),
    'regtr_circle_match': (_I, [_P, _P, _P]),
    'regtr_circle_fwd': (_I, [_P, _P, _P]),
    'regtr_circle_finalize': (_I, [_P, _P, _P, _P]),
    'regtr_circle_bwd': (_I, [_P, _P, _P, _P]),
    'regtr_dropout_keep_mask': (_I, [_P, _I, _I, _I, _I, _P, _P]),
    'regtr_dropout_rows': (_I, [_P, _I, _I, _P, _I, _P, _P]),
    'regtr_status_clear': (_I, [_P, _P]),
}

_ERR = {-1: 'REGTR_ERR_ARG (rejected argument)', -2: 'REGTR_ERR_WORKSPACE (workspace too small)',
        -3: 'REGTR_ERR_UNSUPPORTED (shape outside the hot path)'}

_lib = None


def header_symbols():
    """Every function name declared in include/regtr_b200.h."""
    text = open(HEADER).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(regtr_[a-z0-9_]+)\s*\(', text)))


def load():
    """Load (building first if the .so is absent and nvcc exists).  Raises RegtrLibError."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        try:
            from . import build as _build
            _build.build()
        except Exception as exc:
            raise RegtrLibError(f'{LIB_PATH} is missing and could not be built: {exc}') from exc
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as exc:
        raise RegtrLibError(f'cannot load {LIB_PATH}: {exc}') from exc
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as exc:
            raise RegtrLibError(f'{LIB_PATH} does not export {name}') from exc
        fn.restype = res
        fn.argtypes = args
    if lib.regtr_version() != 1:
        raise RegtrLibError('ABI version mismatch')
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc == 0:
        return
    if rc <= -1000:
        raise RegtrLibError(f'{what}: CUDA error {-rc - 1000} at launch')
    raise RegtrLibError(f'{what}: {_ERR.get(rc, rc)}')
