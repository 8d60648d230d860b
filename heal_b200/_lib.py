"""ctypes loader for the C-ABI library.  The product path has NO fallback: if libheal_b200.so is
missing or fails to load, importing this module raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libheal_b200.so")

_c = ctypes
_vp, _i, _sz = _c.c_void_p, _c.c_int, _c.c_size_t


class HealAct(ctypes.Structure):
    """heal_act_t of include/heal_b200.h"""
    _fields_ = [("data", _vp), ("fmt", _i), ("cstride", _i), ("coffset", _i), ("plane_stride", _sz)]


_ap = ctypes.POINTER(HealAct)


class HealStackSource(ctypes.Structure):
    """heal_stack_source_t of include/heal_b200.h"""
    _fields_ = [("map", HealAct), ("images", _i), ("height", _i), ("width", _i), ("center_crop", _i)]


class HealCavHeads(ctypes.Structure):
    """heal_cav_heads_t of include/heal_b200.h"""
    _fields_ = [("cls", _ap), ("reg", _ap), ("dir", _ap), ("iou", _ap), ("anchors", _vp), ("transform4x4_host", ctypes.POINTER(ctypes.c_float))]

# name -> (restype, argtypes); must list every symbol include/heal_b200.h declares
SIGNATURES = {
    "heal_abi_version": (_i, []),
    "heal_device_check": (_i, []),
    "heal_launch_count": (_c.c_longlong, []),
    "heal_voxelize_workspace": (_sz, [_i, _i, _i]),
    "heal_voxelize": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_mask_points_workspace": (_sz, [_i]),
    "heal_mask_points": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "heal_mean_vfe": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "heal_pillar_vfe_scatter": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _ap, _vp]),
    "heal_pillar_scatter": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _ap, _vp]),
    "heal_pillar_idmap": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "heal_sparse_stem": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _ap, _ap, _vp]),
    "heal_sparse_stem_tc": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _ap, _ap, _vp]),
    "heal_conv2d_simt": (_i, [_ap, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _i, _i, _i, _ap, _ap, _i, _i, _i,
                              _i, _i, _i, _i, _vp]),
    "heal_conv2d_tc": (_i, [_vp, _sz, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i,
                            _vp, _sz, _vp, _i, _i, _vp, _sz, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "heal_conv3x3_narrow_tc": (_i, [_ap, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _ap, _vp]),
    "heal_bottleneck_tc": (_i, [_vp, _sz, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _sz, _i, _i, _vp]),
    "heal_gconv_reduce_tc": (_i, [_vp, _sz, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _sz, _i, _i, _i, _vp, _sz, _i, _i,
                                  _vp]),
    "heal_dwconv_layernorm": (_i, [_ap, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _c.c_float, _ap, _vp]),
    "heal_maxpool3x3s2": (_i, [_ap, _i, _i, _i, _i, _i, _ap, _vp]),
    "heal_pyramid_fuse_level": (_i, [_ap, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _ap, _vp]),
    "heal_att_fuse": (_i, [_ap, _vp, _i, _i, _i, _i, _ap, _vp]),
    "heal_max_fuse": (_i, [_ap, _vp, _i, _i, _i, _i, _ap, _vp]),
    "heal_warp_affine": (_i, [_ap, _vp, _vp, _i, _i, _i, _i, _ap, _vp]),
    "heal_v2v_aggregate": (_i, [_ap, _ap, _ap, _vp, _vp, _i, _i, _i, _i, _i, _i, _ap, _vp]),
    "heal_gru_gate": (_i, [_ap, _c.c_longlong, _i, _ap, _vp]),
    "heal_ego_mha": (_i, [_ap, _ap, _vp, _vp, _vp, _i, _i, _i, _i, _i, _ap, _vp]),
    "heal_swap_attention": (_i, [_ap, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _ap, _vp]),
    "heal_mean_layernorm": (_i, [_ap, _i, _i, _i, _i, _i, _vp, _vp, _c.c_float, _ap, _vp]),
    "heal_window_attention": (_i, [_ap, _i, _i, _i, _i, _i, _i, _vp, _ap, _vp]),
    "heal_cav_attention": (_i, [_ap, _vp, _i, _i, _i, _i, _i, _ap, _vp]),
    "heal_split_attn_workspace": (_sz, [_i, _i]),
    "heal_split_attn": (_i, [_ap, _ap, _i, _i, _i, _i, _vp, _vp, _vp, _c.c_float, _vp, _vp, _sz, _ap, _vp]),
    "heal_sttf_resample": (_i, [_ap, _vp, _i, _i, _i, _i, _ap, _vp]),
    "heal_act_convert": (_i, [_ap, _ap, _sz, _i, _vp]),
    "heal_agent_stack": (_i, [ctypes.POINTER(HealStackSource), _i, _vp, _vp, _i, _i, _ap, _i, _i, _vp]),
    "heal_postprocess_workspace": (_sz, [_i, _i, _i, _i]),
    "heal_box_decode_nms": (_i, [_ap, _ap, _ap, _vp, _i, _i, _i, _c.c_float, _c.c_float, _i, _vp, _i, _c.c_float, _i,
                                 _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_box_decode_nms_multi": (_i, [ctypes.POINTER(HealCavHeads), _i, _i, _i, _i, _c.c_float, _c.c_float, _i, _i, _c.c_float, _i,
                                       _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_box_decode_nms_late": (_i, [_ap, _ap, _ap, _vp, _vp, _i, _i, _i, _i, _c.c_float, _c.c_float, _i, _i, _c.c_float, _i,
                                      _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_eval_workspace": (_sz, [_i, _i]),
    "heal_eval_tp_fp": (_i, [_vp, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_eval_tp_fp_counted": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_spconv_table_size": (_sz, [_i]),
    "heal_spconv_build_table": (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "heal_spconv_subm_neighbors": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp]),
    "heal_spconv_strided_workspace": (_sz, [_i, _i, _i]),
    "heal_spconv_strided_rulebook": (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "heal_spconv_gather_gemm": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "heal_spconv_gather_gemm_tc": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _vp, _vp,
                                        _c.c_longlong, _c.c_longlong, _c.c_longlong, _c.c_longlong, _vp]),
    "heal_stem_rulebook": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "heal_rows_to_split": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "heal_sparse_to_bev": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "heal_p2p_push": (_i, [_vp, _vp, _i, _i, _sz, _vp]),
    "heal_p2p_signal_wait": (_i, [_vp, _i, _i, _vp, _vp]),
    "heal_lss_camera_matrices": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "heal_lss_cell_index": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "heal_lss_pool_sorted_workspace": (_sz, [_i, _i, _i, _i, _i, _i]),
    "heal_lss_pool_sorted": (_i, [_vp, _c.c_longlong, _c.c_longlong, _c.c_longlong, _vp, _c.c_longlong, _c.c_longlong, _c.c_longlong,
                                  _vp, _i, _i, _i, _i, _i, _i, _i, _ap, _vp, _sz, _vp]),
    "heal_lss_pool": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "heal_stem_conv_swish": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "heal_dwconv_bn_swish_workspace": (_sz, [_i, _i, _i, _i]),
    "heal_dwconv_bn_swish": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "heal_se_gate": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "heal_pwconv": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "heal_upsample2x_concat": (_i, [_ap, _ap, _i, _i, _i, _i, _i, _ap, _i, _vp]),
    "heal_camera_input": (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
}

ERRORS = {-1: "HEAL_ERR_ARG", -2: "HEAL_ERR_WORKSPACE", -3: "HEAL_ERR_LAUNCH", -4: "HEAL_ERR_UNSUPPORTED",
          -5: "HEAL_ERR_DRIVER"}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -m heal_b200.build` (nvcc, sm_90a). "
            "heal_b200 has no CPU / PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(code: int, what: str):
    if code != 0:
        raise RuntimeError(f"{what} failed: {ERRORS.get(code, code)}")
