"""ctypes binding of ``libesb200.so`` (C ABI declared in ``include/esb200.h``).

The product path fails loudly when the CUDA library is missing: there is no CPU fallback.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libesb200.so')

_CT = {'p': ctypes.c_void_p, 'q': ctypes.c_longlong, 'i': ctypes.c_int, 'f': ctypes.c_float, 'z': ctypes.c_size_t}

# name -> (argument codes, return code).  p=pointer q=long long i=int f=float z=size_t
SIGNATURES = {
    'esb_last_error': ('', 'p'),
    'esb_voxelize_points': ('pqiifpp', 'i'),
    'esb_hash_capacity': ('q', 'q'),
    'esb_coord_unique_workspace_bytes': ('q', 'z'),
    'esb_coord_unique': ('pqippqppppzp', 'i'),
    'esb_hash_build': ('pqppqp', 'i'),
    'esb_hash_lookup': ('pqppqpp', 'i'),
    'esb_interp_features': ('pqppqpiiipp', 'i'),
    'esb_kernel_map': ('pqpippqpp', 'i'),
    'esb_kernel_map_transpose': ('piqqpp', 'i'),
    'esb_kmap_pairs_workspace_bytes': ('iq', 'z'),
    'esb_kmap_pairs': ('piqppppzp', 'i'),
    'esb_generative_children': ('pqipp', 'i'),
    'esb_spconv_fwd': ('ppppqiiiiip', 'i'),
    'esb_spconv_wgrad': ('ppppppqiiiip', 'i'),
    'esb_spconv_wgrad_slot': ('ppppppqiiiip', 'i'),
    'esb_kmap_tile_masks': ('piqpp', 'i'),
    'esb_spconv_tc_fwd': ('pppppqiiiip', 'i'),
    'esb_spconv_tc_wgrad': ('ppppppqiiip', 'i'),
    'esb_spconv_tc_wgrad_slot': ('ppppppqiiip', 'i'),
    'esb_maxpool_fwd': ('ppppqiiip', 'i'),
    'esb_maxpool_bwd': ('pppqiip', 'i'),
    'esb_norm_fwd': ('ppppiqiippfppfipppip', 'i'),
    'esb_batchnorm_fwd_fused': ('ppqippfppfippip', 'i'),
    'esb_norm_apply': ('pppqippppipip', 'i'),
    'esb_norm_bwd': ('pppppiqiipppippppiip', 'i'),
    'esb_bias_act_fwd': ('ppppqiiip', 'i'),
    'esb_act_bwd': ('pppqiip', 'i'),
    'esb_gather2_rows': ('ppqpppqiip', 'i'),
    'esb_conv2d_tma_fwd': ('ppppp' + 'iiiiiiiiii' + 'p', 'i'),
    'esb_conv2d_tma_wgrad': ('ppp' + 'iiiiiiiii' + 'p', 'i'),
    'esb_conv2d_tma_dgrad': ('ppp' + 'iiiiiiiii' + 'p', 'i'),
    'esb_conv3d_tma_fwd': ('ppppp' + 'iiiiiiiiii' + 'p', 'i'),
    'esb_conv3d_tma_dgrad': ('ppp' + 'iiiiiiiii' + 'p', 'i'),
    'esb_conv3d_tma_wgrad': ('ppp' + 'iiiiiiiii' + 'p', 'i'),
    'esb_stem7x7_tc': ('pppp' + 'iiii' + 'p', 'i'),
    'esb_conv2d_direct_fwd': ('ppppp' + 'iiiiiiiiiii' + 'p', 'i'),
    'esb_conv2d_direct_dgrad': ('ppp' + 'iiiiiiiiii' + 'p', 'i'),
    'esb_conv2d_direct_wgrad': ('ppp' + 'iiiiiiiiii' + 'p', 'i'),
    'esb_maxpool2d_nhwc': ('pp' + 'iiiiiiii' + 'p', 'i'),
    'esb_attn_fwd': ('pppppp' + 'iiii' + 'f' + 'p', 'i'),
    'esb_attn_bwd': ('ppppppppppp' + 'iiii' + 'f' + 'p', 'i'),
    'esb_paint_meta_bytes': ('', 'i'),
    'esb_paint_fwd': ('pppqfppipiiiffppip', 'i'),
    'esb_paint_bwd': ('pppqfppipiiiffpip', 'i'),
    'esb_fcaf3d_targets_workspace_bytes': ('iii', 'z'),
    'esb_fcaf3d_targets': ('ppiippppp' + 'iiiii' + 'pppp' + 'pzp', 'i'),
    'esb_focal_loss_fwd': ('ppqiffppip', 'i'),
    'esb_focal_loss_bwd': ('ppqiffpppip', 'i'),
    'esb_bbox_cd_loss': ('ppppp' + 'iiii' + 'ppp', 'i'),
    'esb_chamfer_fwd': ('pp' + 'iiiii' + 'ppppp', 'i'),
    'esb_chamfer_bwd': ('pppppp' + 'iiiii' + 'ppp', 'i'),
    'esb_nms_bev_segmented': ('ppiifipp', 'i'),
    'esb_iou_bev_pairwise': ('pipiipp', 'i'),
    'esb_box3d_overlap': ('pipippp', 'i'),
    'esb_box3d_best_overlap': ('pippppppp', 'i'),
    'esb_rotated_iou3d_fwd': ('pipiqpp', 'i'),
    'esb_rotated_iou3d_bwd': ('pipiqpppp', 'i'),
    'esb_nms3d_9dof_workspace_bytes': ('iii', 'z'),
    'esb_nms3d_9dof': ('pppp' + 'ii' + 'ff' + 'ii' + 'ppp' + 'zp', 'i'),
    'esb_hungarian_batch': ('ppiiippp', 'i'),
    'esb_img_normalize': ('piiiiippiipip', 'i'),
    'esb_img_resize_linear_u8': ('piiiiipp', 'i'),
    'esb_unproject_depth_workspace_bytes': ('iii', 'z'),
    'esb_unproject_depth': ('piiifpppppzp', 'i'),
    'esb_grad_clip_coef': ('pqffpp', 'i'),
    'esb_adamw_step_groups': ('ppppppiqfffifpp', 'i'),
    'esb_cast_f32_to_bf16': ('ppqp', 'i'),
}

_lib = None

# kernels launched per C-ABI call (for bench.py's `gpu_launches`; memsets are not counted)
KERNELS_PER_CALL = {
    'esb_voxelize_points': 1, 'esb_coord_unique': 6, 'esb_hash_build': 2, 'esb_hash_lookup': 1, 'esb_kernel_map': 1,
    'esb_kernel_map_transpose': 2, 'esb_kmap_pairs': 3, 'esb_generative_children': 1, 'esb_spconv_fwd': 1,
    'esb_spconv_wgrad': 1, 'esb_spconv_wgrad_slot': 1, 'esb_maxpool_fwd': 1, 'esb_maxpool_bwd': 1, 'esb_norm_fwd': 5, 'esb_norm_apply': 1,
    'esb_norm_bwd': 2, 'esb_batchnorm_fwd_fused': 2, 'esb_paint_fwd': 1, 'esb_paint_bwd': 1, 'esb_fcaf3d_targets': 5,
    'esb_focal_loss_fwd': 1, 'esb_focal_loss_bwd': 1, 'esb_nms_bev_segmented': 1, 'esb_iou_bev_pairwise': 1,
    'esb_img_normalize': 1, 'esb_unproject_depth': 3, 'esb_grad_clip_coef': 2, 'esb_adamw_step_groups': 1,
    'esb_cast_f32_to_bf16': 1, 'esb_spconv_tc_fwd': 1, 'esb_spconv_tc_wgrad': 1, 'esb_spconv_tc_wgrad_slot': 1,
    'esb_kmap_tile_masks': 1,
    'esb_chamfer_fwd': 2, 'esb_chamfer_bwd': 4, 'esb_nms3d_9dof': 2,
}
launch_counter = {'kernels': 0, 'calls': 0, 'by_name': {}}


def exported_symbols():
    return list(SIGNATURES.keys())


def lib():
    """Load the library (once). Raises if it was not built — never falls back to a CPU path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f'{LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                '(esb200 has no CPU fallback)')
        handle = ctypes.CDLL(LIB_PATH)
        for name, (args, ret) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.argtypes = [_CT[c] for c in args]
            fn.restype = _CT[ret]
        _lib = handle
    return _lib


def last_error():
    p = lib().esb_last_error()
    return ctypes.cast(p, ctypes.c_char_p).value.decode() if p else ''


def ptr(t):
    """Device (or host) pointer of a tensor, None -> NULL."""
    if t is None:
        return None
    return t.data_ptr()


def stream():
    """Raw handle of the current CUDA stream (torch.cuda.current_stream() builds a Stream object per call: ~14 us, 2000
    calls per step)."""
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def call(name, *args):
    launch_counter['calls'] += 1
    launch_counter['kernels'] += KERNELS_PER_CALL.get(name, 1)
    launch_counter['by_name'][name] = launch_counter['by_name'].get(name, 0) + 1
    rc = getattr(lib(), name)(*args)
    if rc != 0:
        raise RuntimeError(f'{name} failed ({rc}): {last_error()}')


def query(name, *args):
    return getattr(lib(), name)(*args)


def dtype_code(dtype):
    if dtype == torch.float32:
        return 0
    if dtype == torch.bfloat16:
        return 1
    raise TypeError(f'esb200 kernels take float32 or bfloat16 features, got {dtype}')
