"""ctypes binding of libsgb200.so (the C ABI declared in include/sgb200.h).

Importing this module never initialises CUDA (DataLoader workers call voxelization_idx on the CPU,
reference softgroup/data/custom.py:239). There is NO fallback: if the library is missing or a call fails,
an exception is raised.
"""
import ctypes
import os
from ctypes import c_double, c_float, c_int, c_longlong, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), 'libsgb200.so')

_P = c_void_p
_INTP = ctypes.POINTER(c_int)

# name -> (restype, argtypes); mirrors include/sgb200.h one to one
SIGNATURES = {
    'sgb_last_error': (ctypes.c_char_p, []),
    'sgb_abi_version': (c_int, []),
    'sgb_device_available': (c_int, []),
    'sgb_launch_count': (c_longlong, []),
    'sgb_voxelize_idx_workspace_bytes': (c_size_t, [c_int]),
    'sgb_voxelize_idx_count': (c_int, [_P, c_int, c_int, c_int, _P, _P, c_size_t, _INTP, _INTP, _P]),
    'sgb_voxelize_idx_fill': (c_int, [_P, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    'sgb_voxelize_idx_cpu_begin': (_P, [_P, c_int, c_int, c_int, _P, _INTP, _INTP]),
    'sgb_voxelize_idx_cpu_finish': (c_int, [_P, _P, _P, _P]),
    'sgb_voxelize_fp': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'sgb_voxelize_bp': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'sgb_ballquery_workspace_bytes': (c_size_t, [c_int]),
    'sgb_ballquery_batch_p': (c_longlong, [c_int, c_int, c_float, _P, _P, _P, c_int, _P, _P, _P, c_size_t, _P]),
    'sgb_ballquery_batch_p_async': (c_int, [c_int, c_longlong, c_float, _P, _P, _P, c_int, _P, _P, _P, _P, c_size_t,
                                            _P]),
    'sgb_octree_workspace_bytes': (c_size_t, [c_int]),
    'sgb_octree_build': (c_int, [_P, c_int, _P, _P, _P, _P, _P, c_size_t, _P]),
    'sgb_octree_ball_query': (c_longlong, [_P, _P, _P, _P, c_int, c_int, c_float, _P, _P, _P, _P]),
    'sgb_bfs_cluster_workspace_bytes': (c_size_t, [c_int]),
    'sgb_bfs_cluster_count': (c_int, [_P, _P, c_int, c_float, _P, _P, _P, _P, c_size_t, _INTP, _INTP, _P]),
    'sgb_bfs_cluster_scratch_bytes': (c_size_t, [c_int, c_int]),
    'sgb_bfs_cluster_fill': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, _P, c_size_t, _P, c_size_t, _P]),
    'sgb_sec_mean': (c_int, [_P, _P, _P, c_int, c_int, _P]),
    'sgb_sec_min': (c_int, [_P, _P, _P, c_int, c_int, _P]),
    'sgb_sec_max': (c_int, [_P, _P, _P, c_int, c_int, _P]),
    'sgb_global_avg_pool_fp': (c_int, [_P, _P, _P, c_int, c_int, _P]),
    'sgb_global_avg_pool_bp': (c_int, [_P, _P, _P, c_int, c_int, _P]),
    'sgb_get_mask_iou': (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, _P]),
    'sgb_get_mask_label': (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_float, _P, _P]),
    'sgb_rulebook_workspace_bytes': (c_size_t, [c_int]),
    'sgb_rulebook_subm3': (c_int, [_P, c_int, _P, _P, c_size_t, _P]),
    'sgb_rulebook_down2_count': (c_int, [_P, c_int, _INTP, _P, c_size_t, _P]),
    'sgb_rulebook_down2_fill': (c_int, [_P, c_int, c_int, _P, _P, _P, _P, c_size_t, _P]),
    'sgb_spconv_forward': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, _P, _P, _P, c_int, c_int, _P,
                                   _P, c_int, c_int, _P]),
    'sgb_spconv_tc_packed_floats': (c_longlong, [c_int, c_int, c_int]),
    'sgb_spconv_lo_shift': (c_int, []),
    'sgb_spconv_overflow': (c_int, [_INTP, _P]),
    'sgb_spconv_tc_plan': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, _INTP]),
    'sgb_act_pack': (c_int, [_P, c_int, c_int, _P, _P, c_int, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'sgb_spconv_forward_tc': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, _P, _P, c_int,
                                      c_int, _P, c_int, c_int, _P, _P, c_int, c_int, _P]),
    'sgb_spconv_forward_tc_ex': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, _P, c_int, c_int, _P, _P, c_int,
                                         c_int, _P, c_int, c_int, _P, _P, c_int, c_int, c_int, _P]),
    'sgb_spconv_kernel_choice': (c_int, [c_int, c_int, c_int, c_int, c_int]),
    'sgb_group_entries_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'sgb_group_entries': (c_int, [_P, c_int, c_int, _INTP, c_int, c_float, c_int, _P, c_int, _P, _P, _P, _P, _P, _P, _P, _P,
                                  c_size_t, _P]),
    'sgb_unet_run': (c_int, [_P, c_int, _P, _P, _P, _P, _P, c_int, _P]),
    'sgb_bn_relu': (c_int, [_P, c_int, _P, _P, c_int, _P, c_int, c_int, c_int, _P]),
    'sgb_gather_rows': (c_int, [_P, _P, _P, c_int, c_int, _P]),
    'sgb_inst_count': (c_int, [_P, _P, c_int, c_int, c_int, c_float, _P, c_int, _P]),
    'sgb_bitmap_words': (c_size_t, [c_int]),
    'sgb_inst_scatter': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_float, _P, _P, c_int, c_int, _P]),
    'sgb_bitmap_set': (c_int, [_P, _P, c_longlong, _P, c_int, c_int, c_int, _P]),
    'sgb_rle_workspace_bytes': (c_size_t, [c_int, c_int]),
    'sgb_rle_count': (c_longlong, [_P, c_int, c_int, _P, c_size_t, _P]),
    'sgb_rle_fill': (c_int, [_P, c_int, c_int, c_int, _P, _P, _P, c_size_t, _P]),
    'sgb_rle_format_runs': (c_longlong, [_P, _P, c_int, _P, c_longlong, _P]),
    'sgb_bitmap_intersections': (c_int, [_P, c_int, c_int, _P, c_int, _P, _P, _P, _P]),
    'sgb_panoptic_paste': (c_int, [_P, c_int, _P, _P, c_int, c_double, _P, _P, _P, _P]),
    'sgb_bitmap_ids_workspace_bytes': (c_size_t, [c_int, c_int]),
    'sgb_bitmap_ids_count': (c_int, [_P, c_int, c_int, _P, _P, c_size_t, _P]),
    'sgb_bitmap_ids_fill': (c_int, [_P, c_int, c_int, _P, _P, c_size_t, _P]),
    'sgb_class_bitmaps': (c_int, [_P, c_int, _P, c_int, _P, c_int, _P, _P]),
    'sgb_id_lists_reduce_workspace_bytes': (c_size_t, [c_longlong, c_int]),
    'sgb_id_lists_reduce': (c_int, [_P, _P, c_int, c_longlong, c_int, _P, c_longlong, c_int, c_int, _P, _P, _P, _P, _P, c_size_t,
                                    _P]),
    'sgb_id_lists_point_map_workspace_bytes': (c_size_t, [c_int]),
    'sgb_id_lists_point_map': (c_int, [_P, _P, c_int, c_longlong, c_int, _P, _P, _P, c_size_t, _P]),
    'sgb_id_lists_fps_workspace_bytes': (c_size_t, [c_int, c_longlong]),
    'sgb_id_lists_fps': (c_int, [_P, _P, c_int, c_longlong, c_int, _P, c_longlong, c_int, _P, _P, c_size_t, _P]),
    'sgb_affine3_f64': (c_int, [_P, _P, _P, c_int, _P]),
    'sgb_rle_format_ids': (c_longlong, [_P, _P, c_int, _P, c_longlong, _P]),
}

_lib = None


class SgbError(RuntimeError):
    pass


def lib():
    """Load libsgb200.so; raises if it has not been built (python softgroup_b200/build.py)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SgbError('libsgb200.so not found at %s -- build it with `python -m softgroup_b200.build` '
                           '(there is no CPU/PyTorch fallback)' % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc, what=''):
    """Raise on a negative status; returns rc otherwise."""
    if rc is None:
        raise SgbError('%s returned NULL: %s' % (what, lib().sgb_last_error().decode()))
    if rc < 0:
        raise SgbError('%s failed (%d): %s' % (what, rc, lib().sgb_last_error().decode()))
    return rc


def ptr(t):
    """Device/host pointer of a tensor (None -> NULL)."""
    return None if t is None else c_void_p(t.data_ptr())


def stream():
    """Handle of torch's current CUDA stream, the `stream` argument of every entry point."""
    # the raw-handle call avoids ~10 us of Python per launch
    try:
        return c_void_p(torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice()))
    except Exception:  # older torch: public (slower) path
        return c_void_p(torch.cuda.current_stream().cuda_stream)


def workspace(nbytes, device):
    """Uninitialised device scratch of `nbytes` bytes (the `d_ws` / `d_scratch` arguments)."""
    return torch.empty(int(nbytes), dtype=torch.uint8, device=device)
