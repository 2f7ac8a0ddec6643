"""
ctypes binding of libneurite_b200.so (the C ABI declared in include/neurite_b200.h).

There is no CPU fallback: if the shared library is missing, importing this module raises;
if a tensor is not on a CUDA device, the op wrappers raise.  PyTorch is only the device
allocator / stream provider -- tensors cross the boundary as raw pointers.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libneurite_b200.so')

c_i32, c_i64, c_f32, c_vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p
c_u64 = ctypes.c_uint64
P_I32 = ctypes.POINTER(ctypes.c_int32)

# name -> (restype, argtypes); mirrors include/neurite_b200.h one to one
SIGNATURES = {
    'nrt_version': (ctypes.c_int, []),
    'nrt_last_error_string': (ctypes.c_char_p, []),
    'nrt_status_string': (ctypes.c_char_p, [ctypes.c_int]),
    'nrt_interpn_f32': (ctypes.c_int, [c_vp, P_I32, ctypes.c_int, ctypes.c_int, c_vp, c_i64, ctypes.c_int,
                                        ctypes.c_int, c_f32, c_vp, c_vp]),
    'nrt_interpn_grid_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, P_I32, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_f32,
                                             ctypes.c_int, c_vp]),
    'nrt_warp_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, ctypes.c_int, P_I32, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_int, c_f32, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp, c_vp]),
    'nrt_warp_strided_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, ctypes.c_int, P_I32, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int, c_f32, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp, c_i64, c_i64, c_i64, c_vp]),
    'nrt_resize_f32': (ctypes.c_int, [c_vp, c_vp, ctypes.c_int, P_I32, P_I32, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_int, c_vp]),
    'nrt_dice_workspace_bytes': (c_i64, [ctypes.c_int, ctypes.c_int]),
    'nrt_dice_sums_f32': (ctypes.c_int, [c_vp, c_vp, ctypes.c_int, c_i64, ctypes.c_int, c_i64, c_i64,
                                          ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, c_i64, c_vp]),
    'nrt_dice_label_sums_i32': (ctypes.c_int, [c_vp, c_vp, ctypes.c_int, c_i64, ctypes.c_int, c_i64, c_i64,
                                                c_vp, c_vp, c_i64, c_vp]),
    'nrt_argmax_f32': (ctypes.c_int, [c_vp, c_i64, ctypes.c_int, c_vp, c_vp]),
    'nrt_dice_finalize_f32': (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_f32, c_vp, c_vp]),
    'nrt_cce_workspace_bytes': (c_i64, []),
    'nrt_cce_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.c_int, ctypes.c_int, c_f32,
                                    c_vp, c_vp, c_vp, c_i64, c_vp]),
    'nrt_warp_bwd_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_int, P_I32, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_int, ctypes.c_int, c_vp]),
    'nrt_interpn_bwd_f32': (ctypes.c_int, [c_vp, P_I32, ctypes.c_int, ctypes.c_int, c_vp, c_i64, ctypes.c_int,
                                            ctypes.c_int, c_vp, c_vp, c_vp, c_vp]),
    'nrt_resize_bwd_f32': (ctypes.c_int, [c_vp, c_vp, ctypes.c_int, P_I32, P_I32, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, c_vp]),
    'nrt_dice_bwd_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, ctypes.c_int, c_i64, ctypes.c_int, c_f32,
                                         c_vp, c_vp, c_vp]),
    'nrt_cce_bwd_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, ctypes.c_int, ctypes.c_int, c_f32,
                                        c_vp, c_f32, c_vp, c_vp, c_vp]),
    'nrt_lc3d_fwd_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, ctypes.c_int, P_I32, ctypes.c_int,
                                         ctypes.c_int, P_I32, P_I32, ctypes.c_int, ctypes.c_int,
                                         c_i64, c_i64, c_vp]),
    'nrt_lc3d_bwd_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_int, P_I32, ctypes.c_int,
                                         ctypes.c_int, P_I32, P_I32, ctypes.c_int, c_i64, c_i64, c_vp]),
    'nrt_mi_workspace_bytes': (c_i64, [ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    'nrt_mi_hist_f32': (ctypes.c_int, [c_vp, c_i64, c_i64, ctypes.c_int, ctypes.c_int, c_vp,
                                        c_vp, c_i64, c_i64, ctypes.c_int, ctypes.c_int, c_vp,
                                        ctypes.c_int, ctypes.c_int, c_i64, c_f32, c_f32, c_f32,
                                        c_vp, c_vp, c_vp, c_i64, c_vp]),
    'nrt_mi_finalize_f32': (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_f32, c_vp, c_vp]),
    'nrt_mi_finalize_bwd_f32': (ctypes.c_int, [c_vp, c_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_f32, c_vp, c_vp]),
    'nrt_mi_bwd_workspace_bytes': (c_i64, [ctypes.c_int]),
    'nrt_mi_bwd_f32': (ctypes.c_int, [c_vp, c_i64, c_i64, ctypes.c_int, ctypes.c_int, c_vp,
                                       c_vp, c_i64, c_i64, ctypes.c_int, ctypes.c_int, c_vp,
                                       ctypes.c_int, ctypes.c_int, c_i64, c_f32, c_f32, c_f32,
                                       c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    'nrt_mi_minmax_bwd_f32': (ctypes.c_int, [c_vp, c_i64, c_vp, c_vp, ctypes.c_int, c_vp, c_vp]),
    'nrt_mi_bin_centers_f32': (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp]),
    'nrt_soft_quantize_f32': (ctypes.c_int, [c_vp, c_i64, c_vp, ctypes.c_int, c_f32, c_f32, c_f32,
                                              ctypes.c_int, c_vp, c_vp]),
    'nrt_sepconv_axis_f32': (ctypes.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int, c_i64, c_vp]),
    'nrt_gather_axis_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp]),
    'nrt_philox_uniform_f32': (ctypes.c_int, [c_u64, c_i64, c_f32, c_f32, c_vp, c_vp]),
    'nrt_philox_normal_f32': (ctypes.c_int, [c_u64, P_I32, P_I32, ctypes.c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    'nrt_item_stats_workspace_bytes': (c_i64, [ctypes.c_int, c_i64]),
    'nrt_item_stats_f32': (ctypes.c_int, [c_vp, ctypes.c_int, c_i64, ctypes.c_int, c_vp, c_vp, c_i64, c_vp]),
    'nrt_level_combine_f32': (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_i64, c_vp, c_vp, c_vp, c_vp]),
    'nrt_philox_normal_background_f32': (ctypes.c_int, [c_u64, ctypes.c_int, c_i64, ctypes.c_int, c_vp, c_vp, c_vp,
                                                         c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_f32, c_vp, c_vp]),
    'nrt_labels_to_image_workspace_bytes': (c_i64, []),
    'nrt_labels_to_image_f32': (ctypes.c_int, [c_vp, ctypes.c_int, c_i64, ctypes.c_int, c_i64, c_i64, c_i64, c_i64,
                                                c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, c_vp, ctypes.c_int,
                                                c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    'nrt_norm_gamma_f32': (ctypes.c_int, [c_vp, ctypes.c_int, c_i64, ctypes.c_int, c_vp, c_vp, c_f32, c_f32, c_vp,
                                           c_vp]),
    'nrt_label_map_f32': (ctypes.c_int, [c_vp, ctypes.c_int, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, ctypes.c_int,
                                          ctypes.c_int, c_vp, c_vp]),
    'nrt_label_map_i32': (ctypes.c_int, [c_vp, ctypes.c_int, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, ctypes.c_int,
                                          c_vp, c_vp]),
    'nrt_crop_window_f32': (ctypes.c_int, [c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp]),
    'nrt_crop_window_i32': (ctypes.c_int, [c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp]),
    'nrt_warp_labels_affine_f32': (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, ctypes.c_int, ctypes.c_int, P_I32, P_I32,
                                                   c_vp]),
}


class NeuriteB200Error(RuntimeError):
    """A C-ABI call returned a non-zero status."""


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            'neurite_b200: %s is missing -- build it with `python -c "import __graft_entry__ as g; g.build()"` '
            'or `make -C neurite_b200/csrc`.  There is no CPU fallback.' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the header and the library diverge
        fn.restype = res
        fn.argtypes = args
    if lib.nrt_version() != 2:
        raise ImportError('neurite_b200: ABI version mismatch (library %d, binding 2)' % lib.nrt_version())
    return lib


lib = _load()

NRT_LINEAR, NRT_NEAREST = 0, 1
NRT_STAT_SD, NRT_STAT_MAX, NRT_STAT_ABSMAX, NRT_STAT_MINMAX = 0, 1, 2, 3
ACTIVATIONS = {None: 0, 'linear': 0, 'relu': 1, 'sigmoid': 2, 'tanh': 3}


def check(status):
    if status != 0:
        raise NeuriteB200Error('%s: %s' % (lib.nrt_status_string(status).decode(),
                                           lib.nrt_last_error_string().decode()))


def method_id(interp_method):
    # reference: AssertionError on anything but linear / nearest (utils.py:194-195)
    assert interp_method in ('linear', 'nearest'), \
        'method should be linear or nearest, got: %s' % interp_method
    return NRT_LINEAR if interp_method == 'linear' else NRT_NEAREST


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise NeuriteB200Error('neurite_b200 ops need CUDA tensors (got device %s); there is no CPU path' % t.device)


def ptr(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def i32_array(vals):
    return (ctypes.c_int32 * len(vals))(*[int(v) for v in vals])
