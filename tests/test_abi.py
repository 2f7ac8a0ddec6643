"""
CPU tests of the drop-in boundary: the C-ABI library loads here (no GPU), exports every
symbol include/neurite_b200.h declares, the ctypes binding covers the header one to one,
argument validation returns status codes (never throws, never touches the device), and the
python wrappers refuse CPU tensors instead of falling back.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT

HEADER = os.path.join(ROOT, 'include', 'neurite_b200.h')


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(nrt_[a-z0-9_]+)\s*\(', src)))


def test_library_loads_at_abi_version_2_and_exports_every_declared_symbol():
    from neurite_b200 import _lib
    names = declared_symbols()
    assert len(names) >= 14
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), 'libneurite_b200.so does not export %s' % n
    assert sorted(_lib.SIGNATURES) == names, 'ctypes binding and header diverge'
    assert _lib.lib.nrt_version() == 2
    assert _lib.lib.nrt_status_string(0) == b'ok'


def test_entry_points_return_status_codes_on_bad_arguments():
    from neurite_b200 import _lib
    lib = _lib.lib
    null = ctypes.c_void_p(0)
    shape = _lib.i32_array([4, 4, 4])
    assert lib.nrt_interpn_f32(null, shape, 3, 1, null, 0, 0, 0, 0.0, null, null) == -1      # null pointers
    assert b'null' in lib.nrt_last_error_string()
    one = ctypes.c_void_p(16)
    assert lib.nrt_interpn_f32(one, _lib.i32_array([2] * 6), 6, 1, one, 0, 0, 0, 0.0, one, null) == -1   # D = 6 (built for 1..5)
    assert lib.nrt_interpn_f32(one, shape, 3, 1, one, 0, 7, 0, 0.0, one, null) == -1         # bad method
    assert b'linear or nearest' in lib.nrt_last_error_string()
    assert lib.nrt_warp_f32(one, one, one, 1, shape, 3, 1, 0, 0, 0.0, 0, 9, 0, 4, 0, null, null) == -1   # src planes > volume
    assert lib.nrt_dice_workspace_bytes(4, 16) == 4 * 2048 * 3 * 16 * 4
    assert lib.nrt_dice_sums_f32(one, one, 1, 10, 4, 5, 9, 0, 0, one, null, one, 1 << 30, null) == -1   # voxel range
    k = _lib.i32_array([3, 3, 3])
    assert lib.nrt_lc3d_fwd_f32(one, one, null, one, 1, _lib.i32_array([2, 8, 8]), 1, 1, k, k, 0, 0, 0, 1, null) == -1
    with pytest.raises(_lib.NeuriteB200Error, match='bad argument'):
        _lib.check(-1)
    # the MI / convolution entry points validate before touching the device too
    f = ctypes.c_float
    inf = float('inf')
    assert lib.nrt_mi_hist_f32(null, 1, 1, 1, 16, one, one, 1, 1, 1, 16, one, 1, 1, 10, f(1.0), f(-inf), f(inf),
                               one, null, one, 1 << 30, null) == -1                                     # null x
    assert lib.nrt_mi_hist_f32(one, 1, 1, 1, 65, one, one, 1, 1, 1, 16, one, 1, 1, 10, f(1.0), f(-inf), f(inf),
                               one, null, one, 1 << 30, null) == -2                                     # 65 bins
    assert b'bins' in lib.nrt_last_error_string()
    assert lib.nrt_mi_hist_f32(one, 1, 1, 1, 16, null, one, 1, 1, 1, 16, one, 1, 1, 10, f(1.0), f(-inf), f(inf),
                               one, null, one, 1 << 30, null) == -1                                     # quantise without centres
    assert lib.nrt_mi_hist_f32(one, 1, 1, 0, 16, null, one, 1, 1, 0, 16, null, 1, 3, 10, f(1.0), f(-inf), f(inf),
                               one, null, one, 1 << 30, null) == -1                                     # channels need two quantised operands
    assert lib.nrt_mi_hist_f32(one, 1, 1, 1, 16, one, one, 1, 1, 1, 16, one, 1, 1, 10, f(1.0), f(-inf), f(inf),
                               one, null, one, 16, null) == -1                                          # workspace too small
    assert lib.nrt_mi_workspace_bytes(2, 16, 16) == 2 * 592 * (256 + 32) * 4
    assert lib.nrt_mi_bwd_f32(one, 1, 1, 1, 33, one, one, 1, 1, 1, 16, one, 1, 1, 10, f(1.0), f(-inf), f(inf),
                              one, one, one, null, null, 0, null) == -2                                 # gradient: <= 32 bins
    assert lib.nrt_mi_bwd_f32(one, 1, 1, 1, 16, one, one, 1, 1, 1, 16, one, 1, 1, 10, f(1.0), f(-inf), f(inf),
                              one, null, null, null, null, 0, null) == -1                               # no gradient requested
    assert lib.nrt_item_stats_f32(one, 1, 0, _lib.NRT_STAT_MINMAX, one, one, 1 << 20, null) == -1         # empty tensor
    assert lib.nrt_sepconv_axis_f32(one, one, 1, 8, 1, one, 3, 1, 1, 1, 8, null) == -1                  # in place
    assert b'in-place' in lib.nrt_last_error_string()
    two = ctypes.c_void_p(32)
    assert lib.nrt_sepconv_axis_f32(one, two, 1, 8, 1, one, 0, 1, 1, 0, 8, null) == -1                  # K = 0
    assert lib.nrt_gather_axis_f32(one, null, two, 1, 8, 1, 8, null) == -1


def test_no_cpu_fallback():
    import neurite_b200 as ne
    vol = torch.zeros(4, 4, 4)
    loc = torch.zeros(2, 3)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.utils.interpn(vol, loc)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.losses.Dice().loss(torch.zeros(1, 4, 4, 2), torch.zeros(1, 4, 4, 2))
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.layers.SpatialTransformer()([torch.zeros(1, 4, 4, 4, 1), torch.zeros(1, 4, 4, 4, 3)])
    # the 'next' rows: mutual information, soft quantisation, blur, subsample, separable convolution
    v = torch.rand(1, 4, 4, 4, 1)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.metrics.MutualInformation().volumes(v, v)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.metrics.MutualInformation().segs(torch.rand(1, 8, 3), torch.rand(1, 8, 3))
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.utils.soft_quantize(v)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.layers.GaussianBlur(sigma=1.0)(v)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.layers.Subsample(seed=0)(v)
    with pytest.raises(ne._lib.NeuriteB200Error, match='no CPU path'):
        ne.utils.separable_conv(v, torch.ones(3), batched=True)


def test_mi_blur_subsample_argument_checks_and_configs():
    """reference-side checks that do not need a device: metrics.py:69-114, layers.py:268-343, 380-423."""
    import neurite_b200 as ne
    m = ne.metrics.MutualInformation()
    assert m.nb_bins == 16 and np.float32(m.soft_bin_alpha) == np.float32(1) / (np.float32(2) * np.float32(0.5 / 15) ** 2)
    with pytest.raises(AssertionError, match='cannot provide both'):
        ne.metrics.MutualInformation(bin_centers=np.linspace(0, 1, 4), nb_bins=4)
    c = ne.metrics.MutualInformation(bin_centers=np.linspace(0, 1, 5))
    assert c.nb_bins == 5 and abs(float(c.soft_bin_alpha) - 1 / (2 * (0.5 * 0.25) ** 2)) < 1e-3
    assert ne.losses.MutualInformation is ne.metrics.MutualInformation          # losses.py:40-43 re-export

    with pytest.raises(AssertionError, match='sigma or level'):
        ne.layers.GaussianBlur()
    with pytest.raises(AssertionError, match='only sigma or level'):
        ne.layers.GaussianBlur(sigma=1, level=2)
    with pytest.raises(ValueError, match='isotropy is implicitly'):
        ne.layers.GaussianBlur(sigma=1, isotropic=True)
    with pytest.raises(ValueError, match='must not be less than 1'):
        ne.layers.GaussianBlur(level=0.5)
    g = ne.layers.GaussianBlur(sigma=[1.0, 2.0, 0.0], name='blur')
    cfg = g.get_config()
    assert cfg == {'name': 'blur', 'sigma': [1.0, 2.0, 0.0], 'random': False, 'min_sigma': 0, 'isotropic': False, 'seed': None}
    assert ne.layers.GaussianBlur.from_config(cfg).sigma == [1.0, 2.0, 0.0]
    g.build((1, 8, 8, 8, 1))
    assert g.sigma == [1.0, 2.0, 0.0] and g.min_sigma == [0, 0, 0]
    with pytest.raises(ValueError, match='1 or 3 sigmas expected'):
        ne.layers.GaussianBlur(sigma=[1.0, 2.0]).build((1, 8, 8, 8, 1))
    with pytest.raises(ValueError, match='must not be less than 0'):
        ne.layers.GaussianBlur(sigma=-1.0).build((1, 8, 8, 1))
    x = torch.zeros(1, 4, 4, 1)
    assert ne.layers.GaussianBlur(sigma=0)(x) is x                            # layers.py:347-348: no positive sigma -> input

    k = ne.utils.gaussian_kernel(1.0)
    assert k.shape == (7,) and abs(float(k.sum()) - 1) < 1e-6 and torch.equal(k, k.flip(0))
    ks = ne.utils.gaussian_kernel([0.5, 2.0], separate=True)
    assert [int(t.numel()) for t in ks] == [5, 13]
    assert ne.utils.gaussian_kernel([1.0, 1.0]).shape == (7, 7)
    with pytest.raises(ValueError, match='differ in length'):
        ne.utils.gaussian_kernel([1.0, 2.0], windowsize=[3])

    s = ne.layers.Subsample(stride_min=2, stride_max=4, axes=[1, 3], prob=0.5, upsample=False, seed=7)
    assert s.get_config() == {'name': 'subsample', 'stride_min': 2, 'stride_max': 4, 'axes': [1, 3], 'prob': 0.5,
                              'upsample': False, 'seed': 7}
    s.build((1, 8, 8, 8, 2))
    assert s.axes == [1, 3]
    with pytest.raises(ValueError):
        ne.layers.Subsample(axes=[4]).build((1, 8, 8, 8, 2))                   # the channel axis is not spatial
    assert ne.layers.Subsample(stride_max=1)(x) is x and ne.layers.Subsample(prob=0)(x) is x
    idx = ne.utils.subsample_indices(10, 2.0)
    assert idx.tolist() == [0, 0, 2, 2, 5, 5, 7, 7, 9, 9]


def test_reference_exceptions_and_config_round_trip():
    import neurite_b200 as ne
    with pytest.raises(Exception, match='does not match volume dimension'):
        ne.utils.interpn(torch.zeros(3, 3, 3, 3, 3), torch.zeros(2, 2))
    with pytest.raises(AssertionError, match='method should be linear or nearest'):
        ne.utils.interpn(torch.zeros(3, 3), torch.zeros(2, 2), 'cubic')
    with pytest.raises(AssertionError):
        ne.utils.resize(torch.zeros(3), [2, 2])
    with pytest.raises(AssertionError):
        ne.metrics.Dice(input_type='one_hot')
    with pytest.raises(AssertionError, match='need nb_labels'):
        ne.metrics.Dice(dice_type='hard', input_type='max_label')
    with pytest.raises(ValueError, match='only "valid" is supported'):
        ne.layers.LocallyConnected3D(4, 3, padding='same')
    with pytest.raises(ValueError, match='Unrecognized implementation mode'):
        ne.layers.LocallyConnected3D(4, 3, implementation=4)
    with pytest.raises(ValueError, match='Label weights must be of len 3, but got 2'):
        ne.losses.CategoricalCrossentropy(label_weights=[1., 2.]).loss(torch.zeros(1, 2, 3), torch.zeros(1, 2, 3))
    r = ne.layers.Resize(2, interp_method='nearest')
    cfg = r.get_config()
    assert cfg['zoom_factor'] == 2 and cfg['interp_method'] == 'nearest'
    r.build((None, 8, 9, 10, 2))
    assert r.compute_output_shape((None, 8, 9, 10, 2)) == (None, 16, 18, 20, 2)
    with pytest.raises(AssertionError, match='zoom factor length'):
        ne.layers.Resize([2, 2]).build((None, 8, 9, 10, 2))
    lc = ne.layers.LocallyConnected3D(64, (3, 3, 3))
    lc.build((None, 32, 32, 32, 3))
    # docstring known answer, layers.py:825-835
    assert lc.compute_output_shape((None, 32, 32, 32, 3)) == (None, 30, 30, 30, 64)
    assert tuple(lc.kernel.shape) == (30 ** 3, 27 * 3, 64) and tuple(lc.bias.shape) == (30, 30, 30, 64)
    assert sorted(dict(lc.named_parameters())) == ['bias', 'kernel']
    cfg = lc.get_config()
    assert cfg['filters'] == 64 and cfg['kernel_size'] == (3, 3, 3) and cfg['implementation'] == 1
    assert ne.utils.flatten_axes(torch.zeros(3, 4, 5, 6), [1, 2]).shape == (3, 20, 6)   # utils.py:1200-1201
