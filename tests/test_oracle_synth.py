"""CPU tests of the label-to-image generator's host side: crop bounds, LUTs, argument checks."""
import numpy as np
import pytest

import neurite_b200 as ne
from oracle import synth as osynth

F32 = np.float32


@pytest.mark.parametrize('prop_low,prop_cen', [(0.0, 1.0), (0.0, 0.8), (0.1, 0.7), (0.25, 0.5), (0.3333, 0.0),
                                               (0.05, 0.95), (0.19999, 0.80001)])
def test_crop_bounds_match_bruteforce_fp32_mask(prop_low, prop_cen):
    raised = 0
    for width in range(1, 513):
        mask = osynth.crop_mask_bruteforce(width, prop_low, prop_cen)
        if mask.size != width:
            with pytest.raises(ValueError, match='cannot reshape'):
                ne.augment.crop_bounds(width, prop_low, prop_cen)
            raised += 1
            continue
        lo, hi = ne.augment.crop_bounds(width, prop_low, prop_cen)
        ref = np.zeros(width, bool)
        ref[lo:hi] = True
        assert np.array_equal(mask, ref), (width, lo, hi)
    assert raised > 0                                   # e.g. width 61: ceil(1 / fp32(1/61)) = 62


def test_crop_length_mismatch_width_raises():
    assert ne.augment.tf_range_f32(61).size == 62
    with pytest.raises(ValueError):
        ne.augment.crop_bounds(61, 0.0, 1.0)


def test_draw_crop_mask_numpy_and_draws():
    x = np.zeros((2, 8, 10, 12, 1), F32)
    m = ne.augment.draw_crop_mask(x, crop_min=0.2, crop_max=0.5, axis=(1, 2, 3), seed=4)
    assert m.dtype == np.float32 and m.ndim == 5 and sum(s > 1 for s in m.shape) == 1
    assert np.array_equal(m, ne.augment.draw_crop_mask(x, crop_min=0.2, crop_max=0.5, axis=(1, 2, 3), seed=4))
    ax = int(np.argmax(m.shape))
    kept = int(m.sum())
    assert ax in (1, 2, 3) and 0.5 * x.shape[ax] - 1 <= kept <= 0.8 * x.shape[ax] + 1
    m0 = ne.augment.draw_crop_mask(x, prob=0, seed=1)                                 # prob 0: nothing cropped
    assert m0.sum() == max(m0.shape) == x.shape[int(np.argmax(m0.shape))]
    with pytest.raises(AssertionError, match='invalid proportions'):
        ne.augment.draw_crop_mask(x, crop_min=0.6, crop_max=0.5)
    with pytest.raises(AssertionError, match='not a probability'):
        ne.augment.draw_crop_mask(x, prob=2)
    assert ne.utils.augment.draw_crop_mask is ne.augment.draw_crop_mask


def test_generation_and_output_luts():
    _, gen, lut = ne.models.generation_lut([0, 2, 5])
    ind = {g: i for i, g in enumerate({0, 2, 5})}
    assert lut == [ind[0], 0, ind[2], 0, 0, ind[5]]
    d = {0: 'bg', 1: 'ctx', 3: 'ctx', 4: 'wm'}
    _, gen, lut = ne.models.generation_lut(d)
    ind = {g: i for i, g in enumerate(set(d.values()))}       # the reference's own expression: set order
    assert len(gen) == 3 and lut == [ind['bg'], ind['ctx'], 0, ind['ctx'], ind['wm']]
    assert ne.models.output_lut([0, 1, 2], None, True) == (None, 3)                      # identity: no gather
    lut, m = ne.models.output_lut([0, 1, 2, 3], {1: 1, 3: 1}, True)
    assert m == 1 and lut == [-1, 0, -1, 0]
    lut, m = ne.models.output_lut([0, 1, 2, 3], {1: 7, 3: 9}, False)
    assert m == 2 and lut == [0, 7, 0, 9]


def test_generator_reference_asserts_and_scope_cut():
    f = ne.models.labels_to_image_new
    with pytest.raises(AssertionError, match='gamma value'):
        f(range(3), in_shape=(8, 8), gamma=1.5)
    with pytest.raises(AssertionError, match='unknown seeds'):
        f(range(3), in_shape=(8, 8), seeds={'bogus': 1})
    with pytest.raises(AssertionError, match='unknown seeds'):
        f(range(3), in_shape=(8, 8), seeds={'warp': 1}, warp_max=0)          # no warp layer pops 'warp'
    with pytest.raises(AssertionError, match='non-isotropic'):
        f(range(3), in_shape=(8, 10), axes_swap=True)
    for kw in ({'aff_shift': 1}, {'aff_rotate': 5}, {'aff_scale': 0.1}, {'aff_shear': 0.1}, {'axes_flip': True},
               {'axes_swap': True}, {'input_model': object()}):
        with pytest.raises(NotImplementedError, match=list(kw)[0]):
            f(range(3), in_shape=(8, 8), **kw)
    g = f({0: 0, 1: 1, 2: 1}, in_shape=(8, 8), seeds=['mean', 'noise'], num_chan=2)
    assert g.cfg['seeds']['mean'] == hash('mean') and g.cfg['num_chan'] == 2
    assert f(range(3), in_shape=(8, 8), seeds={'shift': 1, 'rot': 2}).cfg['seeds']['warp'] is None


def test_random_crop_config_round_trip():
    r = ne.layers.RandomCrop(crop_min=0.1, crop_max=0.3, axis=2, prob=0.5, bilateral=True, seed=3, name='crop')
    cfg = r.get_config()
    assert cfg == {'name': 'crop', 'crop_min': 0.1, 'crop_max': 0.3, 'axis': 2, 'prob': 0.5, 'bilateral': True,
                   'seed': 3}
    assert ne.layers.RandomCrop.from_config(cfg).get_config() == cfg
    r.build((1, 8, 8, 8, 1))
    assert r.axis == (2,)
    r2 = ne.layers.RandomCrop()
    r2.build((1, 8, 8, 8, 1))
    assert r2.axis == (1, 2, 3)
    with pytest.raises(IndexError):
        ne.layers.RandomCrop(axis=4).build((1, 8, 8, 8, 1))


# ---------------------------------------------------------------------------------------
# the reference's own code on replayed draws (tests/golden/synth_*, crop_*, minmax_*)
# ---------------------------------------------------------------------------------------
import ast  # noqa: E402
import glob  # noqa: E402
import os  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _fixtures(prefix):
    return sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, prefix + '*.npz')))


def _load(name):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    return fx, [fx['q%d' % i] for i in range(int(fx['nq']))] if 'nq' in fx.files else []


@pytest.mark.parametrize('name', _fixtures('synth_'))
def test_oracle_reproduces_synth_fixture_bit_for_bit(name):
    fx, q = _load(name)
    kw = ast.literal_eval(str(fx['kwargs']))
    c, p = osynth.decode_synth(kw, fx['labels'], q)
    r = osynth.synth_from_plan(fx['labels'], c, p)
    outs = osynth.synth_outputs(kw, r, p)
    assert len(outs) == int(fx['nout'])
    for i, o in enumerate(outs):
        assert np.array_equal(np.asarray(o), fx['out%d' % i]), (name, i)
    # the fp32 evaluation lies inside the interval bound of the image
    lo, hi = osynth.image_interval(r, c, p)
    im = r['image'].astype(np.float64)
    assert np.all((im >= lo) & (im <= hi))


@pytest.mark.parametrize('name', _fixtures('crop_'))
def test_oracle_reproduces_crop_fixture_bit_for_bit(name):
    fx, q = _load(name)
    kw = ast.literal_eval(str(fx['kwargs']))
    x = fx['x']
    if name == 'crop_mask_fixed_prop':                     # draw_crop_mask itself, axis None: any axis
        (ax, lo, hi), k = osynth.crop_from_draws(q, 0, x.shape, kw['crop_min'], kw['crop_max'], None, 1, False)
        ref = np.zeros([1] * x.ndim, np.float32) + osynth.crop_window(np.ones(x.shape[ax], np.float32), 0, lo, hi) \
            .reshape([x.shape[ax] if d == ax else 1 for d in range(x.ndim)])
    else:
        axis = kw.get('axis')
        axis = list(range(1, x.ndim - 1)) if axis is None else axis
        (ax, lo, hi), k = osynth.crop_from_draws(q, 0, x.shape, kw.get('crop_min', 0), kw.get('crop_max', 0.5),
                                                 axis, kw.get('prob', 1), kw.get('bilateral', False))
        ref = osynth.crop_window(x, ax, lo, hi)
    assert k == len(q)
    assert np.array_equal(ref, fx['out'])


@pytest.mark.parametrize('name', _fixtures('minmax_'))
def test_oracle_reproduces_minmax_fixture_bit_for_bit(name):
    fx, _ = _load(name)
    axis = ast.literal_eval(str(fx['axis']))
    assert np.array_equal(osynth.minmax_norm(fx['x'], axis=axis), fx['out'])
