"""CPU tests of the generator's affine augmentation: the oracle against the reference's own generator
(tests/golden/affsynth_*), the host draw and composition, their statistics, and the argument and seed rules."""
import ast
import glob
import os

import numpy as np
import pytest

import neurite_b200 as ne
from oracle import affine as oaff, synth as osynth

F32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
AFFSYNTH = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, 'affsynth_*.npz')))
SYNTH = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, 'synth_*.npz')))


def _load(name):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    return fx, ast.literal_eval(str(fx['kwargs'])), [fx['q%d' % i] for i in range(int(fx['nq']))]


def _shapes(kw):
    in_shape = np.asarray(kw['in_shape'])
    half = kw.get('half_res', False)
    out = np.array(in_shape if kw.get('out_shape') is None else kw['out_shape']) // (2 if half else 1)
    return in_shape, out, half


def _ulps(a, ref):
    """|a - ref| in units of the fp32 spacing of each row's largest entry (entries near 0 are judged on the row)."""
    ref = np.asarray(ref, np.float64)
    scale = np.spacing(np.max(np.abs(ref), axis=-1, keepdims=True).astype(F32)).astype(np.float64)
    return np.abs(np.asarray(a, np.float64) - ref) / scale


def test_fixture_cases_cover_the_issue_matrix():
    assert len(AFFSYNTH) >= 10
    kws = [_load(n)[1] for n in AFFSYNTH]
    assert any(len(k['in_shape']) == 2 for k in kws) and any(len(k['in_shape']) == 3 for k in kws)
    for key in ('aff_shift', 'aff_rotate', 'aff_scale', 'aff_shear', 'axes_flip', 'axes_swap', 'half_res'):
        assert any(k.get(key) for k in kws), key
    assert any(k.get('warp_max', 2) == 0 for k in kws) and any(k.get('out_shape') for k in kws)
    assert any(any(k.get(n) for n in ('aff_normal_shift', 'aff_normal_rotate', 'aff_normal_scale')) for k in kws)


@pytest.mark.parametrize('name', AFFSYNTH)
def test_oracle_reproduces_affsynth_fixture_bit_for_bit(name):
    fx, kw, q = _load(name)
    labels = fx['labels']
    c, p, aff = oaff.decode(kw, labels, q)
    in_shape, out_shape, half = _shapes(kw)
    # the reference composes in fp32 matmuls; the fp64 composition of the decoded draws is within a few ulp
    full = oaff.compose(aff['aff'], in_shape, out_shape, half, aff['flip'], aff['swap'])
    assert np.max(_ulps(fx['trans'], full[:, :len(in_shape)])) <= 8
    r = oaff.synth(labels, c, p, fx['trans'])
    outs = oaff.outputs(kw, r, p, aff['aff'])
    assert len(outs) == int(fx['nout'])
    for i, o in enumerate(outs):
        assert np.array_equal(np.asarray(o), fx['out%d' % i]), (name, i)
    lo, hi = osynth.image_interval(r, c, p)
    im = r['image'].astype(np.float64)
    assert np.all((im >= lo) & (im <= hi))


@pytest.mark.parametrize('name', AFFSYNTH)
def test_host_matrices_match_fixture_draws(name):
    """The generator's host code on the fixture's decoded parameters: A within 1 ulp of the reference's, the final
    matrix within 2 ulp of the fp64 composition."""
    fx, kw, q = _load(name)
    c, p, aff = oaff.decode(kw, fx['labels'], q)
    n = len(kw['in_shape'])
    a = ne.models.affine_matrix(aff['params'], n)
    assert a.dtype == np.float32 and np.max(_ulps(a, aff['aff'])) <= 1
    in_shape, out_shape, half = _shapes(kw)
    gen = ne.models.labels_to_image_new(vxm_affine=True,
                                        **{k: v for k, v in kw.items() if not k.startswith('return')})
    trans = ne.models.compose_affine(a, gen.cfg['aff_pre'], gen.cfg['aff_post'], aff['flip'], aff['swap'])
    full = oaff.compose(a, in_shape, out_shape, half, aff['flip'], aff['swap'])
    assert trans.dtype == np.float32 and trans.shape == (fx['labels'].shape[0], n, n + 1)
    assert np.max(_ulps(trans, full[:, :n])) <= 2


@pytest.mark.parametrize('name', SYNTH)
def test_oracle_affine_warp_is_the_old_chain_at_identity(name):
    """At the identity affine the fixed-order dense shift, composed and sampled, is the existing synth_* chain."""
    fx, kw, q = _load(name)
    labels = fx['labels']
    c, p = osynth.decode_synth(kw, labels, q)
    ref = osynth.synth_from_plan(labels, c, p)
    in_shape, out_shape, half = _shapes(kw)
    eye = np.eye(len(in_shape) + 1)[None].repeat(labels.shape[0], 0)
    mats = oaff.compose(eye, in_shape, out_shape, half)[:, :len(in_shape)].astype(F32)
    r = oaff.synth(labels, c, p, mats)
    assert np.array_equal(r['warped'], ref['warped']) and np.array_equal(r['map'], ref['map'])


@pytest.mark.parametrize('ndims', [2, 3])
def test_host_composition_within_2_ulp_of_fp64(ndims):
    rng = np.random.default_rng(ndims)
    params = ne.models.affine_params(64, ndims, dict(shift=30, rot=180, scale=0.5, shear=0.3),
                                     dict(shift=False, rot=False, scale=False, shear=False),
                                     dict(shift=1, rot=2, scale=3, shear=4))
    a = ne.models.affine_matrix(params, ndims)
    assert np.max(_ulps(a, oaff.affine_matrix(params, ndims))) <= 1
    for in_shape, out_shape, half in (((40,) * ndims, (40,) * ndims, False),
                                      ((48, 40, 56)[:ndims], (44, 36, 50)[:ndims], False),
                                      ((48, 40, 56)[:ndims], (20, 18, 26)[:ndims], True)):
        gen = ne.models.labels_to_image_new(range(3), in_shape=in_shape, out_shape=out_shape, half_res=half)
        s = gen.cfg['out_shape']
        flip = ne.models.flip_matrix(rng.random(ndims) > 0.5, s)
        swap = ne.models.swap_matrix(rng.permutation(ndims)) if in_shape == out_shape else None
        trans = ne.models.compose_affine(a, gen.cfg['aff_pre'], gen.cfg['aff_post'], flip, swap)
        full = oaff.compose(a, in_shape, s, half, flip, swap)[:, :ndims]
        assert np.max(_ulps(trans, full)) <= 2


def test_identity_affine_is_exact():
    for ndims in (2, 3):
        p = ne.models.affine_params(3, ndims, dict(shift=0, rot=0, scale=0, shear=0),
                                    dict(shift=True, rot=True, scale=True, shear=True), {})
        assert p.shape == (3, 6 if ndims == 2 else 12) and not p.any()
        assert np.array_equal(ne.models.affine_matrix(p, ndims), np.broadcast_to(np.eye(ndims + 1, dtype=F32),
                                                                                  (3, ndims + 1, ndims + 1)))


@pytest.mark.parametrize('kind', ['shift', 'rot', 'scale', 'shear'])
def test_draw_statistics(kind):
    b = {'shift': 7.0, 'rot': 30.0, 'scale': 0.2, 'shear': 0.1}[kind]
    zero = dict(shift=0, rot=0, scale=0, shear=0)
    col = {'shift': slice(0, 3), 'rot': slice(3, 6), 'scale': slice(6, 9), 'shear': slice(9, 12)}[kind]
    off = dict(shift=False, rot=False, scale=False, shear=False)
    u = ne.models.affine_params(20000, 3, dict(zero, **{kind: b}), off, {kind: 5})
    x = u[:, col].astype(np.float64)
    assert not np.delete(u, np.arange(12)[col], 1).any()                 # the other kinds draw nothing
    assert x.min() >= -b and x.max() <= b
    assert abs(x.mean()) < 0.02 * b and abs(x.std() / (b / np.sqrt(3)) - 1) < 0.02
    z = ne.models.affine_params(20000, 3, dict(zero, **{kind: b}), dict(off, **{kind: True}), {kind: 6})[:, col]
    z = z.astype(np.float64) / b
    assert abs(z.mean()) < 0.03
    if kind == 'scale':                                                  # truncated at 2 SD by redrawing
        assert np.abs(z).max() <= 2 and np.abs(z).max() > 1.95
        assert abs(z.std() / 0.8796 - 1) < 0.02                          # SD of N(0, 1) truncated to [-2, 2]
    else:
        assert abs(z.std() - 1) < 0.02 and np.abs(z).max() > 3
    # the draw depends on the kind's seed only
    again = ne.models.affine_params(20000, 3, dict(zero, **{kind: b}), off, {kind: 5})
    assert np.array_equal(again, u)
    assert not np.array_equal(ne.models.affine_params(20000, 3, dict(zero, **{kind: b}), off, {kind: 4}), u)


def test_flip_and_swap_draws():
    flips = np.array([ne.models.draw_flip(s, 3) for s in range(4000)])
    assert np.all(np.abs(flips.mean(0) - 0.5) < 0.03)
    perms = {tuple(ne.models.draw_swap(s, 3)) for s in range(200)}
    assert len(perms) == 6
    assert {tuple(ne.models.draw_swap(s, 2)) for s in range(50)} == {(0, 1), (1, 0)}
    m = ne.models.flip_matrix(np.array([True, False, True]), [10, 12, 14])
    pt = m @ np.array([2, 3, 4, 1.0])
    assert np.array_equal(pt, [7, 3, 9, 1])                              # x -> (out_shape - 1) - x
    p = ne.models.swap_matrix(np.array([2, 0, 1]))
    assert p[0, 2] == p[1, 0] == p[2, 1] == p[3, 3] == 1 and p.sum() == 4


def test_generator_affine_switch_seeds_and_bounds():
    """vxm_affine=True enables the affine arguments; without it they raise as before.  Seeds and bound rules."""
    f = ne.models.labels_to_image_new
    for kw in ({'aff_shift': 1}, {'aff_rotate': 5}, {'aff_scale': 0.1}, {'aff_shear': 0.1}, {'axes_flip': True},
               {'axes_swap': True}):
        with pytest.raises(NotImplementedError, match='vxm_affine=True'):
            f(range(3), in_shape=(8, 8), **kw)
        assert f(range(3), in_shape=(8, 8), vxm_affine=True, **kw).cfg['num_dim'] == 2
    with pytest.raises(AssertionError, match='non-isotropic'):
        f(range(3), in_shape=(8, 10), axes_swap=True, vxm_affine=True)
    with pytest.raises(AssertionError, match='unknown seeds'):
        f(range(3), in_shape=(8, 8), seeds={'flip': 1}, vxm_affine=True)                   # flip without axes_flip
    with pytest.raises(AssertionError, match='unknown seeds'):
        f(range(3), in_shape=(8, 8), seeds={'swap': 1}, axes_flip=True, vxm_affine=True)   # swap without axes_swap
    for name in ('aff_shift', 'aff_rotate', 'aff_scale', 'aff_shear'):
        for switch in (False, True):
            with pytest.raises(NotImplementedError, match=name):
                f(range(3), in_shape=(8, 8), vxm_affine=switch, **{name: [1, 2]})
    g = f(range(3), in_shape=(8, 8, 8), aff_shift=3, aff_rotate=30, aff_scale=0.1, aff_shear=0.1, axes_flip=True,
          axes_swap=True, vxm_affine=True, seeds={'shift': 1, 'rot': 2, 'scale': 3, 'shear': 4, 'flip': 5, 'swap': 6})
    assert {k: g.cfg['seeds'][k] for k in ('shift', 'rot', 'scale', 'shear', 'flip', 'swap')} == \
        dict(shift=1, rot=2, scale=3, shear=4, flip=5, swap=6)
