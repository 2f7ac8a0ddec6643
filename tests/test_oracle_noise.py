"""
CPU tests of the noise oracle (oracle/noise.py): the numpy fp32 restatement reproduces every perlin / blur_rescale
/ gaussnoise fixture (the reference's own draw_perlin_full, random_blur_rescale, PerlinNoise and GaussianNoise on
tools/tfshim.py with replayed draws), the fp64 graph bounds an fp32 evaluation, and the numpy Philox4x32-10
matches known answers.
"""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import noise as onoise

# Philox4x32-10 known answers: (key, block j, the four words of counter {j, 0, 0, 0}).  Generated once from
# at::Philox4_32(seed=key, subsequence=0, offset=j) of PyTorch's ATen/core/PhiloxRNGEngine.h, an independent
# implementation; the first row is also Random123's published zero-key, zero-counter answer.
PHILOX_KAT = [
    (0x0, 0, (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    (0x0, 1, (0xf8e4cca4, 0x5cb200db, 0xb1a574eb, 0x097eff67)),
    (0x0, 1000003, (0x9592c3f8, 0x1087d23f, 0x7bc9e8f7, 0xef3a448f)),
    (0x123456789abcdef, 0, (0xb850222e, 0xc58cb04b, 0x14a7a020, 0x7a84fff9)),
    (0x123456789abcdef, 1, (0xadca1466, 0x523e0d85, 0x65401425, 0xb299da3f)),
    (0x123456789abcdef, 1000003, (0xcfcdfaf8, 0x4a69f54c, 0xa6a0ee7b, 0x2f6bca5f)),
    (0x7fffffffffffffff, 0, (0x32e74fa9, 0x93ebecf5, 0xf8ec7334, 0x0d8e8ffd)),
    (0x7fffffffffffffff, 1, (0x0831d704, 0xc53c3983, 0xc909c241, 0x8cb94662)),
    (0x7fffffffffffffff, 1000003, (0x6cefb196, 0x6bea4f54, 0x887dd07c, 0x9ee83311)),
]

PERLIN = golden_names('perlin_')
GAUSS = golden_names('gaussnoise_')


def test_fixtures_exist():
    assert len(PERLIN) >= 8 and len(GAUSS) >= 4


@pytest.mark.parametrize('key,j,words', PHILOX_KAT)
def test_philox_known_answers(key, j, words):
    assert tuple(int(w) for w in onoise.philox4x32_10(key, [j])[0]) == words


def test_philox_streams():
    w = onoise.philox_words(12345, 4001)
    assert np.array_equal(w[:4000], onoise.philox_words(12345, 4000))          # a prefix is the shorter draw
    u = onoise.u01(w)
    assert u.dtype == np.float32 and u.min() > 0 and u.max() <= 1
    assert np.array_equal(onoise.u01(np.array([0, 0xFFFFFFFF], np.uint32)), np.array([2.0 ** -24, 1.0], np.float32))
    z = onoise.philox_normal64(7, 1 << 16)
    assert abs(z.mean()) < 0.02 and abs(z.std() - 1) < 0.02


@pytest.mark.parametrize('name', PERLIN)
def test_oracle_matches_perlin_fixture(name):
    d = onoise.decode_perlin(load_golden(name))
    out = onoise.perlin_from_draws(d['noise'], d['sigmas'], d['std_max'], d['reduce'])
    np.testing.assert_array_equal(out, d['out'])


@pytest.mark.parametrize('name', GAUSS)
def test_oracle_matches_gaussnoise_fixture(name):
    fx = load_golden(name)
    u, z, kw = onoise.decode_gaussian(fx)
    np.testing.assert_array_equal(onoise.gaussian_noise_from_draws(fx['x'], u, z, **kw), fx['out'])


@pytest.mark.parametrize('name', PERLIN)
def test_fp64_bound_holds_for_fp32(name):
    d = onoise.decode_perlin(load_golden(name))
    ref, parts = onoise.torch_perlin64(d['noise'], d['sigmas'], d['std_max'], d['reduce'])
    scale, k = onoise.perlin_bounds(parts, d['reduce'])
    err = (torch.as_tensor(d['out']).double() - ref).abs()
    assert bool((err <= 4 * k * 2.0 ** -24 * scale).all())
