"""CPU tests of what tests/test_gpu_prepost_edges.py compares the kernels with, and of the host code that feeds the resize kernel.

 * The Gaussian taps of CenterPad's anti-aliasing filter are computed on the host (csrc/dvc_api.cu: resize_taps) and read back
   through dvc_debug_resize_taps, which needs no GPU.  They must be scipy.ndimage._gaussian_kernel1d's: numpy's pairwise sum, not a
   left-to-right one (the two differ in the last bit from radius 5 up, and the truncation to uint8 sees it on flat areas).  exp
   is libm's; numpy evaluates exp with its own vector code on CPUs that have the instructions, which can differ from libm in
   the last bit of some taps, so the bit-for-bit comparison with scipy is made wherever the two exps agree, and a bound of a few ulps
   (one from each exp, the rest through the sum) holds everywhere.
 * The fp32 restatements of resize_half / upsample2 (oracle/prepost_oracle.py) against F.interpolate, and their fused
   multiply-add against exact rational arithmetic.
 * The luminance -> guide thresholds and the continuity of the colour oracles across their branch thresholds.
"""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dvc_oracle as O
from oracle import prepost_oracle as P

# (in_len, out_len) of every CenterPad case of tests/test_gpu_prepost_edges.py, and the factors of the defect table
FACTORS = [(1440, 432), (2560, 768), (2160, 432), (3840, 768), (1080, 432), (1920, 768), (2160, 216), (3840, 384), (1000, 64), (3000, 192),
           (1280, 768), (720, 432), (500, 50), (2000, 200), (360, 108), (640, 192), (540, 108), (960, 192), (1080, 108), (1920, 192), (4000, 2)]


def _scipy_taps(in_len, out_len):
    from scipy.ndimage._filters import _gaussian_kernel1d

    sigma = (in_len / out_len - 1.0) / 2.0
    return _gaussian_kernel1d(sigma, 0, int(4.0 * sigma + 0.5))


def _exp_agrees(in_len, out_len):
    """numpy's exp equals libm's on every argument of this axis' taps (true on any CPU where numpy falls back to libm)."""
    sigma = (in_len / out_len - 1.0) / 2.0
    r = int(4.0 * sigma + 0.5)
    args = -0.5 / (sigma * sigma) * np.arange(-r, r + 1) ** 2
    return np.array_equal(np.exp(args), np.array([math.exp(a) for a in args]))


def test_taps_probe_geometry():
    import dvc

    assert dvc.resize_taps(100, 100) == [] and dvc.resize_taps(100, 200) == []          # no down-scale, no filter
    assert len(dvc.resize_taps(360, 108)) == 11 and len(dvc.resize_taps(1920, 192)) == 37
    for pair in ((5, 4), (360, 108), (10000, 7)):
        t = np.array(dvc.resize_taps(*pair))
        assert np.array_equal(t, t[::-1]) and abs(t.sum() - 1.0) < 1e-15 and (t > 0).all()


@pytest.mark.parametrize("in_len,out_len", FACTORS)
def test_resize_taps_are_scipys_bit_for_bit(in_len, out_len):
    """Fails with a left-to-right sum: at 360 -> 108 (sigma 1.1667, radius 5) the sums are 2.9243960115037066 (numpy) and
    ...706 (sequential), and every tap moves by one ulp."""
    import dvc

    taps = np.array(dvc.resize_taps(in_len, out_len))
    assert np.array_equal(taps, P.resize_taps_twin(in_len, out_len))
    ref = _scipy_taps(in_len, out_len)
    assert taps.shape == ref.shape
    if _exp_agrees(in_len, out_len):
        assert np.array_equal(taps, ref)
    assert (np.abs(taps - ref) <= 8 * np.spacing(ref)).all()


def test_resize_taps_sweep():
    """Every tap count from 1 to beyond numpy's 128-element blocks and its recursion: the sum order changes at 8 and at 129."""
    import dvc

    exact = 0
    pairs = [(i, 64) for i in range(65, 64 * 40, 7)] + [(i, 3) for i in range(4, 400)] + [(8000, 5), (6000, 3), (4095, 4)]
    for in_len, out_len in pairs:
        taps = np.array(dvc.resize_taps(in_len, out_len))
        assert np.array_equal(taps, P.resize_taps_twin(in_len, out_len)), (in_len, out_len)
        ref = _scipy_taps(in_len, out_len)
        if _exp_agrees(in_len, out_len):
            assert np.array_equal(taps, ref), (in_len, out_len)
            exact += 1
        assert (np.abs(taps - ref) <= 8 * np.spacing(ref)).all(), (in_len, out_len)
    assert max(len(dvc.resize_taps(*p)) for p in pairs) > 4096 and exact > 0


def test_fma_f32_is_the_single_rounding():
    rng = np.random.default_rng(5)
    a = rng.standard_normal(4000).astype(np.float32)
    b = rng.standard_normal(4000).astype(np.float32)
    c = (rng.standard_normal(4000) * np.float32(2.0) ** rng.integers(-30, 30, 4000)).astype(np.float32)
    # products that land exactly half-way between two float32 with a small addend deciding the direction (where rounding the
    # float64 sum a second time goes wrong), and subnormal results
    a[:4] = b[:4] = np.float32(1 + 2.0 ** -12)
    c[:4] = np.array([2.0 ** -60, -2.0 ** -60, 0.0, 2.0 ** -100], np.float32)
    a[4:8], b[4:8] = np.float32(3e-39), np.float32(0.5)
    c[4:8] = np.array([1e-45, 0.0, -3e-39, 1.5e-39], np.float32)
    got = P.fma_f32(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        lo, hi = np.nextafter(g, np.float32(-np.inf)), np.nextafter(g, np.float32(np.inf))
        err = abs(Fraction(float(g)) - exact)
        assert err <= abs(Fraction(float(lo)) - exact) and err <= abs(Fraction(float(hi)) - exact), (x, y, z, g)
    assert got[0] != got[1]  # the tie is broken by the addend's sign, which a float64 sum rounded twice would lose


@pytest.mark.parametrize("shape", [(1, 1, 2, 2), (1, 1, 2, 4096), (3, 5, 6, 10), (2, 3, 432, 768)])
def test_resize_half_restatement_matches_interpolate(shape):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(21)) * 40
    mine = P.resize_half_f32(x.numpy())
    ref = F.interpolate(x, scale_factor=0.5, mode="bilinear").numpy()
    assert mine.shape == ref.shape and mine.dtype == np.float32
    assert np.abs(mine - ref).max() <= 1e-6 * float(x.abs().max())
    block = x.double().numpy().reshape(shape[0], shape[1], shape[2] // 2, 2, shape[3] // 2, 2).mean((3, 5))
    assert np.abs(mine - block).max() <= 2e-7 * float(x.abs().max())


@pytest.mark.parametrize("shape", [(1, 2, 1, 1), (1, 2, 1, 7), (1, 2, 7, 1), (5, 3, 3, 5), (2, 2, 216, 384)])
def test_upsample2_restatement_matches_interpolate(shape):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(22)) * 60
    mine = P.upsample2_scaled_f32(x.numpy(), 1.25)
    ref = (F.interpolate(x.double(), scale_factor=2, mode="bilinear") * 1.25).numpy()
    assert mine.shape == ref.shape and mine.dtype == np.float32
    assert np.abs(mine - ref).max() <= 3e-7 * float(x.abs().max())  # three roundings of values <= max|x|, one of the scaled result


def _f32(fr):
    """The float32 nearest to a rational, ties to the even neighbour."""
    c = np.float32(float(fr))
    cands = (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf)))
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - fr), int(v.view(np.int32)) & 1))


def guide_threshold_inputs():
    """For k = 0..255 the float32 nearest to k * 100 / 255 - 50 (where the guide steps to k) and its +-1, +-2 ulp neighbours,
    plus the far ends."""
    base = (np.arange(256, dtype=np.float64) * 100 / 255 - 50).astype(np.float32)
    vals = [base]
    for _ in range(2):
        vals = [np.nextafter(vals[0], np.float32(-np.inf))] + vals + [np.nextafter(vals[-1], np.float32(np.inf))]
    return np.concatenate(vals + [np.array([-1e9, -50.0, 50.0, 1e9], np.float32)])


def test_guide_threshold_table():
    l = guide_threshold_inputs()
    g = P.l_to_guide8(l)
    # the same three float32 operations in exact arithmetic, each rounded by the float32 constructor
    for li, gi in zip(l[:-4], g[:-4]):
        v = _f32(Fraction(float(li)) + 50)
        v = _f32(Fraction(float(v)) * 255)
        v = _f32(Fraction(float(v)) / 100)
        assert gi == min(max(math.trunc(float(v)), 0), 255), li
    assert g[-4:].tolist() == [0, 0, 255, 255]
    order = np.argsort(l, kind="stable")
    assert (np.diff(g[order].astype(int)) >= 0).all() and set(g.tolist()) == set(range(256))
    k = np.arange(256)
    assert (np.abs(g[2 * 256:3 * 256].astype(int) - k) <= 1).all()  # at the nominal threshold: k, or k - 1 when rounding fell short


def test_colour_oracles_are_continuous_across_their_thresholds():
    # the piecewise definitions meet at their thresholds
    assert abs(0.2068966 ** 3 - (0.2068966 - 16 / 116) / 7.787) < 1e-6
    assert abs((1.055 * 0.0031308 ** (1 / 2.4) - 0.055) - 0.0031308 * 12.92) < 1e-6
    assert abs(((0.04045 + 0.055) / 1.055) ** 2.4 - 0.04045 / 12.92) < 1e-6
    assert abs(0.008856 ** (1 / 3) - (7.787 * 0.008856 + 16 / 116)) < 1e-6
    # and so do the oracles: grey Lab inputs on either side of f = 0.2068966 (L = 116 f - 16) and of v = 0.0031308 give the
    # same bytes, and the L of the 256 greys rises without a jump through 0.04045 (bytes 10 | 11) and 0.008856
    for f in (0.2068966, 7.787 * 0.0031308 + 16 / 116):
        L = np.float32(116 * f - 16 - 50)
        l = torch.tensor([np.nextafter(L, np.float32(-100)), L, np.nextafter(L, np.float32(100))]).view(3, 1, 1, 1)
        rgb = O.lab_to_rgb8(l, torch.zeros(3, 2, 1, 1))
        assert (rgb == rgb[0]).all()
    g = torch.arange(256, dtype=torch.uint8).view(1, 1, 256, 1).expand(1, 1, 256, 3).contiguous()
    L = O.rgb8_to_lab(g)[0, 0, 0].numpy()
    step = np.diff(L)
    assert (step > 0.2).all() and (step < 0.52).all() and np.abs(np.diff(step)).max() < 0.025
    assert abs(L[0] + 50) < 1e-6 and abs(L[255] - 50) < 1e-4
