"""GPU: pre / post-processing kernels around the nets (SURVEY.md §8f row 1) against the CPU oracle
(the reference does these with torch.nn.functional.interpolate at test.py:58,71,100-102)."""
import numpy as np
import pytest
import torch

from oracle import dvc_oracle as O
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(1, 3, 32, 48), (2, 3, 432, 768), (1, 1, 6, 4)])
def test_resize_half_matches_interpolate(ctx, shape):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1)) * 40
    ref = O.resize_half(x)
    out = ctx.resize_half(x.cuda()).cpu()
    assert out.shape == ref.shape
    assert (out - ref).abs().max() <= 1e-5 * x.abs().max()


@pytest.mark.parametrize("shape", [(1, 2, 16, 24), (2, 2, 216, 384), (1, 2, 1, 1), (1, 2, 3, 5)])
def test_upsample2_scaled_matches_interpolate(ctx, shape):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(2)) * 60
    ref = O.upsample2_scaled(x, 1.25)
    out = ctx.upsample2_scaled(x.cuda(), 1.25).cpu()
    assert out.shape == ref.shape
    assert (out - ref).abs().max() <= 1e-5 * x.abs().max()


def test_half_resolution_pipeline_roundtrip(ctx):
    """test.py data flow: 432x768 Lab frame -> 1/2 -> colourise -> x2 * 1.25."""
    big = make_lab(5, 1, 64, 96)
    IB = ctx.resize_half(make_lab(6, 1, 64, 96).cuda())
    ctx.set_exemplar(IB)
    IA = ctx.resize_half(big.cuda())
    ab = ctx.colorize_frames(IA[:, 0:1].contiguous(), torch.zeros(1, 3, 32, 48, device="cuda"))
    up = ctx.upsample2_scaled(ab)
    assert up.shape == (1, 2, 64, 96) and torch.isfinite(up).all()
    assert torch.allclose(up.cpu(), O.upsample2_scaled(ab.cpu()), atol=1e-4)


@pytest.mark.parametrize("shape", [(1, 32, 48), (2, 216, 384), (1, 1, 1)])
def test_lab_to_rgb8_matches_float64_oracle(ctx, shape):
    """Output conversion of test.py:116-119 (utils/util.py:140-151): float64 skimage-style Lab -> sRGB -> uint8
    truncation.  CUDA's and numpy's double pow() may differ in the last ulp, which can flip a truncation only when
    v * 255 sits within ~1e-13 of an integer: allow one level on at most 1e-5 of the values."""
    B, H, W = shape
    g = torch.Generator().manual_seed(11)
    l = torch.rand(B, 1, H, W, generator=g) * 100 - 50
    ab = (torch.rand(B, 2, H, W, generator=g) * 2 - 1) * 110  # includes out-of-gamut colours (clipped channels)
    ref = O.lab_to_rgb8(l, ab)
    out = ctx.lab_to_rgb8(l.cuda(), ab.cuda()).cpu()
    assert out.shape == ref.shape == (B, H, W, 3) and out.dtype == torch.uint8
    d = (out.int() - ref.int()).abs()
    assert int(d.max()) <= 1
    assert float((d > 0).float().mean()) <= 1e-5


def test_post_processing_chain_on_device(ctx):
    """test.py:99-119 without the WLS filter: ab x2 * 1.25 -> Lab -> RGB uint8, all on the device."""
    big = make_lab(7, 1, 64, 96)
    ab = torch.randn(1, 2, 32, 48, generator=torch.Generator().manual_seed(3)) * 20
    up = ctx.upsample2_scaled(ab.cuda())
    rgb = ctx.lab_to_rgb8(big[:, 0:1].cuda(), up).cpu()
    ref = O.lab_to_rgb8(big[:, 0:1], O.upsample2_scaled(ab))
    d = (rgb.int() - ref.int()).abs()
    assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 1e-3  # fp32 up-sampling differs by ~1e-6 before truncation


@pytest.mark.parametrize("shape", [(1, 32, 48), (2, 216, 384)])
def test_rgb8_to_lab_matches_float64_oracle(ctx, shape):
    """Ingest conversion of test.py:44-45 (skimage rgb2lab in float64 -> float32 -> L - 50)."""
    B, H, W = shape
    rgb = torch.randint(0, 256, (B, H, W, 3), generator=torch.Generator().manual_seed(12), dtype=torch.uint8)
    ref = O.rgb8_to_lab(rgb)
    out = ctx.rgb8_to_lab(rgb.cuda()).cpu()
    assert out.shape == ref.shape == (B, 3, H, W)
    assert (out - ref).abs().max() <= 2e-5  # one fp32 ulp at |Lab| <= 128 is 7.6e-6


def test_colour_round_trip_on_device(ctx):
    """rgb8 -> Lab -> rgb8 reproduces every 8-bit colour of a ramp up to one level (truncating output conversion)."""
    g = torch.arange(0, 256, dtype=torch.uint8)
    rgb = torch.stack((g, g.flip(0), (g.int() * 7 % 256).to(torch.uint8)), -1).view(1, 16, 16, 3)
    lab = ctx.rgb8_to_lab(rgb.cuda())
    back = ctx.lab_to_rgb8(lab[:, 0:1].contiguous(), lab[:, 1:3].contiguous()).cpu()
    assert int((back.int() - rgb.int()).abs().max()) <= 1


# ------------------------------------------------------------------------------------------ §8f rows 2-3
def test_fgs_filter_vs_oracle(ctx):
    """test.py:105-112 at the reference's own "large" size (432 x 768), lambda = 500, sigma_color = 4: every fp32 operation
    of the kernel is the oracle's, so the two agree bit for bit (oracle/prepost_oracle.py; parity with OpenCV unpinned)."""
    from oracle import prepost_oracle as P

    rng = np.random.default_rng(3)
    for H, W in ((432, 768), (37, 50)):
        l = make_lab(90 + H, 1, H, W)[0, 0].numpy()
        guide = P.l_to_guide8(l)
        g_dev = ctx.l_to_guide8(torch.from_numpy(l).cuda())
        assert np.array_equal(g_dev.cpu().numpy(), guide)
        src = (rng.standard_normal((2, H, W)) * 30).astype(np.float32)
        out = ctx.fgs_filter(g_dev, torch.from_numpy(src).cuda()).cpu().numpy()
        ref = P.fgs_filter(guide, src, 500.0, 4.0)
        assert np.isfinite(out).all()
        assert np.array_equal(out, ref), np.abs(out - ref).max()
        assert abs(out.sum() - src.sum()) < 1e-3 * np.abs(src).sum()


@pytest.mark.parametrize("hs,ws,size", [(540, 960, (432, 768)), (480, 640, (432, 768)), (300, 900, (216, 384)), (216, 384, (216, 384)),
                                        (100, 120, (216, 384))])
def test_centerpad_resize_vs_scipy(ctx, hs, ws, size):
    """CenterPad + CenterCrop (test.py:44-46) on the device vs the scipy.ndimage arithmetic skimage.transform.resize uses."""
    from oracle import prepost_oracle as P

    rng = np.random.default_rng(hs + ws)
    img = (rng.random((hs // 4 + 1, ws // 4 + 1, 3)) * 255).astype(np.uint8)
    img = np.kron(img, np.ones((4, 4, 1), np.uint8))[:hs, :ws]  # blocky content + noise: edges and flats
    img = np.clip(img.astype(np.int32) + rng.integers(-9, 10, img.shape), 0, 255).astype(np.uint8)
    ref = P.centerpad_transform(img, size, P.skimage_resize)
    out = ctx.centerpad_rgb8(torch.from_numpy(img).cuda(), size).cpu().numpy()
    diff = np.abs(out.astype(np.int32) - ref.astype(np.int32))
    # float64 on both sides, same operation order; a value within 1e-13 of an integer could still truncate differently
    assert diff.max() <= 1 and (diff > 0).mean() < 1e-5, (diff.max(), (diff > 0).mean())
