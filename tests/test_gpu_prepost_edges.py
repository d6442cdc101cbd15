"""GPU: edge-case parity of the stand-alone pre / post-processing entry points (csrc/prepost.cu and the colour / resampling
kernels of csrc/elementwise.cu).  Every video path is proved equal to the chain of these calls, so what ties its bytes to the
reference is these calls' own parity.  Each comparison is against a CPU reference in float64 or in explicitly ordered float32
numpy (oracle/prepost_oracle.py, oracle/dvc_oracle.py) on seeded or constructed inputs.

Exact (array_equal) where the kernel is a fixed sequence of correctly rounded operations: the Fast Global Smoother, l_to_guide8,
resize_half, upsample2_scaled, and CenterPad's resize whenever the host's taps are scipy's (always the case for their sum; the
taps' exp is libm's, numpy's own exp can differ from it in the last bit, and then a byte may differ by one level where the filtered
value lies on an integer -- that is what is asserted, pixel by pixel).  The colour conversions go through pow / cbrt in double,
which CUDA and numpy may round differently in the last ulp, so they keep the acceptance of tests/test_gpu_prepost.py.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import dvc_oracle as O
from oracle import prepost_oracle as P
from oracle.weights import make_lab
from test_prepost_edges_oracle import _scipy_taps, guide_threshold_inputs

pytestmark = pytest.mark.gpu

DVC_ERR_ARG, DVC_ERR_SHAPE = -1, -2


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------------ Fast Global Smoother
def _guide(kind, H, W, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "flat":
        return np.full((H, W), 93, np.uint8)
    if kind == "vedge":
        return np.where(np.arange(W)[None, :] < W // 2, 0, 255).astype(np.uint8).repeat(H, 0)
    if kind == "hedge":
        return np.where(np.arange(H)[:, None] < H // 2, 0, 255).astype(np.uint8).repeat(W, 1)
    if kind == "checker":
        return (((np.arange(H)[:, None] + np.arange(W)[None, :]) & 1) * 255).astype(np.uint8)
    if kind == "ramp":
        return ((np.arange(H)[:, None] * 3 + np.arange(W)[None, :] * 2) % 256).astype(np.uint8)
    if kind == "random":
        return rng.integers(0, 256, (H, W), dtype=np.uint8)
    assert kind == "luminance"
    return P.l_to_guide8(make_lab(seed + 7, 1, H, W)[0, 0].numpy())


def _planes(n, H, W, seed):
    return (np.random.default_rng(seed).standard_normal((n, H, W)) * 30).astype(np.float32)


def _fgs_exact(ctx, guide, src, lam=500.0, sigma=4.0, att=0.25, it=3):
    out = ctx.fgs_filter(_dev(guide), _dev(src), lam, sigma, att, it).cpu().numpy()
    ref = P.fgs_filter(guide, src, lam, sigma, att, it)
    assert np.isfinite(ref).all()
    bad = out.view(np.int32) != ref.view(np.int32)
    assert not bad.any(), (int(bad.sum()), float(np.abs(out - ref).max()), np.argwhere(bad)[:4].tolist())
    return out


@pytest.mark.parametrize("H,W", [(2, 2), (2, 33), (33, 2), (31, 31), (32, 32), (33, 33), (32, 64), (65, 97), (432, 768), (1080, 1920)])
def test_fgs_shapes_bit_exact(ctx, H, W):
    """Below / at / one past the 32-column tiles and 32-row groups of the horizontal sweep, the smallest sizes the entry point
    takes, the network size and the source-resolution size."""
    _fgs_exact(ctx, _guide("random", H, W, H + W), _planes(2, H, W, H * W))


@pytest.mark.parametrize("planes", [1, 2, 3, 18])
@pytest.mark.parametrize("H,W", [(2, 2), (33, 33), (65, 97)])
def test_fgs_plane_counts_bit_exact(ctx, planes, H, W):
    """Every plane shares the one guide, also past the 8 entries of the kernels' plane table (18 planes = 9 guide lookups)."""
    _fgs_exact(ctx, _guide("luminance", H, W, planes), _planes(planes, H, W, planes))


@pytest.mark.parametrize("kind", ["flat", "vedge", "hedge", "checker", "ramp", "random", "luminance"])
def test_fgs_guides_bit_exact(ctx, kind):
    _fgs_exact(ctx, _guide(kind, 65, 97, 3), _planes(2, 65, 97, 4))


@pytest.mark.parametrize("sigma", [0.25, 4.0, 1000.0])
@pytest.mark.parametrize("lam", [0.0, 1e-3, 500.0, 1e5])
def test_fgs_parameters_bit_exact(ctx, lam, sigma):
    """sigma 0.25 makes most weights subnormal or zero, sigma 1000 makes them all ~1; lambda 1e5 on the flat guide is the
    worst-conditioned system the filter can be given.  lambda = 0 must return the input bits."""
    src = _planes(2, 33, 65, 9)
    for kind in ("ramp", "flat"):
        out = _fgs_exact(ctx, _guide(kind, 33, 65), src, lam, sigma)
        if lam == 0.0:
            assert np.array_equal(out.view(np.int32), src.view(np.int32))


@pytest.mark.parametrize("it,att", [(1, 0.25), (5, 0.25), (3, 1.0), (5, 1.0)])
def test_fgs_iterations_and_attenuation_bit_exact(ctx, it, att):
    _fgs_exact(ctx, _guide("luminance", 37, 50), _planes(3, 37, 50, it), 500.0, 4.0, att, it)


def test_fgs_in_place_and_workspace_reuse(ctx):
    """dev_dst == dev_src through the C ABI gives the out-of-place bits; a small call between two large ones on the same
    workspaces changes nothing (each is compared with the oracle, which has no state)."""
    g, src = _guide("random", 65, 97, 1), _planes(4, 65, 97, 2)
    ref = _fgs_exact(ctx, g, src)
    buf, gd = _dev(src), _dev(g)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = ctypes.c_void_p(buf.data_ptr())
    rc = ctx.lib.dvc_fgs_filter(ctx.h, ctypes.c_void_p(gd.data_ptr()), p, 4, 65, 97, 500.0, 4.0, 0.25, 3, p, s)
    assert rc == 0 and np.array_equal(buf.cpu().numpy().view(np.int32), ref.view(np.int32))
    big_g, big = _guide("luminance", 432, 768), _planes(2, 432, 768, 5)
    first = _fgs_exact(ctx, big_g, big)
    _fgs_exact(ctx, _guide("ramp", 33, 33), _planes(2, 33, 33, 6))
    assert np.array_equal(_fgs_exact(ctx, big_g, big).view(np.int32), first.view(np.int32))


def test_fgs_solves_the_wls_systems(ctx):
    """Against what the filter must compute (float64 sparse solve per line), with the bound the oracle itself is held to."""
    H, W = 64, 96
    g = _guide("random", H, W, 11)
    g[10:20] = g[10:11]  # a flat band: weights exactly 1 along it
    src = _planes(2, H, W, 12)
    out = ctx.fgs_filter(_dev(g), _dev(src)).cpu().numpy()
    ref = P.fgs_reference_f64(g, src, 500, 4)
    assert np.abs(out - ref).max() <= 2e-5 * np.abs(ref).max()
    # flat guide, lambda = 1e5: every line's system is I + lambda_n L with L the path Laplacian, eigenvalues in [1, 1 + 4 lambda_n],
    # so its condition number is below 1 + 4 lambda_n.  Six solves (lambda_n = 1e5, 2.5e4, 6250, two sweeps each), each
    # a contraction in the max norm, each allowed cond * eps32 relative error: 2 * sum(1 + 4 lambda_n) * 2^-24 ~ 0.063.
    flat = _guide("flat", H, W)
    out = ctx.fgs_filter(_dev(flat), _dev(src), 1e5, 4.0).cpu().numpy()
    ref = P.fgs_reference_f64(flat, src, 1e5, 4)
    bound = 2 * sum(1 + 4 * 1e5 * 0.25 ** n for n in range(3)) * 2.0 ** -24
    err = np.abs(out - ref).max() / np.abs(src).max()
    assert err <= bound, (err, bound)
    assert out.std() < 0.05 * src.std()


def test_fgs_invariants_on_device(ctx):
    g = _guide("random", 24, 40, 1)
    const = np.full((1, 24, 40), 7.25, np.float32)
    assert np.abs(ctx.fgs_filter(_dev(g), _dev(const)).cpu().numpy() - 7.25).max() < 1e-3    # constants are fixed points
    src = _planes(3, 24, 40, 2)
    out = ctx.fgs_filter(_dev(g), _dev(src)).cpu().numpy().astype(np.float64)
    assert (np.abs(out.sum((1, 2)) - src.astype(np.float64).sum((1, 2))) < 1e-3 * np.abs(src).sum((1, 2))).all()  # 1^T (I + lam L) = 1^T
    assert torch.equal(ctx.fgs_filter(_dev(g), _dev(src), 0.0, 4.0).cpu(), torch.from_numpy(src))          # lambda = 0: the input bits


# ------------------------------------------------------------------------------------------------ colour
def _all_colours():
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack(((v >> 16) & 255, (v >> 8) & 255, v & 255), -1).astype(np.uint8).reshape(1, 4096, 4096, 3)


def test_every_srgb_colour_to_lab_and_back(ctx):
    """All 2^24 colours in one 4096 x 4096 image: rgb8_to_lab against the float64 oracle; then the device's own Lab back
    through lab_to_rgb8 against the oracle's conversion of that same Lab, and against the colour it came from."""
    rgb = _all_colours()
    lab_dev = ctx.rgb8_to_lab(_dev(rgb))
    back_dev = ctx.lab_to_rgb8(lab_dev[:, 0:1].contiguous(), lab_dev[:, 1:3].contiguous()).cpu().numpy()
    lab = lab_dev.cpu()
    worst, worst_at, differing = 0.0, None, 0
    for r0 in range(0, 4096, 512):  # the float64 oracles, 2^21 colours at a time
        sl = slice(r0, r0 + 512)
        d = (lab[:, :, sl] - O.rgb8_to_lab(torch.from_numpy(rgb[:, sl]))).abs()
        if float(d.max()) > worst:
            worst = float(d.max())
            _, _, y, x = np.unravel_index(int(d.argmax()), d.shape)
            worst_at = rgb[0, r0 + y, x].tolist()
        ref_back = O.lab_to_rgb8(lab[:, 0:1, sl], lab[:, 1:3, sl]).numpy()
        dd = np.abs(back_dev[:, sl].astype(np.int16) - ref_back.astype(np.int16))
        assert dd.max() <= 1
        differing += int((dd > 0).sum())
    assert worst <= 2e-5, (worst, worst_at)  # one fp32 ulp at |Lab| <= 128 is 7.6e-6
    print(f"rgb8_to_lab worst |error| {worst:.3g} at colour {worst_at}; round trip: {differing} of {3 << 24} values differ from the oracle")
    assert differing <= 1e-5 * (3 << 24), differing  # pow's last ulp, see test_gpu_prepost.py
    assert np.abs(back_dev.astype(np.int16) - rgb.astype(np.int16)).max() <= 1  # truncating output conversion


def _check_lab_to_rgb8(ctx, l, ab, what):
    ref = O.lab_to_rgb8(l, ab)
    out = ctx.lab_to_rgb8(l.cuda(), ab.cuda()).cpu()
    assert out.shape == ref.shape and out.dtype == torch.uint8
    d = (out.int() - ref.int()).abs()
    n = int((d > 0).sum())
    print(f"lab_to_rgb8 {what}: {n} of {d.numel()} values differ from the float64 oracle")
    # CUDA's and numpy's double pow() may differ in the last ulp, which flips a truncation only when v * 255 sits within
    # ~1e-13 of an integer: one level, on at most 1e-5 of the values (none at all for a small input)
    assert int(d.max()) <= 1 and n <= 1e-5 * d.numel(), (what, int(d.max()), n)


def test_lab_to_rgb8_lattice(ctx):
    L = torch.linspace(-50, 50, 101)
    a = torch.linspace(-128, 127, 65)
    l = L.view(101, 1, 1).expand(101, 65, 65).reshape(1, 1, 101, 65 * 65).contiguous()
    ab = torch.stack((a.view(1, 65, 1).expand(101, 65, 65), a.view(1, 1, 65).expand(101, 65, 65))).reshape(1, 2, 101, 65 * 65).contiguous()
    _check_lab_to_rgb8(ctx, l, ab, "lattice")


def test_lab_to_rgb8_at_its_thresholds(ctx):
    """Inputs a few float32 ulps on either side of each branch: f = 0.2068966 in each of f_x, f_y, f_z (the cube / linear
    switch), f_z = 0 (the clamp), v = 0.0031308 (the gamma switch, reached on a grey), black and white, the corners of ab."""
    thr = 0.2068966
    fy_mid = (50.0 + 16.0) / 116.0
    cases = [(116 * thr - 16 - 50, 0.0, 0.0),                       # f_y (and with ab = 0 f_x, f_z) at the threshold
             (0.0, 500 * (thr - fy_mid), 0.0),                      # f_x
             (0.0, 0.0, 200 * (fy_mid - thr)),                      # f_z
             (0.0, 0.0, 200 * fy_mid),                              # f_z = 0
             (-40.0, 0.0, 200 * (10.0 + 16.0) / 116.0),             # f_z = 0 with a dark L
             (116 * (7.787 * 0.0031308 + 16 / 116) - 16 - 50, 0.0, 0.0),  # v = 0.0031308 on a grey
             (-50.0, 0.0, 0.0)]  # white is checked below: its channels sit on 1.0 to the last bit, either side of the truncation
    pts = []
    for c in cases:
        c32 = np.array(c, np.float32)
        for k in range(3):
            lo = hi = c32[k]
            for _ in range(3):
                lo, hi = np.nextafter(lo, np.float32(-1e9)), np.nextafter(hi, np.float32(1e9))
                for v in (lo, hi):
                    q = c32.copy()
                    q[k] = v
                    pts.append(q)
        pts.append(c32)
    for L in (-50.0, 0.0, 50.0):
        for a in (-128.0, 127.0):
            for b in (-128.0, 127.0):
                pts.append(np.array((L, a, b), np.float32))
    pts = torch.from_numpy(np.stack(pts))
    n = pts.shape[0]
    _check_lab_to_rgb8(ctx, pts[:, 0].reshape(1, 1, 1, n).contiguous(), pts[:, 1:3].t().reshape(1, 2, 1, n).contiguous(), "thresholds")
    black_white = ctx.lab_to_rgb8(torch.tensor([-50.0, 50.0]).view(2, 1, 1, 1).cuda(), torch.zeros(2, 2, 1, 1).cuda()).cpu()
    assert black_white[0].tolist() == [[[0, 0, 0]]] and black_white[1].min() >= 254


@pytest.mark.parametrize("shape", [(1, 1, 1), (3, 7, 13), (9, 5, 7), (12, 5, 7), (2, 1080, 1920)])
def test_lab_to_rgb8_batches_and_shapes(ctx, shape):
    """More batches than the 8 entries of the kernel's plane table (batch b must read L plane b), H * W below and not a
    multiple of the block, and the source-resolution size."""
    B, H, W = shape
    g = torch.Generator().manual_seed(B * H + W)
    l = torch.rand(B, 1, H, W, generator=g) * 100 - 50
    ab = (torch.rand(B, 2, H, W, generator=g) * 2 - 1) * 110
    _check_lab_to_rgb8(ctx, l, ab, str(shape))
    rgb = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    assert (ctx.rgb8_to_lab(rgb.cuda()).cpu() - O.rgb8_to_lab(rgb)).abs().max() <= 2e-5


def test_l_to_guide8_at_every_threshold(ctx):
    l = guide_threshold_inputs()
    l = np.concatenate([l, np.zeros(-len(l) % 37, np.float32)]).reshape(37, -1)
    assert np.array_equal(ctx.l_to_guide8(_dev(l)).cpu().numpy(), P.l_to_guide8(l))


# ------------------------------------------------------------------------------------------------ resize_half / upsample2
def _awkward(shape, seed):
    """Normal values, plus zeros, magnitudes near the top of the range (a sum of two halves, or 1.25 x one value, still
    finite) and subnormals."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(shape) * 40).astype(np.float32)
    pick = rng.integers(0, 12, shape)
    x[pick == 0] = 0.0
    x[pick == 1] *= np.float32(5e35)
    x[pick == 2] *= np.float32(1e-40)
    x[pick == 3] = np.float32(1e-45)
    return x


@pytest.mark.parametrize("shape", [(1, 1, 2, 2), (1, 1, 2, 4096), (3, 5, 6, 10), (8, 3, 432, 768), (2, 3, 1080, 1920)])
def test_resize_half_bit_exact(ctx, shape):
    """(8, 3, 432, 768) and (2, 3, 1080, 1920) have more outputs than the launch has threads: the grid-stride loop repeats."""
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(31)) * 40
    out = ctx.resize_half(x.cuda()).cpu()
    assert torch.equal(out, torch.from_numpy(P.resize_half_f32(x.numpy())))
    assert (out - O.resize_half(x)).abs().max() <= 1e-5 * x.abs().max()
    y = _awkward(shape, 32)
    out = ctx.resize_half(_dev(y)).cpu().numpy()
    assert np.array_equal(out.view(np.int32), P.resize_half_f32(y).view(np.int32))


def test_resize_half_refuses_a_misaligned_pointer(ctx):
    """A contiguous view at an odd float offset is not 8-byte aligned: the C entry point refuses it before any launch (the
    kernel loads pairs of floats), and the Python call copies it to an aligned tensor first."""
    base = torch.randn(1 + 3 * 6 * 10, generator=torch.Generator().manual_seed(33)).cuda()
    view = base[1:].view(1, 3, 6, 10)
    assert view.is_contiguous() and view.data_ptr() % 8 == 4
    out = torch.empty(1, 3, 3, 5, device="cuda")
    n = ctx.launch_count()
    rc = ctx.lib.dvc_resize_half(ctx.h, ctypes.c_void_p(view.data_ptr()), 3, 6, 10, ctypes.c_void_p(out.data_ptr()),
                                 ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == DVC_ERR_ARG and ctx.launch_count() == n
    assert torch.equal(ctx.resize_half(view).cpu(), torch.from_numpy(P.resize_half_f32(view.cpu().numpy())))


@pytest.mark.parametrize("shape", [(1, 2, 1, 1), (1, 2, 1, 7), (1, 2, 7, 1), (5, 3, 3, 5), (16, 2, 216, 384), (2, 2, 540, 960)])
def test_upsample2_scaled_bit_exact(ctx, shape):
    """The kernel fuses one product of every sum into the addition (fmaf), the one spelled out in csrc/elementwise.cu;
    P.upsample2_scaled_f32 states the same sequence, and the separately rounded expression would differ in the last bit."""
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(34)) * 60
    out = ctx.upsample2_scaled(x.cuda(), 1.25).cpu()
    assert torch.equal(out, torch.from_numpy(P.upsample2_scaled_f32(x.numpy(), 1.25)))
    assert (out - O.upsample2_scaled(x, 1.25)).abs().max() <= 1e-5 * x.abs().max()
    y = _awkward(shape, 35)
    for scale in (1.25, 1.0):
        out = ctx.upsample2_scaled(_dev(y), scale).cpu().numpy()
        assert np.array_equal(out.view(np.int32), P.upsample2_scaled_f32(y, scale).view(np.int32))


# ------------------------------------------------------------------------------------------------ CenterPad
def _content(kind, hs, ws, seed=0):
    rng = np.random.default_rng(seed)
    if kind in ("0", "128", "255"):
        return np.full((hs, ws, 3), int(kind), np.uint8)
    if kind == "blocks":
        img = rng.integers(0, 256, (hs // 20 + 1, ws // 20 + 1, 3), dtype=np.uint8)
        return np.kron(img, np.ones((20, 20, 1), np.uint8))[:hs, :ws]
    if kind == "split":
        img = np.zeros((hs, ws, 3), np.uint8)
        img[:, ws // 2:] = 255
        img[hs // 2:, :, 1] = 255 - img[hs // 2:, :, 1]
        return img
    if kind == "ramp":
        return ((np.arange(hs)[:, None, None] + np.arange(ws)[None, :, None] * 2 + np.arange(3) * 85) % 256).astype(np.uint8)
    assert kind == "noise"
    return rng.integers(0, 256, (hs, ws, 3), dtype=np.uint8)


def _taps_are_scipys(in_len, out_len):
    import dvc

    return in_len <= out_len or np.array_equal(np.array(dvc.resize_taps(in_len, out_len)), _scipy_taps(in_len, out_len))


def _resize_crop(ctx, img, Hr, Wr, oy, ox, Ho, Wo):
    src, out = _dev(img), torch.empty(Ho, Wo, 3, device="cuda", dtype=torch.uint8)
    rc = ctx.lib.dvc_resize_antialias_crop_rgb8(ctx.h, ctypes.c_void_p(src.data_ptr()), img.shape[0], img.shape[1], Hr, Wr, oy, ox,
                                                ctypes.c_void_p(out.data_ptr()), Ho, Wo,
                                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return rc, out.cpu().numpy()


def _check_against_scipy(out, img, Hr, Wr, oy, ox, what):
    """The CenterPad guarantee: the bytes of scipy's arithmetic exactly whenever the host's taps are scipy's and no axis is
    up-scaled; otherwise at most one level, and only where scipy's float64 value lies on an integer (flat areas).  The two
    causes: numpy's exp differing from libm's in some tap's last bit, and, when up-scaling, the sample points before the first
    and after the last source pixel, which scipy mirrors into the image before it splits them into index and weight while
    zoom_crop_kernel splits first and mirrors the index (the same neighbours, weights one rounding apart)."""
    Ho, Wo = out.shape[:2]
    full = P.skimage_resize(img, (Hr, Wr))
    assert full.shape == (Hr, Wr, 3)
    val = np.zeros((Ho, Wo, 3))
    ys, xs = np.arange(Ho) + oy, np.arange(Wo) + ox
    my, mx = (ys >= 0) & (ys < Hr), (xs >= 0) & (xs < Wr)
    val[np.ix_(my, mx)] = full[np.ix_(ys[my], xs[mx])]
    ref = np.clip(np.trunc(val), 0, 255).astype(np.uint8)
    if _taps_are_scipys(img.shape[0], Hr) and _taps_are_scipys(img.shape[1], Wr) and img.shape[0] >= Hr and img.shape[1] >= Wr:
        bad = out != ref
        assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4].tolist())
        return
    d = np.abs(out.astype(np.int16) - ref.astype(np.int16))
    assert d.max() <= 1, (what, int(d.max()))
    off = np.abs(val[d > 0] - np.rint(val[d > 0]))
    print(f"centerpad {what}: not held to exact equality; {int((d > 0).sum())} bytes one level off, all on integers")
    assert off.size == 0 or off.max() <= 1e-9, (what, float(off.max()))


BIG = [((1440, 2560), (432, 768)), ((1000, 3000), (64, 96))]
OTHER = [((2160, 3840), (432, 768)), ((1080, 1920), (432, 768)), ((2160, 3840), (216, 384)), ((1280, 720), (432, 768)), ((360, 640), (108, 192))]
CASES = [(s, t, k) for s, t in BIG for k in ("0", "255", "128", "blocks", "split", "ramp", "noise")] + \
        [(s, t, k) for s, t in OTHER for k in ("255", "blocks", "noise")]


@pytest.mark.parametrize("src,size,kind", CASES)
def test_centerpad_large_downscales_vs_scipy(ctx, src, size, kind):
    """Down-scales of 2.5x to 31x (radius 3 to 61) on flat, blocky, split, ramp and noisy content: flat areas put the filtered
    value on an integer, where the truncation to uint8 sees the taps' last bit."""
    from dvc.prepost import centerpad_geometry

    img = _content(kind, src[0], src[1], src[0] + size[0])
    Hr, Wr, oy, ox = centerpad_geometry(src[0], src[1], size)
    out = ctx.centerpad_rgb8(_dev(img), size).cpu().numpy()
    _check_against_scipy(out, img, Hr, Wr, oy, ox, (src, size, kind))
    if kind == "noise" and size == (64, 96):
        assert np.abs(P.centerpad_transform(img, size, P.skimage_resize).astype(np.int16) - out).max() <= 1


@pytest.mark.parametrize("src,resized,window", [
    ((1, 500), (1, 50), (-1, 5, 4, 40)),        # one source row (the mirror of a 1-pixel axis), window partly above and beside
    ((500, 1), (50, 1), (10, -2, 30, 6)),       # one source column
    ((3, 2000), (1, 100), (0, 0, 1, 100)),      # radius 4 on a 3-pixel axis: the mirror wraps more than a period
    ((3, 2000), (1, 100), (-2, 90, 5, 20)),     # partly outside on every side
    ((40, 60), (20, 30), (-5, -7, 30, 44)),     # the resized image strictly inside the window
    ((40, 60), (20, 30), (23, 0, 8, 8)),        # wholly outside: zeros
    ((3, 4000), (3, 2), (0, 0, 3, 2)),          # 7997 taps, just inside the 8192 the entry point accepts
])
def test_resize_crop_geometry_through_the_c_abi(ctx, src, resized, window):
    oy, ox, Ho, Wo = window
    for kind in ("noise", "255"):
        img = _content(kind, src[0], src[1], 5)
        rc, out = _resize_crop(ctx, img, resized[0], resized[1], oy, ox, Ho, Wo)
        assert rc == 0
        _check_against_scipy(out, img, resized[0], resized[1], oy, ox, (src, resized, window, kind))
        if oy >= resized[0]:
            assert not out.any()


def test_resize_refuses_more_than_8192_taps(ctx):
    img = _content("noise", 3, 5000)
    n = ctx.launch_count()
    rc, _ = _resize_crop(ctx, img, 3, 2, 0, 0, 3, 2)   # 5000 -> 2: sigma 1249.5, radius 4998, 9997 taps
    assert rc == DVC_ERR_SHAPE and ctx.launch_count() == n
