"""Per-layer parity of the convolution engines (run with -m gpu on an H100): ONE nn.Conv2d of the reference
(NonlocalNet.py:235-255,364-423; ColorVidNet.py:96-143) through dvc_debug_conv2d -- the same engine, operand planes and
epilogue the layer programs use -- against F.conv2d evaluated in float64 on the CPU with the same seeded weights.

What this pins that the network-level goldens cannot: the channel tile is FORCED (tc_force_bn = 256 / 128 / 64), so the
256-channel CTA-pair tile that the 480x864 bench runs on (and that the launcher's heuristic never picks at the golden
sizes) is compared with the oracle at small M, and then again at the bench's own geometry (208 pixel tiles = two rounds
of the persistent grid; 108 tiles of the 512-channel layers).

Tolerances: max|y - y64| <= 4e-6 * max|y64| (fp32-class accumulation over K = 9 * Cin <= 4608 products: the
reference's own fp32 F.conv2d is printed beside it); InstanceNorm sums (of the stored fp32 values, against fp64 sums of
the fp64 values): 1e-5 relative to the sum of |values|.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

VGG, WARP, COLOR = 0, 1, 2
NETKEY = {VGG: "vgg", WARP: "warp", COLOR: "color"}


def ref_conv(sd, name, x, dil=1, stride=1, act=0, slope=0.0, reflect=False, upconv=False, add=None, dtype=torch.float64):
    w, b = sd[name + ".weight"].to(dtype), sd[name + ".bias"].to(dtype)
    x = x.to(dtype)
    if upconv:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    k = w.shape[2]
    if k == 3:
        x = F.pad(x, (dil,) * 4, mode="reflect" if reflect else "constant")
    y = F.conv2d(x, w, b, stride=stride, dilation=dil)
    if add is not None:
        y = y + add.to(dtype)
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = F.leaky_relu(y, slope)
    return y


def make_input(seed, B, C, H, W, nonneg):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, H, W, generator=g)
    # per-channel gains over two decades, like real feature maps; ReLU outputs are non-negative
    x = x * torch.logspace(-1, 1, C).view(1, C, 1, 1)[:, torch.randperm(C, generator=g)]
    return x.abs() if nonneg else x


@pytest.fixture(params=["pair", "single"])
def engine(request, ctx):
    import dvc

    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    ctx.debug_flag("tc_cluster", 2 if request.param == "pair" else 1)
    yield request.param
    ctx.debug_flag("tc_cluster", 2)
    ctx.debug_flag("tc_force_bn", 0)


# (id, net, weight name, Cin, Cout, H, W, kwargs)
LAYERS = [
    ("vgg_conv3_2_relu", VGG, "conv3_2", 256, 256, 24, 40, dict(act=1, nonneg=True)),
    ("vgg_conv4_2_relu", VGG, "conv4_2", 512, 512, 16, 24, dict(act=1, nonneg=True)),
    ("warp_res_conv1_reflect_stats", WARP, "layer.0.conv1", 256, 256, 24, 32, dict(reflect=True, want_stats=True)),
    ("warp_theta_1x1_stats", WARP, "theta", 256, 256, 24, 32, dict(want_stats=True)),
    ("warp_head_stride2", WARP, "layer2_1.5", 128, 64, 32, 48, dict(stride=2, reflect=True, want_stats=True)),
    ("color_conv5_2_dil2", COLOR, "conv5_2", 512, 512, 16, 24, dict(act=1, dil=2, nonneg=True)),
    ("color_conv6_3_dil2_stats", COLOR, "conv6_3", 512, 512, 16, 24, dict(act=1, dil=2, nonneg=True, want_stats=True)),
    ("color_conv8_1_upconv_add", COLOR, "conv8_1.1", 512, 256, 12, 16, dict(act=1, upconv=True, with_add=True)),
    ("color_conv9_1_upconv_add", COLOR, "conv9_1.1", 256, 128, 12, 16, dict(act=1, upconv=True, with_add=True)),
    ("color_conv3_3_short", COLOR, "conv3_3_short", 256, 256, 24, 32, dict()),
    ("color_conv10_2_fused_tail", COLOR, "conv10_2", 128, 128, 24, 32, dict(act=2, slope=0.2, fuse_tail=True, nonneg=True)),
]


_REF = {}  # the CPU fp64 / fp32 references are shared by the engine / tile variants of a layer


def reference(sds, net, name, cin, cout, H, W, B, seed, nonneg, with_add, fuse_tail, kw, sd=None):
    key = (net, name, H, W, B, seed, nonneg, with_add, fuse_tail, tuple(sorted(kw.items())))
    if key not in _REF:
        sd = sds[NETKEY[net]] if sd is None else sd
        assert tuple(sd[name + ".weight"].shape[:2]) == (cout, cin), (name, sd[name + ".weight"].shape)
        x = make_input(1234 + seed, B, cin, H, W, nonneg)
        add = None
        if with_add:  # an addend of the output's shape
            st = kw.get("stride", 1)
            Ho, Wo = (2 * H, 2 * W) if kw.get("upconv") else ((H + st - 1) // st, (W + st - 1) // st)
            add = torch.randn(B, cout, Ho, Wo, generator=torch.Generator().manual_seed(99 + seed)) * 3
        with torch.no_grad():
            y64 = ref_conv(sd, name, x, add=add, **kw)
            y32 = ref_conv(sd, name, x, add=add, dtype=torch.float32, **kw)
            if fuse_tail:  # ColorVidNet.py:143-144
                tail = lambda y: torch.tanh(F.conv2d(y, sds["color"]["conv10_ab.weight"].to(y.dtype), sds["color"]["conv10_ab.bias"].to(y.dtype))) * 128
                y64, y32 = tail(y64), tail(y32)
        _REF[key] = (x, add, y64, y32)
    return _REF[key]


def run_layer(ctx, sds, net, name, cin, cout, H, W, B=1, seed=0, out_planes=False, sd=None, in_bound=None, **kw):
    """One layer through dvc_debug_conv2d against fp64.  sd: the layer's own state dict (synthetic layers loaded under
    test-only names) instead of the network's.  Returns (max error, reference fp32 floor), both relative to max |y64|."""
    kw = dict(kw)
    nonneg, with_add, want_stats = kw.pop("nonneg", False), kw.pop("with_add", False), kw.pop("want_stats", False)
    fuse_tail = kw.pop("fuse_tail", False)
    x, add, y64, y32 = reference(sds, net, name, cin, cout, H, W, B, seed, nonneg, with_add, fuse_tail, kw, sd)
    res = ctx.debug_conv2d(net, name, x.cuda(), cout, dil=kw.get("dil", 1), stride=kw.get("stride", 1), act=kw.get("act", 0),
                           slope=kw.get("slope", 0.0), reflect=kw.get("reflect", False), upconv=kw.get("upconv", False),
                           fuse_tail=fuse_tail, out_planes=out_planes, add=add.cuda() if add is not None else None,
                           want_stats=want_stats, in_bound=in_bound)
    y, st = res if want_stats else (res, None)
    y = y.cpu().double()
    scale = y64.abs().max().item()
    err, floor = (y - y64).abs().max().item() / scale, (y32.double() - y64).abs().max().item() / scale
    if st is not None:
        st = st.cpu()
        s64 = torch.stack((y64.sum((2, 3)), (y64 * y64).sum((2, 3))), -1)
        a64 = torch.stack((y64.abs().sum((2, 3)), (y64 * y64).sum((2, 3))), -1)
        serr = ((st - s64).abs() / a64.clamp_min(1e-30)).max().item()
        assert serr < 1e-5, ("InstanceNorm sums", name, serr)
    return err, floor


@pytest.mark.parametrize("force_bn", [0, 256, 128, 64])
@pytest.mark.parametrize("layer", LAYERS, ids=[l[0] for l in LAYERS])
def test_layer_vs_fp64_conv2d(ctx, sds, engine, layer, force_bn):
    _, net, name, cin, cout, H, W, kw = layer
    ctx.debug_flag("tc_force_bn", force_bn)
    err, floor = run_layer(ctx, sds, net, name, cin, cout, H, W, **kw)
    # the fused tail ends in tanh * 128: compare absolute (|ab| <= 128)
    assert err <= 4e-6, (layer[0], force_bn, engine, err, floor)


@pytest.mark.parametrize("force_bn", [0, 256, 64])
@pytest.mark.parametrize("layer", [l for l in LAYERS if l[7].get("act") == 1 and not l[7].get("want_stats")], ids=lambda l: l[0])
def test_layer_device_scaled_output_planes(ctx, sds, engine, layer, force_bn):
    """The conv -> ReLU -> conv chains store fp16 hi/lo planes with an exponent derived on the device: read back
    through those planes, the layer must be as close to fp64 as through the fp32 store."""
    _, net, name, cin, cout, H, W, kw = layer
    ctx.debug_flag("tc_force_bn", force_bn)
    err, floor = run_layer(ctx, sds, net, name, cin, cout, H, W, out_planes=True, **kw)
    assert err <= 4e-6, (layer[0], force_bn, engine, err, floor)


def test_layer_batch2_tiles_straddle_images(ctx, sds, engine):
    """B = 2: pixel tiles that straddle the image boundary take the per-pixel statistics path."""
    ctx.debug_flag("tc_force_bn", 256)
    err, _ = run_layer(ctx, sds, WARP, "layer.1.conv2", 256, 256, 20, 24, B=2, reflect=True, want_stats=True)
    assert err <= 4e-6, err


# ---- the bench's own geometry (480x864 frame: 120x216 quarter-resolution, 60x108 eighth-resolution maps) ----
BENCH = [
    # layers with more than 64 output channels run on the 128 x 128 tile unless another tile is forced (conv_tc.cu)
    ("quarter_256_208tiles", VGG, "conv3_2", 256, 256, 120, 216, dict(act=1, nonneg=True), 128),
    ("quarter_256_reflect_stats", WARP, "layer.0.conv1", 256, 256, 120, 216, dict(reflect=True, want_stats=True), 128),
    ("eighth_512_108tiles", VGG, "conv4_2", 512, 512, 60, 108, dict(act=1, nonneg=True), 128),
    ("eighth_512_dil2_stats", COLOR, "conv5_3", 512, 512, 60, 108, dict(act=1, dil=2, nonneg=True, want_stats=True), 128),
    ("half_128", VGG, "conv2_2", 128, 128, 240, 432, dict(act=1, nonneg=True), 128),
    # the four phases of conv8_1 each see 54 pixel tiles of the 1/8-resolution input: the launcher narrows to 128 channels
    ("quarter_upconv_256", COLOR, "conv8_1.1", 512, 256, 60, 108, dict(act=1, upconv=True, with_add=True), 128),
]


@pytest.mark.parametrize("force_bn", [256, 128])
@pytest.mark.parametrize("layer", BENCH[:4], ids=[l[0] for l in BENCH[:4]])
def test_layer_at_bench_geometry_forced_tile(ctx, sds, layer, force_bn):
    """The 64 x 256 and 128 x 128 tiles at the bench's geometry."""
    import dvc

    _, net, name, cin, cout, H, W, kw, _ = layer
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    ctx.debug_flag("tc_cluster", 2)
    ctx.debug_flag("tc_force_bn", force_bn)
    try:
        err, floor = run_layer(ctx, sds, net, name, cin, cout, H, W, **kw)
    finally:
        ctx.debug_flag("tc_force_bn", 0)
    assert err <= 4e-6, (layer[0], force_bn, err, floor)


@pytest.mark.parametrize("layer", BENCH, ids=[l[0] for l in BENCH])
def test_layer_at_bench_geometry(ctx, sds, layer):
    """Default engine, the launcher's own tile choice (asserted to be the bench's), full-size layer vs fp64."""
    import dvc

    _, net, name, cin, cout, H, W, kw, expect_bn = layer
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    ctx.debug_flag("tc_force_bn", 0)
    ctx.debug_flag("tc_cluster", 2)
    ctx.profile_conv(True)
    ctx.conv_profile(0, reset=True)
    try:
        err, floor = run_layer(ctx, sds, net, name, cin, cout, H, W, **kw)
        torch.cuda.synchronize()
        n_expected = ctx.conv_profile(expect_bn)[0]
    finally:
        ctx.conv_profile(0, reset=True)
        ctx.profile_conv(False)
    assert n_expected >= 1, f"the launcher did not pick the {expect_bn}-channel tile at the bench geometry"
    print(f"{layer[0]}: |y - y64| / max = {err:.2e} (reference fp32 conv2d: {floor:.2e})")
    assert err <= 4e-6, (layer[0], err, floor)
