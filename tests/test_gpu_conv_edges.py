"""Edge-case parity of the convolution engines (run with -m gpu on an H100).

test_gpu_conv_layers.py checks the real layers of the three nets at friendly sizes (H, W multiples of 8, Cin and Cout
multiples of 64).  This module runs the shapes where the engines' bookkeeping can go wrong, on seeded synthetic layers
loaded under test-only names ("edge.c<cin>_o<cout>_k<k>" of NET_COLOR, which no layer program reads) and on the real
up-convolution and fused-tail layers, each against an fp64 F.conv2d:

  - channel padding: Cout 32 / 40 / 72 / 200 / 264 / 320 (the tensor-core weight block is padded to 64 / 128 / 512, so
    whole channel tiles lie past Cout) and Cin 32 / 96 / 160 (fp16 operands with 64-byte K rows) as well as 64 / 256;
  - pixel tails: B * Hp * Wp below one tile, at and just past 128 * k (126, 128, 129, 255, 259 -- 127 and 257 are prime,
    so no B * Hp * Wp with Hp, Wp >= 3 reaches them), odd tile counts under 2-CTA clusters (the peer CTA's tile lies
    wholly past the last pixel), B = 3 / 5 with image boundaries inside 64- and 128-pixel tiles;
  - geometry: zero / reflect 3x3, 1x1, stride 2 on odd sizes, dilation 2 with reflect padding at W = 3, dilation 3 and 4,
    up-convolution phases at 1 x N, 1 x 1 and odd x odd low-resolution sizes, the fused conv10_2 -> conv10_ab tail;
  - epilogues: none / ReLU / LeakyReLU 0.2 and 3, skip addend, InstanceNorm sums;
  - engines: every case under each channel tile that divides its padded Cout and under single CTAs and 2-CTA clusters,
    with one of fp16 planes (default), tf32 planes, 64-byte K rows, the tail split of 256-channel launches, device-scaled
    fp16 output planes, or the exact-fp32 CUDA-core engine.

Then the exact invariants the engine promises (split-K, clusters, batch), the first-layer kernel at widths that are not
multiples of 8, and the scale-bound adversaries of oracle/conv_adversary.py, whose outputs reach the bound that sizes
the device-scaled fp16 store.  Tolerances are test_gpu_conv_layers.py's: max |y - y64| <= 4e-6 max |y64|, InstanceNorm
sums 1e-5 of the sums of |values|; the reference's own fp32 error is printed beside each result.
"""
import math

import pytest
import torch

from oracle import conv_adversary as ADV
from test_gpu_conv_layers import COLOR, VGG, ref_conv, run_layer

pytestmark = pytest.mark.gpu

TOL = 4e-6
_LOADED = set()


@pytest.fixture(autouse=True)
def defaults(ctx):
    """Every test starts and ends on the library's default engine settings."""
    import dvc

    def reset():
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        for flag, v in (("tc_cluster", 2), ("tc_force_bn", 0), ("tc_f16", 1), ("tc_kbytes", 128), ("tc_tail", 0),
                        ("tc_splits", 1)):
            ctx.debug_flag(flag, v)

    reset()
    yield
    reset()


def load_synthetic(ctx, cin, cout, k=3):
    """(name, state dict) of a seeded synthetic layer, loaded into NET_COLOR once per session (bias first: the
    weight's upload copies the bias it has seen)."""
    import dvc

    name, sd = ADV.synthetic_layer(cin, cout, k)
    if name not in _LOADED:
        ctx.set_weights(dvc.NET_COLOR, {name + ".bias": sd[name + ".bias"], name + ".weight": sd[name + ".weight"]})
        _LOADED.add(name)
    return name, sd


def cout_pad_tc(cout):
    bn = 256 if cout >= 256 else (128 if cout > 64 else 64)  # conv_tc.cu: conv_tc_pick_bn
    return (cout + bn - 1) // bn * bn


# (id, layer, H, W, B, kwargs, engine).  layer: (cin, cout, k) synthetic, or (name, cin, cout) of ColorVidNet.
# engine: "f16" default fp16 planes, "tf32" tc_f16 = 0, "kb64" tc_kbytes = 64, "tail16" tc_tail = 16 (the 256 / 128
# tail split with 16 pretend SM pairs), "planes" device-scaled fp16 output planes, "fp32" the CUDA-core engine.
CASES = [
    # channel padding and tiny pixel counts
    ("c32_o32_1x1", (32, 32, 3), 1, 1, 1, dict(act=1), "f16"),
    ("c96_o40_1x9_b5_lrelu_stats", (96, 40, 3), 1, 9, 5, dict(act=2, slope=0.2, want_stats=True), "f16"),
    ("c160_o72_3x3_b3_reflect_add_stats", (160, 72, 3), 3, 3, 3, dict(reflect=True, with_add=True, want_stats=True), "tf32"),
    ("c64_o200_5x13_b3_relu_stats", (64, 200, 3), 5, 13, 3, dict(act=1, want_stats=True), "kb64"),
    ("c256_o264_7x17_reflect_stats", (256, 264, 3), 7, 17, 1, dict(reflect=True, want_stats=True), "f16"),
    ("c32_o320_11x29_lrelu3", (32, 320, 3), 11, 29, 1, dict(act=2, slope=3.0), "planes"),
    ("c160_o264_11x29_b2_relu", (160, 264, 3), 11, 29, 2, dict(act=1, nonneg=True), "planes"),
    # 1x1
    ("k1_c64_o72_5x13_b2_relu_stats", (64, 72, 1), 5, 13, 2, dict(act=1, want_stats=True), "f16"),
    ("k1_c96_o264_7x17_add", (96, 264, 1), 7, 17, 1, dict(with_add=True), "tf32"),
    ("k1_c32_o200_1x9_b3_stats", (32, 200, 1), 1, 9, 3, dict(want_stats=True), "planes"),
    # stride 2 on odd sizes
    ("s2_c64_o40_7x17_b2_reflect_stats", (64, 40, 3), 7, 17, 2, dict(stride=2, reflect=True, want_stats=True), "f16"),
    ("s2_c160_o200_11x29_relu", (160, 200, 3), 11, 29, 1, dict(stride=2, act=1), "tf32"),
    ("s2_c256_o72_5x13_b3_add_stats", (256, 72, 3), 5, 13, 3, dict(stride=2, with_add=True, want_stats=True), "kb64"),
    # dilation 2 with reflect padding at the smallest width, dilation 3 and 4
    ("d2_c64_o72_5x3_b3_reflect_lrelu_stats", (64, 72, 3), 5, 3, 3, dict(dil=2, reflect=True, act=2, slope=0.2, want_stats=True), "f16"),
    ("d2_c256_o320_3x3_b2_reflect_relu", (256, 320, 3), 3, 3, 2, dict(dil=2, reflect=True, act=1), "planes"),
    ("d3_c64_o72_7x17_relu", (64, 72, 3), 7, 17, 1, dict(dil=3, act=1), "f16"),
    ("d3_c96_o32_11x29_lrelu3", (96, 32, 3), 11, 29, 1, dict(dil=3, act=2, slope=3.0), "tf32"),
    ("d4_c256_o200_5x13_b2_stats", (256, 200, 3), 5, 13, 2, dict(dil=4, want_stats=True), "f16"),
    ("d4_c32_o264_3x3_b5_relu", (32, 264, 3), 3, 3, 5, dict(dil=4, act=1), "planes"),
    # B * Hp * Wp around one and two 128-pixel tiles
    ("m126_c64_o40_5x7_b2_relu_stats", (64, 40, 3), 5, 7, 2, dict(act=1, want_stats=True), "f16"),
    ("m128_c256_o72_6x6_b2_stats", (256, 72, 3), 6, 6, 2, dict(want_stats=True), "f16"),
    ("m129_c32_o200_1x41_relu", (32, 200, 3), 1, 41, 1, dict(act=1), "tf32"),
    ("m255_c160_o264_1x15_b5_stats", (160, 264, 3), 1, 15, 5, dict(want_stats=True), "f16"),
    ("m255_c96_o200_3x15_b3_relu_add", (96, 200, 3), 3, 15, 3, dict(act=1, with_add=True), "kb64"),
    ("m259_c64_o320_5x35_lrelu_stats", (64, 320, 3), 5, 35, 1, dict(act=2, slope=0.2, want_stats=True), "f16"),
    # 256-channel launch split into whole rounds of the 256-channel tile and a 128-channel tail (39 pixel tiles)
    ("tail_c64_o256_61x77_stats", (64, 256, 3), 61, 77, 1, dict(want_stats=True), "tail16"),
    # up-convolution phases (nearest x2 + 3x3 as four 2x2 convolutions) with the skip addend
    ("up8_1x5", ("conv8_1.1", 512, 256), 1, 5, 1, dict(act=1, upconv=True, with_add=True), "f16"),
    ("up8_5x7_b2", ("conv8_1.1", 512, 256), 5, 7, 2, dict(act=1, upconv=True, with_add=True), "tf32"),
    ("up9_3x5_b3", ("conv9_1.1", 256, 128), 3, 5, 3, dict(act=1, upconv=True, with_add=True), "planes"),
    ("up9_1x1_b2", ("conv9_1.1", 256, 128), 1, 1, 2, dict(act=1, upconv=True, with_add=True), "kb64"),
    # the fused conv10_2 -> LeakyReLU -> conv10_ab -> tanh * 128 tail with a pixel tail (105 and 3 x 171 pixels)
    ("tail10_5x13", ("conv10_2", 128, 128), 5, 13, 1, dict(act=2, slope=0.2, fuse_tail=True, nonneg=True), "f16"),
    ("tail10_7x17_b3", ("conv10_2", 128, 128), 7, 17, 3, dict(act=2, slope=0.2, fuse_tail=True, nonneg=True), "tf32"),
    # the exact-fp32 CUDA-core engine
    ("fp32_c32_o40_3x3_b3_reflect_lrelu3_stats", (32, 40, 3), 3, 3, 3, dict(reflect=True, act=2, slope=3.0, want_stats=True), "fp32"),
    ("fp32_c256_o264_7x17_b2_s2_add", (256, 264, 3), 7, 17, 2, dict(stride=2, with_add=True), "fp32"),
    ("fp32_c96_o72_1x9_d3", (96, 72, 3), 1, 9, 1, dict(dil=3), "fp32"),
    ("fp32_c160_o320_5x13_b5_d4_relu_stats", (160, 320, 3), 5, 13, 5, dict(dil=4, act=1, want_stats=True), "fp32"),
    ("fp32_k1_c64_o200_11x29", (64, 200, 1), 11, 29, 1, dict(), "fp32"),
]


def variants(case):
    """(force_bn, cluster) pairs a case runs under: every channel tile that divides the padded Cout, both cluster modes."""
    _, layer, _, _, _, kw, eng = case
    if eng == "fp32":
        return [(0, 1)]
    if eng == "tail16":
        return [(256, 2)]  # the split only exists for 256-channel tiles in clusters
    if kw.get("fuse_tail"):
        return [(0, 1), (0, 2)]  # the fused tail always runs the 128-channel tile
    cpt = cout_pad_tc(layer[2] if isinstance(layer[0], str) else layer[1])
    return [(bn, cl) for bn in (0, 64, 128, 256) if bn == 0 or cpt % bn == 0 for cl in (1, 2)]


GRID = [(c, bn, cl) for c in CASES for bn, cl in variants(c)]


def run_case(ctx, sds, case, force_bn, cluster):
    import dvc

    cid, layer, H, W, B, kw, eng = case
    ctx.debug_flag("tc_force_bn", force_bn)
    ctx.debug_flag("tc_cluster", cluster)
    if eng == "tf32":
        ctx.debug_flag("tc_f16", 0)
    elif eng == "kb64":
        ctx.debug_flag("tc_kbytes", 64)
    elif eng == "tail16":
        ctx.debug_flag("tc_tail", 16)
    elif eng == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP16X3)
    if isinstance(layer[0], str):
        name, cin, cout = layer
        sd = None
    else:
        cin, cout, k = layer
        name, sd = load_synthetic(ctx, cin, cout, k)
    return run_layer(ctx, sds, COLOR, name, cin, cout, H, W, B=B, sd=sd, out_planes=eng == "planes", **kw)


@pytest.mark.parametrize("case,force_bn,cluster", GRID, ids=[f"{c[0]}-{c[6]}-bn{bn}-cl{cl}" for c, bn, cl in GRID])
def test_edge_vs_fp64(ctx, sds, case, force_bn, cluster):
    err, floor = run_case(ctx, sds, case, force_bn, cluster)
    print(f"{case[0]} [{case[6]}, bn {force_bn}, cluster {cluster}]: |y - y64| / max = {err:.2e} (reference fp32: {floor:.2e})")
    assert err <= TOL, (case[0], case[6], force_bn, cluster, err, floor)


def test_cout_not_multiple_of_8_is_rejected(ctx):
    """The tensor-core epilogue stores channel pairs of 8-channel groups: Cout = 36 must fail before any launch."""
    import dvc

    name, _ = load_synthetic(ctx, 64, 36)
    x = torch.randn(1, 64, 5, 7, generator=torch.Generator().manual_seed(3)).cuda()
    with pytest.raises(dvc.DvcError, match="multiple of 8"):
        ctx.debug_conv2d(dvc.NET_COLOR, name, x, 36)


# ---- exact invariants ---------------------------------------------------------------------------------------------
# B * Hp * Wp = 3 * 7 * 15 = 315: 3 pixel tiles of 128 and 5 of 64 (odd counts: under clusters the last peer tile lies
# wholly past the last pixel), image boundaries inside tiles of both heights.
INV_LAYER, INV_H, INV_W, INV_B = (256, 200), 5, 13, 3


def raw(ctx, x, in_bound=None, **kw):
    """(y, stats) of the invariant layer (InstanceNorm sums always on)."""
    import dvc

    name, _ = load_synthetic(ctx, *INV_LAYER)
    y, st = ctx.debug_conv2d(dvc.NET_COLOR, name, x.cuda(), INV_LAYER[1], want_stats=True, in_bound=in_bound, **kw)
    torch.cuda.synchronize()
    return y.cpu(), st.cpu()


def inv_input(B=INV_B):
    return torch.randn(B, INV_LAYER[0], INV_H, INV_W, generator=torch.Generator().manual_seed(77)) * 2


@pytest.mark.parametrize("f16", [1, 0])
@pytest.mark.parametrize("force_bn", [128, 256])
@pytest.mark.parametrize("splits", [2, 3, 8])
def test_split_k_is_bit_identical(ctx, f16, force_bn, splits):
    """Split s of S continues the fp32 register totals split s-1 left in the workspace: same chunks, same order, so the
    outputs keep every bit (conv_tc.cu, split-K).  The InstanceNorm sums do not: every tile adds its share to the
    per-image sums with a double atomicAdd, in the order the tiles finish, and tiles that straddle an image boundary add
    exact double squares v * v per pixel, whose double sum rounds -- so the last bits of those sums follow the tile
    completion order, which splitting changes (two runs without splitting can differ the same way).  They must agree to
    the rounding of that sum."""
    ctx.debug_flag("tc_f16", f16)
    ctx.debug_flag("tc_force_bn", force_bn)
    x = inv_input()
    y1, s1 = raw(ctx, x, act=2, slope=0.2)
    ctx.debug_flag("tc_splits", splits)
    yS, sS = raw(ctx, x, act=2, slope=0.2)
    assert torch.equal(y1, yS), (splits, (y1 - yS).abs().max().item())
    a = torch.stack((y1.double().abs().sum((2, 3)), (y1.double() ** 2).sum((2, 3))), -1)
    assert ((s1 - sS).abs() / a).max().item() < 1e-13, (splits, (s1 - sS).abs().max().item())


@pytest.mark.parametrize("f16", [1, 0])
@pytest.mark.parametrize("force_bn", [64, 128, 256])
def test_cluster_is_bit_identical(ctx, f16, force_bn):
    """2-CTA clusters only share the weight tile by multicast: the arithmetic, and every output bit, is that of single CTAs."""
    ctx.debug_flag("tc_f16", f16)
    ctx.debug_flag("tc_force_bn", force_bn)
    x = inv_input()
    ctx.debug_flag("tc_cluster", 1)
    y1, _ = raw(ctx, x, act=1)
    ctx.debug_flag("tc_cluster", 2)
    y2, _ = raw(ctx, x, act=1)
    assert torch.equal(y1, y2), (y1 - y2).abs().max().item()


@pytest.mark.parametrize("force_bn", [0, 64, 128, 256])
def test_batch_image_matches_single_image(ctx, force_bn):
    """Image b of a batch of 3 has the bits of a batch-of-1 call on that image (same static operand scale: the fp16
    planes' exponent follows in_bound, which is fixed here).  The InstanceNorm sums add the same values in another
    order across tiles, so they only agree within the tolerance."""
    ctx.debug_flag("tc_force_bn", force_bn)
    x = inv_input()
    bound = float(x.abs().max())
    y3, s3 = raw(ctx, x, in_bound=bound, reflect=True)
    for b in range(INV_B):
        y1, s1 = raw(ctx, x[b:b + 1], in_bound=bound, reflect=True)
        assert torch.equal(y3[b:b + 1], y1), (b, (y3[b:b + 1] - y1).abs().max().item())
        a = torch.stack((y1.double().abs().sum((2, 3)), (y1.double() ** 2).sum((2, 3))), -1)
        assert ((s3[b:b + 1] - s1).abs() / a.clamp_min(1e-30)).max().item() < 1e-5, b


# ---- the first layers: conv_first_kernel (tensor-core mode) and the CUDA-core engine (fp32 mode) --------------------
FIRST = [("vgg_conv1_1", VGG, "conv1_1", 3, 64), ("color_conv1_1_0", COLOR, "conv1_1.0", 7, 32)]


@pytest.mark.parametrize("mode", ["first_kernel", "first_kernel_planes", "fp32"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("W", [1, 5, 8, 13, 17])
@pytest.mark.parametrize("layer", FIRST, ids=[f[0] for f in FIRST])
def test_first_layer_vs_fp64(ctx, sds, layer, W, B, mode):
    """One thread per 8-pixel octet: dead lanes past the last octet and the right-edge guard at W % 8 != 0; the planes
    variant stores device-scaled fp16 planes with the input's max measured on the device (in_bound < 0)."""
    import dvc

    _, net, name, cin, cout = layer
    if mode == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP16X3)
    planes = mode == "first_kernel_planes"
    err, floor = run_layer(ctx, sds, net, name, cin, cout, 5, W, B=B, act=1, out_planes=planes,
                           in_bound=-1.0 if planes else None)
    print(f"{name} W={W} B={B} [{mode}]: |y - y64| / max = {err:.2e} (reference fp32: {floor:.2e})")
    assert err <= TOL, (name, W, B, mode, err, floor)


# ---- scale-bound adversaries (oracle/conv_adversary.py) --------------------------------------------------------------
@pytest.mark.parametrize("case", list(ADV.CASES))
def test_adversary_reaches_bound_without_saturating(ctx, case):
    """Output planes of a layer whose target output attains the bound that sizes the fp16 store: read back, the layer
    must still match fp64 (a clamp at 65504 or an inf from the first-layer kernel would not), and the device must have
    chosen the exponent of the library's own bound formula."""
    import dvc

    adv = ADV.build(case)
    net, name, kw = adv["net"], adv["name"], adv["kw"]
    if name.startswith("edge."):
        ctx.set_weights(net, {name + ".bias": adv["sd"][name + ".bias"], name + ".weight": adv["sd"][name + ".weight"]})
    y = ctx.debug_conv2d(net, name, adv["x"].cuda(), adv["cout"], dil=kw["dil"], act=kw["act"], slope=kw["slope"],
                         upconv=kw["upconv"], in_bound=adv["in_bound"], out_planes=True,
                         add=adv["add"].cuda() if adv["add"] is not None else None)
    scaled = ctx.debug_buffer("dbg.y")  # the stored planes, hi + lo, in units of 2^-e
    y = y.cpu().double()
    sd = adv["sd"]
    y64 = ref_conv(sd, name, adv["x"], dil=kw["dil"], act=kw["act"], slope=kw["slope"], upconv=kw["upconv"], add=adv["add"])
    y32 = ref_conv(sd, name, adv["x"], dil=kw["dil"], act=kw["act"], slope=kw["slope"], upconv=kw["upconv"], add=adv["add"],
                   dtype=torch.float32)
    o, py, px = adv["target"]
    attained = abs(y64[0, o, py, px].item())
    e_dev = round(math.log2(abs(scaled[0, o, py, px].item()) / attained))
    e_lib = ADV.e16_from_bound(adv["bound"])
    scale = y64.abs().max().item()
    err, floor = (y - y64).abs().max().item() / scale, (y32.double() - y64).abs().max().item() / scale
    print(f"{case}: |y*| / bound = {attained / adv['bound']:.5f}, device exponent {e_dev} (bound formula {e_lib}), "
          f"|y*| * 2^e = {attained * 2.0 ** e_dev:.1f}; |y - y64| / max = {err:.2e} (reference fp32: {floor:.2e})")
    assert torch.isfinite(y).all(), case
    assert e_dev == e_lib, (case, e_dev, e_lib)
    assert attained * 2.0 ** e_dev <= 32768.0, case
    assert err <= TOL, (case, err, floor)
