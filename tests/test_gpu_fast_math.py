"""DVC_MATH_FP16X1 (include/dvc.h): the convolutions of the tensor-core engine with ONE MMA per product, hi * hi, on the
operand planes the default mode already stores (run with -m gpu on an H100).

1. Per layer, against an exact-rounding oracle: the layers of test_gpu_conv_layers.py (reflect, stride 2, dilation 2,
   up-convolution phases with the skip addend, the fused conv10_ab + tanh tail, InstanceNorm sums) and a few synthetic
   edge shapes, under every channel tile, single CTAs and 2-CTA clusters, row-shared taps, tf32 planes, 64-byte K rows
   and split-K, through dvc_debug_conv2d, against an fp64 F.conv2d of the ROUNDED operands
   x~ = fp16_rn(x * 2^e_x) * 2^-e_x, w~ = fp16_rn(w * 2^e_w) * 2^-e_w (tf32 planes: cvt.rna), with the exponents of
   dvc_api.cu's e16_for restated here.  Gate: the fp32-class 4e-6 * max |y64| of test_gpu_conv_layers.py.  The same
   results against the UNROUNDED fp64 conv must exceed that gate on at least one layer per net (one pass really ran),
   and stay within the one-pass bound 2.01 * 2^-11 * (|x| * |w|) plus the fp16 subnormal floor.
2. End to end: the fused frame at the default 216x384 and 480x864 goldens, against fp64, compared with the "reference on
   a GPU" emulated by the fp64 oracle with every convolution operand rounded to TF32 (tf32_reference.py).
3. Every driver (clip from host and device buffers, clip of K exemplars, video) gives the chained per-frame calls' bits
   in this mode; the drop-in modules run in it, within the end-to-end envelope of 2.
4. Mode hygiene: determinism, switching back to the default bits, exemplar invalidation, refused corr_math.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from oracle import dvc_oracle as O
from oracle.weights import make_lab
from tf32_reference import tf32_conv_operands
from test_gpu_conv_edges import load_synthetic
from test_gpu_conv_layers import COLOR, LAYERS, NETKEY, ref_conv, make_input

pytestmark = pytest.mark.gpu

TOL = 4e-6
T = 1e-10


@pytest.fixture(autouse=True)
def fast(ctx):
    """Every test runs in FP16X1 and leaves the library's default settings behind."""
    import dvc

    def reset():
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        for flag, v in (("tc_cluster", 2), ("tc_force_bn", 0), ("tc_f16", 1), ("tc_kbytes", 128), ("tc_splits", 1),
                        ("tc_rowshare", 0)):
            ctx.debug_flag(flag, v)

    reset()
    ctx.set_math(conv=dvc.MATH_FP16X1, corr=dvc.MATH_FP16X3)
    yield
    reset()


# ---- exact-rounding oracle ------------------------------------------------------------------------------------------
def e16_for(bound):
    """dvc_api.cu: e16_for -- largest e with bound * 2^e <= 2^15, clamped to [-14, 14]."""
    if not bound > 0:
        return 14
    return max(-14, min(14, math.floor(math.log2(32768.0 / bound))))


def round16(t, e):
    """The fp16 hi plane of t * 2^e (round to nearest even, subnormals kept), descaled: fp32 in, fp64 out."""
    return (t.float() * 2.0 ** e).half().double() * 2.0 ** -e


def round_tf32_rna(t):
    """cvt.rna.tf32.f32 (nearest, ties away from zero) of fp32 values, as fp64."""
    u = t.float().contiguous().view(torch.int32)
    return ((u + 0x1000) & ~0x1FFF).view(torch.float32).double()


def phase_weights(w):
    """dvc_api.cu: the four 2x2 kernels of nearest-x2 + 3x3 (sums of the 3x3 taps, fp32, ky then kx ascending)."""
    out = []
    for ph in range(4):
        a, b = ph >> 1, ph & 1
        wp = torch.zeros(w.shape[0], w.shape[1], 2, 2, dtype=torch.float32)
        for r in range(2):
            for cc in range(2):
                v = torch.zeros(w.shape[0], w.shape[1], dtype=torch.float32)
                for ky in range(3):
                    rin = (ky <= 1 if r == 0 else ky == 2) if a else (ky == 0 if r == 0 else ky >= 1)
                    if not rin:
                        continue
                    for kx in range(3):
                        cin_ = (kx <= 1 if cc == 0 else kx == 2) if b else (kx == 0 if cc == 0 else kx >= 1)
                        if cin_:
                            v = v + w[:, :, ky, kx]
                wp[:, :, r, cc] = v
        out.append(wp)
    return out


def conv_rounded(x, w, b, fmt, dil=1, stride=1, reflect=False, upconv=False):
    """fp64 conv (no activation) of the rounded operands the engine multiplies; x, w fp32."""
    if fmt == "f16":
        rx = lambda t: round16(t, e16_for(float(x.abs().max())))  # noqa: E731
        rw = lambda t: round16(t, e16_for(float(t.abs().max())))  # noqa: E731
    else:
        rx = rw = round_tf32_rna
    xr = rx(x)
    b = b.double()
    if upconv:
        xp = F.pad(xr, (1, 1, 1, 1))
        H, W = x.shape[2], x.shape[3]
        y = torch.empty(x.shape[0], w.shape[0], 2 * H, 2 * W, dtype=torch.float64)
        for ph, wp in enumerate(phase_weights(w)):
            a, bb = ph >> 1, ph & 1
            r0, c0 = (0 if a else -1), (0 if bb else -1)
            y[:, :, a::2, bb::2] = F.conv2d(xp[:, :, 1 + r0:1 + r0 + H + 1, 1 + c0:1 + c0 + W + 1], rw(wp), b)
        return y
    if w.shape[2] == 3:
        xr = F.pad(xr, (dil,) * 4, mode="reflect" if reflect else "constant")
    return F.conv2d(xr, rw(w), b, stride=stride, dilation=dil)


def epilogue(y, act, slope, add):
    if add is not None:
        y = y + add.double()
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = F.leaky_relu(y, slope)
    return y


def tail(sds, y):
    """ColorVidNet.py:143-144, fp64."""
    return torch.tanh(F.conv2d(y, sds["color"]["conv10_ab.weight"].double(), sds["color"]["conv10_ab.bias"].double())) * 128


_REF = {}


def run_fast_layer(ctx, sds, net, name, cin, cout, H, W, fmt="f16", B=1, sd=None, **kw):
    """One layer in FP16X1 through dvc_debug_conv2d.  Returns (error vs the rounded-operand oracle, error vs the exact
    fp64 conv, one-pass bound violation), the first two relative to max |y64|; InstanceNorm sums are checked here."""
    kw = dict(kw)
    nonneg, with_add, want_stats = kw.pop("nonneg", False), kw.pop("with_add", False), kw.pop("want_stats", False)
    fuse_tail = kw.pop("fuse_tail", False)
    dil, stride, act, slope = kw.get("dil", 1), kw.get("stride", 1), kw.get("act", 0), kw.get("slope", 0.0)
    reflect, upconv = kw.get("reflect", False), kw.get("upconv", False)
    sd = sds[NETKEY[net]] if sd is None else sd
    key = (net, name, H, W, B, fmt, tuple(sorted(kw.items())), nonneg, with_add, fuse_tail)
    if key not in _REF:
        x = make_input(1234, B, cin, H, W, nonneg)
        add = None
        if with_add:
            Ho, Wo = (2 * H, 2 * W) if upconv else ((H + stride - 1) // stride, (W + stride - 1) // stride)
            add = torch.randn(B, cout, Ho, Wo, generator=torch.Generator().manual_seed(99)) * 3
        w, b = sd[name + ".weight"].float(), sd[name + ".bias"].float()
        with torch.no_grad():
            yr = epilogue(conv_rounded(x, w, b, fmt, dil, stride, reflect, upconv), act, slope, add)
            y64 = ref_conv(sd, name, x, add=add, **kw)
            # |x| * |w| (the bound of the operand rounding), and the subnormal floor of the fp16 planes
            absd = {name + ".weight": w.abs(), name + ".bias": torch.zeros_like(b)}
            A = ref_conv(absd, name, x.abs(), dil=dil, stride=stride, reflect=reflect, upconv=upconv)
            floor = 0.0
            if fmt == "f16":
                ex, ew = e16_for(float(x.abs().max())), e16_for(float(w.abs().max()))
                taps = w.shape[2] * w.shape[3]
                floor = 2.0 ** -25 * (2.0 ** -ex * float(w.abs().sum((1, 2, 3)).max()) * (4 if upconv else 1)
                                      + 2.0 ** -ew * taps * cin * float(x.abs().max()) * (4 if upconv else 1))
            bound = 2.01 * 2.0 ** -11 * A + floor
            if fuse_tail:  # LeakyReLU (slope <= 1) and the 1x1 conv10_ab, then tanh * 128 (1-Lipschitz * 128)
                bound = 128 * F.conv2d(bound, sds["color"]["conv10_ab.weight"].double().abs())
                yr, y64 = tail(sds, yr), tail(sds, y64)
        _REF[key] = (x, add, yr, y64, bound)
    x, add, yr, y64, bound = _REF[key]
    res = ctx.debug_conv2d(net, name, x.cuda(), cout, dil=dil, stride=stride, act=act, slope=slope, reflect=reflect,
                           upconv=upconv, fuse_tail=fuse_tail, add=add.cuda() if add is not None else None,
                           want_stats=want_stats)
    y, st = res if want_stats else (res, None)
    y = y.cpu().double()
    scale = yr.abs().max().item()
    err_r, err_x = (y - yr).abs().max().item() / scale, (y - y64).abs().max().item() / scale
    over = ((y - y64).abs() - bound - TOL * scale).max().item()
    if st is not None:
        st = st.cpu()
        s64 = torch.stack((yr.sum((2, 3)), (yr * yr).sum((2, 3))), -1)
        a64 = torch.stack((yr.abs().sum((2, 3)), (yr * yr).sum((2, 3))), -1)
        serr = ((st - s64).abs() / a64.clamp_min(1e-30)).max().item()
        assert serr < 1e-5, ("InstanceNorm sums", name, serr)
    return err_r, err_x, over


# (engine id, flags, format of the operand planes)
ENGINES = [
    ("pair", {}, "f16"),
    ("single", {"tc_cluster": 1}, "f16"),
    ("rowshare", {"tc_rowshare": 1}, "f16"),
    ("rowshare_single", {"tc_rowshare": 1, "tc_cluster": 1}, "f16"),
    ("tf32", {"tc_f16": 0}, "tf32"),
    ("kb64", {"tc_kbytes": 64}, "f16"),
    ("splitk3", {"tc_splits": 3}, "f16"),
]
GRID = [(l, bn, e) for l in LAYERS for e in ENGINES for bn in ((0, 64, 128, 256) if e[0] in ("pair", "single") else (0,))
        if not (l[7].get("fuse_tail") and bn)]


@pytest.mark.parametrize("layer,force_bn,engine", GRID, ids=[f"{l[0]}-{e[0]}-bn{bn}" for l, bn, e in GRID])
def test_layer_vs_rounded_operand_oracle(ctx, sds, layer, force_bn, engine):
    lid, net, name, cin, cout, H, W, kw = layer
    eid, flags, fmt = engine
    for f, v in flags.items():
        ctx.debug_flag(f, v)
    ctx.debug_flag("tc_force_bn", force_bn)
    err_r, err_x, over = run_fast_layer(ctx, sds, net, name, cin, cout, H, W, fmt=fmt, **kw)
    print(f"{lid} [{eid}, bn {force_bn}]: vs rounded operands {err_r:.2e}, vs exact {err_x:.2e}, bound margin {over:.2e}")
    assert err_r <= TOL, (lid, eid, force_bn, err_r, err_x)
    assert over <= 0, (lid, eid, force_bn, over)


# synthetic shapes of test_gpu_conv_edges.py: Cin 32 / 96 / 160 (64-byte K rows on fp16 planes), pixel tails, batches
EDGES = [
    ("c32_o32_1x1", (32, 32, 3), 1, 1, 1, dict(act=1)),
    ("c96_o40_1x9_b5_lrelu_stats", (96, 40, 3), 1, 9, 5, dict(act=2, slope=0.2, want_stats=True)),
    ("c160_o72_3x3_b3_reflect_add_stats", (160, 72, 3), 3, 3, 3, dict(reflect=True, with_add=True, want_stats=True)),
    ("c256_o264_7x17_reflect_stats", (256, 264, 3), 7, 17, 1, dict(reflect=True, want_stats=True)),
    ("k1_c96_o264_7x17_add", (96, 264, 1), 7, 17, 1, dict(with_add=True)),
    ("s2_c160_o200_11x29_relu", (160, 200, 3), 11, 29, 1, dict(stride=2, act=1)),
    ("d2_c64_o72_5x3_b3_reflect_lrelu_stats", (64, 72, 3), 5, 3, 3, dict(dil=2, reflect=True, act=2, slope=0.2, want_stats=True)),
    ("m259_c64_o320_5x35_lrelu_stats", (64, 320, 3), 5, 35, 1, dict(act=2, slope=0.2, want_stats=True)),
]


@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("fmt", ["f16", "tf32"])
@pytest.mark.parametrize("case", EDGES, ids=[c[0] for c in EDGES])
def test_edge_shapes_vs_rounded_operand_oracle(ctx, sds, case, fmt, cluster):
    cid, (cin, cout, k), H, W, B, kw = case
    ctx.debug_flag("tc_cluster", cluster)
    ctx.debug_flag("tc_f16", 1 if fmt == "f16" else 0)
    name, sd = load_synthetic(ctx, cin, cout, k)
    err_r, err_x, over = run_fast_layer(ctx, sds, COLOR, name, cin, cout, H, W, fmt=fmt, B=B, sd=sd, **kw)
    print(f"{cid} [{fmt}, cluster {cluster}]: vs rounded operands {err_r:.2e}, vs exact {err_x:.2e}")
    assert err_r <= TOL, (cid, fmt, cluster, err_r)
    assert over <= 0, (cid, fmt, cluster, over)


def test_one_pass_is_visible_in_every_net(ctx, sds):
    """Against the exact operands at least one layer of each net misses the fp32-class gate: one MMA per product ran."""
    worst = {}
    for lid, net, name, cin, cout, H, W, kw in LAYERS:
        _, err_x, _ = run_fast_layer(ctx, sds, net, name, cin, cout, H, W, **kw)
        worst[net] = max(worst.get(net, 0.0), err_x)
    print("max |y - y64(exact operands)| / max per net:", {NETKEY[k]: f"{v:.2e}" for k, v in worst.items()})
    assert all(v > TOL for v in worst.values()), worst


# ---- end to end ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["default_216x384", "default_480x864"])
def test_fused_frame_vs_emulated_gpu_reference(ctx, sds, name):
    """Mean |ab - ab64| <= 1.5 x that of the reference's TF32 convolutions (emulated in fp64), and argmax rows that
    differ from fp64 <= 1.5 x the emulation's + 2."""
    g = load_golden(name)
    if "IA_lab" in g:
        IA, IB, last = (torch.from_numpy(g[k]) for k in ("IA_lab", "IB_lab", "IA_last_lab"))
    else:  # inputs regenerated from the stored seed (test_gpu_headline.py)
        seed, (H, W) = int(g["seed"]), g["ab64"].shape[2:]
        IA, IB, last = make_lab(seed, 1, H, W), make_lab(seed + 1, 1, H, W), make_lab(seed + 2, 1, H, W) * 0.5
    ab64 = torch.from_numpy(g["ab64"]).double()
    ctx.set_exemplar(IB)
    ab, warp, _ = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T, want_warp=True)
    ab = ab.cpu().double()
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    ex, ex_e = {}, {}
    with torch.no_grad():
        fB = O.exemplar_features(sds64["vgg"], IB.double())
        ab_x, _, _, _ = O.frame_colorization(sds64, IA.double(), IB.double(), last.double(), fB, extras=ex)
        with tf32_conv_operands():
            fBe = O.exemplar_features(sds64["vgg"], IB.double())
            ab_e, _, _, _ = O.frame_colorization(sds64, IA.double(), IB.double(), last.double(), fBe, extras=ex_e)
    assert (ab_x - ab64).abs().max().item() < 1e-9  # the oracle reproduces its golden
    am64, am_e = ex["argmax"], ex_e["argmax"]
    # at T -> 0 the warp of a query row is the pooled exemplar colour of its argmax: a row counts as different when
    # its colour is not fp64's (indices of equal colours are ambiguous)
    V = ex["V"][0]  # [N, 3] pooled exemplar colours
    wd = warp.cpu().double()[0, :, ::4, ::4].reshape(3, -1).t()
    off = lambda c: int(((c - V[am64[0]]).abs().max(-1).values > 1e-4).sum())  # noqa: E731
    diff_dev, diff_e = off(wd), off(V[am_e[0]])
    m_dev, m_e = float((ab - ab64).abs().mean()), float((ab_e - ab64).abs().mean())
    print(f"{name}: mean |ab - ab64| fast {m_dev:.3e}, emulated TF32 reference {m_e:.3e}; "
          f"argmax rows != fp64: fast {diff_dev}, emulated {diff_e} (of {am64.numel()})")
    assert m_dev <= 1.5 * m_e, (m_dev, m_e)
    assert diff_dev <= 1.5 * diff_e + 2, (diff_dev, diff_e)


# ---- drivers ---------------------------------------------------------------------------------------------------------
def test_clip_drivers_equal_chained_frames(ctx):
    g = load_golden("clip3_32x48")
    L = torch.from_numpy(g["frames_lab"])[:, 0:1].contiguous()
    F_, _, H, W = L.shape
    IB = torch.from_numpy(g["IB_lab"])
    ctx.set_exemplar(IB)
    out = ctx.colorize_clip(L.pin_memory())
    assert torch.equal(ctx.colorize_clip(L.cuda()).cpu(), out.cpu())
    last = torch.zeros(1, 3, H, W, device="cuda")
    for t in range(F_):
        Lt = L[t:t + 1].cuda()
        ab = ctx.colorize_frames(Lt, last)
        assert torch.equal(ab.cpu(), out[t:t + 1].cpu()), t
        last = torch.cat((Lt, ab), 1)
    IBk = make_lab(90, 2, H, W)
    ctx.set_exemplars(IBk)
    outk = ctx.colorize_clip_exemplars(L.pin_memory())
    assert torch.equal(ctx.colorize_clip_exemplars(L.cuda()).cpu(), outk.cpu())
    last = torch.zeros(2, 3, H, W, device="cuda")
    for t in range(F_):
        Lt = L[t:t + 1].cuda()
        ab = ctx.colorize_frames_exemplars(Lt, last)
        assert torch.equal(ab.cpu(), outk[:, t].cpu()), t
        last = torch.cat((Lt.expand(2, 1, H, W), ab), 1)


@pytest.mark.parametrize("K", [1, 2])
def test_video_equals_composition(ctx, K):
    from test_gpu_video import _composition, _frames, _set_exemplars

    Hs, Ws, Ho, Wo = 100, 90, 64, 96
    _set_exemplars(ctx, K, Ho // 2, Wo // 2)
    frames = _frames(5 + K, 3, Hs, Ws)
    ref, _, _ = _composition(ctx, frames, (Ho, Wo), K)
    out = ctx.colorize_video_rgb8(frames.pin_memory(), (Ho, Wo), T)
    assert torch.equal(out.cpu(), ref)


def test_dropin_modules_run_in_the_selected_mode(ctx, sds):
    """The drop-in modules driven as in test_gpu_dropin.py follow the context's conv mode.  Their glue normalises the
    features in torch, not in the fused path's kernel, so at T -> 0 near-tie rows may pick other exemplar positions than
    the fused path does; they are held to the end-to-end envelope of test_fused_frame_vs_emulated_gpu_reference."""
    import dvc
    from models.ColorVidNet import ColorVidNet
    from models.NonlocalNet import VGG19_pytorch, WarpNet

    nonlocal_net, colornet, vggnet = WarpNet(1), ColorVidNet(7), VGG19_pytorch()
    vggnet.load_state_dict(sds["vgg"])
    nonlocal_net.load_state_dict(sds["warp"])
    colornet.load_state_dict(sds["color"])
    for m in (nonlocal_net, colornet, vggnet):
        m.eval()
        m.cuda()
    g = load_golden("small_32x48")
    IA, IB, last = (torch.from_numpy(g[k]).cuda() for k in ("IA_lab", "IB_lab", "IA_last_lab"))

    def modules():
        with torch.no_grad():
            rgb = O.tensor_lab2rgb(torch.cat((O.uncenter_l(IB[:, 0:1]), IB[:, 1:3]), dim=1).cpu()).cuda()
            features_B = vggnet(rgb, ["r12", "r22", "r32", "r42", "r52"], preprocess=True)
            IA_l = IA[:, 0:1]
            fA = vggnet(O.gray2rgb_batch(IA_l), ["r12", "r22", "r32", "r42", "r52"], preprocess=True)
            An = [O.feature_normalize(t) for t in fA[1:]]
            Bn = [O.feature_normalize(t) for t in features_B[1:]]
            warped, sim = nonlocal_net(IB, *An, *Bn, temperature=1e-10)
            return fA, colornet(torch.cat((IA_l, warped[:, 1:3], sim, last), dim=1))

    fA, ab = modules()
    fA2, ab2 = modules()
    assert all(torch.equal(a, b) for a, b in zip(fA, fA2)) and torch.equal(ab, ab2)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    fA_d, ab_d = modules()
    assert not torch.equal(fA[1], fA_d[1])  # the VGG features of the module path changed with the mode
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    with torch.no_grad():
        with tf32_conv_operands():
            ab_e, _, _, _ = O.frame_colorization(sds64, IA.cpu().double(), IB.cpu().double(), last.cpu().double(),
                                                 O.exemplar_features(sds64["vgg"], IB.cpu().double()))
    ab64 = torch.from_numpy(g["ab64"]).double()
    m_fast, m_def = float((ab.cpu().double() - ab64).abs().mean()), float((ab_d.cpu().double() - ab64).abs().mean())
    m_e = float((ab_e - ab64).abs().mean())
    print(f"drop-in modules, mean |ab - ab64|: fast {m_fast:.3e}, default {m_def:.3e}, emulated TF32 reference {m_e:.3e}")
    assert m_fast <= 1.5 * m_e + 1e-3, (m_fast, m_e)


# ---- mode hygiene ----------------------------------------------------------------------------------------------------
def _frame(ctx, seed=5, H=32, W=48):
    IA, IB, last = make_lab(seed, 1, H, W), make_lab(seed + 1, 1, H, W), make_lab(seed + 2, 1, H, W)
    ctx.set_exemplar(IB)
    return ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T).cpu()


def test_mode_switches(ctx):
    import dvc

    a1, a2 = _frame(ctx), _frame(ctx)
    assert torch.equal(a1, a2)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    d1 = _frame(ctx)
    assert not torch.equal(d1, a1)
    ctx.set_math(conv=dvc.MATH_FP16X1, corr=dvc.MATH_FP16X3)
    assert torch.equal(_frame(ctx), a1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    assert torch.equal(_frame(ctx), d1)


def test_exemplar_is_refused_after_a_mode_change(ctx):
    import dvc

    IA, IB, last = make_lab(11, 1, 32, 48), make_lab(12, 1, 32, 48), make_lab(13, 1, 32, 48)
    ctx.set_exemplar(IB)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    with pytest.raises(dvc.DvcError):
        ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T)


def test_corr_fp16x1_is_refused_and_changes_nothing(ctx):
    import dvc

    IA, IB, last = make_lab(21, 1, 32, 48), make_lab(22, 1, 32, 48), make_lab(23, 1, 32, 48)
    ctx.set_exemplar(IB)
    ref = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T).cpu()
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    for conv in (dvc.MATH_FP16X1, dvc.MATH_TF32X3):
        with pytest.raises(dvc.DvcError) as e:
            ctx.set_math(conv=conv, corr=dvc.MATH_FP16X1)
        assert "(-1)" in str(e.value)  # DVC_ERR_ARG
    assert ctx.launch_count() == n0
    # the context is as it was: same conv mode, the exemplar still cached
    assert torch.equal(ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T).cpu(), ref)
