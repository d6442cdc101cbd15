"""Stage-by-stage parity of the layer programs (run with -m gpu on an H100).

The convolution and correlation engines have suites of their own; this one checks the code between them -- the glue
kernels of csrc/elementwise.cu (InstanceNorm apply, PReLU, reflect / zero borders, nearest x2, the stride-2 pick of
the *_ss layers, the residual add, the r5 row repair, the fp32 / tf32-split / fp16-plane stores, pixnorm, the pools,
the NCHW prologues and epilogues) and the wiring of the layer programs of dvc_api.cu (which weights, stride, dilation,
padding mode, InstanceNorm count and static fp16 exponent each stage gets).

Method: run a layer program once, download every intermediate buffer by name (Context.debug_buffer), and recompute
each stage in float64 on the CPU from the library's OWN input buffer of that stage.  The error measured is then only
that stage's rounding, so the gates are per-element bounds derived from the kernel's arithmetic (u = 2^-24):

  prologues          bit-identical to the fp32 oracle (same operations), or a propagated bound (Lab -> sRGB)
  max-pools          exact (in scaled units on fp16 planes); a tf32 split within 2^-22 |x|
  pixnorm            |ref| * ((C / 64 + 8) u) + store
  InstanceNorm apply the statistics are one-pass sums of fp32 tile partials (conv epilogues) kept in double:
                     gain * (rstd * u * (K a1 + |mean| + |v - mean|) + |z| * u * K (m2 + 2 |mean| a1) / (2 var) + 3u |z|)
                     + u |out| (residual add) + store, K = 128 (longest fp32 partial sum), a1 = mean |v|, m2 = mean v^2
  convolutions       test_gpu_conv_layers.py's 4e-6 * max |y64| on the stored padded input (fp32 / tf32 engines, and
                     every fp16-engine convolution whose input exponent is static)
  store              fp32: exact; tf32 or fp16 hi/lo: 2^-21 |out|; fp16 planes also 2^-24 * 2^-e (the lo plane's floor)

The fp16 planes are descaled with the static exponents restated here (e16_for and each call site's bound), so a changed
exponent fails.  Each gate class is also evaluated on one plausible WRONG reference on the same downloaded data, which
must fail it (replicate border, unbiased variance, shifted row repair, missing *_ss scale, offset pool window,
exponent off by one): every gate is shown able to fail.  The reference's own fp32 evaluation of a stage is printed
beside the library's error; run with -s for the per-gate report.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import dvc_oracle as O
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
K_PARTIAL = 128
CONV_TOL = 4e-6
ENGINES = ["fp32", "tf32", "fp16"]
# (H, W, B): smallest legal frame (r52 2x2); rowpad with r52 2x3 and pools 40 -> 20 -> 10 -> 5 -> 2; rowpad, r52 3x5
# and odd ColorVidNet stride-2 picks (56 -> 28 -> 14 -> 7); image boundaries inside pixel tiles with per-image statistics
SHAPES = [(32, 32, 1), (40, 48, 2), (56, 80, 1), (64, 96, 3)]
SHAPE_IDS = ["32x32x1", "40x48x2", "56x80x1", "64x96x3"]


def e16_for(bound):
    """dvc_api.cu: e16_for -- largest e with bound * 2^e <= 2^15, clamped to [-14, 14]."""
    if not bound > 0:
        return 14
    return max(-14, min(14, math.floor(math.log2(32768.0 / bound))))


@pytest.fixture(autouse=True)
def defaults(ctx):
    import dvc

    def reset():
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        for flag, v in (("tc_cluster", 2), ("tc_force_bn", 0), ("tc_f16", 1), ("tc_kbytes", 128), ("tc_tail", 0),
                        ("tc_splits", 1), ("keep_stages", 0)):
            ctx.debug_flag(flag, v)

    reset()
    yield
    reset()


def set_engine(ctx, eng):
    """fp32: CUDA-core engine (st4 / ld4 fp32 stores); tf32: tensor cores on tf32 hi/lo planes (tc_f16 = 0); fp16: the
    default fp16 hi/lo planes (st4h / dst_h16 stores, ld4h loads)."""
    import dvc

    if eng == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32)
    else:
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        ctx.debug_flag("tc_f16", 0 if eng == "tf32" else 1)


# ---------------------------------------------------------------------------------------------------- gate bookkeeping
class Gates:
    """Collects (stage, error / gate, reference fp32 error / gate) and the sensitivity margins of one run."""

    def __init__(self, label):
        self.label, self.rows, self.sens, self.bad = label, [], [], []

    def check(self, stage, lib, ref, tol, ref32=None):
        lib, ref = lib.double(), ref.double()
        tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(ref).clamp_min(1e-300)  # zero gate: exact
        assert lib.shape == ref.shape, (stage, lib.shape, ref.shape)
        r = ((lib - ref).abs() / tol).max().item() if lib.numel() else 0.0
        f = ((ref32.double() - ref).abs() / tol).max().item() if ref32 is not None else float("nan")
        self.rows.append((stage, r, f))
        if not r <= 1.0:
            self.bad.append((stage, r))
        return r

    def exact(self, stage, lib, ref):
        ok = torch.equal(lib, ref.to(lib.dtype))
        self.rows.append((stage, 0.0 if ok else float("inf"), float("nan")))
        if not ok:
            self.bad.append((stage, (lib.double() - ref.double()).abs().max().item()))

    def wrong(self, stage, lib, wrong, tol):
        """A plausible wrong reference must fail the same gate."""
        lib, wrong = lib.double(), wrong.double()
        tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(wrong).clamp_min(1e-300)
        r = ((lib - wrong).abs() / tol).max().item()
        self.sens.append((stage, r))
        if not r > 1.0:
            self.bad.append(("sensitivity " + stage, r))

    def finish(self):
        for stage, r, f in self.rows:
            print(f"[{self.label}] {stage:40s} err/gate {r:9.3e}   ref-fp32 err/gate {f:9.3e}")
        for stage, r in self.sens:
            print(f"[{self.label}] wrong reference {stage:24s} err/gate {r:9.3e} (must be > 1)")
        assert not self.bad, self.bad


def store_tol(ref, eng, e=None):
    """Rounding of the store: fp32 exact; hi/lo planes 2^-21 relative; fp16 planes also the lo plane's floor."""
    t = torch.zeros_like(ref) if eng == "fp32" else ref.abs() * 2.0 ** -21
    if e is not None:
        t = t + 2.0 ** -24 * 2.0 ** -e
    return t


class Buffers:
    def __init__(self, ctx, eng):
        self.ctx, self.eng = ctx, eng

    def get(self, name, border=False, e=None, fp16=False):
        """fp64 copy of a buffer; e: the static exponent of fp16 planes (descaled here)."""
        t = self.ctx.debug_buffer(name, keep_border=border, fp16=fp16).double().cpu()
        return t * 2.0 ** -e if e is not None else t

    def plane_e(self, bound):
        """Static exponent of an fp16-plane buffer in the fp16 engine (None: the buffer holds fp32 values)."""
        return e16_for(bound) if self.eng == "fp16" else None


def reflect1(x):
    return F.pad(x, (1, 1, 1, 1), mode="reflect")


def zpad(x, p):
    return F.pad(x, (p, p, p, p))


def up(x, k):
    return x if k == 1 else F.interpolate(x, scale_factor=k, mode="nearest")


def prelu(x, s):
    return torch.where(x > 0, x, x * s)


# ------------------------------------------------------------------------------------------------- stage references
def inorm_ref(v, unbiased=False):
    """fp64 two-pass instance norm (eps 1e-5, biased like F.instance_norm) and the per-element bound of the library's
    evaluation of it (module docstring), before gain and store."""
    n = v.shape[2] * v.shape[3]
    mean = v.mean((2, 3), keepdim=True)
    var = ((v - mean) ** 2).sum((2, 3), keepdim=True) / (n - 1 if unbiased else n)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    z = (v - mean) * rstd
    a1, m2 = v.abs().mean((2, 3), keepdim=True), (v * v).mean((2, 3), keepdim=True)
    tol = rstd * U * (K_PARTIAL * a1 + mean.abs() + (v - mean).abs()) \
        + z.abs() * U * K_PARTIAL * (m2 + 2 * mean.abs() * a1) / (2 * (var + 1e-5)) + 3 * U * z.abs()
    return z, tol


def conv64(sd, name, xpad, stride=1, dil=1):
    w, b = sd[name + ".weight"].double(), sd[name + ".bias"].double()
    return F.conv2d(xpad[:, :w.shape[1]], w, b, stride=stride, dilation=dil)


def check_conv(g, stage, lib, ref):
    g.check(stage, lib, ref, CONV_TOL * max(ref.abs().max().item(), 1e-30))


def check_border(g, stage, lib_padded, interior_to_padded, p):
    """The stored border equals the reference padding of the stored interior."""
    inner = lib_padded[:, :, p:-p, p:-p]
    g.exact(stage + " border", lib_padded, interior_to_padded(inner))


def check_pixnorm(g, bufs, stage, r, n_name, e):
    """feature_normalize (util.py:155-158) of a stored VGG map, reflect pad 1 (scale-invariant: r may be scaled)."""
    C = r.shape[1]
    ref = reflect1(r / (torch.sqrt((r * r).sum(1, keepdim=True)) + O.EPS))
    r32 = r.float()
    ref32 = reflect1(r32 / (torch.norm(r32, 2, 1, keepdim=True) + O.EPS))
    lib = bufs.get(n_name, border=True, e=e)
    tol = ref.abs() * (C / 64 + 8) * U + store_tol(ref, bufs.eng, e)
    g.check(stage, lib, ref, tol, ref32)
    g.wrong(stage + " replicate", lib, F.pad(ref[:, :, 1:-1, 1:-1], (1, 1, 1, 1), mode="replicate"), tol)
    if e is not None:
        g.wrong(stage + " exponent+1", bufs.get(n_name, border=True, e=e + 1), ref, tol)


def check_pool(g, bufs, stage, src, dst_name, e_scaled):
    """max_pool2d (floor on odd sizes) of the stored input, zero border.  e_scaled: compare in scaled units."""
    lib = bufs.get(dst_name, border=True)
    ref = zpad(F.max_pool2d(src, 2), 1)
    if bufs.eng == "tf32":
        g.check(stage, lib, ref, ref.abs() * 2.0 ** -22 + 1e-300)
    else:
        g.exact(stage, lib, ref)
    shifted = zpad(F.max_pool2d(F.pad(src, (0, 1, 0, 1))[:, :, 1:, 1:], 2)[:, :, :ref.shape[2] - 2, :ref.shape[3] - 2], 1)
    g.wrong(stage + " window+1", lib, shifted, ref.abs() * 2.0 ** -22 + 1e-30)


def vgg_stages(g, bufs, sd, tag, x0, last="r52"):
    """Trunk of NonlocalNet.py:228-256 from the stored x0: every conv (fp32 / tf32 engines), every pool."""
    eng = bufs.eng
    cur, block, idx = x0, 1, 1
    for name in O.VGG_ORDER:
        if name == "P":
            key = f"p{block}"
            check_pool(g, bufs, f"{tag}.{key} maxpool", cur, f"{tag}.{key}", None)
            cur = bufs.get(f"{tag}.{key}", border=True)[:, :, 1:-1, 1:-1]
            block, idx = block + 1, 1
        else:
            key = f"r{block}{idx}"
            lib = bufs.get(f"{tag}.{key}", border=True)
            if eng != "fp16":  # fp16 planes carry a device-derived exponent: checked through pools and pixnorm only
                ref = torch.relu(conv64(sd, name, zpad(cur, 1)))
                check_conv(g, f"{tag}.{key} conv", lib[:, :, 1:-1, 1:-1], ref)
                check_border(g, f"{tag}.{key}", lib, lambda t: zpad(t, 1), 1)
            cur = lib[:, :, 1:-1, 1:-1]
            idx += 1
        if key == last:
            break


def warp_side_stages(g, bufs, sd, tag, n_names, n_e, rows_name, proj, H, W):
    """NonlocalNet.py:451-476 for one side from the stored n{k}: heads, row repair, concat, residual blocks, projection."""
    eng = bufs.eng
    h, w = H // 4, W // 4
    heads = [("layer2_1.1", "layer2_1.3", "layer2_1.5", "layer2_1.7", 2, 1, 1),
             ("layer3_1.1", "layer3_1.3", "layer3_1.5", "layer3_1.7", 1, 1, 1),
             ("layer4_1.1", "layer4_1.3", "layer4_1.5", "layer4_1.7", 1, 1, 2),
             ("layer5_1.1", "layer5_1.3", "layer5_1.6", "layer5_1.8", 1, 2, 2)]
    slope = lambda k: float(sd[k + ".weight"])
    cat_bound = max(math.sqrt(h * w) * max(1.0, abs(slope(hd[3]))) for hd in heads)
    e_cat = bufs.plane_e(cat_bound)
    cat = bufs.get(f"{tag}.cat", border=True)
    cat16 = bufs.get(f"{tag}.cat", border=True, e=e_cat, fp16=True) if e_cat is not None else None
    for k, (c1, s1, c2, s2, stride2, up_mid, up_end) in enumerate(heads):
        t = f"{tag}.h{k}"
        x = bufs.get(n_names[k], border=True, e=n_e)
        raw1 = bufs.get(t + ".raw1")
        check_conv(g, f"{t}.raw1 conv", raw1, conv64(sd, c1, x))
        # mid = reflect(up(PReLU(IN(raw1))))
        z, tz = inorm_ref(raw1)
        g1 = max(1.0, abs(slope(s1)))
        e_mid = bufs.plane_e(math.sqrt(raw1.shape[2] * raw1.shape[3]) * g1)
        ref = reflect1(up(prelu(z, slope(s1)), up_mid))
        tol = reflect1(up(tz * g1, up_mid)) + store_tol(ref, eng, e_mid)
        r32 = reflect1(up(F.prelu(F.instance_norm(raw1.float(), eps=1e-5), torch.tensor([slope(s1)])), up_mid))
        mid = bufs.get(t + ".mid", border=True, e=e_mid)
        g.check(f"{t}.mid IN/PReLU/up/reflect", mid, ref, tol, r32)
        if k == 0:
            zu, _ = inorm_ref(raw1, unbiased=True)
            g.wrong(f"{t}.mid unbiased var", mid, reflect1(prelu(zu, slope(s1))), tol)
            g.wrong(f"{t}.mid replicate", mid, F.pad(prelu(z, slope(s1)), (1, 1, 1, 1), mode="replicate"), tol)
            if e_mid is not None:
                g.wrong(f"{t}.mid exponent-1", bufs.get(t + ".mid", border=True, e=e_mid - 1), ref, tol)
        raw2 = bufs.get(t + ".raw2")
        check_conv(g, f"{t}.raw2 conv stride {stride2}", raw2, conv64(sd, c2, mid, stride=stride2))
        # cat slice: up(PReLU(IN(raw2))), rows replicated by one on the r5 head when the heights disagree, then reflect
        z2, tz2 = inorm_ref(raw2)
        g2 = max(1.0, abs(slope(s2)))
        f = up(prelu(z2, slope(s2)), up_end)
        ft = up(tz2 * g2, up_end)
        if f.shape[2] != h:
            f, ft = F.pad(f, (0, 0, 1, 1), mode="replicate"), F.pad(ft, (0, 0, 1, 1), mode="replicate")
        sl = slice(64 * k, 64 * k + 64)
        ref, tol = reflect1(f), reflect1(ft)
        f32 = up(F.prelu(F.instance_norm(raw2.float(), eps=1e-5), torch.tensor([slope(s2)])), up_end)
        if f32.shape[2] != h:
            f32 = F.pad(f32, (0, 0, 1, 1), mode="replicate")
        g.check(f"{t} cat slice", cat[:, sl], ref, tol + store_tol(ref, "fp32" if eng == "fp16" else eng), reflect1(f32))
        if cat16 is not None:
            g.check(f"{t} cat slice fp16 planes", cat16[:, sl], ref, tol + store_tol(ref, eng, e_cat))
        if k == 3 and up(z2, up_end).shape[2] != h:
            fs = F.pad(up(prelu(z2, slope(s2)), up_end), (0, 0, 0, 2), mode="replicate")  # repair shifted by one row
            g.wrong(f"{t} rowpad shifted", cat[:, sl], reflect1(fs), tol + 1e-30)
    # residual blocks (NonlocalNet.py:341-352); the convolutions read the fp16 planes of cat / out when they exist, the
    # residual add reads the fp32 plane
    xa, xa16 = cat, cat16 if cat16 is not None else cat
    chain = cat_bound
    for i in range(3):
        r = f"{tag}.res{i}"
        sl_ = float(sd[f"layer.{i}.prelu.weight"])
        gi = max(1.0, abs(sl_))
        raw1 = bufs.get(r + ".raw1")
        check_conv(g, f"{r}.raw1 conv", raw1, conv64(sd, f"layer.{i}.conv1", xa16))
        z, tz = inorm_ref(raw1)
        e_mid = bufs.plane_e(math.sqrt(h * w) * gi)
        ref = reflect1(prelu(z, sl_))
        mid = bufs.get(r + ".mid", border=True, e=e_mid)
        r32 = reflect1(F.prelu(F.instance_norm(raw1.float(), eps=1e-5), torch.tensor([sl_])))
        g.check(f"{r}.mid", mid, ref, reflect1(tz * gi) + store_tol(ref, eng, e_mid), r32)
        raw2 = bufs.get(r + ".raw2")
        check_conv(g, f"{r}.raw2 conv", raw2, conv64(sd, f"layer.{i}.conv2", mid))
        z2, tz2 = inorm_ref(raw2)
        add = xa[:, :, 1:-1, 1:-1]
        pre = z2 + add
        ref = reflect1(prelu(pre, sl_))
        tol = reflect1((tz2 + U * pre.abs()) * gi) + store_tol(ref, "fp32" if eng == "fp16" else eng)
        out = bufs.get(r + ".out", border=True)
        r32 = reflect1(F.prelu(F.instance_norm(raw2.float(), eps=1e-5) + add.float(), torch.tensor([sl_])))
        g.check(f"{r}.out IN + residual / PReLU", out, ref, tol, r32)
        chain = (chain + math.sqrt(h * w)) * gi
        e_out = bufs.plane_e(chain)
        xa, xa16 = out, out
        if e_out is not None:
            xa16 = bufs.get(r + ".out", border=True, e=e_out, fp16=True)
            g.check(f"{r}.out fp16 planes", xa16, ref, tol + store_tol(ref, eng, e_out))
            g.wrong(f"{r}.out exponent+1", bufs.get(r + ".out", border=True, e=e_out + 1, fp16=True), ref,
                    tol + store_tol(ref, eng, e_out))
        if i == 0:
            g.wrong(f"{r}.out no residual", out, reflect1(prelu(z2, sl_)), tol)
    # projection, centring over positions, unit L2 norm (NonlocalNet.py:468-476)
    praw = bufs.get(f"{tag}.proj_raw")
    check_conv(g, f"{tag} {proj} conv 1x1", praw, conv64(sd, proj, xa16[:, :, 1:-1, 1:-1]))
    B = praw.shape[0]
    v = praw.view(B, 256, -1)
    mean = v.mean(-1, keepdim=True)
    t = v - mean
    nrm = torch.sqrt((t * t).sum(1, keepdim=True))
    ref = (t / (nrm + O.EPS)).permute(0, 2, 1)
    ec = U * (K_PARTIAL * v.abs().mean(-1, keepdim=True) + mean.abs() + t.abs())
    tol = (ec / nrm + (t / nrm).abs() * (torch.sqrt((ec * ec).sum(1, keepdim=True)) / nrm + 12 * U)).permute(0, 2, 1)
    v32 = praw.float().view(B, 256, -1)
    t32 = v32 - v32.mean(-1, keepdim=True)
    ref32 = (t32 / (torch.norm(t32, 2, 1, keepdim=True) + O.EPS)).permute(0, 2, 1)
    rows = bufs.ctx.debug_buffer(rows_name, act=False).double().cpu()[:B * h * w * 256].view(B, h * w, 256)
    g.check(f"{tag} {proj} rows centre/normalise", rows, ref, tol, ref32)
    g.wrong(f"{tag} {proj} rows uncentred", rows, (v / torch.sqrt((v * v).sum(1, keepdim=True))).permute(0, 2, 1), tol)


COLOR_SEQ = ["conv1_1.0", "conv1_1.2", "conv1_2", "n1", "d1", "conv2_1", "conv2_2", "n2", "d2", "conv3_1", "conv3_2", "conv3_3",
             "n3", "d3", "conv4_1", "conv4_2", "conv4_3", "n4", "conv5_1", "conv5_2", "conv5_3", "n5", "conv6_1", "conv6_2",
             "conv6_3", "n6", "conv7_1", "conv7_2", "conv7_3", "conv3_3_short", "conv8_1.1", "conv8_1.1.in", "conv8_2",
             "conv8_3", "conv2_2_short", "conv9_1.1", "conv9_1.1.in", "conv9_2", "conv1_2_short", "conv10_1.1",
             "conv10_1.1.in", "conv10_2"]


def colorvid_stages(g, bufs, sd, tag, in0, ab):
    """ColorVidNet.py:96-144 from the stored buffers: the fp32 / tf32 engines' convolutions (with the reference's
    dilation and padding), every InstanceNorm apply with its stride-2 / *_ss scale / nearest x2, the output tail."""
    eng = bufs.eng
    nm = {s: f"{tag}.{s}#{i}" for i, s in enumerate(COLOR_SEQ)}
    B = in0.shape[0]
    # (output, weights, input, dilation, addend, activation); the stored border of the input is the conv's padding
    convs = [("conv1_1.0", "in0", 1), ("conv1_1.2", "conv1_1.0", 1), ("conv1_2", "conv1_1.2", 1), ("conv2_1", "d1", 1),
             ("conv2_2", "conv2_1", 1), ("conv3_1", "d2", 1), ("conv3_2", "conv3_1", 1), ("conv3_3", "conv3_2", 1),
             ("conv4_1", "d3", 1), ("conv4_2", "conv4_1", 1), ("conv4_3", "conv4_2", 1), ("conv5_1", "n4", 2),
             ("conv5_2", "conv5_1", 2), ("conv5_3", "conv5_2", 2), ("conv6_1", "n5", 2), ("conv6_2", "conv6_1", 2),
             ("conv6_3", "conv6_2", 2), ("conv7_1", "n6", 1), ("conv7_2", "conv7_1", 1), ("conv7_3", "conv7_2", 1),
             ("conv3_3_short", "n3", 1), ("conv8_2", "conv8_1.1", 1), ("conv8_3", "conv8_2", 1), ("conv2_2_short", "n2", 1),
             ("conv9_2", "conv9_1.1", 1), ("conv1_2_short", "n1", 1)]
    # norms: (name, source raw, sub, up, scale vector, border)
    norms = [("n1", "conv1_2", 1, 1, None, 1), ("d1", "conv1_2", 2, 1, "conv1_2norm_ss", 1),
             ("n2", "conv2_2", 1, 1, None, 1), ("d2", "conv2_2", 2, 1, "conv2_2norm_ss", 1),
             ("n3", "conv3_3", 1, 1, None, 1), ("d3", "conv3_3", 2, 1, "conv3_3norm_ss", 1),
             ("n4", "conv4_3", 1, 1, None, 2), ("n5", "conv5_3", 1, 1, None, 2), ("n6", "conv6_3", 1, 1, None, 1),
             ("conv8_1.1.in", "conv7_3", 1, 1 if eng != "fp32" else 2, None, 1),
             ("conv9_1.1.in", "conv8_3", 1, 1 if eng != "fp32" else 2, None, 1),
             ("conv10_1.1.in", "conv9_2", 1, 1 if eng != "fp32" else 2, None, 1)]
    raw = lambda s: bufs.get(nm[s])  # convolutions with InstanceNorm statistics store fp32 without a border
    for name, src, sub, upk, ss, p in norms:
        v = raw(src)
        z, tz = inorm_ref(v)
        gain = torch.ones(1, v.shape[1], 1, 1, dtype=torch.float64)
        scale_abs = 1.0
        if ss is not None:
            s = sd[ss + ".weight"].double().view(1, -1, 1, 1)
            z, tz, gain, scale_abs = z * s, tz * s.abs(), s.abs(), max(1e-3, s.abs().max().item())
        e = bufs.plane_e(math.sqrt(v.shape[2] * v.shape[3]) * scale_abs)
        ref = zpad(up(z[:, :, ::sub, ::sub], upk), p)
        tol = zpad(up(tz[:, :, ::sub, ::sub], upk), p) + store_tol(ref, eng, e)
        lib = bufs.get(nm[name], border=True, e=e)
        f32 = F.instance_norm(v.float(), eps=1e-5)
        if ss is not None:
            f32 = F.conv2d(f32, sd[ss + ".weight"], None, stride=2, groups=f32.shape[1])
        g.check(f"{tag}.{name} IN" + (" stride-2 *_ss" if ss else "") + (" up" if upk > 1 else ""), lib, ref, tol,
                zpad(up(f32, upk), p))
        if name == "d1":
            g.wrong(f"{tag}.d1 missing *_ss scale", lib, zpad((z / sd[ss + ".weight"].double().view(1, -1, 1, 1))[:, :, ::2, ::2], p), tol)
            g.wrong(f"{tag}.d1 odd pick", lib, zpad(F.pad(z, (0, 1, 0, 1))[:, :, 1::2, 1::2], p), tol)
            if e is not None:
                g.wrong(f"{tag}.d1 exponent+1", bufs.get(nm[name], border=True, e=e + 1), ref, tol)
    if eng == "fp16":
        return  # the conv -> ReLU -> conv chains carry device-derived exponents
    stored = {"in0": in0}
    get_in = lambda s: stored[s] if s in stored else bufs.get(nm[s], border=True)
    for out, src, dil in convs:
        x = get_in(src)
        ref = torch.relu(conv64(sd, out, x, dil=dil)) if not out.endswith("_short") else conv64(sd, out, x, dil=dil)
        lib = bufs.get(nm[out], border=True)
        pl = (lib.shape[2] - ref.shape[2]) // 2
        check_conv(g, f"{tag}.{out} conv dil {dil}", lib[:, :, pl:lib.shape[2] - pl, pl:lib.shape[3] - pl], ref)
        if pl:
            check_border(g, f"{tag}.{out}", lib, lambda t, pl=pl: zpad(t, pl), pl)
    # decoder up-convolutions: relu(conv(up(IN(raw))) + short)
    for out, nin, short in (("conv8_1.1", "conv8_1.1.in", "conv3_3_short"), ("conv9_1.1", "conv9_1.1.in", "conv2_2_short"),
                            ("conv10_1.1", "conv10_1.1.in", "conv1_2_short")):
        x = bufs.get(nm[nin], border=True)[:, :, 1:-1, 1:-1]
        xu = zpad(up(x, 2 if eng != "fp32" else 1), 1)
        ref = torch.relu(conv64(sd, out, xu) + bufs.get(nm[short]))
        lib = bufs.get(nm[out], border=True)
        check_conv(g, f"{tag}.{out} up-conv + skip", lib[:, :, 1:-1, 1:-1], ref)
    # tail: tanh(conv10_ab(LeakyReLU(conv10_2(u), 0.2))) * 128
    wab, bab = sd["conv10_ab.weight"].double(), sd["conv10_ab.bias"].double()
    u = bufs.get(nm["conv10_1.1"], border=True)
    # final_ab (fp32 engine): 4-term lane sums, a 5-level butterfly, the bias, tanhf (<= 2 ulp), * 128
    if eng == "fp32":
        y = bufs.get(nm["conv10_2"])
        check_conv(g, f"{tag}.conv10_2 conv", y, F.leaky_relu(conv64(sd, "conv10_2", u), 0.2))
        conv_err = torch.zeros(1)
    else:  # fused into conv10_2's epilogue: its outputs are not stored, their conv gate enters through |conv10_ab|
        y = F.leaky_relu(conv64(sd, "conv10_2", u), 0.2)
        conv_err = wab.abs().sum((1, 2, 3)).view(1, 2, 1, 1) * CONV_TOL * y.abs().max()
    s = F.conv2d(y, wab, bab)
    dot = F.conv2d(y.abs(), wab.abs())
    t = torch.tanh(s)
    ref = t * 128
    tol = 128 * ((12 * U * dot + U * s.abs() + conv_err) * (1 - t * t) + 4 * U * t.abs()) + U * ref.abs() + 1e-30
    g.check(f"{tag} conv10_ab + tanh * 128", ab.double(), ref, tol)
    g.wrong(f"{tag} tail without tanh", ab.double(), s.clamp(-1, 1) * 128, tol)


# ------------------------------------------------------------------------------------------------------- the runs
def frame_inputs(H, W, B, flat=False, seed=0):
    IA, IB, last = make_lab(90 + seed, B, H, W), make_lab(91 + seed, 1, H, W), make_lab(92 + seed, B, H, W)
    if flat:  # a fade / letterbox bar: constant luminance plus 1e-3 noise
        IA[:, 0:1] = 10.0 + 1e-3 * torch.randn(B, 1, H, W, generator=torch.Generator().manual_seed(seed))
    return IA, IB, last


def check_prologues(g, bufs, IA, IB):
    B, _, H, W = IA.shape
    x0 = bufs.get("fr.x0", border=True).float()
    ref = zpad(F.pad(O.vgg_preprocess(O.gray2rgb_batch(IA[:, 0:1])), (0, 0, 0, 0, 0, 5)), 1)
    g.exact("fr.x0 gray prologue", x0, ref)
    g.wrong("fr.x0 RGB-order means", x0.double(), zpad(F.pad((O.gray2rgb_batch(IA[:, 0:1]) - torch.tensor(
        [0.48501961, 0.45795686, 0.40760392]).view(1, 3, 1, 1)) * 255, (0, 0, 0, 0, 0, 5)), 1), 1e-30)
    # Lab -> sRGB -> preprocess (util.py:379-414, 347-352): fp32 with powf; the per-element bound propagates u-sized
    # errors of f = (L+16)/116 etc. through the cube (3 f^2), the matrix (sum |lin m|), the sRGB gamma (slope <= 12.92)
    lab = torch.cat((O.uncenter_l(IB[:, 0:1]), IB[:, 1:3]), 1).double()
    L, a, b = lab[:, 0:1], lab[:, 1:2], lab[:, 2:3]
    fy = (L + 16) / 116
    fs = [a / 500 + fy, fy, (fy - b / 200).clamp_min(0)]
    dfy = 4 * U * fy.abs()
    dfs = [dfy + 2 * U * ((a / 500).abs() + fs[0].abs()), dfy, dfy + 2 * U * ((b / 200).abs() + fs[2].abs())]
    white = [0.95047, 1.0, 1.08883]
    lin, dlin = [], []
    for f, df, wt in zip(fs, dfs, white):
        big = f > 0.2068966
        lv = torch.where(big, f ** 3, (f - 16 / 116) / 7.787) * wt
        dl = torch.where(big, 3 * f * f * df + 3 * U * f.abs() ** 3, (df + U * f.abs()) / 7.787) * wt + 2 * U * lv.abs()
        lin.append(lv), dlin.append(dl)
    M = O._RGB_FROM_XYZ
    out_tol = []
    for j in range(3):
        r = sum(lin[i] * M[i][j] for i in range(3))
        dr = sum(dlin[i] * abs(M[i][j]) + 3 * U * (lin[i] * M[i][j]).abs() for i in range(3))
        slope = torch.where(r > 0.0031308, 1.055 / 2.4 * r.clamp_min(0.0031308) ** (-7 / 12), torch.full_like(r, 12.92))
        out_tol.append(255 * (slope.clamp_max(12.92) * dr + 8 * U) + 255 * U)
    ref64 = O.vgg_preprocess(O.tensor_lab2rgb(lab))
    tol = torch.cat(out_tol[::-1], 1) + 2 * U * ref64.abs()
    exl = bufs.get("ex.x0", border=True)
    ref32 = O.vgg_preprocess(O.tensor_lab2rgb(lab.float()))
    g.check("ex.x0 Lab->sRGB prologue", exl[:, :3, 1:-1, 1:-1], ref64, tol, ref32)
    g.exact("ex.x0 channels 3..7 and border", torch.cat((exl[:, 3:].flatten(), exl[:, :, 0].flatten(), exl[:, :, -1].flatten(),
                                                          exl[:, :, :, 0].flatten(), exl[:, :, :, -1].flatten())),
            torch.zeros(exl[:, 3:].numel() + 2 * exl[:, :, 0].numel() + 2 * exl[:, :, :, 0].numel(), dtype=torch.float64))
    g.wrong("ex.x0 without sRGB gamma", exl[:, :3, 1:-1, 1:-1], O.vgg_preprocess(lab / torch.tensor([100., 1, 1]).view(1, 3, 1, 1).double()), tol)


def check_pooled_exemplar(g, V, IB, stage):
    """avg_pool2d(4) of the Lab map as rows (L, a, b, 1): 16-term fp32 sums."""
    ref = F.avg_pool2d(IB.double(), 4).flatten(2).permute(0, 2, 1).reshape(-1, 3)
    n = ref.shape[0]
    V = V.double().reshape(-1, 4)
    tol = 15 * U * F.avg_pool2d(IB.double().abs(), 4).flatten(2).permute(0, 2, 1).reshape(-1, 3) + U * ref.abs() + 1e-30
    g.check(stage + " avg_pool2d(4)", V[:n, :3], ref, tol)
    g.exact(stage + " 4th lane", V[:n, 3], torch.ones(n, dtype=torch.float64))
    g.wrong(stage + " window+1", V[:n, :3], F.avg_pool2d(F.pad(IB.double(), (0, 1, 0, 1), mode="replicate")[:, :, 1:, 1:], 4)
            .flatten(2).permute(0, 2, 1).reshape(-1, 3), tol)


def run_fused(ctx, sds, eng, H, W, B, flat=False):
    set_engine(ctx, eng)
    ctx.debug_flag("keep_stages", 1)
    IA, IB, last = frame_inputs(H, W, B, flat)
    ctx.set_exemplar(IB)
    ab, warp, sim = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), 1e-10, want_warp=True)
    torch.cuda.synchronize()
    bufs = Buffers(ctx, eng)
    g = Gates(f"fused {eng} {H}x{W}x{B}" + (" flat" if flat else ""))
    check_prologues(g, bufs, IA, IB)
    n_e = 14 if eng == "fp16" else None
    for side, tag, src in (("ex", "ex", "ex.x0"), ("fr", "fr", "fr.x0")):
        vgg_stages(g, bufs, sds["vgg"], tag, bufs.get(src, border=True)[:, :, 1:-1, 1:-1])
        for k, key in enumerate(("r22", "r32", "r42", "r52")):
            check_pixnorm(g, bufs, f"{tag}.n{k} feature_normalize/reflect", bufs.get(f"{tag}.{key}"), f"{tag}.n{k}", n_e)
        warp_side_stages(g, bufs, sds["warp"], tag, [f"{tag}.n{k}" for k in range(4)], n_e,
                         "ex.phi" if tag == "ex" else "fr.theta", "phi" if tag == "ex" else "theta", H, W)
    check_pooled_exemplar(g, ctx.debug_buffer("ex.V", act=False).cpu().view(-1, 4), IB, "ex.V")
    # correlation rows -> NCHW (nearest x4) and the ColorVidNet input (FrameColor.py:63-64)
    h, w = H // 4, W // 4
    yrows = ctx.debug_buffer("fr.yrows", act=False).cpu()[:B * h * w * 4].view(B, h, w, 4).permute(0, 3, 1, 2)
    simrows = ctx.debug_buffer("fr.simrows", act=False).cpu()[:B * h * w].view(B, 1, h, w)
    g.exact("warp = nearest x4 of the rows", warp.cpu(), up(yrows[:, :3], 4))
    g.exact("sim = nearest x4 of the rows", sim.cpu(), up(simrows, 4))
    in0 = bufs.get("fr.in0", border=True)
    ref_in0 = zpad(torch.cat((IA[:, 0:1], up(yrows[:, 1:3], 4), up(simrows, 4), last, torch.zeros(B, 1, H, W)), 1), 1)
    g.exact("fr.in0 cat(L, warped ab, sim, last)", in0, ref_in0.double())
    colorvid_stages(g, bufs, sds["color"], "fr", in0, ab.cpu())
    g.finish()
    return ab, warp, sim


def run_modules(ctx, sds, eng, H, W, B):
    set_engine(ctx, eng)
    ctx.debug_flag("keep_stages", 1)
    IA, IB, last = frame_inputs(H, W, B, seed=5)
    bufs = Buffers(ctx, eng)
    g = Gates(f"modules {eng} {H}x{W}x{B}")
    # VGG19 module (preprocess)
    rgb = O.gray2rgb_batch(IA[:, 0:1])
    keys = ["r22", "r32", "r42", "r52"]
    ctx.vgg19_forward(rgb.cuda(), keys, preprocess=True)
    torch.cuda.synchronize()
    g.exact("mvgg.x0 preprocess", bufs.get("mvgg.x0", border=True).float(), zpad(F.pad(O.vgg_preprocess(rgb), (0, 0, 0, 0, 0, 5)), 1))
    vgg_stages(g, bufs, sds["vgg"], "mvgg", bufs.get("mvgg.x0", border=True)[:, :, 1:-1, 1:-1])
    # WarpNet module on oracle features: n{k} are reflect-padded copies of the caller's maps
    with torch.no_grad():
        An = [O.feature_normalize(t) for t in O.vgg19_forward(sds["vgg"], rgb)[1:]]
        Bn = [O.feature_normalize(t) for t in O.exemplar_features(sds["vgg"], IB.expand(B, 3, H, W).contiguous())[1:]]
    IBb = IB.expand(B, 3, H, W).contiguous()
    y, sim = ctx.warpnet_forward(IBb.cuda(), [t.cuda() for t in An], [t.cuda() for t in Bn], 1e-10)
    torch.cuda.synchronize()
    for tag, feats, rows, proj in (("mwarpA", An, "mwarp.theta", "theta"), ("mwarpB", Bn, "mwarp.phi", "phi")):
        for k in range(4):
            lib = bufs.get(f"{tag}.n{k}", border=True)
            ref = reflect1(feats[k].double())
            if eng == "fp32":
                g.exact(f"{tag}.n{k} reflect copy", lib, ref)
            else:
                g.check(f"{tag}.n{k} reflect copy (tf32 split)", lib, ref, store_tol(ref, "tf32") + 1e-300)
        warp_side_stages(g, bufs, sds["warp"], tag, [f"{tag}.n{k}" for k in range(4)], None, rows, proj, H, W)
    check_pooled_exemplar(g, ctx.debug_buffer("mwarp.V", act=False).cpu().view(-1, 4), IBb, "mwarp.V")
    # ColorVidNet module
    x = torch.cat((IA[:, 0:1], IA[:, 1:3] * 0.5, torch.rand(B, 1, H, W, generator=torch.Generator().manual_seed(3)), last), 1)
    ab = ctx.colorvidnet_forward(x.cuda())
    torch.cuda.synchronize()
    in0 = bufs.get("mcolor.in0", border=True)
    g.exact("mcolor.in0 copy", in0, zpad(F.pad(x, (0, 0, 0, 0, 0, 1)), 1).double())
    colorvid_stages(g, bufs, sds["color"], "mcolor", in0, ab.cpu())
    g.finish()


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("eng", ENGINES)
def test_fused_path_stages(ctx, sds, eng, shape):
    run_fused(ctx, sds, eng, *shape)


@pytest.mark.parametrize("eng", ENGINES)
def test_fused_path_stages_near_flat_frame(ctx, sds, eng):
    """(v - mean) cancels: the InstanceNorm gates are in ulps of |v| (and of v^2 / var for the one-pass variance)."""
    run_fused(ctx, sds, eng, 40, 48, 1, flat=True)


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("eng", ENGINES)
def test_module_entry_stages(ctx, sds, eng, shape):
    run_modules(ctx, sds, eng, *shape)


def test_keep_stages_is_bit_identical(ctx):
    """keep_stages only changes which buffers WarpNet's residual chain writes: ab, warp and sim keep every bit."""
    IA, IB, last = frame_inputs(40, 48, 2)
    outs = []
    for keep in (0, 1, 0):
        ctx.debug_flag("keep_stages", keep)
        ctx.set_exemplar(IB)
        outs.append(ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), 1e-10, want_warp=True))
    for other in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], other))


# ---------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("eng", ["fp32", "fp16"])
def test_colorize_frames_vs_fp64_oracle_at_stage_shapes(ctx, sds, eng, shape):
    """The stage shapes end to end against the fp64 oracle computed here, with the gates of test_gpu_parity.py's
    test_oracle_on_the_fly_64x64: sim 2e-5, warp exact on rows with a clear winner, ab within max(1e-3, 2x the
    reference's own fp32 error) -- one fp32 sample of ColorVidNet's chaotic amplification is the yardstick, so the
    factor 1.25 of the golden tests (a fixed, pinned sample) does not carry over: the fp32 engine lands at 1.28x at
    56x80."""
    H, W, B = shape
    set_engine(ctx, eng)
    IA, IB, last = frame_inputs(H, W, B, seed=20)
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    ex = {}
    batch = lambda ts: [t.expand(B, *t.shape[1:]) for t in ts]  # one exemplar for the whole batch
    with torch.no_grad():
        fB = O.exemplar_features(sds64["vgg"], IB.double())
        ab64, warped64, sim64, _ = O.frame_colorization(sds64, IA.double(), IB.expand(B, 3, H, W).double(), last.double(),
                                                        batch(fB), extras=ex)
        fB32 = O.exemplar_features(sds["vgg"], IB)
        ab32, _, _, _ = O.frame_colorization(sds, IA, IB.expand(B, 3, H, W), last, batch(fB32))
    gap = O.top2_gap(ex["theta_hat"], ex["phi_hat"])
    ctx.set_exemplar(IB)
    ab, warp, sim = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), 1e-10, want_warp=True)
    assert (sim.cpu().double() - sim64).abs().max() < 2e-5
    h, w = H // 4, W // 4
    clear = (gap > 1e-5).view(B, 1, h, w).expand(B, 3, h, w)
    assert (warp.cpu()[:, :, ::4, ::4][clear].double() - warped64[:, :, ::4, ::4][clear]).abs().max() < 1e-4
    floor = (ab32.double() - ab64).abs().max().item()
    err, tol = (ab.cpu().double() - ab64).abs().max().item(), max(1e-3, 2 * floor)
    print(f"e2e {eng} {H}x{W}x{B}: |ab - ab64| = {err:.3e}, gate {tol:.3e}")
    assert err <= tol, (err, tol)


# ---------------------------------------------------------------------------------------------- illegal shapes
@pytest.mark.parametrize("H,W", [(16, 64), (24, 64), (32, 16)])
def test_frames_below_32_are_rejected_before_any_launch(ctx, H, W):
    """The reference cannot run these (VGG19's fifth max-pool raises): every entry point fails before launching."""
    import dvc

    z = lambda *s: torch.zeros(*s, device="cuda")
    feats = [z(1, c, max(1, H // d), max(1, W // d)) for c, d in ((128, 2), (256, 4), (512, 8), (512, 16))]
    calls = {
        "set_exemplar": lambda: ctx.set_exemplar(z(1, 3, H, W)),
        "warpnet_forward": lambda: ctx.warpnet_forward(z(1, 3, H, W), feats, feats, 1e-10),
        "vgg19_forward": lambda: ctx.vgg19_forward(z(1, 3, H, W), ["r52"]),
        "exemplar_import": lambda: ctx.exemplar_import(z(max(1, (H // 4) * (W // 4) * 260)), H, W),
    }
    torch.cuda.synchronize()
    for what, call in calls.items():
        n0 = ctx.launch_count()
        with pytest.raises(dvc.DvcError, match=">= 32"):
            call()
        assert ctx.launch_count() == n0, what
