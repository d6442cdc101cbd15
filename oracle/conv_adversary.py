"""Worst-case inputs for the device-scaled fp16 store of the convolution engines (dvc_internal.cuh: dyn_out_exponent).

A conv -> ReLU -> conv chain stores its activations as fp16 hi / lo planes of y * 2^e.  The exponent e is derived on the
device from a bound of |y|:

    bound = (max|x| * L1 + max|bias| + max|add|) * gain * 1.0001,   L1 = max_o sum |w[o]|,  gain = max(1, |slope|)

and e16_from_bound() takes the largest e with bound * 2^e <= 2^15, one binade below the fp16 maximum.  The tensor-core
epilogue clamps to +-65504 and the first-layer kernel does not clamp at all, so a bound that is too small shows up only
as saturated (or infinite) activations.  Random inputs sit about sqrt(K) below the L1 bound, so no random test can see
a wrong bound; the inputs built here reach it:

  o* = the output channel whose attainable |y| is largest, one output pixel of it is the target;
  the 3x3 (dilated) neighbourhood of that pixel is A * s * sign(w[o*]) over every input channel and tap, with s chosen
  so that the bias adds to the sum (or, for LeakyReLU with a slope > 1, so that the sum lands on the negative branch);
  the addend, where there is one, is +max|add| at the target; everything else is noise of at most A / 64.

A is a power of two: the static input bound of the debug hook is 32768 * 2^-e16(A), which equals A exactly only then
(any other amplitude would be rounded up by as much as 2x and hide a factor-2 error in the bound).  For the up-convolution
(nearest x2 + 3x3, evaluated as four 2x2 phase convolutions on the low-resolution map) the same is done with the phase
whose summed weights have the largest L1 norm; the library bounds all four phases with the largest phase L1.

Where a case has a free magnitude (the addend of the up-convolution, the bias of the synthetic LeakyReLU layer) it is
chosen so that this term carries at least 3/4 of the bound and the bound sits at 0.7 of its binade: dropping the term
(or the gain of 3) from the bound then moves e up by two and the attained value past 65504.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.weights import make_state_dict

VGG, WARP, COLOR = 0, 1, 2
NETKEY = {VGG: "vgg", WARP: "warp", COLOR: "color"}
NOISE = 1.0 / 64  # |x| elsewhere <= A * NOISE, |add| elsewhere <= max|add| * NOISE
BINADE_POS = 0.7  # where a tuned bound sits in its binade (a third of it is still below the binade under it)


def synthetic_layer(cin, cout, k=3, seed=0):
    """Seeded conv layer under a name no layer program reads: ("edge.c<cin>_o<cout>_k<k>", state dict)."""
    name = f"edge.c{cin}_o{cout}_k{k}"
    g = torch.Generator().manual_seed(7_000_003 + 1009 * cin + 31 * cout + k + 100_003 * seed)
    bound = 1.0 / math.sqrt(cin * k * k)
    w = torch.empty(cout, cin, k, k).uniform_(-bound, bound, generator=g)
    b = torch.empty(cout).uniform_(-bound, bound, generator=g)
    return name, {name + ".weight": w, name + ".bias": b}


def library_l1max(w):
    """ConvW::l1max as dvc_set_weight / upload_w16 compute it: float(max_o sum |w[o]| (double) * (1 + 1e-6))."""
    return float(np.float32(w.double().abs().flatten(1).sum(1).max().item() * (1.0 + 1e-6)))


def phase_weights(w):
    """[Cout,Cin,3,3] -> [4,Cout,Cin,2,2]: phase (a, b) of Upsample(2, nearest) + 3x3 conv (zero pad 1) is a 2x2 conv
    on the low-resolution rows {i-1, i} (a = 0) or {i, i+1} (a = 1), and likewise for columns; its taps are float32 sums
    of the 3x3 taps that land on the same source pixel, in dvc_set_weight's order (ky outer, kx inner)."""
    rows = {0: ([0], [1, 2]), 1: ([0, 1], [2])}
    out = torch.zeros(4, w.shape[0], w.shape[1], 2, 2, dtype=torch.float32)
    for ph in range(4):
        a, b2 = ph >> 1, ph & 1
        for r in range(2):
            for cc in range(2):
                v = torch.zeros(w.shape[0], w.shape[1], dtype=torch.float32)
                for ky in rows[a][r]:
                    for kx in rows[b2][cc]:
                        v = v + w[:, :, ky, kx].float()
                out[ph, :, :, r, cc] = v
    return out


def device_bound(ain, l1, bmax, aadd, gain):
    """dyn_out_exponent's bound in float32: (fmaf(ain, l1, bmax) + aadd) * gain * 1.0001f."""
    f = np.float32
    fma = f(float(f(ain)) * float(f(l1)) + float(f(bmax)))
    return float((fma + f(aadd)) * f(gain) * f(1.0001))


def e16_from_bound(bound):
    """dvc_internal.cuh e16_from_bound: e = 15 - (frexp exponent of bound), so bound * 2^e lies in (2^14, 2^15] (2^14
    for an exact power of two), clamped to [-100, 24]."""
    if not bound > 0:
        return 24
    _, ex = math.frexp(bound)  # bound = m * 2^ex, m in [0.5, 1)
    return max(-100, min(24, 15 - ex))


def _tuned(base, scale):
    """The free term t >= 3 * base that puts (base + t) * scale at BINADE_POS of a binade."""
    top = 2.0 ** math.ceil(math.log2(4 * base * scale / BINADE_POS))
    return BINADE_POS * top / scale - base


def _sign(t):
    return torch.where(t >= 0, 1.0, -1.0)


def _noise(g, shape, amp):
    return (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * amp


def build(case):
    """Case dict -> dict(net, name, sd, cin, cout, x, add, kw, in_bound, A, target, bound_terms)."""
    c = dict(CASES[case])
    net, A, H, W = c["net"], c["A"], c["H"], c["W"]
    act, slope, dil = c.get("act", 0), c.get("slope", 0.0), c.get("dil", 1)
    if "synthetic" in c:
        name, sd = synthetic_layer(*c["synthetic"])
        sd = {k: v.clone() for k, v in sd.items()}
    else:
        name = c["name"]
        full = make_state_dict(NETKEY[net], seed=0)
        sd = {name + ".weight": full[name + ".weight"], name + ".bias": full[name + ".bias"]}
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    cout, cin = w.shape[:2]
    gain = max(1.0, abs(slope)) if act == 2 else 1.0
    g = torch.Generator().manual_seed(4242 + sum(map(ord, case)))
    x = _noise(g, (1, cin, H, W), A * NOISE)
    add = None
    upconv = c.get("upconv", False)
    if upconv:
        pw = phase_weights(w).double()
        l1 = pw.abs().flatten(2).sum(2)  # [4, Cout]
        l1max = float(np.float32(l1.max().item() * (1.0 + 1e-6)))
        score = A * l1 + b.double()[None]  # ReLU: the positive branch
        ph, o = divmod(int(score.argmax()), cout)
        i, j = H // 2, W // 2
        a, b2 = ph >> 1, ph & 1
        r0, c0 = (0 if a else -1), (0 if b2 else -1)
        x[0, :, i + r0:i + r0 + 2, j + c0:j + c0 + 2] = A * _sign(pw[ph, o])
        bmax = b.abs().max().item()
        M = _tuned(A * l1max + bmax, 1.0001)
        add = _noise(g, (1, cout, 2 * H, 2 * W), M * NOISE)
        target = (o, 2 * i + a, 2 * j + b2)
        add[0, o, target[1], target[2]] = M
        aadd = M
    else:
        l1 = w.double().abs().flatten(1).sum(1)
        l1max = library_l1max(w)
        if act == 2 and slope > 1:
            s = -torch.ones(cout, dtype=torch.float64)  # the negative branch: |y| = slope * |pre|
        elif act == 1:
            s = torch.ones(cout, dtype=torch.float64)
        else:
            s = _sign(b.double())
        if c.get("tune_bias"):  # the bias of the target channel carries >= 3/4 of the bound, with the sign of s
            o = int(l1.argmax())
            b[o] = float(s[o]) * _tuned(A * l1max, gain * 1.0001)
            name += "_adv"  # not the untuned synthetic layer of the same shape
            sd = {name + ".weight": w, name + ".bias": b}
        score = A * l1 + s * b.double()
        o = int(score.argmax())
        i, j = H // 2, W // 2
        k = w.shape[2]
        for ky in range(k):
            for kx in range(k):
                yy, xx = i + (ky - k // 2) * dil, j + (kx - k // 2) * dil
                x[0, :, yy, xx] = float(s[o]) * A * _sign(w[o, :, ky, kx].double())
        target = (o, i, j)
        bmax = b.abs().max().item()
        aadd = 0.0
    first = cin <= 8
    kw = dict(act=act, slope=slope, dil=dil, upconv=upconv)
    return dict(case=case, net=net, name=name, sd=sd, cin=cin, cout=cout, x=x.float(), add=None if add is None else add.float(),
                kw=kw, in_bound=-1.0 if first else A, A=A, target=target,
                bound=device_bound(A, l1max, bmax, aadd, gain), terms=dict(l1max=l1max, bmax=bmax, aadd=aadd, gain=gain))


def forward64(adv):
    """The case's layer in float64: (pad / up-sample), conv, bias, addend, activation -> y [1, Cout, Ho, Wo]."""
    w, b = adv["sd"][adv["name"] + ".weight"].double(), adv["sd"][adv["name"] + ".bias"].double()
    kw, x = adv["kw"], adv["x"].double()
    if kw["upconv"]:
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    y = F.conv2d(F.pad(x, (kw["dil"],) * 4), w, b, dilation=kw["dil"])
    if adv["add"] is not None:
        y = y + adv["add"].double()
    if kw["act"] == 1:
        y = F.relu(y)
    elif kw["act"] == 2:
        y = F.leaky_relu(y, kw["slope"])
    return y


CASES = {
    # a ReLU layer of the VGG trunk (conv -> ReLU -> conv on device-scaled planes)
    "vgg_conv3_2_relu": dict(net=VGG, name="conv3_2", H=7, W=9, A=4, act=1),
    # a dilated ColorVidNet layer
    "color_conv5_2_dil2_relu": dict(net=COLOR, name="conv5_2", H=7, W=7, A=2, act=1, dil=2),
    # the decoder up-convolution with its skip addend (max|add| carries 3/4 of the bound)
    "color_conv8_1_upconv_add": dict(net=COLOR, name="conv8_1.1", H=5, W=7, A=2, act=1, upconv=True),
    # LeakyReLU with slope 3 on its negative branch (gain 3), the bias carrying 3/4 of the bound
    "synthetic_lrelu3_bias": dict(net=COLOR, synthetic=(64, 72, 3), H=5, W=9, A=8, act=2, slope=3.0, tune_bias=True),
    # the first layers (conv_first_kernel: no clamp in its fp16 store), bound measured on the device
    "vgg_conv1_1_first": dict(net=VGG, name="conv1_1", H=5, W=13, A=64, act=1),
    "color_conv1_1_0_first": dict(net=COLOR, name="conv1_1.0", H=5, W=13, A=64, act=1),
}
