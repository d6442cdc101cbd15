"""CPU oracle for the exemplar-colorization forward path.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this file; the product (libdvc.so and the drop-in modules) never does.

What this is: a functional, parameter-dict restatement of the reference's forward path,
  models/FrameColor.py:5-67      (warp_color, frame_colorization)
  models/NonlocalNet.py:228-256  (VGG19_pytorch.forward)
  models/NonlocalNet.py:330-352  (ResidualBlock.forward)
  models/NonlocalNet.py:427-502  (WarpNet.forward)
  models/ColorVidNet.py:96-144   (ColorVidNet.forward)
  utils/util.py:63,97-101,155-158,347-352,379-414 (helpers)
written against torch CPU ops (the arithmetic of the reference lives in PyTorch, a
third-party dependency that requirements.txt:11 leaves unpinned; this container's torch
2.11.0 is the de-facto pinned version).  Every function is dtype-generic: pass fp32
parameters/inputs for the "reference fp32" oracle and fp64 for the "truth" oracle.

Pinning: oracle/make_golden.py imports the real reference modules from a checkout of the
reference named by DVC_REFERENCE_ROOT, runs both on the same seeded weights/inputs, asserts agreement and
writes tests/golden/*.npz.  tests/test_oracle_golden.py re-checks this file against those
vectors on every run (CPU).  The reference itself ships no tests and no golden vectors
(SURVEY.md §4), so these generated vectors are the only pin available.

PARITY UNPINNED for two helpers outside the net path: `lab_to_rgb8` and `rgb8_to_lab` (the colour conversions of
test.py:44-45,116-119) restate skimage.color.{lab2rgb,rgb2lab}, a dependency that is NOT installed in this image
(SURVEY.md 8c) and whose outputs therefore cannot be generated here; they are anchored on closed-form values, the
round trip and the reference's own fp32 torch twin tensor_lab2rgb (tests/test_oracle_golden.py).  Everything on the
net path is pinned as described above.

The N x N correlation is evaluated in query-row chunks (`row_chunk`) so that 480x864
(N=25920) and larger fit in host memory; per-row results are identical to the unchunked
formulation because every row of NonlocalNet.py:477-497 is independent.
"""
import math
import sys

import torch
import torch.nn.functional as F

EPS = sys.float_info.epsilon  # util.py:156, NonlocalNet.py:470,475

VGG_ORDER = [
    "conv1_1", "conv1_2", "P", "conv2_1", "conv2_2", "P", "conv3_1", "conv3_2", "conv3_3", "conv3_4", "P",
    "conv4_1", "conv4_2", "conv4_3", "conv4_4", "P", "conv5_1", "conv5_2", "conv5_3", "conv5_4", "P",
]


def _cast(sd, dtype):
    return {k: v.to(dtype) for k, v in sd.items()}


# ----------------------------------------------------------------------------- helpers
def uncenter_l(l):
    """util.py:63 with l_norm=1, l_mean=50 (util.py:15-18)."""
    return l * 1.0 + 50.0


def gray2rgb_batch(l):
    """util.py:97-101: (L+50)/100 replicated to three channels."""
    g = uncenter_l(l) / (2 * 50.0)
    return torch.cat((g, g, g), dim=1)


def vgg_preprocess(x):
    """util.py:347-352: RGB in [0,1] -> BGR, minus mean, times 255."""
    bgr = torch.cat((x[:, 2:3], x[:, 1:2], x[:, 0:1]), dim=1)
    mean = torch.tensor([0.40760392, 0.45795686, 0.48501961], dtype=torch.float32).to(x.dtype).view(1, 3, 1, 1)
    return (bgr - mean) * 255


def feature_normalize(x):
    """util.py:155-158: divide by (L2 norm over channels + eps)."""
    return x / (torch.norm(x, 2, 1, keepdim=True) + EPS)


_RGB_FROM_XYZ = [
    [3.24048134, -0.96925495, 0.05564664],
    [-1.53715152, 1.87599, -0.20404134],
    [-0.49853633, 0.04155593, 1.05731107],
]


def tensor_lab2rgb(lab):
    """util.py:379-414.  lab = [n,3,h,w] with un-centred L; returns sRGB in [0,1]."""
    t = lab.permute(0, 2, 3, 1)
    L, a, b = t[..., 0:1], t[..., 1:2], t[..., 2:3]
    y = (L + 16.0) / 116.0
    x = a / 500.0 + y
    z = y - b / 200.0
    z = torch.where(z < 0, torch.zeros_like(z), z)
    xyz = torch.cat((x, y, z), dim=3)
    # The transcendental branches are evaluated on the COMPACTED selected elements, like the
    # reference's boolean-mask assignments (util.py:391-394,404-407): torch's vectorised pow and its
    # scalar tail can differ in the last ulp, so where an element sits in the compacted vector
    # matters for bit-exactness of the pin.
    big = xyz > 0.2068966
    lin = torch.empty_like(xyz)
    lin[big] = torch.pow(xyz[big], 3.0)
    lin[~big] = (xyz[~big] - 16.0 / 116.0) / 7.787
    lin[..., 0] = lin[..., 0] * 0.95047
    lin[..., 2] = lin[..., 2] * 1.08883
    # the reference converts the float64 numpy matrix with .type_as(xyz) (util.py:399)
    m = torch.tensor(_RGB_FROM_XYZ, dtype=torch.float64).to(lab.dtype)
    rgb = torch.mm(lin.reshape(-1, 3), m).view(lab.size(0), lab.size(2), lab.size(3), 3)
    rgb = rgb.permute(0, 3, 1, 2)
    hi = rgb > 0.0031308
    out = torch.empty_like(rgb)
    out[hi] = 1.055 * torch.pow(rgb[hi], 1 / 2.4) - 0.055
    out[~hi] = rgb[~hi] * 12.92
    return out.clamp(0.0, 1.0)


# ----------------------------------------------------------------------------- VGG19
def vgg19_forward(sd, x, out_keys=("r12", "r22", "r32", "r42", "r52"), preprocess=True):
    """NonlocalNet.py:228-256.  All 16 convs are evaluated like the reference does."""
    if preprocess:
        x = vgg_preprocess(x)
    out = {}
    block, idx = 1, 1
    for name in VGG_ORDER:
        if name == "P":
            x = F.max_pool2d(x, kernel_size=2, stride=2)
            out[f"p{block}"] = x
            block, idx = block + 1, 1
        else:
            x = F.relu(F.conv2d(x, sd[name + ".weight"], sd[name + ".bias"], padding=1))
            out[f"r{block}{idx}"] = x
            idx += 1
    return [out[k] for k in out_keys]


# ----------------------------------------------------------------------------- WarpNet
def _in_norm(x):
    return F.instance_norm(x, eps=1e-5)


def _rconv(x, sd, key, stride=1):
    """ReflectionPad2d(1) + valid 3x3 conv (NonlocalNet.py:365-366 and siblings)."""
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), sd[key + ".weight"], sd[key + ".bias"], stride=stride)


def _up(x, k):
    return F.interpolate(x, scale_factor=k, mode="nearest")


def warp_head(sd, name, x):
    """The four feature heads, NonlocalNet.py:364-410."""
    if name == "layer2_1":
        x = F.prelu(_in_norm(_rconv(x, sd, "layer2_1.1")), sd["layer2_1.3.weight"])
        x = F.prelu(_in_norm(_rconv(x, sd, "layer2_1.5", stride=2)), sd["layer2_1.7.weight"])
    elif name == "layer3_1":
        x = F.prelu(_in_norm(_rconv(x, sd, "layer3_1.1")), sd["layer3_1.3.weight"])
        x = F.prelu(_in_norm(_rconv(x, sd, "layer3_1.5")), sd["layer3_1.7.weight"])
    elif name == "layer4_1":
        x = F.prelu(_in_norm(_rconv(x, sd, "layer4_1.1")), sd["layer4_1.3.weight"])
        x = F.prelu(_in_norm(_rconv(x, sd, "layer4_1.5")), sd["layer4_1.7.weight"])
        x = _up(x, 2)
    elif name == "layer5_1":
        x = F.prelu(_in_norm(_rconv(x, sd, "layer5_1.1")), sd["layer5_1.3.weight"])
        x = _up(x, 2)
        x = F.prelu(_in_norm(_rconv(x, sd, "layer5_1.6")), sd["layer5_1.8.weight"])
        x = _up(x, 2)
    else:
        raise KeyError(name)
    return x


def residual_block(sd, i, x):
    """NonlocalNet.py:341-352: one shared PReLU slope per block."""
    slope = sd[f"layer.{i}.prelu.weight"]
    out = F.prelu(_in_norm(_rconv(x, sd, f"layer.{i}.conv1")), slope)
    out = _in_norm(_rconv(out, sd, f"layer.{i}.conv2"))
    return F.prelu(out + x, slope)


def warp_features(sd, r2, r3, r4, r5):
    """NonlocalNet.py:451-465 for one side (A or B): heads, height repair, concat, 3 residual blocks."""
    f2 = warp_head(sd, "layer2_1", r2)
    f3 = warp_head(sd, "layer3_1", r3)
    f4 = warp_head(sd, "layer4_1", r4)
    f5 = warp_head(sd, "layer5_1", r5)
    if f5.shape[2] != f2.shape[2] or f5.shape[3] != f2.shape[3]:
        f5 = F.pad(f5, (0, 0, 1, 1), "replicate")  # NonlocalNet.py:461-463 (rows only)
    x = torch.cat((f2, f3, f4, f5), 1)
    for i in range(3):
        x = residual_block(sd, i, x)
    return x


def project_normalize(sd, which, feat):
    """NonlocalNet.py:468-476: 1x1 conv, centre over positions, unit L2 norm over channels. -> [B,256,N]"""
    B = feat.shape[0]
    t = F.conv2d(feat, sd[which + ".weight"], sd[which + ".bias"]).view(B, 256, -1)
    t = t - t.mean(dim=-1, keepdim=True)
    return t / (torch.norm(t, 2, 1, keepdim=True) + EPS)


def corr_softmax_warp(theta_hat, phi_hat, V, temperature, row_chunk=4096, return_argmax=False):
    """NonlocalNet.py:477-498 restated per query-row chunk.

    theta_hat [B,C,NA], phi_hat [B,C,NB], V [B,NB,ch].  Returns y [B,NA,ch], sim [B,NA]
    (sim = row max of f BEFORE the temperature, NonlocalNet.py:481-483)."""
    B, C, NA = theta_hat.shape
    ys, sims, idxs = [], [], []
    for r0 in range(0, NA, row_chunk):
        th = theta_hat[:, :, r0:r0 + row_chunk].permute(0, 2, 1)  # [B,rows,C]
        f = torch.matmul(th, phi_hat)  # [B,rows,NB]
        m, idx = torch.max(f, -1)
        p = F.softmax(f / temperature, dim=-1)
        ys.append(torch.matmul(p, V))
        sims.append(m)
        idxs.append(idx)
    y, sim = torch.cat(ys, 1), torch.cat(sims, 1)
    if return_argmax:
        return y, sim, torch.cat(idxs, 1)
    return y, sim


def top2_gap(theta_hat, phi_hat, row_chunk=4096):
    """Gap between the best and second-best correlation per query row (tie-aware metric, SURVEY.md §8c)."""
    B, C, NA = theta_hat.shape
    gaps = []
    for r0 in range(0, NA, row_chunk):
        f = torch.matmul(theta_hat[:, :, r0:r0 + row_chunk].permute(0, 2, 1), phi_hat)
        t2 = torch.topk(f, 2, dim=-1).values
        gaps.append(t2[..., 0] - t2[..., 1])
    return torch.cat(gaps, 1)


def warpnet_forward(sd, B_lab_map, A_feats, B_feats, temperature=0.005, row_chunk=4096, extras=None):
    """WarpNet.forward, NonlocalNet.py:427-502.  A_feats/B_feats = (r2,r3,r4,r5) already feature_normalize()d."""
    B, ch, H, W = B_lab_map.shape
    h, w = int(H / 4), int(W / 4)
    fa = warp_features(sd, *A_feats)
    fb = warp_features(sd, *B_feats)
    theta = project_normalize(sd, "theta", fa)
    phi = project_normalize(sd, "phi", fb)
    V = F.avg_pool2d(B_lab_map, 4).view(B, ch, -1).permute(0, 2, 1)
    y, sim, idx = corr_softmax_warp(theta, phi, V, temperature, row_chunk, return_argmax=True)
    if extras is not None:
        extras.update(theta_hat=theta, phi_hat=phi, V=V, argmax=idx, y_rows=y, sim_rows=sim)
    y = y.permute(0, 2, 1).contiguous().view(B, ch, h, w)
    sim = sim.view(B, 1, h, w)
    return _up(y, 4), _up(sim, 4)


# ----------------------------------------------------------------------------- ColorVidNet
def colorvidnet_forward(sd, x):
    """ColorVidNet.forward, ColorVidNet.py:96-144 (nearest+conv 'deconvs' 81-83, InstanceNorm 86-94)."""

    def c(name, t, dil=1, relu=True):
        t = F.conv2d(t, sd[name + ".weight"], sd[name + ".bias"], padding=dil, dilation=dil)
        return F.relu(t) if relu else t

    def ss(name, t):  # depthwise 1x1, stride 2, no bias
        return F.conv2d(t, sd[name + ".weight"], None, stride=2, groups=t.shape[1])

    t = c("conv1_1.2", c("conv1_1.0", x))          # Sequential(conv, ReLU, conv) then relu1_1
    t = c("conv1_2", t)
    n1 = _in_norm(t)
    t = c("conv2_2", c("conv2_1", ss("conv1_2norm_ss", n1)))
    n2 = _in_norm(t)
    t = c("conv3_3", c("conv3_2", c("conv3_1", ss("conv2_2norm_ss", n2))))
    n3 = _in_norm(t)
    t = c("conv4_3", c("conv4_2", c("conv4_1", ss("conv3_3norm_ss", n3))))
    t = _in_norm(t)
    t = _in_norm(c("conv5_3", c("conv5_2", c("conv5_1", t, 2), 2), 2))
    t = _in_norm(c("conv6_3", c("conv6_2", c("conv6_1", t, 2), 2), 2))
    t = _in_norm(c("conv7_3", c("conv7_2", c("conv7_1", t))))
    t = F.relu(c("conv8_1.1", _up(t, 2), relu=False) + c("conv3_3_short", n3, relu=False))
    t = _in_norm(c("conv8_3", c("conv8_2", t)))
    t = F.relu(c("conv9_1.1", _up(t, 2), relu=False) + c("conv2_2_short", n2, relu=False))
    t = _in_norm(c("conv9_2", t))
    t = F.relu(c("conv10_1.1", _up(t, 2), relu=False) + c("conv1_2_short", n1, relu=False))
    t = F.leaky_relu(c("conv10_2", t, relu=False), 0.2)
    t = F.conv2d(t, sd["conv10_ab.weight"], sd["conv10_ab.bias"])
    return torch.tanh(t) * 128


# ----------------------------------------------------------------------------- per-frame glue
def exemplar_features(vgg_sd, IB_lab):
    """test.py:61-66: Lab exemplar -> sRGB -> VGG maps (computed once per exemplar)."""
    rgb = tensor_lab2rgb(torch.cat((uncenter_l(IB_lab[:, 0:1]), IB_lab[:, 1:3]), dim=1))
    return vgg19_forward(vgg_sd, rgb)


def frame_colorization(sds, IA_lab, IB_lab, IA_last_lab, features_B, temperature=1e-10, row_chunk=4096,
                       extras=None):
    """FrameColor.py:41-67 (+ warp_color 5-38) with feature_noise = luminance_noise = 0.

    sds = {"vgg":..., "warp":..., "color":...}.  Returns (ab_predict, warped_lab, sim, features_A)."""
    IA_l = IA_lab[:, 0:1]
    fA = vgg19_forward(sds["vgg"], gray2rgb_batch(IA_l))
    An = [feature_normalize(t) for t in fA[1:]]
    Bn = [feature_normalize(t) for t in features_B[1:]]
    warped, sim = warpnet_forward(sds["warp"], IB_lab, An, Bn, temperature, row_chunk, extras)
    color_in = torch.cat((IA_l, warped[:, 1:3], sim, IA_last_lab), dim=1)
    ab = colorvidnet_forward(sds["color"], color_in)
    return ab, warped, sim, fA


def colorize_clip(sds, frames_lab, IB_lab, temperature=1e-10, row_chunk=4096):
    """test.py:57-96 per segment: frames processed in order, frame t-1's prediction feeds frame t."""
    fB = exemplar_features(sds["vgg"], IB_lab)
    last = torch.zeros_like(frames_lab[0:1])  # test.py:80
    outs = []
    for t in range(frames_lab.shape[0]):
        IA = frames_lab[t:t + 1]
        ab, _, _, _ = frame_colorization(sds, IA, IB_lab, last, fB, temperature, row_chunk)
        last = torch.cat((IA[:, 0:1], ab), dim=1)  # test.py:96
        outs.append(ab)
    return torch.cat(outs, 0)


def resize_half(x):
    """test.py:58,71: F.interpolate(x, scale_factor=0.5, mode="bilinear")."""
    return F.interpolate(x, scale_factor=0.5, mode="bilinear")


def upsample2_scaled(ab, scale=1.25):
    """test.py:100-102: F.interpolate(ab, scale_factor=2, mode="bilinear") * 1.25."""
    return F.interpolate(ab, scale_factor=2, mode="bilinear") * scale


def lab_to_rgb8(l, ab):
    """utils/util.py:140-151 (`batch_lab2rgb_transpose_mc`, one image per batch entry): Lab = (l + 50, ab) in float64 ->
    skimage.color.lab2rgb -> clip -> * 255 -> uint8 (truncation), returned as [B,H,W,3].

    PARITY UNPINNED for this function: `skimage` is not installed in this image (SURVEY.md 8c), so the conversion is
    restated from skimage.color.colorconv (lab2xyz: D65 / observer "2" white point (0.95047, 1, 1.08883), z < 0 -> 0,
    threshold 0.2068966, (t - 16/116) / 7.787; xyz2rgb: rgb_from_xyz = inv(xyz_from_rgb), gamma threshold 0.0031308)
    and anchored on the reference's own torch twin `tensor_lab2rgb` (utils/util.py:379-414, pinned bit-exactly by
    tests/golden) in tests/test_oracle_golden.py."""
    import numpy as np

    lab = np.concatenate([l.double().numpy() + 50.0, ab.double().numpy()], axis=1).transpose(0, 2, 3, 1)  # [B,H,W,3]
    L, A, Bq = lab[..., 0], lab[..., 1], lab[..., 2]
    y = (L + 16.0) / 116.0
    x = (A / 500.0) + y
    z = y - (Bq / 200.0)
    z = np.where(z < 0, 0.0, z)
    out = np.stack([x, y, z], axis=-1)
    mask = out > 0.2068966
    out = np.where(mask, np.power(out, 3.0), (out - 16.0 / 116.0) / 7.787)
    out = out * np.array([0.95047, 1.0, 1.08883])
    xyz_from_rgb = np.array([[0.412453, 0.357580, 0.180423], [0.212671, 0.715160, 0.072169], [0.019334, 0.119193, 0.950227]])
    arr = out @ np.linalg.inv(xyz_from_rgb).T
    mask = arr > 0.0031308
    arr = np.where(mask, 1.055 * np.power(np.where(mask, arr, 1.0), 1 / 2.4) - 0.055, arr * 12.92)
    return torch.from_numpy((np.clip(arr, 0, 1) * 255).astype("uint8"))


def rgb8_to_lab(rgb):
    """test.py:44-45: RGB2Lab (util_distortion.py:18-23, skimage.color.rgb2lab in float64) -> ToTensor (lib/functional.py:
    85-103, `.float()` without /255) -> Normalize (util_distortion.py:85-92: L - 50).  rgb: uint8 [B,H,W,3] -> float32
    [B,3,H,W].  PARITY UNPINNED (skimage absent): restated from skimage.color.colorconv (rgb2xyz: uint8 / 255, inverse
    gamma threshold 0.04045; xyz2lab: D65 / observer "2" white point, threshold 0.008856, np.cbrt, 7.787 t + 16/116)."""
    import numpy as np

    arr = rgb.numpy().astype(np.float64) / 255.0
    mask = arr > 0.04045
    arr = np.where(mask, np.power((np.where(mask, arr, 1.0) + 0.055) / 1.055, 2.4), arr / 12.92)
    xyz_from_rgb = np.array([[0.412453, 0.357580, 0.180423], [0.212671, 0.715160, 0.072169], [0.019334, 0.119193, 0.950227]])
    xyz = arr @ xyz_from_rgb.T
    t = xyz / np.array([0.95047, 1.0, 1.08883])
    mask = t > 0.008856
    f = np.where(mask, np.cbrt(t), 7.787 * t + 16.0 / 116.0)
    x, y, z = f[..., 0], f[..., 1], f[..., 2]
    lab = np.stack([116.0 * y - 16.0, 500.0 * (x - y), 200.0 * (y - z)], axis=1)  # [B,3,H,W] float64
    out = torch.from_numpy(lab).float()
    out[:, 0:1] = out[:, 0:1] - 50.0
    return out


def legal_shape(H, W):
    """Shapes the reference's full path accepts (SURVEY.md fact 2): H % 8 == 0 and W % 16 == 0 (NonlocalNet.py:464), and
    H, W >= 32: below that VGG19's fifth max-pool (NonlocalNet.py:255) gets a 1-pixel input and raises."""
    return H % 8 == 0 and W % 16 == 0 and H >= 32 and W >= 32


def corr_flops(NA, NB, C=256, ch=3):
    """Algorithmic FLOPs of the correlation + warp (SURVEY.md §8d): 2*NA*NB*(C+ch)."""
    return 2.0 * NA * NB * (C + ch)


def contextual_loss_forward(X_features, Y_features, h=0.1, feature_centering=True):
    """ContextualLoss_forward.forward, models/ContextualLoss.py:82-126, line by line (train.py's default matching direction).
    X_features, Y_features [B,C,h,w]; returns the per-sample loss [B]."""
    batch_size, feature_depth = X_features.shape[0], X_features.shape[1]
    if feature_centering:
        mean_y = Y_features.view(batch_size, feature_depth, -1).mean(dim=-1).unsqueeze(dim=-1).unsqueeze(dim=-1)
        X_features = X_features - mean_y
        Y_features = Y_features - mean_y
    X = feature_normalize(X_features).view(batch_size, feature_depth, -1)
    Y = feature_normalize(Y_features).view(batch_size, feature_depth, -1)
    d = 1 - torch.matmul(X.permute(0, 2, 1), Y)
    d_norm = d / (torch.min(d, dim=-1, keepdim=True)[0] + 1e-5)
    w = torch.exp((1 - d_norm) / h)
    A_ij = w / torch.sum(w, dim=-1, keepdim=True)
    CX = torch.mean(torch.max(A_ij, dim=-1)[0], dim=1)
    return -torch.log(CX)
