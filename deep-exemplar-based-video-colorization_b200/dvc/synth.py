"""Deterministic, portable synthetic weights and frames for the three networks of the hot path.

Used by bench.py, __graft_entry__.smoke() and (through oracle/weights.py) by the tests: the CUDA path and the
CPU oracle must see the very same tensors.  Pretrained checkpoints are not in the reference tree
(the reference's .gitignore:4 excludes *.pth) and cannot be downloaded, so every parity
test uses seeded random weights.  The generator below does not depend on module
construction order or on the global RNG: each tensor is drawn from its own
`torch.Generator` seeded with (seed, index-of-key), which makes the result identical in
this container and on the GPU box (torch CPU generators are platform independent).

The distribution mirrors what the reference's constructors would give through
`nn.Conv2d` defaults (kaiming_uniform(a=sqrt(5)) == U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for
weight and bias).  PReLU slopes (reference default 0.25, NonlocalNet.py:336,368) are drawn
from U(0.1, 0.4) so that a mis-wired slope parameter is detected by the parity tests.

Key names / shapes are the reference's `state_dict()` contract:
  VGG19_pytorch  (models/NonlocalNet.py:197-226)   32 tensors
  WarpNet        (models/NonlocalNet.py:355-425)   43 tensors
  ColorVidNet    (models/ColorVidNet.py:6-94)      65 tensors
"""
import math
from collections import OrderedDict

import torch

VGG_CFG = [
    ("conv1_1", 3, 64), ("conv1_2", 64, 64),
    ("conv2_1", 64, 128), ("conv2_2", 128, 128),
    ("conv3_1", 128, 256), ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256),
    ("conv4_1", 256, 512), ("conv4_2", 512, 512), ("conv4_3", 512, 512), ("conv4_4", 512, 512),
    ("conv5_1", 512, 512), ("conv5_2", 512, 512), ("conv5_3", 512, 512), ("conv5_4", 512, 512),
]


def vgg_shapes():
    out = OrderedDict()
    for name, ci, co in VGG_CFG:
        out[name + ".weight"] = (co, ci, 3, 3)
        out[name + ".bias"] = (co,)
    return out


def warp_shapes():
    out = OrderedDict()

    def head(name, c_in, c_mid, second_idx):
        out[f"{name}.1.weight"] = (c_mid, c_in, 3, 3)
        out[f"{name}.1.bias"] = (c_mid,)
        out[f"{name}.3.weight"] = (1,)
        out[f"{name}.{second_idx}.weight"] = (64, c_mid, 3, 3)
        out[f"{name}.{second_idx}.bias"] = (64,)
        out[f"{name}.{second_idx + 2}.weight"] = (1,)

    head("layer2_1", 128, 128, 5)
    head("layer3_1", 256, 128, 5)
    head("layer4_1", 512, 256, 5)
    head("layer5_1", 512, 256, 6)
    for i in range(3):
        out[f"layer.{i}.conv1.weight"] = (256, 256, 3, 3)
        out[f"layer.{i}.conv1.bias"] = (256,)
        out[f"layer.{i}.prelu.weight"] = (1,)
        out[f"layer.{i}.conv2.weight"] = (256, 256, 3, 3)
        out[f"layer.{i}.conv2.bias"] = (256,)
    for n in ("theta", "phi"):
        out[f"{n}.weight"] = (256, 256, 1, 1)
        out[f"{n}.bias"] = (256,)
    return out


COLOR_CFG = [
    # name, cin, cout, k, has_bias
    ("conv1_1.0", 7, 32, 3, True), ("conv1_1.2", 32, 64, 3, True), ("conv1_2", 64, 64, 3, True),
    ("conv1_2norm_ss", None, 64, 1, False),
    ("conv2_1", 64, 128, 3, True), ("conv2_2", 128, 128, 3, True),
    ("conv2_2norm_ss", None, 128, 1, False),
    ("conv3_1", 128, 256, 3, True), ("conv3_2", 256, 256, 3, True), ("conv3_3", 256, 256, 3, True),
    ("conv3_3norm_ss", None, 256, 1, False),
    ("conv4_1", 256, 512, 3, True), ("conv4_2", 512, 512, 3, True), ("conv4_3", 512, 512, 3, True),
    ("conv5_1", 512, 512, 3, True), ("conv5_2", 512, 512, 3, True), ("conv5_3", 512, 512, 3, True),
    ("conv6_1", 512, 512, 3, True), ("conv6_2", 512, 512, 3, True), ("conv6_3", 512, 512, 3, True),
    ("conv7_1", 512, 512, 3, True), ("conv7_2", 512, 512, 3, True), ("conv7_3", 512, 512, 3, True),
    ("conv8_1.1", 512, 256, 3, True), ("conv3_3_short", 256, 256, 3, True),
    ("conv8_2", 256, 256, 3, True), ("conv8_3", 256, 256, 3, True),
    ("conv9_1.1", 256, 128, 3, True), ("conv2_2_short", 128, 128, 3, True), ("conv9_2", 128, 128, 3, True),
    ("conv10_1.1", 128, 128, 3, True), ("conv1_2_short", 64, 128, 3, True), ("conv10_2", 128, 128, 3, True),
    ("conv10_ab", 128, 2, 1, True),
]


def color_shapes():
    out = OrderedDict()
    for name, ci, co, k, has_bias in COLOR_CFG:
        if ci is None:  # depthwise 1x1 stride-2 "norm_ss" (ColorVidNet.py:12,16,21)
            out[name + ".weight"] = (co, 1, 1, 1)
        else:
            out[name + ".weight"] = (co, ci, k, k)
        if has_bias:
            out[name + ".bias"] = (co,)
    return out


NET_IDS = {"vgg": 0, "warp": 1, "color": 2}
_SHAPES = {"vgg": vgg_shapes, "warp": warp_shapes, "color": color_shapes}


def net_shapes(net):
    return _SHAPES[net]()


def make_state_dict(net, seed=0, dtype=torch.float32):
    """Seeded state_dict for `net` in {"vgg","warp","color"} with the reference's keys."""
    shapes = net_shapes(net)
    sd = OrderedDict()
    for idx, (key, shape) in enumerate(shapes.items()):
        g = torch.Generator(device="cpu")
        g.manual_seed(1_000_003 * (seed + 1) + 7919 * NET_IDS[net] + idx)
        if len(shape) == 1 and shape[0] == 1:  # PReLU slope
            t = torch.empty(shape, dtype=torch.float32).uniform_(0.1, 0.4, generator=g)
        else:
            if key.endswith(".weight"):
                fan_in = shape[1] * shape[2] * shape[3]
            else:  # bias: fan_in of the matching weight
                wshape = shapes[key[: -len(".bias")] + ".weight"]
                fan_in = wshape[1] * wshape[2] * wshape[3]
            bound = 1.0 / math.sqrt(fan_in)
            t = torch.empty(shape, dtype=torch.float32).uniform_(-bound, bound, generator=g)
        sd[key] = t.to(dtype)
    return sd


def make_lab(seed, B, H, W, dtype=torch.float32):
    """Synthetic centred-Lab tensor [B,3,H,W]: L-50, a, b ~ U(-50,50) (SURVEY.md §8d).

    A smooth low-frequency component is mixed in so that neighbouring pixels correlate the way
    image content does (pure white noise makes every VGG feature look alike).
    """
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    noise = torch.empty(B, 3, H, W, dtype=torch.float32).uniform_(-50.0, 50.0, generator=g)
    coarse = torch.empty(B, 3, max(H // 8, 1), max(W // 8, 1), dtype=torch.float32).uniform_(-50.0, 50.0, generator=g)
    smooth = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False)
    return (0.5 * noise + 0.5 * smooth).to(dtype)
