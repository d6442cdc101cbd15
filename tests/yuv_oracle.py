"""OpenCV's BT.601 limited-range 4:2:0 conversions (cv2.cvtColor COLOR_YUV2RGB_I420 / COLOR_RGB2YUV_I420) restated in numpy with
int64 arithmetic: 20-bit fixed point, rounding by + 2^19, arithmetic >> 20, saturation to [0, 255].

An I420 frame of H x W pixels (H, W even) is [3H/2, W] uint8: the Y plane [H, W], then U [(H/2) (W/2)], then V, as cv2 lays it out.
Chroma is nearest-neighbour: each (u, v) serves its 2 x 2 block, and RGB -> I420 takes the block's top-left pixel (no averaging).
Leading batch dimensions are allowed in both directions."""
import numpy as np

SHIFT = 20
HALF = 1 << (SHIFT - 1)
Y2RGB, V2R, V2G, U2G, U2B = 1220542, 1673527, -852492, -409993, 2116026
R2Y, G2Y, B2Y = 269484, 528482, 102760
R2U, G2U, B2U = -155188, -305135, 460324
R2V, G2V, B2V = 460324, -385875, -74448


def _sat(x):
    return np.clip(x, 0, 255).astype(np.uint8)


def split_planes(yuv):
    """[..., 3H/2, W] -> Y [..., H, W], U and V [..., H/2, W/2]."""
    yuv = np.asarray(yuv, dtype=np.uint8)
    H, W = yuv.shape[-2] * 2 // 3, yuv.shape[-1]
    lead = yuv.shape[:-2]
    flat = yuv.reshape(*lead, -1)
    n, q = H * W, (H // 2) * (W // 2)
    return (flat[..., :n].reshape(*lead, H, W), flat[..., n:n + q].reshape(*lead, H // 2, W // 2),
            flat[..., n + q:n + 2 * q].reshape(*lead, H // 2, W // 2))


def join_planes(y, u, v):
    """Y [..., H, W], U, V [..., H/2, W/2] -> [..., 3H/2, W]."""
    lead, (H, W) = y.shape[:-2], y.shape[-2:]
    flat = np.concatenate([y.reshape(*lead, -1), u.reshape(*lead, -1), v.reshape(*lead, -1)], axis=-1)
    return flat.reshape(*lead, 3 * H // 2, W)


def i420_to_rgb(yuv):
    """[..., 3H/2, W] uint8 -> [..., H, W, 3] uint8 (COLOR_YUV2RGB_I420)."""
    y, u, v = split_planes(yuv)
    y = np.maximum(y.astype(np.int64) - 16, 0) * Y2RGB
    d = np.repeat(np.repeat(u.astype(np.int64) - 128, 2, axis=-2), 2, axis=-1)
    e = np.repeat(np.repeat(v.astype(np.int64) - 128, 2, axis=-2), 2, axis=-1)
    r = (y + HALF + V2R * e) >> SHIFT
    g = (y + HALF + V2G * e + U2G * d) >> SHIFT
    b = (y + HALF + U2B * d) >> SHIFT
    return np.stack([_sat(r), _sat(g), _sat(b)], axis=-1)


def rgb_to_i420(rgb):
    """[..., H, W, 3] uint8 -> [..., 3H/2, W] uint8 (COLOR_RGB2YUV_I420)."""
    rgb = np.asarray(rgb).astype(np.int64)
    R, G, B = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    y = _sat((R2Y * R + G2Y * G + B2Y * B + HALF + (16 << SHIFT)) >> SHIFT)
    r, g, b = R[..., ::2, ::2], G[..., ::2, ::2], B[..., ::2, ::2]
    u = _sat((R2U * r + G2U * g + B2U * b + HALF + (128 << SHIFT)) >> SHIFT)
    v = _sat((R2V * r + G2V * g + B2V * b + HALF + (128 << SHIFT)) >> SHIFT)
    return join_planes(y, u, v)
