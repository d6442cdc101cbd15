"""The numpy I420 conversions of tests/yuv_oracle.py against cv2.cvtColor, byte for byte, and the Y4M header parser and writer of
tools/colorize_y4m.py.  CPU only: the oracle pins the arithmetic that csrc/prepost.cu's I420 kernels restate, so the GPU tests
can compare the device with it."""
import io
import os
import sys

import numpy as np
import pytest
import torch

import yuv_oracle as Y
from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import colorize_y4m as T  # noqa: E402

cv2 = pytest.importorskip("cv2")

SIZES = [(2, 2), (2, 34), (2, 2 * 97), (36, 2), (2 * 53, 2), (6, 34), (36, 50), (432, 768), (1080, 1920)]


def _yuv_random(rng, H, W):
    return rng.integers(0, 256, (3 * H // 2, W), dtype=np.uint8)


def _yuv_clamps(H, W):
    """Every (y, u, v) corner and edge of the byte range: y below 16 and above 235, u and v at 0 and 255 (every R, G and B clamp,
    low and high, is reached), tiled over the frame."""
    rng = np.random.default_rng(H * 7919 + W)
    vals = np.array([0, 1, 15, 16, 17, 128, 235, 236, 254, 255], dtype=np.uint8)
    y = vals[rng.integers(0, len(vals), (H, W))]
    u = vals[rng.integers(0, len(vals), (H // 2, W // 2))]
    v = vals[rng.integers(0, len(vals), (H // 2, W // 2))]
    return Y.join_planes(y, u, v)


@pytest.mark.parametrize("H,W", SIZES, ids=lambda v: str(v))
def test_i420_to_rgb_equals_cv2(H, W):
    rng = np.random.default_rng(H * 31 + W)
    for yuv in (_yuv_random(rng, H, W), _yuv_clamps(H, W)):
        assert np.array_equal(Y.i420_to_rgb(yuv), cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_I420))


@pytest.mark.parametrize("H,W", SIZES, ids=lambda v: str(v))
def test_rgb_to_i420_equals_cv2(H, W):
    rng = np.random.default_rng(H * 37 + W)
    extremes = np.array([0, 1, 254, 255], dtype=np.uint8)
    for rgb in (rng.integers(0, 256, (H, W, 3), dtype=np.uint8), extremes[rng.integers(0, 4, (H, W, 3))]):
        assert np.array_equal(Y.rgb_to_i420(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420))


def test_clamps_are_reached():
    """The clamp content drives every RGB channel below 0 and above 255 before saturation, and the decoded frame still matches."""
    yuv = _yuv_clamps(36, 50)
    y, u, v = Y.split_planes(yuv)
    yy = np.maximum(y.astype(np.int64) - 16, 0) * Y.Y2RGB
    d = np.repeat(np.repeat(u.astype(np.int64) - 128, 2, 0), 2, 1)
    e = np.repeat(np.repeat(v.astype(np.int64) - 128, 2, 0), 2, 1)
    for raw in ((yy + Y.HALF + Y.V2R * e) >> 20, (yy + Y.HALF + Y.V2G * e + Y.U2G * d) >> 20, (yy + Y.HALF + Y.U2B * d) >> 20):
        assert raw.min() < 0 and raw.max() > 255
    assert (y < 16).any() and (y > 235).any() and (u == 0).any() and (u == 255).any() and (v == 0).any() and (v == 255).any()


def test_batched():
    rng = np.random.default_rng(5)
    yuv = rng.integers(0, 256, (3, 2, 9, 10), dtype=np.uint8)
    rgb = Y.i420_to_rgb(yuv)
    assert rgb.shape == (3, 2, 6, 10, 3)
    for i in range(3):
        for j in range(2):
            assert np.array_equal(rgb[i, j], cv2.cvtColor(yuv[i, j], cv2.COLOR_YUV2RGB_I420))
            assert np.array_equal(Y.rgb_to_i420(rgb)[i, j], cv2.cvtColor(rgb[i, j], cv2.COLOR_RGB2YUV_I420))


# ------------------------------------------------------------------------------------------ Y4M headers and frames
def test_header_round_trip():
    src = T.parse_header(b"YUV4MPEG2 W1920 H1080 F30000:1001 Ip A1:1 C420mpeg2 XYSCSS=420MPEG2\n")
    assert (src["W"], src["H"], src["F"], src["I"], src["A"], src["C"], src["X"]) == (1920, 1080, "30000:1001", "p", "1:1", "420mpeg2",
                                                                                     ["YSCSS=420MPEG2"])
    out = T.parse_header(T.format_header(768, 432, src))
    assert (out["W"], out["H"], out["F"], out["I"], out["A"], out["C"]) == (768, 432, "30000:1001", "p", "1:1", "420mpeg2")
    # no C / A / I tag: progressive 4:2:0 by default, written as C420jpeg
    bare = T.parse_header(b"YUV4MPEG2 W4 H2 F25:1")
    assert T.format_header(4, 2, bare) == b"YUV4MPEG2 W4 H2 F25:1 Ip C420jpeg\n"
    for c in T.CHROMA_420:
        assert T.parse_header(f"YUV4MPEG2 W2 H2 C{c}".encode())["C"] == c


@pytest.mark.parametrize("line", [
    b"YUV4MPEG2 W64 H48 C444", b"YUV4MPEG2 W64 H48 Cmono", b"YUV4MPEG2 W64 H48 C420p10", b"YUV4MPEG2 W64 H48 C422",
    b"YUV4MPEG2 W64 H48 It", b"YUV4MPEG2 W64 H48 Ib", b"YUV4MPEG2 W64 H48 Im", b"YUV4MPEG2 H48", b"YUV4MPEG2 W64",
    b"YUV4MPEG2 W64 Hx", b"YUV4MPEG2 W0 H48", b"YUV4MPEG2 W63 H48", b"YUV4MPEG2 W64 H47", b"YUV4MPEG W64 H48",
    b"YUV4MPEG2  W64 H48",
], ids=lambda b: b.decode())
def test_header_refusals(line):
    with pytest.raises(T.Y4MError):
        T.parse_header(line)


def test_frames_read_in_chunks():
    rng = np.random.default_rng(7)
    frames = [rng.integers(0, 256, (6, 4), dtype=np.uint8) for _ in range(5)]
    # frame 1 carries a frame parameter, which is allowed and ignored
    r = T.Y4MReader(io.BytesIO(b"YUV4MPEG2 W4 H4 F25:1 C420jpeg\n" + b"".join(
        (b"FRAME Ixyz\n" if t == 1 else b"FRAME\n") + f.tobytes() for t, f in enumerate(frames))))
    buf = torch.zeros(2, 6, 4, dtype=torch.uint8)
    got = []
    while True:
        n = r.read_into(buf)
        if not n:
            break
        got += [buf[t].numpy().copy() for t in range(n)]
    assert len(got) == 5 and all(np.array_equal(a, b) for a, b in zip(got, frames))
    # the writer's frames read back
    out = io.BytesIO()
    out.write(T.format_header(4, 4, r.header))
    T.write_frames([out], [torch.from_numpy(np.stack(frames))], 5)
    out.seek(0)
    r2 = T.Y4MReader(out)
    buf = torch.zeros(8, 6, 4, dtype=torch.uint8)
    assert r2.read_into(buf) == 5 and np.array_equal(buf[:5].numpy(), np.stack(frames))


@pytest.mark.parametrize("case", ["bad-marker", "no-newline-marker", "truncated", "truncated-marker"])
def test_frame_refusals(case):
    f = np.zeros((6, 4), np.uint8)
    head = b"YUV4MPEG2 W4 H4\n"
    data = {
        "bad-marker": head + b"FRAME\n" + f.tobytes() + b"FRAMX\n" + f.tobytes(),
        "no-newline-marker": head + b"FRAME\n" + f.tobytes() + b"FRAME",
        "truncated": head + b"FRAME\n" + f.tobytes() + b"FRAME\n" + f.tobytes()[:-1],
        "truncated-marker": head + b"FRAME\n" + f.tobytes() + b"FRAMEFRAME\n",
    }[case]
    r = T.Y4MReader(io.BytesIO(data))
    with pytest.raises(T.Y4MError):
        r.read_into(torch.zeros(4, 6, 4, dtype=torch.uint8))


def test_reader_refusals():
    for data in (b"", b"YUV4MPEG2 W4 H4", b"YUV4MPEG2 W4 H4 C444\n"):
        with pytest.raises(T.Y4MError):
            T.Y4MReader(io.BytesIO(data))
