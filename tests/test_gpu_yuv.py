"""Planar YUV 4:2:0 (I420) on the device (include/dvc.h: dvc_i420_to_rgb8, dvc_rgb8_to_i420, dvc_colorize_videos_i420).

The conversions are cv2's BT.601 ones, restated in tests/yuv_oracle.py (pinned to cv2 by tests/test_yuv_oracle.py).  An I420
clip has one correct output: what the sRGB calls return for its frames converted by the oracle, and, with I420 output, the
oracle's conversion of those frames back.  Every check compares by torch.equal: bytes, last_lab_out and launch counts."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import yuv_oracle as Y
from conftest import ROOT
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu
T = 1e-10
WLS = (500.0, 4.0)
SIZE = (64, 96)  # networks at 32 x 48
CANARY = 0xA5


def _yuv(seed, F, Hs, Ws):
    """I420 frames [F,3Hs/2,Ws]: blocky luma with noise that reaches below 16 and above 235, chroma over the whole byte range."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1)) * 255).astype(np.int32)
    y = np.clip(np.kron(coarse, np.ones((1, 8, 8), np.int32))[:, :Hs, :Ws] + rng.integers(-30, 31, (F, Hs, Ws)), 0, 255)
    u = rng.integers(0, 256, (F, Hs // 2, Ws // 2))
    v = np.clip(255 - u + rng.integers(-60, 61, u.shape), 0, 255)
    return torch.from_numpy(Y.join_planes(y.astype(np.uint8), u.astype(np.uint8), v.astype(np.uint8)))


def _to_rgb(yuv):
    return torch.from_numpy(Y.i420_to_rgb(yuv.cpu().numpy()))


def _to_i420(rgb):
    return torch.from_numpy(Y.rgb_to_i420(rgb.cpu().numpy()))


def _side(on_device):
    return (lambda t: t.cuda()) if on_device else (lambda t: t.pin_memory())


def _counted(ctx, fn):
    torch.cuda.synchronize()
    ctx.launch_count(reset=True)
    res = fn()
    torch.cuda.synchronize()
    return res, ctx.launch_count()


def _footprints(clips, size):
    import dvc
    from dvc.prepost import centerpad_geometry

    fps = []
    for c in clips:
        Hs, Ws = c.shape[1] * 2 // 3, c.shape[2]
        fps.append(dvc.source_footprint(Hs, Ws, *centerpad_geometry(Hs, Ws, size), *size)[2:])
    return fps


def _check(ctx, clips, K, size=SIZE, source=False, on_device=False, wls=WLS, first_last=None, fmt="rgb"):
    """The I420 call against the sRGB call on the oracle-converted frames; returns the I420 call's output and last state."""
    side = _side(on_device)
    yuv = [side(c) for c in clips]
    rgb = [side(_to_rgb(c)) for c in clips]
    fl = None if first_last is None else side(first_last)
    kw = dict(first_last_lab=fl, wls=wls, return_last=True)
    ctx.colorize_videos_i420(yuv, K, size, T, first_last_lab=fl, wls=wls, source_resolution=source, out_format=fmt)  # one-off launches
    if source:
        (ref, ref_last), n_ref = _counted(ctx, lambda: ctx.colorize_videos_source_rgb8(rgb, K, size, T, **kw))
        sizes = len(set(_footprints(clips, size)))
    else:
        (ref, ref_last), n_ref = _counted(ctx, lambda: ctx.colorize_videos_exemplars_rgb8(rgb, K, size, T, **kw))
        ref, sizes = list(torch.split(ref, K)), 1
    (got, last), n_got = _counted(ctx, lambda: ctx.colorize_videos_i420(yuv, K, size, T, source_resolution=source, out_format=fmt, **kw))
    assert len(got) == len(ref) and all(a.is_cuda == on_device for a in got)
    for a, b in zip(got, ref):
        assert torch.equal(a.cpu(), b.cpu() if fmt == "rgb" else _to_i420(b))
    assert torch.equal(last.cpu(), ref_last.cpu())
    S, F_ = len(clips), clips[0].shape[0]  # per frame step: one conversion per clip, and one per output size with I420 output
    assert n_got == n_ref + F_ * (S + (sizes if fmt == "i420" else 0)), (n_got, n_ref, S, sizes)
    return got, last


# ------------------------------------------------------------------------------------------ stand-alone kernels
KSIZES = [(2, 2), (2, 34), (36, 2), (6, 34), (36, 50), (432, 768), (1080, 1920)]


@pytest.mark.parametrize("H,W", KSIZES, ids=lambda v: str(v))
def test_kernels_equal_oracle(ctx, H, W):
    B, pad = 3, 64
    rng = np.random.default_rng(H * 7 + W)
    yuv = torch.from_numpy(rng.integers(0, 256, (B, 3 * H // 2, W), dtype=np.uint8))
    yuv[0, :H, : W // 2] = torch.tensor([0, 15, 16, 235, 236, 255], dtype=torch.uint8).repeat(W)[: W // 2]  # luma clamps
    rgb = torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8))
    rgb[1, ::2, ::2] = torch.tensor([[0, 0, 255], [255, 255, 0]], dtype=torch.uint8).repeat(H * W, 1)[: (H // 2) * (W // 2)].view(
        H // 2, W // 2, 3)
    vp, stream = ctypes.c_void_p, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    n_rgb, n_yuv = B * H * W * 3, B * H * W * 3 // 2
    out_rgb = torch.full((n_rgb + pad,), CANARY, dtype=torch.uint8, device="cuda")
    out_yuv = torch.full((n_yuv + pad,), CANARY, dtype=torch.uint8, device="cuda")
    dyuv, drgb = yuv.cuda(), rgb.cuda()
    n = ctx.launch_count()
    assert ctx.lib.dvc_i420_to_rgb8(ctx.h, vp(dyuv.data_ptr()), B, H, W, vp(out_rgb.data_ptr()), stream) == 0
    assert ctx.lib.dvc_rgb8_to_i420(ctx.h, vp(drgb.data_ptr()), B, H, W, vp(out_yuv.data_ptr()), stream) == 0
    assert ctx.launch_count() == n + 2
    torch.cuda.synchronize()
    assert torch.equal(out_rgb[:n_rgb].cpu().view(B, H, W, 3), torch.from_numpy(Y.i420_to_rgb(yuv.numpy())))
    assert torch.equal(out_yuv[:n_yuv].cpu().view(B, 3 * H // 2, W), torch.from_numpy(Y.rgb_to_i420(rgb.numpy())))
    assert (out_rgb[n_rgb:] == CANARY).all() and (out_yuv[n_yuv:] == CANARY).all()
    # the Python wrappers
    assert torch.equal(ctx.i420_to_rgb8(dyuv).cpu(), out_rgb[:n_rgb].cpu().view(B, H, W, 3))
    assert torch.equal(ctx.rgb8_to_i420(drgb).cpu(), out_yuv[:n_yuv].cpu().view(B, 3 * H // 2, W))


def test_kernel_refusals(ctx):
    vp, stream = ctypes.c_void_p, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.full((4096,), CANARY, dtype=torch.uint8, device="cuda")
    p = vp(buf.data_ptr())
    n = ctx.launch_count()
    for fn in (ctx.lib.dvc_i420_to_rgb8, ctx.lib.dvc_rgb8_to_i420):
        for B, H, W, want in ((1, 3, 4, -2), (1, 4, 5, -2), (1, 0, 4, -2), (0, 4, 4, -1)):
            assert fn(ctx.h, p, B, H, W, p, stream) == want, (B, H, W)
        assert fn(ctx.h, vp(0), 1, 4, 4, p, stream) == -1
    assert ctx.launch_count() == n
    torch.cuda.synchronize()
    assert (buf == CANARY).all()


# ------------------------------------------------------------------------------------------ I420 in, sRGB or I420 out
@pytest.mark.parametrize("fmt", ["rgb", "i420"])
@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
@pytest.mark.parametrize("K", [[1], [3], [1, 2, 1]], ids=lambda K: "K" + "-".join(map(str, K)))
def test_counts_and_outputs(ctx, K, source, fmt):
    R = sum(K)
    shapes = ((90, 150), (48, 80), (100, 90))
    if R == 1:
        ctx.set_exemplar(make_lab(600, 1, 32, 48))
    else:
        ctx.set_exemplars(make_lab(600, R, 32, 48))
    clips = [_yuv(601 + s, 3, *shapes[s]) for s in range(len(K))]
    _check(ctx, clips, K, source=source, on_device=R % 2 == 0, fmt=fmt)


GEOMETRIES = {
    "window-size": ((64, 96), SIZE),
    "crop-4to3-into-16to9": ((480, 640), (144, 256)),
    "zero-pad": ((40, 50), SIZE),
    "small-upscale": ((18, 24), SIZE),
}


@pytest.mark.parametrize("fmt", ["rgb", "i420"])
@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_geometries(ctx, geom, source, fmt):
    (Hs, Ws), size = GEOMETRIES[geom]
    ctx.set_exemplar(make_lab(610, 1, size[0] // 2, size[1] // 2))
    _check(ctx, [_yuv(611, 3, Hs, Ws)], [1], size=size, source=source, on_device=source, fmt=fmt)


@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
def test_wls_off_first_last(ctx, source):
    K = [2, 1]
    ctx.set_exemplars(make_lab(620, 3, 32, 48))
    clips = [_yuv(621, 3, 72, 120), _yuv(622, 3, 34, 48)]
    _check(ctx, clips, K, source=source, wls=None, first_last=make_lab(623, 3, 32, 48))
    _check(ctx, clips, K, source=source, on_device=True, first_last=make_lab(624, 3, 32, 48), fmt="i420")


@pytest.mark.parametrize("fmt", ["rgb", "i420"])
@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
def test_chunks_continue_exactly(ctx, source, fmt):
    F_, a, K = 6, 4, [2, 1]
    ctx.set_exemplars(make_lab(630, 3, 32, 48))
    clips = [_yuv(631, F_, 72, 120).pin_memory(), _yuv(632, F_, 100, 90).pin_memory()]
    kw = dict(source_resolution=source, out_format=fmt, return_last=True)
    whole, last = ctx.colorize_videos_i420(clips, K, SIZE, T, **kw)
    head, l1 = ctx.colorize_videos_i420([f[:a] for f in clips], K, SIZE, T, **kw)
    tail, l2 = ctx.colorize_videos_i420([f[a:] for f in clips], K, SIZE, T, first_last_lab=l1, **kw)
    for w, h, t in zip(whole, head, tail):
        assert torch.equal(torch.cat([h, t], 1), w)
    assert torch.equal(l2, last)


def test_device_memory_does_not_grow_with_F(ctx):
    K = [1, 2]
    ctx.set_exemplars(make_lab(640, 3, 32, 48))
    shapes = ((120, 200), (92, 92))

    def run(F_):
        clips = [_yuv(641 + s, F_, *shapes[s]).pin_memory() for s in range(2)]
        for source in (False, True):
            for fmt in ("rgb", "i420"):
                ctx.colorize_videos_i420(clips, K, SIZE, T, source_resolution=source, out_format=fmt)
        torch.cuda.synchronize()

    run(8)
    free0, _ = torch.cuda.mem_get_info()
    run(40)
    free1, _ = torch.cuda.mem_get_info()
    assert free1 >= free0, (free0, free1)


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(ctx):
    import dvc
    from dvc.prepost import centerpad_geometry

    K, F_ = [1, 2], 2
    clips = [_yuv(650, F_, 48, 80).pin_memory(), _yuv(651, F_, 64, 96).pin_memory()]
    geoms = [(48, 80, 57, 96, 0, 0), (64, 96, 64, 96, 0, 0)]
    # a source whose footprint has an odd side: CenterPad crops a 70 x 120 frame to the 105 middle columns
    odd = (70, 120, *centerpad_geometry(70, 120, SIZE))
    assert dvc.source_footprint(*odd, *SIZE)[2:] == (70, 105)
    ctx.set_exemplars(make_lab(652, 3, 32, 48))
    pad = 1 << 16
    outs = [torch.full((k * F_ * 200 * 400 * 3 + pad,), CANARY, dtype=torch.uint8).pin_memory() for k in K]
    big = torch.full((F_ * odd[0] * odd[1] * 3 // 2,), 0, dtype=torch.uint8).pin_memory()
    torch.cuda.synchronize()
    vp = ctypes.c_void_p

    def call(S=2, Kc=K, frames="clips", gm=geoms, source=0, oi=0, out="auto", fr_list=None):
        o = outs if out == "auto" else out
        optrs = None if o is None else (vp * 2)(*[t.data_ptr() if t is not None else 0 for t in o])
        fl = fr_list if fr_list is not None else [f.data_ptr() for f in clips]
        fr = None if frames is None else (vp * 2)(*fl)
        g = (ctypes.c_int * 12)(*[v for gg in gm for v in gg])
        return ctx.lib.dvc_colorize_videos_i420(ctx.h, S, (ctypes.c_int * 2)(*Kc), fr, F_, g, SIZE[0], SIZE[1], T, vp(0), 1, 500.0,
                                                4.0, source, oi, optrs, vp(0), vp(torch.cuda.current_stream().cuda_stream))

    cases = [
        ({"frames": None}, -1), ({"out": None}, -1), ({"out": [outs[0], None]}, -1), ({"gm": [geoms[0], (64, 96, 70, 96, 7, 0)]}, -2),
        ({"S": 0}, -1), ({"S": 9}, -1), ({"Kc": [2, 2]}, -2), ({"oi": 2}, -1), ({"oi": -1}, -1),
        ({"gm": [geoms[0], (63, 96, 64, 96, 0, 0)]}, -2), ({"gm": [geoms[0], (64, 95, 64, 96, 0, 0)]}, -2),
    ]
    for kw, want in cases:
        for source in (0, 1):
            for oi in (0, 1):
                kw2 = {"source": source, "oi": oi, **kw}
                n = ctx.launch_count()
                assert call(**kw2) == want, kw2
                assert ctx.launch_count() == n, kw2
    # I420 output of an odd footprint: refused at source resolution only
    n = ctx.launch_count()
    assert call(gm=[geoms[0], odd], source=1, oi=1, fr_list=[clips[0].data_ptr(), big.data_ptr()]) == -2
    assert ctx.launch_count() == n
    torch.cuda.synchronize()
    for t in outs:
        assert (t == CANARY).all()  # nothing was written
    # the context still works after the refusals, and writes nothing past its outputs
    assert call(oi=1) == 0
    win = SIZE[0] * SIZE[1] * 3 // 2
    for k, t in zip(K, outs):
        assert (t[k * F_ * win:] == CANARY).all()
    # the odd footprint is fine with sRGB output
    assert call(gm=[geoms[0], odd], source=1, oi=0, fr_list=[clips[0].data_ptr(), big.data_ptr()]) == 0


def test_python_shapes_and_types(ctx):
    import dvc

    ctx.set_exemplar(make_lab(660, 1, 32, 48))
    y = _yuv(661, 2, 50, 70).cuda()
    a = ctx.colorize_videos_i420([y], [1], SIZE, T)
    b = ctx.colorize_videos_i420([y], [1], SIZE, T, out_format="i420")
    assert a[0].shape == (1, 2, *SIZE, 3) and b[0].shape == (1, 2, SIZE[0] * 3 // 2, SIZE[1])
    for bad in (y.to(torch.int16), y[:, :-1], y[..., None], y.float()):
        with pytest.raises(dvc.DvcError):
            ctx.colorize_videos_i420([bad], [1], SIZE, T)
    with pytest.raises(dvc.DvcError):
        ctx.colorize_videos_i420([y], [1], SIZE, T, out_format="nv12")
    with pytest.raises(dvc.DvcError):
        ctx.colorize_videos_i420([y], [1], SIZE, T, out=[torch.empty(1, 2, *SIZE, 3, dtype=torch.uint8, device="cuda")],
                                 out_format="i420")


# ------------------------------------------------------------------------------------------ the Y4M tool
def _write_y4m(path, frames, tags="F25:1 Ip A1:1 C420mpeg2"):
    F_, R, W = frames.shape
    with open(path, "wb") as f:
        f.write(f"YUV4MPEG2 W{W} H{R * 2 // 3} {tags}\n".encode())
        for t in range(F_):
            f.write(b"FRAME\n" + frames[t].numpy().tobytes())


def _read_y4m(data):
    head, _, body = data.partition(b"\n")
    tags = {p[:1].decode(): p[1:].decode() for p in head.split(b" ")[1:]}
    W, H = int(tags["W"]), int(tags["H"])
    n = H * W * 3 // 2
    frames = []
    while body:
        marker, _, body = body.partition(b"\n")
        assert marker == b"FRAME"
        frames.append(np.frombuffer(body[:n], np.uint8).reshape(H * 3 // 2, W))
        body = body[n:]
    return tags, torch.from_numpy(np.stack(frames))


def _tool(args, **kw):
    cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_y4m.py"), "--seeded-weights", "--chunk", "3", "--image-size",
           str(SIZE[0]), str(SIZE[1]), *map(str, args)]
    return subprocess.run(cmd, check=True, stdout=subprocess.PIPE, **kw).stdout


def test_colorize_y4m(ctx, tmp_path):
    """The tool's streams equal one direct colorize_videos_i420 call over all frames, with the exemplars prepared as the folder
    tool prepares them; window and source output, two exemplars into a folder, and stdin / stdout piping."""
    from PIL import Image

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from colorize_folder import exemplars_lab

    F_, Hs, Ws = 8, 96, 128
    frames = _yuv(670, F_, Hs, Ws)
    src = tmp_path / "in.y4m"
    _write_y4m(src, frames)
    rng = np.random.default_rng(671)
    refs = []
    for i, shape in enumerate(((70, 100, 3), (90, 90, 3))):
        p = tmp_path / f"ref{i}.png"
        Image.fromarray(rng.integers(0, 256, shape, dtype=np.uint8)).save(p)
        refs.append(p)

    def direct(paths, source):
        lab = exemplars_lab(ctx, [str(p) for p in paths], SIZE)
        if len(paths) == 1:
            ctx.set_exemplar(lab)
        else:
            ctx.set_exemplars(lab)
        return ctx.colorize_videos_i420([frames.pin_memory()], [len(paths)], SIZE, T, source_resolution=source, out_format="i420")[0]

    for source in (False, True):
        extra = ["--source-resolution"] if source else []
        want = direct(refs[:1], source)
        out = tmp_path / f"out{int(source)}.y4m"
        _tool(["-i", src, "-o", out, "--ref", refs[0], *extra])
        tags, got = _read_y4m(out.read_bytes())
        h, w = want.shape[2] * 2 // 3, want.shape[3]
        assert (tags["W"], tags["H"], tags["F"], tags["A"], tags["C"], tags["I"]) == (str(w), str(h), "25:1", "1:1", "420mpeg2", "p")
        assert (h, w) == ((86, 128) if source else SIZE)  # the 3:4 source cropped to the 2:3 window's band
        assert torch.equal(got, want[0])
    # two exemplars in one pass, one stream each
    want = direct(refs, False)
    _tool(["-i", src, "-o", tmp_path / "two", "--ref", *refs])
    for k, p in enumerate(refs):
        _, got = _read_y4m((tmp_path / "two" / (p.stem + ".y4m")).read_bytes())
        assert torch.equal(got, want[k])
    # stdin -> stdout, input without a C tag (written back as C420jpeg)
    bare = tmp_path / "bare.y4m"
    _write_y4m(bare, frames, tags="F30000:1001")
    with open(bare, "rb") as f:
        data = _tool(["-i", "-", "-o", "-", "--ref", refs[0]], stdin=f)
    tags, got = _read_y4m(data)
    assert (tags["F"], tags["C"]) == ("30000:1001", "420jpeg") and "A" not in tags
    assert torch.equal(got, direct(refs[:1], False)[0])
