"""Video output at the source resolution (include/dvc.h: dvc_ab_to_source, dvc_colorize_videos_source_rgb8).  The resampling
kernel must be the float32 oracle bit for bit; every output byte of the video call must be the chain of stand-alone entry
points: the window's ab (centerpad_rgb8 -> rgb8_to_lab -> resize_half -> colorize_frames_clips_exemplars chained over the
frames -> upsample2_scaled(1.25)) -> ab_to_source -> rgb8_to_lab of the source footprint, plane 0 -> l_to_guide8 -> fgs_filter
-> lab_to_rgb8; and with sources already at the window size, the bytes of the window-size calls."""
import ctypes
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
import source_oracle as PP
from oracle.weights import make_lab
from test_source_footprint import GEOMETRIES

pytestmark = pytest.mark.gpu
T = 1e-10


def _frames(seed, F, Hs, Ws):
    """Seeded uint8 frames [F,Hs,Ws,3]: blocky content plus noise (edges and flats for the resize and the WLS filter)."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1, 3)) * 255).astype(np.int32)
    img = np.kron(coarse, np.ones((1, 8, 8, 1), np.int32))[:, :Hs, :Ws]
    img = np.clip(img + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
    return torch.from_numpy(img)


def _src(K):
    return [s for s, k in enumerate(K) for _ in range(k)]


def _geometry(frames, size, geometry=None):
    from dvc.prepost import centerpad_geometry

    Hs, Ws = frames.shape[1:3]
    return (Hs, Ws, *(geometry if geometry is not None else centerpad_geometry(Hs, Ws, size)))


def _centerpad_raw(ctx, rgb, geometry, size):
    Hr, Wr, oy, ox = geometry
    out = torch.empty(size[0], size[1], 3, device="cuda", dtype=torch.uint8)
    rc = ctx.lib.dvc_resize_antialias_crop_rgb8(ctx.h, ctypes.c_void_p(rgb.data_ptr()), rgb.shape[0], rgb.shape[1], Hr, Wr, oy, ox,
                                                ctypes.c_void_p(out.data_ptr()), size[0], size[1], ctypes.c_void_p(0))
    ctx._check(rc, "dvc_resize_antialias_crop_rgb8")
    return out


def _chain(ctx, clips, K, size, wls=(500.0, 4.0), first_last=None, geometries=None):
    """Per clip [K[s],F,h_s,w_s,3] uint8 through the stand-alone entry points, and the rows' last state."""
    import dvc

    geometries = geometries or [None] * len(clips)
    L = []
    for frames, g in zip(clips, geometries):
        crops = torch.stack([ctx.centerpad_rgb8(f.cuda(), size) if g is None else _centerpad_raw(ctx, f.cuda(), g, size) for f in frames])
        L.append(ctx.resize_half(ctx.rgb8_to_lab(crops))[:, 0:1].contiguous())
    L = torch.stack(L)  # [S,F,1,h,w]
    src, F_ = _src(K), L.shape[1]
    last = first_last.cuda() if first_last is not None else torch.zeros(len(src), 3, *L.shape[3:], device="cuda")
    abs_ = []
    for t in range(F_):
        ab = ctx.colorize_frames_clips_exemplars(L[:, t].contiguous(), K, last, T)
        abs_.append(ab)
        last = torch.cat((L[src, t], ab), 1)
    abs_ = torch.stack(abs_, 1)  # [R,F,2,h,w]
    outs = [[] for _ in clips]
    for r, s in enumerate(src):
        geom = _geometry(clips[s], size, geometries[s])
        y0, x0, h, w = dvc.source_footprint(*geom, *size)
        Ls = ctx.rgb8_to_lab(clips[s][:, y0:y0 + h, x0:x0 + w].contiguous().cuda())[:, 0:1].contiguous()  # [F,1,h,w]
        ab_src = ctx.ab_to_source(ctx.upsample2_scaled(abs_[r], 1.25), geom, size)
        if wls is not None:
            for t in range(F_):
                ab_src[t] = ctx.fgs_filter(ctx.l_to_guide8(Ls[t, 0]), ab_src[t], wls[0], wls[1])
        outs[s].append(ctx.lab_to_rgb8(Ls, ab_src))
    return [torch.stack(o).cpu() for o in outs], last.cpu()


def _source_raw(ctx, clips, K, geoms, size, outs, wls=1, first_last=None, last=None, lam=500.0, sigma=4.0, S=None, counts="K",
                frames_ptrs=None, out_ptrs="outs"):
    """dvc_colorize_videos_source_rgb8 with explicit geometries; returns the status."""
    S = len(clips) if S is None else S
    n = max(S, 1)
    vp = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    ptrs = (ctypes.c_void_p * n)(*(frames_ptrs if frames_ptrs is not None else [clips[s % len(clips)].data_ptr() for s in range(n)]))
    g = (ctypes.c_int * (6 * n))(*[v for s in range(n) for v in geoms[s % len(geoms)]])
    ck = None if counts is None else (ctypes.c_int * n)(*[K[s % len(K)] for s in range(n)])
    optr = None if out_ptrs is None else (ctypes.c_void_p * n)(
        *([outs[s % len(outs)].data_ptr() for s in range(n)] if out_ptrs == "outs" else out_ptrs))
    F_ = clips[0].shape[0]
    return ctx.lib.dvc_colorize_videos_source_rgb8(ctx.h, S, ck, ptrs, F_, g, size[0], size[1], T, vp(first_last), wls, lam, sigma,
                                                   optr, vp(last), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


# ------------------------------------------------------------------------------------------ the resampling kernel
@pytest.mark.parametrize("geometry,size", GEOMETRIES)
def test_ab_to_source_is_the_oracle_bit_for_bit(ctx, geometry, size):
    P = 3 if size[0] > 100 else 5
    ab = np.random.default_rng(sum(geometry)).standard_normal((P, *size)).astype(np.float32) * np.float32(40)
    got = ctx.ab_to_source(torch.from_numpy(ab).cuda(), geometry, size).cpu().numpy()
    want = PP.ab_to_source(ab, geometry, size)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------------------------------ identity at the window size
@pytest.mark.parametrize("wls", [True, False])
@pytest.mark.parametrize("K", [1, 3])
def test_window_size_sources_give_the_window_calls_bytes(ctx, wls, K):
    size, F_ = (64, 96), 4
    if K == 1:
        ctx.set_exemplar(make_lab(300, 1, 32, 48))
    else:
        ctx.set_exemplars(make_lab(300 + K, K, 32, 48))
    frames = _frames(301 + K, F_, *size).pin_memory()
    w = (500.0, 4.0) if wls else None
    ref = ctx.colorize_video_rgb8(frames, size, T, wls=w)
    (got,) = ctx.colorize_videos_source_rgb8([frames], [K], size, T, wls=w)
    assert got.shape == (K, F_, 64, 96, 3) and not got.is_cuda
    assert torch.equal(got, ref)


@pytest.mark.parametrize("wls", [True, False])
def test_window_size_sources_two_clips(ctx, wls):
    size, F_, K = (64, 96), 3, [1, 2]
    ctx.set_exemplars(make_lab(310, 3, 32, 48))
    clips = [_frames(311, F_, *size).cuda(), _frames(312, F_, *size).cuda()]
    w = (500.0, 4.0) if wls else None
    ref = ctx.colorize_videos_exemplars_rgb8(clips, K, size, T, wls=w)
    got = ctx.colorize_videos_source_rgb8(clips, K, size, T, wls=w)
    assert got[0].is_cuda and torch.equal(got[0], ref[:1]) and torch.equal(got[1], ref[1:])


# ------------------------------------------------------------------------------------------ the chain of stand-alone calls
# (source sizes per clip, K, size, frames, on the device)
CASES = [
    ([(1080, 1920)], [1], (432, 768), 2, False),
    ([(720, 1280)], [3], (432, 768), 2, True),
    ([(480, 640)], [1], (432, 768), 2, False),   # CenterPad crops: the centre band
    ([(50, 60)], [1], (64, 96), 4, False),       # a source smaller than the window
    ([(90, 150), (60, 60)], [1, 2], (64, 96), 4, True),
]


@pytest.mark.parametrize("shapes,K,size,F_,on_device", CASES)
def test_video_source_matches_chain(ctx, shapes, K, size, F_, on_device):
    import dvc

    R = sum(K)
    ctx.set_exemplars(make_lab(320 + R, R, size[0] // 2, size[1] // 2))
    clips = [_frames(321 + s + shapes[s][0], F_, *shapes[s]) for s in range(len(shapes))]
    ref, _ = _chain(ctx, clips, K, size)
    got = ctx.colorize_videos_source_rgb8([f.cuda() if on_device else f.pin_memory() for f in clips], K, size, T)
    for s, (o, f) in enumerate(zip(got, clips)):
        _, _, h, w = dvc.source_footprint(*_geometry(f, size), *size)
        assert o.is_cuda == on_device and o.shape == (K[s], F_, h, w, 3)
        assert torch.equal(o.cpu(), ref[s]), s


@pytest.mark.parametrize("wls", [True, False])
def test_video_source_zero_padded_window_and_first_last(ctx, wls):
    """A 40x64 source whose 64x96 window zero-pads the resized image beside a cropped clip, counts (1, 2), first_last_lab."""
    size, K, F_ = (64, 96), [1, 2], 3
    geoms = [(50, 80, -7, -8), (64, 110, 0, 7)]
    clips = [_frames(330, F_, 40, 64), _frames(331, F_, 70, 120)]
    ctx.set_exemplars(make_lab(332, 3, 32, 48))
    first = make_lab(333, 3, 32, 48)
    w = (500.0, 4.0) if wls else None
    ref, _ = _chain(ctx, clips, K, size, wls=w, first_last=first, geometries=geoms)
    assert ref[0].shape == (1, F_, 40, 64, 3)  # the whole frame
    outs = [torch.empty(r.shape, dtype=torch.uint8).pin_memory() for r in ref]
    src = [f.pin_memory() for f in clips]
    full = [(*f.shape[1:3], *g) for f, g in zip(clips, geoms)]
    ctx._check(_source_raw(ctx, src, K, full, size, outs, wls=1 if wls else 0, first_last=first.pin_memory()),
               "dvc_colorize_videos_source_rgb8")
    for o, r in zip(outs, ref):
        assert torch.equal(o, r)


@pytest.mark.parametrize("on_device", [False, True])
def test_video_source_chunks_continue_exactly(ctx, on_device):
    F_, a, size, K = 7, 3, (64, 96), [2, 1]
    ctx.set_exemplars(make_lab(340, 3, 32, 48))
    clips = [_frames(341, F_, 72, 120), _frames(342, F_, 100, 90)]
    clips = [f.cuda() if on_device else f.pin_memory() for f in clips]
    whole, last = ctx.colorize_videos_source_rgb8(clips, K, size, T, return_last=True)
    head, l1 = ctx.colorize_videos_source_rgb8([f[:a] for f in clips], K, size, T, return_last=True)
    tail, l2 = ctx.colorize_videos_source_rgb8([f[a:] for f in clips], K, size, T, first_last_lab=l1, return_last=True)
    for s in range(2):
        assert torch.equal(torch.cat((head[s], tail[s]), 1), whole[s]), s
    assert torch.equal(l2, last)
    ref, ref_last = _chain(ctx, [f.cpu() for f in clips], K, size)
    for s in range(2):
        assert torch.equal(whole[s].cpu(), ref[s]), s
    assert torch.equal(last.cpu(), ref_last)
    # the recurrence state is the window-size call's
    _, last_w = ctx.colorize_videos_exemplars_rgb8(clips, K, size, T, return_last=True)
    assert torch.equal(last_w, last)


# ------------------------------------------------------------------------------------------ memory
def test_device_memory_does_not_grow_with_F(ctx):
    K, size = [1, 2], (64, 96)
    ctx.set_exemplars(make_lab(350, 3, 32, 48))
    shapes = ((120, 200), (90, 90))
    ctx.colorize_videos_source_rgb8([_frames(351 + s, 8, *shapes[s]).pin_memory() for s in range(2)], K, size, T)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    out = ctx.colorize_videos_source_rgb8([_frames(353 + s, 40, *shapes[s]).pin_memory() for s in range(2)], K, size, T)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert out[0].shape[:2] == (1, 40) and out[1].shape[:2] == (2, 40) and not out[0].is_cuda
    assert free1 >= free0, (free0, free1)


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(ctx):
    import dvc

    size, K = (64, 96), [1, 2]
    clips = [_frames(360, 2, 48, 80).pin_memory(), _frames(361, 2, 64, 96).pin_memory()]
    geoms = [(48, 80, 57, 96, 0, 0), (64, 96, 64, 96, 0, 0)]
    outs = [torch.empty(1, 2, 48, 80, 3, dtype=torch.uint8).pin_memory(), torch.empty(2, 2, 64, 96, 3, dtype=torch.uint8).pin_memory()]
    ctx.set_exemplars(make_lab(362, 3, 32, 48))
    torch.cuda.synchronize()

    def refused(call, want):
        n = ctx.launch_count()
        assert call() == want
        assert ctx.launch_count() == n

    refused(lambda: _source_raw(ctx, clips, K, geoms, size, outs, counts=None), -1)                   # null K
    refused(lambda: _source_raw(ctx, clips, K, geoms, size, outs, out_ptrs=None), -1)                 # null out
    refused(lambda: _source_raw(ctx, clips, K, geoms, size, outs, out_ptrs=[outs[0].data_ptr(), 0]), -1)  # null out[1]
    refused(lambda: _source_raw(ctx, clips, K, geoms, size, outs, frames_ptrs=[clips[0].data_ptr(), 0]), -1)  # null frames[1]
    refused(lambda: _source_raw(ctx, clips, [1, 0], geoms, size, outs), -1)                           # a count below 1
    refused(lambda: _source_raw(ctx, clips, K, geoms, size, outs, S=0), -1)                           # S outside [1, 8]
    refused(lambda: _source_raw(ctx, clips, K, geoms, size, outs, lam=-1.0), -1)                      # bad WLS parameter
    refused(lambda: _source_raw(ctx, clips, [2, 2], geoms, size, outs), -2)                           # 4 rows, 3 cached slots
    refused(lambda: _source_raw(ctx, clips, K, [geoms[0], (64, 96, 70, 96, 7, 0)], size, outs), -2)   # window leaves the image
    refused(lambda: _source_raw(ctx, clips, K, [(48, 80, 86, 144, 3, 0), (64, 96, 80, 128, 0, 0)], (80, 128), outs), -2)  # size
    with pytest.raises(dvc.DvcError):
        ctx.colorize_videos_source_rgb8(clips, K, size, T, out=[outs[1], outs[0]])  # outputs not at the footprints
    with pytest.raises(dvc.DvcError):
        ctx.ab_to_source(torch.zeros(2, 64, 96, device="cuda"), (2, 1, 1536, 768, 552, 0), size)  # no source pixel in the window
    # the context still works after the refusals (CenterPad crops the 48x80 clip to its centre 72 columns)
    got = ctx.colorize_videos_source_rgb8(clips, K, size, T)
    assert got[0].shape == (1, 2, 48, 72, 3) and got[1].shape == (2, 2, 64, 96, 3)


# ------------------------------------------------------------------------------------------ the folder tool
def _run_tool(tmp_path, dirs, refs, out_dir, size, extra=()):
    cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", *map(str, dirs), "--ref", *map(str, refs),
           "--out", str(out_dir), "--seeded-weights", "--chunk", "3", "--image-size", str(size[0]), str(size[1]), *extra]
    subprocess.run(cmd, check=True, cwd=str(tmp_path))


def test_colorize_folder_source_resolution(ctx, tmp_path):
    """Two clip folders: with --source-resolution every PNG has its clip's footprint size and the bytes of the source call
    chunk by chunk; a clip already at the window size writes the same bytes with and without the flag."""
    import dvc
    from dvc.prepost import centerpad_geometry
    from PIL import Image

    size, lens, shapes = (64, 96), (5, 5), ((90, 100), (64, 96))
    dirs, refs, clips = [], [], []
    for s in range(2):
        d = tmp_path / f"clip{s}"
        d.mkdir()
        fr = _frames(370 + s, lens[s], *shapes[s])
        for t in range(lens[s]):
            Image.fromarray(fr[t].numpy()).save(d / f"f{t + 1}.png")
        p = tmp_path / f"ref{s}.png"
        Image.fromarray(_frames(380 + s, 1, 70, 100)[0].numpy()).save(p)
        dirs.append(d), refs.append(p), clips.append(fr)
    _run_tool(tmp_path, dirs, refs, tmp_path / "src", size, ["--source-resolution"])
    _run_tool(tmp_path, dirs, refs, tmp_path / "win", size)
    # the source call chunk by chunk (chunk 3), from the same decoded images
    ref_lab = ctx.resize_half(ctx.rgb8_to_lab(torch.stack([ctx.centerpad_rgb8(
        torch.from_numpy(np.asarray(Image.open(r).convert("RGB")).copy()).cuda(), size) for r in refs])))
    ctx.set_exemplars(ref_lab)
    want, last = [[], []], None
    for a in range(0, 5, 3):
        out, last = ctx.colorize_videos_source_rgb8([c[a:a + 3] for c in clips], [1, 1], size, T, first_last_lab=last, return_last=True)
        for s in range(2):
            want[s] += list(out[s][0])
    for s in range(2):
        _, _, h, w = dvc.source_footprint(*shapes[s], *centerpad_geometry(*shapes[s], size), *size)
        for t in range(lens[s]):
            png = tmp_path / "src" / f"clip{s}" / f"f{t + 1}.png"
            assert Image.open(png).size == (w, h), (s, t)
            buf = io.BytesIO()
            Image.fromarray(want[s][t].numpy()).save(buf, format="PNG")
            assert png.read_bytes() == buf.getvalue(), (s, t)
    for t in range(lens[1]):  # already at the window size
        assert (tmp_path / "src" / "clip1" / f"f{t + 1}.png").read_bytes() == (tmp_path / "win" / "clip1" / f"f{t + 1}.png").read_bytes()
