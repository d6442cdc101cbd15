"""The device JPEG encoder (include/dvc.h: dvc_jpeg_max_bytes, dvc_encode_jpeg, dvc_colorize_videos_jpeg).  Every file must be
byte-equal to Pillow's (libjpeg-turbo) encoding of the same image, and the video call's files must be Pillow's encoding of the
frames the rgb8 calls return."""
import ctypes
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import jpeg_oracle as J
from conftest import ROOT
from oracle.weights import make_lab
from test_jpeg_oracle import LARGE_SIZES, QUALITIES, SMALL_SIZES

pytestmark = pytest.mark.gpu
T = 1e-10
CANARY = 0xA5


def pillow_jpeg(rgb, q):
    from PIL import Image

    buf = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(rgb)).save(buf, "JPEG", quality=q)
    return buf.getvalue()


def _frames(seed, F, Hs, Ws):
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1, 3)) * 255).astype(np.int32)
    img = np.kron(coarse, np.ones((1, 8, 8, 1), np.int32))[:, :Hs, :Ws]
    return torch.from_numpy(np.clip(img + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8))


# ------------------------------------------------------------------------------------------ the stand-alone encoder
@pytest.mark.parametrize("hw", SMALL_SIZES + LARGE_SIZES, ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_encode_jpeg_equals_pillow(ctx, hw):
    """B = 6 images (every kind of content) per call, at every quality; out / sizes alternate between device and page-locked host
    memory.  Each slot is followed by canary bytes, which must survive, and every size is within dvc_jpeg_max_bytes."""
    import dvc

    H, W = hw
    imgs = np.stack([J.content(k, H, W, seed=H + W) for k in J.KINDS])
    rgb = torch.from_numpy(imgs).cuda()
    bound = dvc.jpeg_max_bytes(H, W)
    assert bound == J.max_bytes(H, W)
    stride = bound + 64
    for i, q in enumerate(QUALITIES):
        on_device = i % 2 == 1
        out = torch.full((len(imgs), stride), CANARY, dtype=torch.uint8)
        sizes = torch.full((len(imgs),), -1, dtype=torch.int64)
        out, sizes = (out.cuda(), sizes.cuda()) if on_device else (out.pin_memory(), sizes.pin_memory())
        ctx.encode_jpeg_into(rgb, out[:, :bound], sizes, q)
        torch.cuda.synchronize()
        out, sizes = out.cpu().numpy(), sizes.cpu().numpy()
        for b, img in enumerate(imgs):
            n = int(sizes[b])
            assert 0 < n <= bound, (hw, q, b, n)
            assert out[b, :n].tobytes() == pillow_jpeg(img, q), (hw, q, J.KINDS[b], on_device)
            assert (out[b, n:] == CANARY).all(), (hw, q, b)  # nothing past the file, in its slot or after it


def test_encode_jpeg_list_api(ctx):
    img = torch.from_numpy(J.content("gradient", 37, 53)).cuda()
    (f,) = ctx.encode_jpeg(img, quality=90)
    assert f == pillow_jpeg(img.cpu().numpy(), 90)


def test_encode_jpeg_refusals_launch_nothing(ctx):
    rgb = torch.zeros(2, 16, 16, 3, dtype=torch.uint8, device="cuda")
    bound = J.max_bytes(16, 16)
    out = torch.empty(2, bound, dtype=torch.uint8, device="cuda")
    sizes = torch.empty(2, dtype=torch.int64, device="cuda")
    pageable_out = torch.empty(2, bound, dtype=torch.uint8)
    pageable_sizes = torch.empty(2, dtype=torch.int64)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = ctypes.c_void_p
    torch.cuda.synchronize()

    def call(q=75, o=out, st=bound, sz=sizes, B=2, H=16, W=16):
        return ctx.lib.dvc_encode_jpeg(ctx.h, vp(rgb.data_ptr()), B, H, W, q, vp(o.data_ptr() if o is not None else 0), st,
                                       vp(sz.data_ptr() if sz is not None else 0), s)

    for kw, want in (({"q": 0}, -1), ({"q": 101}, -1), ({"o": None}, -1), ({"sz": None}, -1), ({"B": 0}, -1),
                     ({"o": pageable_out}, -1), ({"sz": pageable_sizes}, -1), ({"st": bound - 1}, -2), ({"H": 0}, -2),
                     ({"W": 70000}, -2)):
        n = ctx.launch_count()
        assert call(**kw) == want, kw
        assert ctx.launch_count() == n, kw
    assert call() == 0
    assert ctx.lib.dvc_jpeg_max_bytes(0, 5) == -2 and ctx.lib.dvc_jpeg_max_bytes(16, 16) == bound


# ------------------------------------------------------------------------------------------ the video call
def _check_video(ctx, clips, K, size, q, source, on_device, wls=(500.0, 4.0), first_last=None):
    """The JPEG call's files against Pillow's encoding of the rgb8 call's frames; returns the JPEG call's last state."""
    import dvc

    side = (lambda f: f.cuda()) if on_device else (lambda f: f.pin_memory())
    clips = [side(f) for f in clips]
    fl = None if first_last is None else side(first_last)
    if source:
        ref, ref_last = ctx.colorize_videos_source_rgb8(clips, K, size, T, first_last_lab=fl, wls=wls, return_last=True)
        ref = [r.cpu() for r in ref]
    else:
        full, ref_last = ctx.colorize_videos_exemplars_rgb8(clips, K, size, T, first_last_lab=fl, wls=wls, return_last=True)
        full, row0, ref = full.cpu(), 0, []
        for k in K:
            ref.append(full[row0:row0 + k])
            row0 += k
    slots, sizes, last = ctx.colorize_videos_jpeg(clips, K, size, quality=q, source_resolution=source, temperature=T,
                                                  first_last_lab=fl, wls=wls, return_last=True)
    assert all(o.is_cuda == on_device for o in slots) and sizes.is_cuda == on_device
    files = dvc.jpeg_files(slots, sizes)
    r = 0
    for s in range(len(clips)):
        for k in range(K[s]):
            for t in range(clips[0].shape[0]):
                frame = ref[s][k, t].numpy()
                assert files[r][t] == pillow_jpeg(frame, q), (s, k, t)
                assert len(files[r][t]) <= dvc.jpeg_max_bytes(*frame.shape[:2])
            r += 1
    assert torch.equal(last.cpu(), ref_last.cpu())  # the recurrence is the rgb8 call's, bit for bit
    return last


@pytest.mark.parametrize("source", [False, True])
@pytest.mark.parametrize("on_device", [False, True])
def test_video_one_clip(ctx, source, on_device):
    size, F_ = (64, 96), 3
    ctx.set_exemplar(make_lab(400, 1, 32, 48))
    _check_video(ctx, [_frames(401, F_, 90, 150)], [1], size, 75, source, on_device)


@pytest.mark.parametrize("source", [False, True])
def test_video_clips_of_different_sizes_two_exemplars_each(ctx, source):
    """K = (2, 2), a cropped footprint (480x640 -> the centre band) beside a 1080p-shaped clip, q95."""
    size, F_, K = (64, 96), 2, [2, 2]
    ctx.set_exemplars(make_lab(410, 4, 32, 48))
    _check_video(ctx, [_frames(411, F_, 480, 640), _frames(412, F_, 108, 192)], K, size, 95, source, on_device=False)


@pytest.mark.parametrize("source", [False, True])
def test_video_zero_padded_window_no_wls_first_last(ctx, source):
    """A source smaller than the window (the window zero-pads it), WLS off, first_last_lab given."""
    size, F_, K = (64, 96), 3, [1, 2]
    ctx.set_exemplars(make_lab(420, 3, 32, 48))
    _check_video(ctx, [_frames(421, F_, 40, 50), _frames(422, F_, 70, 120)], K, size, 50, source, on_device=True, wls=None,
                 first_last=make_lab(423, 3, 32, 48))


@pytest.mark.parametrize("source", [False, True])
def test_video_chunks_continue_exactly(ctx, source):
    import dvc

    F_, a, size, K = 6, 4, (64, 96), [2, 1]
    ctx.set_exemplars(make_lab(430, 3, 32, 48))
    clips = [_frames(431, F_, 72, 120).pin_memory(), _frames(432, F_, 100, 90).pin_memory()]
    whole, ws, last = ctx.colorize_videos_jpeg(clips, K, size, source_resolution=source, return_last=True)
    head, hs, l1 = ctx.colorize_videos_jpeg([f[:a] for f in clips], K, size, source_resolution=source, return_last=True)
    tail, ts, l2 = ctx.colorize_videos_jpeg([f[a:] for f in clips], K, size, source_resolution=source, first_last_lab=l1,
                                            return_last=True)
    fw, fh, ft = dvc.jpeg_files(whole, ws), dvc.jpeg_files(head, hs), dvc.jpeg_files(tail, ts)
    assert [h + t for h, t in zip(fh, ft)] == fw
    assert torch.equal(l2, last)


def test_video_device_memory_does_not_grow_with_F(ctx):
    K, size = [1, 2], (64, 96)
    ctx.set_exemplars(make_lab(440, 3, 32, 48))
    shapes = ((120, 200), (90, 90))
    for source in (False, True):
        ctx.colorize_videos_jpeg([_frames(441 + s, 8, *shapes[s]).pin_memory() for s in range(2)], K, size, source_resolution=source)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    for source in (False, True):
        slots, sizes = ctx.colorize_videos_jpeg([_frames(443 + s, 40, *shapes[s]).pin_memory() for s in range(2)], K, size,
                                                source_resolution=source)
        assert slots[1].shape[:2] == (2, 40) and not slots[0].is_cuda
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert free1 >= free0, (free0, free1)


def test_video_refusals_launch_nothing(ctx):
    import dvc

    size, K, F_ = (64, 96), [1, 2], 2
    clips = [_frames(450, F_, 48, 80).pin_memory(), _frames(451, F_, 64, 96).pin_memory()]
    geoms = [(48, 80, 57, 96, 0, 0), (64, 96, 64, 96, 0, 0)]
    ctx.set_exemplars(make_lab(452, 3, 32, 48))
    stride = dvc.jpeg_max_bytes(*size)
    outs = [torch.empty(k, F_, stride, dtype=torch.uint8).pin_memory() for k in K]
    sizes = torch.empty(3, F_, dtype=torch.int64).pin_memory()
    pageable = [torch.empty(k, F_, stride, dtype=torch.uint8) for k in K]
    torch.cuda.synchronize()
    vp = ctypes.c_void_p

    def call(q=75, source=0, out="outs", st=stride, sz=sizes, Kc=K, gm=geoms):
        o = None if out is None else (vp * 2)(*[t.data_ptr() if t is not None else 0 for t in (outs if out == "outs" else out)])
        ptrs = (vp * 2)(*[f.data_ptr() for f in clips])
        g = (ctypes.c_int * 12)(*[v for gg in gm for v in gg])
        return ctx.lib.dvc_colorize_videos_jpeg(ctx.h, 2, (ctypes.c_int * 2)(*Kc), ptrs, F_, g, size[0], size[1], T, vp(0), 1, 500.0,
                                                4.0, source, q, o, st, vp(sz.data_ptr() if sz is not None else 0), vp(0),
                                                vp(torch.cuda.current_stream().cuda_stream))

    for kw, want in (({"q": 0}, -1), ({"q": 101}, -1), ({"out": None}, -1), ({"out": [outs[0], None]}, -1), ({"sz": None}, -1),
                     ({"out": pageable}, -1), ({"sz": torch.empty(3, F_, dtype=torch.int64)}, -1), ({"st": stride - 1}, -2),
                     ({"Kc": [2, 2]}, -2), ({"gm": [geoms[0], (64, 96, 70, 96, 7, 0)]}, -2)):
        for source in (0, 1):
            n = ctx.launch_count()
            assert call(source=source, **kw) == want, (kw, source)
            assert ctx.launch_count() == n, (kw, source)
    assert call() == 0 and call(source=1) == 0  # the context still works after the refusals


# ------------------------------------------------------------------------------------------ the folder tool
def test_colorize_folder_jpg_is_pillows_encoding_of_the_pngs(tmp_path):
    from PIL import Image

    size, lens, shapes = (64, 96), (4, 4), ((90, 100), (64, 96))
    dirs, refs = [], []
    for s in range(2):
        d = tmp_path / f"clip{s}"
        d.mkdir()
        fr = _frames(460 + s, lens[s], *shapes[s])
        for t in range(lens[s]):
            Image.fromarray(fr[t].numpy()).save(d / f"f{t + 1}.png")
        p = tmp_path / f"ref{s}.png"
        Image.fromarray(_frames(470 + s, 1, 70, 100)[0].numpy()).save(p)
        dirs.append(d), refs.append(p)
    for fmt in ("png", "jpg"):
        for extra in ([], ["--source-resolution"]):
            out = tmp_path / f"{fmt}{len(extra)}"
            cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", *map(str, dirs), "--ref", *map(str, refs),
                   "--out", str(out), "--seeded-weights", "--chunk", "3", "--image-size", str(size[0]), str(size[1]),
                   "--format", fmt, "--jpeg-quality", "85", *extra]
            subprocess.run(cmd, check=True, cwd=str(tmp_path))
    for n in (0, 1):
        for s in range(2):
            for t in range(lens[s]):
                png = np.asarray(Image.open(tmp_path / f"png{n}" / f"clip{s}" / f"f{t + 1}.png").convert("RGB"))
                jpg = (tmp_path / f"jpg{n}" / f"clip{s}" / f"f{t + 1}.jpg").read_bytes()
                assert jpg == pillow_jpeg(png, 85), (n, s, t)
