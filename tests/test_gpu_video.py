"""dvc_colorize_video_rgb8 (include/dvc.h): uint8 frames in, WLS-filtered sRGB frames out, in one pipelined call.  Every
output byte must be what the chain of the stand-alone entry points gives (tools/colorize_folder.py's data flow before it
streamed, restated below): centerpad_rgb8 -> rgb8_to_lab -> resize_half -> colorize_clip(_exemplars) -> upsample2_scaled
(1.25) -> l_to_guide8 -> fgs_filter -> lab_to_rgb8."""
import ctypes
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

T = 1e-10


def _frames(seed, F, Hs, Ws):
    """Seeded uint8 frames [F,Hs,Ws,3]: blocky content plus noise (edges and flats for the resize and the WLS filter)."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1, 3)) * 255).astype(np.int32)
    img = np.kron(coarse, np.ones((1, 8, 8, 1), np.int32))[:, :Hs, :Ws]
    img = np.clip(img + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
    return torch.from_numpy(img)


def _set_exemplars(ctx, K, h, w, seed=40):
    from dvc.synth import make_lab

    IB = make_lab(seed, K, h, w)
    if K == 1:
        ctx.set_exemplar(IB)
    else:
        ctx.set_exemplars(IB)


def _composition(ctx, frames, size, K, wls=(500.0, 4.0), first_last=None, geometry=None):
    """[K,F,Ho,Wo,3] uint8 and the clip's ab [K,F,2,Ho/2,Wo/2] through the stand-alone entry points."""
    if geometry is None:
        crops = torch.stack([ctx.centerpad_rgb8(f.cuda(), size) for f in frames])
    else:
        crops = torch.stack([_centerpad_raw(ctx, f.cuda(), geometry, size) for f in frames])
    lab_large = ctx.rgb8_to_lab(crops)
    L = ctx.resize_half(lab_large)[:, 0:1].contiguous()
    if K == 1:
        fl = first_last.cuda() if first_last is not None else None
        abs_ = ctx.colorize_clip(L, T, first_last_lab=fl)[None]
    else:
        abs_ = ctx.colorize_clip_exemplars(L, T, first_last_lab=first_last.cuda() if first_last is not None else None)
    outs = []
    for ab in abs_:
        ab_large = ctx.upsample2_scaled(ab, 1.25)
        if wls is not None:
            for t in range(len(frames)):
                ab_large[t] = ctx.fgs_filter(ctx.l_to_guide8(lab_large[t, 0]), ab_large[t], wls[0], wls[1])
        outs.append(ctx.lab_to_rgb8(lab_large[:, 0:1].contiguous(), ab_large))
    return torch.stack(outs).cpu(), abs_.cpu(), L.cpu()


def _centerpad_raw(ctx, rgb, geometry, size):
    Hr, Wr, oy, ox = geometry
    out = torch.empty(size[0], size[1], 3, device="cuda", dtype=torch.uint8)
    rc = ctx.lib.dvc_resize_antialias_crop_rgb8(ctx.h, ctypes.c_void_p(rgb.data_ptr()), rgb.shape[0], rgb.shape[1], Hr, Wr, oy, ox,
                                                ctypes.c_void_p(out.data_ptr()), size[0], size[1], ctypes.c_void_p(0))
    ctx._check(rc, "dvc_resize_antialias_crop_rgb8")
    return out


def _video_raw(ctx, frames, geometry, size, out, wls=1, last=None):
    """dvc_colorize_video_rgb8 with an explicit geometry (the Python method computes CenterPad's); returns the status."""
    F_, Hs, Ws = (frames.shape[:3] if frames is not None else (1, 8, 8))
    Hr, Wr, oy, ox = geometry
    vp = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    return ctx.lib.dvc_colorize_video_rgb8(ctx.h, vp(frames), F_, Hs, Ws, Hr, Wr, oy, ox, size[0], size[1], T, None, wls, 500.0, 4.0,
                                           vp(out), vp(last), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


# ------------------------------------------------------------------------------------------ byte equality
# (Hs, Ws, Ho, Wo, K, wls, with first_last, frames on the device)
CASES = [
    (720, 1280, 432, 768, 1, True, False, False),   # test.py's default size from a 720p source
    (720, 1280, 432, 768, 3, True, False, True),
    (50, 60, 64, 96, 1, True, True, False),         # a source smaller than the target
    (90, 150, 80, 128, 3, False, True, True),       # H = 40: H % 16 == 8 (the replicate-pad branch), no WLS
    (100, 90, 64, 96, 2, False, False, False),
]


@pytest.mark.parametrize("Hs,Ws,Ho,Wo,K,wls,use_first,on_device", CASES)
def test_video_matches_composition(ctx, Hs, Ws, Ho, Wo, K, wls, use_first, on_device):
    from dvc.synth import make_lab

    F_ = 3 if Ho > 200 else 5
    _set_exemplars(ctx, K, Ho // 2, Wo // 2)
    frames = _frames(Hs + Ws + K, F_, Hs, Ws)
    first = make_lab(77, K, Ho // 2, Wo // 2) if use_first else None
    w = (500.0, 4.0) if wls else None
    ref, _, _ = _composition(ctx, frames, (Ho, Wo), K, wls=w, first_last=first)
    src = frames.cuda() if on_device else frames.pin_memory()
    fl = None if first is None else (first.cuda() if on_device else first.pin_memory())
    out = ctx.colorize_video_rgb8(src, (Ho, Wo), T, first_last_lab=fl, wls=w)
    assert out.is_cuda == on_device and out.shape == (K, F_, Ho, Wo, 3) and out.dtype == torch.uint8
    assert torch.equal(out.cpu(), ref)


def test_video_zero_padded_window(ctx):
    """A geometry whose output window is larger than the resized image (zero border on every side)."""
    size, geometry = (64, 96), (50, 80, -7, -8)
    _set_exemplars(ctx, 1, 32, 48)
    frames = _frames(5, 4, 40, 64).pin_memory()
    ref, _, _ = _composition(ctx, frames, size, 1, geometry=geometry)
    out = torch.empty(1, 4, 64, 96, 3, dtype=torch.uint8).pin_memory()
    ctx._check(_video_raw(ctx, frames, geometry, size, out), "dvc_colorize_video_rgb8")
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------ chunking
@pytest.mark.parametrize("K,on_device", [(1, False), (2, True)])
def test_chunks_continue_exactly(ctx, K, on_device):
    F_, a, size = 7, 3, (64, 96)
    _set_exemplars(ctx, K, 32, 48)
    frames = _frames(11, F_, 72, 120)
    frames = frames.cuda() if on_device else frames.pin_memory()
    whole, last = ctx.colorize_video_rgb8(frames, size, T, return_last=True)
    head, l1 = ctx.colorize_video_rgb8(frames[:a], size, T, return_last=True)
    tail, l2 = ctx.colorize_video_rgb8(frames[a:], size, T, first_last_lab=l1, return_last=True)
    assert torch.equal(torch.cat((head, tail), 1), whole)
    assert torch.equal(l2, last)
    # last_lab_out = cat(L/2, ab) of the last frame, as the clip computes them
    ref, ab, L = _composition(ctx, frames.cpu(), size, K)
    assert torch.equal(whole.cpu(), ref)
    want = torch.cat((L[-1:].expand(K, 1, 32, 48), ab[:, -1]), 1)
    assert torch.equal(last.cpu(), want)


# ------------------------------------------------------------------------------------------ memory
def test_device_memory_does_not_grow_with_F(ctx):
    _set_exemplars(ctx, 1, 32, 48)
    warm = _frames(3, 8, 48, 80).pin_memory()
    ctx.colorize_video_rgb8(warm, (64, 96), T)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    long_clip = _frames(4, 200, 48, 80).pin_memory()
    out = ctx.colorize_video_rgb8(long_clip, (64, 96), T)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert out.shape == (1, 200, 64, 96, 3) and not out.is_cuda
    assert free1 >= free0, (free0, free1)


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(ctx, sds):
    import dvc

    frames = _frames(6, 2, 48, 80).pin_memory()
    out = torch.empty(1, 2, 64, 96, 3, dtype=torch.uint8).pin_memory()
    geometry = (57, 96, 0, 0)

    def refused(call):
        n = ctx.launch_count()
        rc = call()
        assert rc != 0
        assert ctx.launch_count() == n

    ctx.set_weights(dvc.NET_VGG, sds["vgg"])  # drops the cached exemplar
    refused(lambda: _video_raw(ctx, frames, geometry, (64, 96), out))                  # no exemplar
    _set_exemplars(ctx, 1, 32, 48)
    refused(lambda: _video_raw(ctx, frames, (86, 144, 3, 0), (80, 128), out))          # exemplar size differs
    refused(lambda: _video_raw(ctx, frames, (48, 80, 0, 0), (48, 80), out))            # illegal image size (H = 24)
    refused(lambda: _video_raw(ctx, frames, (64, 100, 0, 0), (64, 100), out))          # W = 50 not a multiple of 16
    refused(lambda: _video_raw(ctx, frames, (64, 96, 0, 0), (65, 96), out))            # odd output height
    refused(lambda: _video_raw(ctx, frames, (70, 96, 7, 0), (64, 96), out))            # window leaves the resized image
    refused(lambda: _video_raw(ctx, frames, (50, 80, 1, 0), (64, 96), out))            # pad window not around it
    refused(lambda: _video_raw(ctx, None, geometry, (64, 96), out))                    # null frames
    refused(lambda: _video_raw(ctx, frames, geometry, (64, 96), None))                 # null out
    with pytest.raises(dvc.DvcError):
        ctx.colorize_video_rgb8(frames, (64, 96), T, first_last_lab=torch.zeros(2, 3, 32, 48))
    # the context still works after the refusals
    assert ctx.colorize_video_rgb8(frames, (64, 96), T).shape == (1, 2, 64, 96, 3)


# ------------------------------------------------------------------------------------------ the folder tool
@pytest.mark.parametrize("n_refs", [1, 2])
def test_colorize_folder_streams_the_same_bytes(ctx, tmp_path, n_refs):
    from PIL import Image

    size = (64, 96)
    clip, out_dir = tmp_path / "clip", tmp_path / "out"
    clip.mkdir()
    frames = _frames(21, 7, 60, 110)
    for t in range(7):
        Image.fromarray(frames[t].numpy()).save(clip / f"f{t + 1}.png")
    refs = []
    for k in range(n_refs):
        p = tmp_path / f"ref{k}.png"
        Image.fromarray(_frames(30 + k, 1, 70, 100)[0].numpy()).save(p)
        refs.append(p)
    cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", str(clip), "--ref", *map(str, refs),
           "--out", str(out_dir), "--seeded-weights", "--chunk", "3", "--image-size", str(size[0]), str(size[1])]
    subprocess.run(cmd, check=True, cwd=str(tmp_path))
    # the composition, from the same decoded images
    ref_lab = ctx.resize_half(ctx.rgb8_to_lab(torch.stack([ctx.centerpad_rgb8(
        torch.from_numpy(np.asarray(Image.open(r).convert("RGB")).copy()).cuda(), size) for r in refs])))
    if n_refs == 1:
        ctx.set_exemplar(ref_lab)
    else:
        ctx.set_exemplars(ref_lab)
    ref, _, _ = _composition(ctx, frames, size, n_refs)
    for k in range(n_refs):
        d = out_dir if n_refs == 1 else out_dir / f"ref{k}"
        for t in range(7):
            buf = io.BytesIO()
            Image.fromarray(ref[k, t].numpy()).save(buf, format="PNG")
            assert (d / f"f{t + 1}.png").read_bytes() == buf.getvalue(), (k, t)
