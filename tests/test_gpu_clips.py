"""Several clips in one pass, one exemplar each (include/dvc.h: dvc_colorize_frames_clips, dvc_colorize_clips,
dvc_colorize_videos_rgb8).  Clip s's results must be those of test.py:68-120 run on clip s alone against exemplar s:
S = 1 bit for bit against the single-exemplar calls; S > 1 against colorize_frames with only that exemplar cached (up to
the InstanceNorm summation order and device-derived fp16 scales a batch shares) and against the fp64 oracle; the clip and
video calls bit for bit against the chain of the calls they are built from."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from oracle import dvc_oracle as O
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu
T = 1e-10


@pytest.fixture(params=["fp32", "tf32x3", "tf32x3-nof16"])
def conv_math(request, ctx):
    """The exact CUDA-core engines, and the tensor-core convolutions with and without the fp16 planes of bounded layers."""
    import dvc

    if request.param == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32)
    else:
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        ctx.debug_flag("tc_f16", 0 if request.param.endswith("nof16") else 1)
    yield request.param
    ctx.debug_flag("tc_f16", 1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)


def _frames(seed, F, Hs, Ws):
    """Seeded uint8 frames [F,Hs,Ws,3]: blocky content plus noise (edges and flats for the resize and the WLS filter)."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1, 3)) * 255).astype(np.int32)
    img = np.kron(coarse, np.ones((1, 8, 8, 1), np.int32))[:, :Hs, :Ws]
    img = np.clip(img + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
    return torch.from_numpy(img)


def _centerpad_raw(ctx, rgb, geometry, size):
    Hr, Wr, oy, ox = geometry
    out = torch.empty(size[0], size[1], 3, device="cuda", dtype=torch.uint8)
    rc = ctx.lib.dvc_resize_antialias_crop_rgb8(ctx.h, ctypes.c_void_p(rgb.data_ptr()), rgb.shape[0], rgb.shape[1], Hr, Wr, oy, ox,
                                                ctypes.c_void_p(out.data_ptr()), size[0], size[1], ctypes.c_void_p(0))
    ctx._check(rc, "dvc_resize_antialias_crop_rgb8")
    return out


def _composition(ctx, clips, size, wls=(500.0, 4.0), first_last=None, geometries=None):
    """[S,F,Ho,Wo,3] uint8 and the clips' ab [S,F,2,Ho/2,Wo/2] through the stand-alone entry points, with colorize_clips as
    the network step."""
    labs = []
    for s, frames in enumerate(clips):
        g = geometries[s] if geometries else None
        crops = torch.stack([ctx.centerpad_rgb8(f.cuda(), size) if g is None else _centerpad_raw(ctx, f.cuda(), g, size) for f in frames])
        labs.append(ctx.rgb8_to_lab(crops))
    L = torch.stack([ctx.resize_half(lab)[:, 0:1].contiguous() for lab in labs])
    abs_ = ctx.colorize_clips(L, T, first_last_lab=first_last.cuda() if first_last is not None else None)
    outs = []
    for s, lab in enumerate(labs):
        ab_large = ctx.upsample2_scaled(abs_[s], 1.25)
        if wls is not None:
            for t in range(lab.shape[0]):
                ab_large[t] = ctx.fgs_filter(ctx.l_to_guide8(lab[t, 0]), ab_large[t], wls[0], wls[1])
        outs.append(ctx.lab_to_rgb8(lab[:, 0:1].contiguous(), ab_large))
    return torch.stack(outs).cpu(), abs_.cpu(), L.cpu()


def _videos_raw(ctx, clips, geoms, size, out, S=None, wls=1, last=None, null_at=None):
    """dvc_colorize_videos_rgb8 with explicit geometries; returns the status."""
    S = len(clips) if S is None else S
    n = max(S, 1)
    ptrs = (ctypes.c_void_p * n)(*[0 if s == null_at else clips[s % len(clips)].data_ptr() for s in range(n)])
    g = (ctypes.c_int * (6 * n))(*[v for s in range(n) for v in (*clips[s % len(clips)].shape[1:3], *geoms[s % len(geoms)])])
    vp = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)  # noqa: E731
    return ctx.lib.dvc_colorize_videos_rgb8(ctx.h, S, ptrs, clips[0].shape[0], g, size[0], size[1], T, None, wls, 500.0, 4.0, vp(out),
                                            vp(last), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


# ------------------------------------------------------------------------------------------ S = 1
def test_one_clip_is_the_single_path(ctx, conv_math):
    g = load_golden("clip3_32x48")
    L, IB = torch.from_numpy(g["frames_lab"])[:, 0:1].contiguous(), torch.from_numpy(g["IB_lab"])
    last = torch.from_numpy(g["frames_lab"][:1]).cuda() * 0.5
    frames = _frames(3, 4, 50, 70)
    ctx.set_exemplar(IB)
    ref_clip = ctx.colorize_clip(L.pin_memory())
    ref_ab, ref_warp, ref_sim = ctx.colorize_frames(L[:1].cuda(), last, want_warp=True)
    ref_video, ref_last = ctx.colorize_video_rgb8(frames.pin_memory(), (64, 96), T, return_last=True)
    for setter in (ctx.set_exemplar, ctx.set_exemplars):
        setter(IB)
        ab, warp, sim = ctx.colorize_frames_clips(L[:1].cuda(), last, want_warp=True)
        assert torch.equal(ab, ref_ab) and torch.equal(warp, ref_warp) and torch.equal(sim, ref_sim)
        assert torch.equal(ctx.colorize_clips(L[None].pin_memory())[0], ref_clip)
        assert torch.equal(ctx.colorize_clips(L[None].cuda())[0].cpu(), ref_clip)
        for src in (frames.pin_memory(), frames.cuda()):
            out, lst = ctx.colorize_videos_rgb8([src], (64, 96), T, return_last=True)
            assert torch.equal(out.cpu(), ref_video) and torch.equal(lst.cpu(), ref_last)


# ------------------------------------------------------------------------------------------ frames
@pytest.mark.parametrize("H,W", [(32, 64), (40, 64)])
@pytest.mark.parametrize("Tc", [1e-10, 0.01])
def test_frame_slots_equal_single_clip_frames(ctx, conv_math, H, W, Tc):
    IB = make_lab(80, 3, H, W)
    L = make_lab(81, 3, H, W)[:, 0:1].cuda()
    last = make_lab(82, 3, H, W).cuda()
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_clips(L, last, Tc, want_warp=True)
    assert ab.shape == (3, 2, H, W) and warp.shape == (3, 3, H, W) and sim.shape == (3, 1, H, W)
    for s in range(3):
        ctx.set_exemplar(IB[s:s + 1])
        ab1, warp1, sim1 = ctx.colorize_frames(L[s:s + 1], last[s:s + 1], Tc, want_warp=True)
        # VGG19 / WarpNet / ColorVidNet at batch S: device-derived scales and InstanceNorm sums differ from batch 1
        # (test_fused_batch_equals_single)
        assert (sim[s:s + 1] - sim1).abs().max() < 2e-6
        if Tc < 1e-9:
            assert torch.equal(warp[s:s + 1], warp1)
        else:
            # unlike the K-exemplar call, each clip's query features come out of the batch-S networks, so the scores move by
            # up to the sim bound and softmax(f / T) scales that by 1 / T: the warped colours agree to ~1e-5 relative
            assert (warp[s:s + 1] - warp1).abs().max() < 1e-3
        assert (ab[s:s + 1] - ab1).abs().max() < 5e-3


def test_frame_clips_vs_oracle_64x64(ctx, conv_math, sds):
    IA, IB, last = make_lab(120, 2, 64, 64), make_lab(121, 2, 64, 64), make_lab(122, 2, 64, 64)
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_clips(IA[:, 0:1].contiguous().cuda(), last.cuda(), want_warp=True)
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    for s in range(2):
        IAs, IBs, lasts = IA[s:s + 1], IB[s:s + 1], last[s:s + 1]
        ex = {}
        with torch.no_grad():
            fB = O.exemplar_features(sds64["vgg"], IBs.double())
            ab64, warped64, sim64, _ = O.frame_colorization(sds64, IAs.double(), IBs.double(), lasts.double(), fB, extras=ex)
            ab32, _, _, _ = O.frame_colorization(sds, IAs, IBs, lasts, O.exemplar_features(sds["vgg"], IBs))
        gap = O.top2_gap(ex["theta_hat"], ex["phi_hat"])
        assert (sim[s:s + 1].cpu().double() - sim64).abs().max() < 2e-5
        clear = (gap > 1e-5).view(1, 1, 16, 16).expand(1, 3, 16, 16)
        assert (warp[s:s + 1].cpu()[:, :, ::4, ::4][clear].double() - warped64[:, :, ::4, ::4][clear]).abs().max() < 1e-4
        floor = (ab32.double() - ab64).abs().max().item()
        assert (ab[s:s + 1].cpu().double() - ab64).abs().max().item() <= max(1e-3, 2 * floor)


# ------------------------------------------------------------------------------------------ clip
def test_clips_equal_chained_frames(ctx, conv_math):
    """S recurrences in one clip call == chaining colorize_frames_clips with last_s = cat(L_s, ab_s), bit for bit, from
    pinned host memory and from device memory, on one and on two phase-A streams, and with --frame_propagate."""
    S, F_, H, W = 3, 4, 32, 48
    L = torch.stack([make_lab(91 + s, F_, H, W)[:, 0:1] for s in range(S)]).contiguous()
    IB = make_lab(90, S, H, W)
    ctx.set_exemplars(IB)
    out = ctx.colorize_clips(L.pin_memory())
    assert out.shape == (S, F_, 2, H, W) and not out.is_cuda
    assert torch.equal(ctx.colorize_clips(L.cuda()).cpu(), out)
    ctx.debug_flag("clip_astreams", 2)
    try:
        out2 = ctx.colorize_clips(L.pin_memory())
    finally:
        ctx.debug_flag("clip_astreams", 1)
    assert torch.equal(out, out2)
    for first, res in ((None, out), (IB, ctx.colorize_clips(L.cuda(), first_last_lab=IB.cuda()).cpu())):
        last = torch.zeros(S, 3, H, W, device="cuda") if first is None else first.cuda()
        for t in range(F_):
            Lt = L[:, t].contiguous().cuda()
            ab = ctx.colorize_frames_clips(Lt, last)
            assert torch.equal(ab.cpu(), res[:, t]), (first is None, t)
            last = torch.cat((Lt, ab), 1)
    assert not torch.equal(res, out)


# ------------------------------------------------------------------------------------------ video
def test_videos_match_composition_720p(ctx):
    """Three clips of different source sizes in one call at test.py's default size, WLS on, from pinned host memory."""
    size, F_ = (432, 768), 3
    clips = [_frames(1, F_, 720, 1280), _frames(2, F_, 50, 60), _frames(3, F_, 100, 90)]
    ctx.set_exemplars(make_lab(40, 3, size[0] // 2, size[1] // 2))
    ref, _, _ = _composition(ctx, clips, size)
    out = ctx.colorize_videos_rgb8([f.pin_memory() for f in clips], size, T)
    assert out.shape == (3, F_, 432, 768, 3) and not out.is_cuda
    assert torch.equal(out, ref)


@pytest.mark.parametrize("wls,on_device", [(True, True), (False, False)])
def test_videos_zero_padded_window_and_first_last(ctx, wls, on_device):
    """A clip whose output window is larger than its resized image (zero border on every side) beside a cropped one, with
    first_last_lab, WLS on and off, host and device buffers."""
    size, geoms = (64, 96), [(50, 80, -7, -8), (64, 110, 0, 7)]
    clips = [_frames(5, 4, 40, 64), _frames(6, 4, 70, 120)]
    ctx.set_exemplars(make_lab(41, 2, 32, 48))
    first = make_lab(77, 2, 32, 48)
    w = (500.0, 4.0) if wls else None
    ref, _, _ = _composition(ctx, clips, size, wls=w, first_last=first, geometries=geoms)
    dev = (lambda t: t.cuda()) if on_device else (lambda t: t.pin_memory())
    out = dev(torch.empty(2, 4, 64, 96, 3, dtype=torch.uint8))
    S = len(clips)
    src = [dev(f) for f in clips]
    ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in src])
    g = (ctypes.c_int * (6 * S))(*[v for s in range(S) for v in (*clips[s].shape[1:3], *geoms[s])])
    fl = dev(first)
    rc = ctx.lib.dvc_colorize_videos_rgb8(ctx.h, S, ptrs, 4, g, 64, 96, T, ctypes.c_void_p(fl.data_ptr()), 1 if wls else 0, 500.0,
                                          4.0, ctypes.c_void_p(out.data_ptr()), None, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    ctx._check(rc, "dvc_colorize_videos_rgb8")
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("on_device", [False, True])
def test_videos_chunks_continue_exactly(ctx, on_device):
    F_, a, size = 7, 3, (64, 96)
    ctx.set_exemplars(make_lab(42, 2, 32, 48))
    clips = [_frames(11, F_, 72, 120), _frames(12, F_, 60, 60)]
    clips = [f.cuda() if on_device else f.pin_memory() for f in clips]
    whole, last = ctx.colorize_videos_rgb8(clips, size, T, return_last=True)
    head, l1 = ctx.colorize_videos_rgb8([f[:a] for f in clips], size, T, return_last=True)
    tail, l2 = ctx.colorize_videos_rgb8([f[a:] for f in clips], size, T, first_last_lab=l1, return_last=True)
    assert torch.equal(torch.cat((head, tail), 1), whole)
    assert torch.equal(l2, last)
    # last_lab_out = cat(L/2, ab) of every clip's last frame, as the clips compute them
    ref, ab, L = _composition(ctx, [f.cpu() for f in clips], size)
    assert torch.equal(whole.cpu(), ref)
    assert torch.equal(last.cpu(), torch.cat((L[:, -1], ab[:, -1]), 1))


def test_videos_device_memory_does_not_grow_with_F(ctx):
    ctx.set_exemplars(make_lab(43, 2, 32, 48))
    ctx.colorize_videos_rgb8([_frames(3, 8, 48, 80), _frames(4, 8, 40, 40)], (64, 96), T)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    out = ctx.colorize_videos_rgb8([_frames(5, 200, 48, 80).pin_memory(), _frames(6, 200, 40, 40).pin_memory()], (64, 96), T)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert out.shape == (2, 200, 64, 96, 3) and not out.is_cuda
    assert free1 >= free0, (free0, free1)


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(ctx):
    import dvc

    H, W, size = 32, 48, (64, 96)
    ctx.set_exemplars(make_lab(44, 2, H, W))
    clips = [_frames(7, 2, 48, 80).pin_memory(), _frames(8, 2, 64, 96).pin_memory()]
    geoms = [(57, 96, 0, 0), (64, 96, 0, 0)]
    out = torch.empty(9, 2, 64, 96, 3, dtype=torch.uint8).pin_memory()
    L = make_lab(45, 9, H, W)[:, 0:1].cuda()
    last = make_lab(46, 9, H, W).cuda()
    ab = torch.empty(9, 2, 2, H, W, device="cuda")
    stream = dvc._stream(ctx.device)
    torch.cuda.synchronize()

    def refused(call, want):
        n = ctx.launch_count()
        assert call() == want
        assert ctx.launch_count() == n

    for S, want in ((0, -1), (9, -1), (3, -2), (1, -2)):  # S outside [1, 8]; S other than the 2 cached exemplars
        refused(lambda: _videos_raw(ctx, clips, geoms, size, out, S=S), want)
        refused(lambda: ctx.lib.dvc_colorize_clips(ctx.h, dvc._ptr(L), 1, H, W, T, None, S, dvc._ptr(ab), stream), want)
        refused(lambda: ctx.lib.dvc_colorize_frames_clips(ctx.h, dvc._ptr(L), dvc._ptr(last), S, H, W, T, dvc._ptr(ab), None, None,
                                                          stream), want)
    refused(lambda: _videos_raw(ctx, clips, [(86, 144, 3, 0), (80, 128, 0, 0)], (80, 128), out), -2)  # frame size != exemplars'
    refused(lambda: ctx.lib.dvc_colorize_clips(ctx.h, dvc._ptr(L), 1, H, 64, T, None, 2, dvc._ptr(ab), stream), -2)
    refused(lambda: _videos_raw(ctx, clips, [geoms[0], (70, 96, 7, 0)], size, out), -2)  # clip 1's window leaves its image
    refused(lambda: _videos_raw(ctx, clips, [(50, 80, 1, 0), geoms[1]], size, out), -2)  # clip 0's pad window not around it
    refused(lambda: _videos_raw(ctx, clips, geoms, size, out, null_at=1), -1)            # a null frame pointer
    with pytest.raises(dvc.DvcError):
        ctx.colorize_videos_rgb8(clips, size, T, first_last_lab=torch.zeros(3, 3, 32, 48))
    # the context still works after the refusals
    assert ctx.colorize_videos_rgb8(clips, size, T).shape == (2, 2, 64, 96, 3)


# ------------------------------------------------------------------------------------------ the folder tool
def test_colorize_folder_several_clips(ctx, tmp_path):
    """Two clips of different lengths and source sizes, one reference each: every frame is written once, and the PNGs are
    the bytes of the call sequence tools/colorize_folder.py documents, restated here."""
    import io

    from PIL import Image

    size, C = (64, 96), 3
    lens, shapes = (7, 4), ((60, 110), (50, 80))
    dirs, clips, refs = [], [], []
    for s in range(2):
        d = tmp_path / f"clip{s}"
        d.mkdir()
        fr = _frames(21 + s, lens[s], *shapes[s])
        for t in range(lens[s]):
            Image.fromarray(fr[t].numpy()).save(d / f"f{t + 1}.png")
        p = tmp_path / f"ref{s}.png"
        Image.fromarray(_frames(30 + s, 1, 70, 100)[0].numpy()).save(p)
        dirs.append(d), clips.append(fr), refs.append(p)
    out_dir = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", *map(str, dirs), "--ref", *map(str, refs),
           "--out", str(out_dir), "--seeded-weights", "--chunk", str(C), "--image-size", str(size[0]), str(size[1])]
    subprocess.run(cmd, check=True, cwd=str(tmp_path))
    # the documented sequence: each call takes n = min(chunk, frames left) frames of every clip that has frames left; a clip
    # that runs out leaves, and the others continue with their exemplars and their rows of last_lab_out
    ref_lab = ctx.resize_half(ctx.rgb8_to_lab(torch.stack([ctx.centerpad_rgb8(
        torch.from_numpy(np.asarray(Image.open(r).convert("RGB")).copy()).cuda(), size) for r in refs])))
    want = {s: [] for s in range(2)}
    pos, active, last = [0, 0], [0, 1], None
    ctx.set_exemplars(ref_lab)
    while active:
        n = min(C, *(lens[s] - pos[s] for s in active))
        out, last = ctx.colorize_videos_rgb8([clips[s][pos[s]:pos[s] + n] for s in active], size, T, first_last_lab=last,
                                             return_last=True)
        for j, s in enumerate(active):
            want[s] += list(out[j])
            pos[s] += n
        keep = [j for j, s in enumerate(active) if pos[s] < lens[s]]
        if len(keep) < len(active):
            active = [active[j] for j in keep]
            last = last[keep]
            if active:
                ctx.set_exemplars(ref_lab[active])
    for s in range(2):
        d = out_dir / dirs[s].name
        assert sorted(os.listdir(d)) == sorted(f"f{t + 1}.png" for t in range(lens[s]))
        for t in range(lens[s]):
            buf = io.BytesIO()
            Image.fromarray(want[s][t].numpy()).save(buf, format="PNG")
            assert (d / f"f{t + 1}.png").read_bytes() == buf.getvalue(), (s, t)
