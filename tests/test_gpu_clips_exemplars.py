"""Several clips in one pass with several exemplars each (include/dvc.h: dvc_colorize_frames_clips_exemplars,
dvc_colorize_clips_exemplars, dvc_colorize_videos_exemplars_rgb8).  Clip s has K[s] exemplar rows; row r = (s, k) must be
test.py:68-120 run on clip s against its exemplar k: the degenerate counts bit for bit against the existing calls, the rows
against the several-clip call that caches exemplar k of every clip, the fp64 oracle, and the clip and video calls bit for
bit against the chain of the calls they are built from."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import dvc_oracle as O
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu
T = 1e-10


def _conv_math(ctx, name):
    import dvc

    if name == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32)
    else:
        ctx.set_math(conv=dvc.MATH_FP16X1 if name == "fp16x1" else dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        ctx.debug_flag("tc_f16", 0 if name.endswith("nof16") else 1)
    yield name
    ctx.debug_flag("tc_f16", 1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)


@pytest.fixture(params=["fp32", "tf32x3", "tf32x3-nof16", "fp16x1"])
def conv_math(request, ctx):
    """Every convolution arithmetic: the exact CUDA-core engines, the tensor-core convolutions with and without the fp16
    planes of bounded layers, and the one-pass fp16 mode."""
    yield from _conv_math(ctx, request.param)


@pytest.fixture(params=["fp32", "tf32x3", "tf32x3-nof16"])
def fp32_conv_math(request, ctx):
    """The fp32-class convolution arithmetics, which the fp64 oracle's gates are set for (MATH_FP16X1 rounds the operands
    to 11 bits, tests/test_gpu_fast_math.py)."""
    yield from _conv_math(ctx, request.param)


@pytest.fixture(params=["fp32", "tf32x3", "bf16x3", "fp16x3", "fp16x3-noscreen"])
def corr_math(request, ctx):
    """Every correlation arithmetic; fp16x3 at T -> 0 screens unless "-noscreen"."""
    import dvc

    name = request.param.replace("-noscreen", "")
    mode = {"fp32": dvc.MATH_FP32, "tf32x3": dvc.MATH_TF32X3, "bf16x3": dvc.MATH_BF16X3, "fp16x3": dvc.MATH_FP16X3}[name]
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=mode)
    ctx.debug_flag("corr_screen", 0 if "noscreen" in request.param else 1)
    yield name
    ctx.debug_flag("corr_screen", 1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)


def _frames(seed, F, Hs, Ws):
    """Seeded uint8 frames [F,Hs,Ws,3]: blocky content plus noise (edges and flats for the resize and the WLS filter)."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1, 3)) * 255).astype(np.int32)
    img = np.kron(coarse, np.ones((1, 8, 8, 1), np.int32))[:, :Hs, :Ws]
    img = np.clip(img + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
    return torch.from_numpy(img)


def _src(K):
    """Clip of every row."""
    return [s for s, k in enumerate(K) for _ in range(k)]


def _centerpad_raw(ctx, rgb, geometry, size):
    Hr, Wr, oy, ox = geometry
    out = torch.empty(size[0], size[1], 3, device="cuda", dtype=torch.uint8)
    rc = ctx.lib.dvc_resize_antialias_crop_rgb8(ctx.h, ctypes.c_void_p(rgb.data_ptr()), rgb.shape[0], rgb.shape[1], Hr, Wr, oy, ox,
                                                ctypes.c_void_p(out.data_ptr()), size[0], size[1], ctypes.c_void_p(0))
    ctx._check(rc, "dvc_resize_antialias_crop_rgb8")
    return out


def _composition(ctx, clips, K, size, wls=(500.0, 4.0), first_last=None, geometries=None):
    """[R,F,Ho,Wo,3] uint8 and the rows' ab [R,F,2,Ho/2,Wo/2] through the stand-alone entry points: colorize_frames_clips_exemplars
    chained over the frames, then per row upsample2_scaled -> fgs_filter with its clip's guide -> lab_to_rgb8 with its clip's L."""
    labs = []
    for s, frames in enumerate(clips):
        g = geometries[s] if geometries else None
        crops = torch.stack([ctx.centerpad_rgb8(f.cuda(), size) if g is None else _centerpad_raw(ctx, f.cuda(), g, size) for f in frames])
        labs.append(ctx.rgb8_to_lab(crops))
    L = torch.stack([ctx.resize_half(lab)[:, 0:1].contiguous() for lab in labs])  # [S,F,1,h,w]
    src, F_ = _src(K), L.shape[1]
    last = first_last.cuda() if first_last is not None else torch.zeros(len(src), 3, *L.shape[3:], device="cuda")
    abs_ = []
    for t in range(F_):
        ab = ctx.colorize_frames_clips_exemplars(L[:, t].contiguous(), K, last, T)
        abs_.append(ab)
        last = torch.cat((L[src, t], ab), 1)
    abs_ = torch.stack(abs_, 1)  # [R,F,2,h,w]
    outs = []
    for r, s in enumerate(src):
        lab = labs[s]
        ab_large = ctx.upsample2_scaled(abs_[r], 1.25)
        if wls is not None:
            for t in range(F_):
                ab_large[t] = ctx.fgs_filter(ctx.l_to_guide8(lab[t, 0]), ab_large[t], wls[0], wls[1])
        outs.append(ctx.lab_to_rgb8(lab[:, 0:1].contiguous(), ab_large))
    return torch.stack(outs).cpu(), abs_.cpu(), L.cpu(), last.cpu()


# ------------------------------------------------------------------------------------------ degenerate counts
def test_degenerate_counts_are_the_existing_calls(ctx, conv_math):
    """Every K[s] = 1 is the several-clip call, one clip the K-exemplar call: bit for bit, frames, clips and videos."""
    H, W, F_, size = 32, 48, 3, (64, 96)
    IB = make_lab(200, 3, H, W)
    Lc = torch.stack([make_lab(201 + s, F_, H, W)[:, 0:1] for s in range(3)]).contiguous()  # [3,F,1,H,W]
    last = make_lab(205, 3, H, W).cuda()
    videos = [_frames(210, F_, 50, 70), _frames(211, F_, 72, 120), _frames(212, F_, 64, 96)]
    ctx.set_exemplars(IB)
    # every K[s] = 1
    ref = ctx.colorize_frames_clips(Lc[:, 0].cuda(), last, want_warp=True)
    got = ctx.colorize_frames_clips_exemplars(Lc[:, 0].cuda(), [1, 1, 1], last, want_warp=True)
    assert all(torch.equal(a, b) for a, b in zip(got, ref))
    assert torch.equal(ctx.colorize_clips_exemplars(Lc.pin_memory(), [1, 1, 1]), ctx.colorize_clips(Lc.pin_memory()))
    pinned = [v.pin_memory() for v in videos]
    ref_v, ref_l = ctx.colorize_videos_rgb8(pinned, size, T, return_last=True)
    got_v, got_l = ctx.colorize_videos_exemplars_rgb8(pinned, [1, 1, 1], size, T, return_last=True)
    assert torch.equal(got_v, ref_v) and torch.equal(got_l, ref_l)
    # one clip, three exemplars
    ref = ctx.colorize_frames_exemplars(Lc[0, :1].cuda(), last, want_warp=True)
    got = ctx.colorize_frames_clips_exemplars(Lc[0, :1].cuda(), [3], last, want_warp=True)
    assert all(torch.equal(a, b) for a, b in zip(got, ref))
    assert torch.equal(ctx.colorize_clips_exemplars(Lc[:1].pin_memory(), [3]), ctx.colorize_clip_exemplars(Lc[0].pin_memory()))
    ref_v, ref_l = ctx.colorize_video_rgb8(pinned[1], size, T, return_last=True)
    got_v, got_l = ctx.colorize_videos_exemplars_rgb8(pinned[1:2], [3], size, T, return_last=True)
    assert torch.equal(got_v, ref_v) and torch.equal(got_l, ref_l)


# ------------------------------------------------------------------------------------------ rows against the S-clip call
@pytest.mark.parametrize("Tc", [1e-10, 0.01])
def test_rows_equal_clip_calls_per_exemplar(ctx, corr_math, Tc):
    """Counts (2, 2, 2): row (s, k) against dvc_colorize_frames_clips with exemplar k of every clip cached.  Phase A is the
    same batch-S computation, so the row maxima are bit-equal and the warped colours follow test_gpu_exemplars' bound."""
    S, Kc, H, W = 3, 2, 32, 64
    IB = make_lab(220, S * Kc, H, W)  # row order: clip 0's exemplars, then clip 1's, ...
    L = make_lab(221, S, H, W)[:, 0:1].contiguous().cuda()
    last = make_lab(222, S * Kc, H, W).cuda()
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_clips_exemplars(L, [Kc] * S, last, Tc, want_warp=True)
    assert ab.shape == (S * Kc, 2, H, W) and warp.shape == (S * Kc, 3, H, W) and sim.shape == (S * Kc, 1, H, W)
    for k in range(Kc):
        rows = [s * Kc + k for s in range(S)]
        ctx.set_exemplars(IB[rows])
        ab1, warp1, sim1 = ctx.colorize_frames_clips(L, last[rows], Tc, want_warp=True)
        assert torch.equal(sim[rows], sim1), k
        if Tc < 1e-9:
            assert torch.equal(warp[rows], warp1), k
        else:
            assert (warp[rows] - warp1).abs().max() < 1e-4, k  # another column-split count: another softmax summation order
        # ColorVidNet at batch R instead of S: InstanceNorm sums and device-derived scales differ (test_fused_batch_equals_single)
        assert (ab[rows] - ab1).abs().max() < 5e-3, k


@pytest.mark.parametrize("K", [(2, 2), (1, 3)])
def test_rows_vs_oracle_64x64(ctx, fp32_conv_math, sds, K):
    S, R = len(K), sum(K)
    IA, IB, last = make_lab(230, S, 64, 64), make_lab(231, R, 64, 64), make_lab(232, R, 64, 64)
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_clips_exemplars(IA[:, 0:1].contiguous().cuda(), list(K), last.cuda(), want_warp=True)
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    for r, s in enumerate(_src(K)):
        IAs, IBr, lastr = IA[s:s + 1], IB[r:r + 1], last[r:r + 1]
        ex = {}
        with torch.no_grad():
            fB = O.exemplar_features(sds64["vgg"], IBr.double())
            ab64, warped64, sim64, _ = O.frame_colorization(sds64, IAs.double(), IBr.double(), lastr.double(), fB, extras=ex)
            ab32, _, _, _ = O.frame_colorization(sds, IAs, IBr, lastr, O.exemplar_features(sds["vgg"], IBr))
        gap = O.top2_gap(ex["theta_hat"], ex["phi_hat"])
        assert (sim[r:r + 1].cpu().double() - sim64).abs().max() < 2e-5, r
        clear = (gap > 1e-5).view(1, 1, 16, 16).expand(1, 3, 16, 16)
        assert (warp[r:r + 1].cpu()[:, :, ::4, ::4][clear].double() - warped64[:, :, ::4, ::4][clear]).abs().max() < 1e-4, r
        floor = (ab32.double() - ab64).abs().max().item()
        assert (ab[r:r + 1].cpu().double() - ab64).abs().max().item() <= max(1e-3, 2 * floor), r


# ------------------------------------------------------------------------------------------ clip
@pytest.mark.parametrize("K", [(2, 2), (3, 1, 2)])
def test_clips_exemplars_equal_chained_frames(ctx, conv_math, K):
    """R recurrences in one clip call == chaining colorize_frames_clips_exemplars with last_r = cat(L_src(r), ab_r), bit for
    bit, from pinned host memory and from device memory, on one and on two phase-A streams, and with first_last_lab."""
    S, R, F_, H, W = len(K), sum(K), 4, 32, 48
    src = _src(K)
    L = torch.stack([make_lab(240 + s, F_, H, W)[:, 0:1] for s in range(S)]).contiguous()
    IB = make_lab(239, R, H, W)
    ctx.set_exemplars(IB)
    out = ctx.colorize_clips_exemplars(L.pin_memory(), list(K))
    assert out.shape == (R, F_, 2, H, W) and not out.is_cuda
    assert torch.equal(ctx.colorize_clips_exemplars(L.cuda(), list(K)).cpu(), out)
    ctx.debug_flag("clip_astreams", 2)
    try:
        out2 = ctx.colorize_clips_exemplars(L.pin_memory(), list(K))
    finally:
        ctx.debug_flag("clip_astreams", 1)
    assert torch.equal(out, out2)
    for first, res in ((None, out), (IB, ctx.colorize_clips_exemplars(L.cuda(), list(K), first_last_lab=IB.cuda()).cpu())):
        last = torch.zeros(R, 3, H, W, device="cuda") if first is None else first.cuda()
        for t in range(F_):
            Lt = L[:, t].contiguous().cuda()
            ab = ctx.colorize_frames_clips_exemplars(Lt, list(K), last)
            assert torch.equal(ab.cpu(), res[:, t]), (first is None, t)
            last = torch.cat((Lt[src], ab), 1)
    assert not torch.equal(res, out)


# ------------------------------------------------------------------------------------------ video
def test_videos_exemplars_match_composition_720p(ctx):
    """A 720x1280 clip with two exemplars beside a small clip with one, at test.py's default size, WLS on, pinned host memory."""
    size, F_, K = (432, 768), 3, [2, 1]
    clips = [_frames(250, F_, 720, 1280), _frames(251, F_, 50, 60)]
    ctx.set_exemplars(make_lab(252, 3, size[0] // 2, size[1] // 2))
    ref, _, _, _ = _composition(ctx, clips, K, size)
    out = ctx.colorize_videos_exemplars_rgb8([f.pin_memory() for f in clips], K, size, T)
    assert out.shape == (3, F_, 432, 768, 3) and not out.is_cuda
    assert torch.equal(out, ref)


@pytest.mark.parametrize("wls,on_device", [(True, True), (False, False)])
def test_videos_exemplars_zero_padded_window_and_first_last(ctx, wls, on_device):
    """A clip whose output window is larger than its resized image (zero border on every side) beside a cropped one, counts
    (1, 3), with first_last_lab, WLS on and off, host and device buffers."""
    size, geoms, K = (64, 96), [(50, 80, -7, -8), (64, 110, 0, 7)], [1, 3]
    clips = [_frames(255, 4, 40, 64), _frames(256, 4, 70, 120)]
    ctx.set_exemplars(make_lab(257, 4, 32, 48))
    first = make_lab(258, 4, 32, 48)
    w = (500.0, 4.0) if wls else None
    ref, _, _, _ = _composition(ctx, clips, K, size, wls=w, first_last=first, geometries=geoms)
    dev = (lambda t: t.cuda()) if on_device else (lambda t: t.pin_memory())
    out = dev(torch.empty(4, 4, 64, 96, 3, dtype=torch.uint8))
    S = len(clips)
    src = [dev(f) for f in clips]
    ptrs = (ctypes.c_void_p * S)(*[f.data_ptr() for f in src])
    g = (ctypes.c_int * (6 * S))(*[v for s in range(S) for v in (*clips[s].shape[1:3], *geoms[s])])
    fl = dev(first)
    rc = ctx.lib.dvc_colorize_videos_exemplars_rgb8(ctx.h, S, (ctypes.c_int * S)(*K), ptrs, 4, g, 64, 96, T, ctypes.c_void_p(fl.data_ptr()),
                                                    1 if wls else 0, 500.0, 4.0, ctypes.c_void_p(out.data_ptr()), None,
                                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    ctx._check(rc, "dvc_colorize_videos_exemplars_rgb8")
    assert torch.equal(out.cpu(), ref)


@pytest.mark.parametrize("on_device", [False, True])
def test_videos_exemplars_chunks_continue_exactly(ctx, on_device):
    F_, a, size, K = 7, 3, (64, 96), [3, 2]
    ctx.set_exemplars(make_lab(260, 5, 32, 48))
    clips = [_frames(261, F_, 72, 120), _frames(262, F_, 60, 60)]
    clips = [f.cuda() if on_device else f.pin_memory() for f in clips]
    whole, last = ctx.colorize_videos_exemplars_rgb8(clips, K, size, T, return_last=True)
    head, l1 = ctx.colorize_videos_exemplars_rgb8([f[:a] for f in clips], K, size, T, return_last=True)
    tail, l2 = ctx.colorize_videos_exemplars_rgb8([f[a:] for f in clips], K, size, T, first_last_lab=l1, return_last=True)
    assert torch.equal(torch.cat((head, tail), 1), whole)
    assert torch.equal(l2, last)
    # last_lab_out = cat(L/2, ab) of every row's last frame, as the stand-alone chain computes it
    ref, _, _, ref_last = _composition(ctx, [f.cpu() for f in clips], K, size)
    assert torch.equal(whole.cpu(), ref)
    assert torch.equal(last.cpu(), ref_last)


def test_videos_exemplars_device_memory_does_not_grow_with_F(ctx):
    K = [1, 3]
    ctx.set_exemplars(make_lab(265, 4, 32, 48))
    ctx.colorize_videos_exemplars_rgb8([_frames(266, 8, 48, 80), _frames(267, 8, 40, 40)], K, (64, 96), T)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    out = ctx.colorize_videos_exemplars_rgb8([_frames(268, 200, 48, 80).pin_memory(), _frames(269, 200, 40, 40).pin_memory()], K,
                                             (64, 96), T)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert out.shape == (4, 200, 64, 96, 3) and not out.is_cuda
    assert free1 >= free0, (free0, free1)


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(ctx):
    import dvc

    H, W, size = 32, 48, (64, 96)
    clips = [_frames(270, 2, 48, 80).pin_memory(), _frames(271, 2, 64, 96).pin_memory()]
    geoms = [(57, 96, 0, 0), (64, 96, 0, 0)]
    out = torch.empty(9, 2, 64, 96, 3, dtype=torch.uint8).pin_memory()
    L = make_lab(272, 9, H, W)[:, 0:1].cuda()
    last = make_lab(273, 9, H, W).cuda()
    ab = torch.empty(9, 2, 2, H, W, device="cuda")
    stream = dvc._stream(ctx.device)

    def ints(K):
        return None if K is None else (ctypes.c_int * max(len(K), 1))(*K)

    def videos(S, K, geo=geoms, sz=size, null_at=None):
        n = max(S, 1)
        ptrs = (ctypes.c_void_p * n)(*[0 if s == null_at else clips[s % 2].data_ptr() for s in range(n)])
        g = (ctypes.c_int * (6 * n))(*[v for s in range(n) for v in (*clips[s % 2].shape[1:3], *geo[s % 2])])
        return ctx.lib.dvc_colorize_videos_exemplars_rgb8(ctx.h, S, ints(K), ptrs, 2, g, sz[0], sz[1], T, None, 1, 500.0, 4.0,
                                                          ctypes.c_void_p(out.data_ptr()), None, stream)

    def clips_call(S, K, w=W):
        return ctx.lib.dvc_colorize_clips_exemplars(ctx.h, dvc._ptr(L), 1, H, w, T, None, S, ints(K), dvc._ptr(ab), stream)

    def frames_call(S, K, w=W):
        return ctx.lib.dvc_colorize_frames_clips_exemplars(ctx.h, dvc._ptr(L), dvc._ptr(last), S, ints(K), H, w, T, dvc._ptr(ab), None,
                                                           None, stream)

    def refused(call, want):
        n = ctx.launch_count()
        assert call() == want
        assert ctx.launch_count() == n

    for slots in (2, 8):  # counts (2, 2) against 2 or 8 cached slots
        ctx.set_exemplars(make_lab(274, slots, H, W))
        torch.cuda.synchronize()
        for call in (videos, clips_call, frames_call):
            refused(lambda: call(2, [2, 2]), -2)
    ctx.set_exemplars(make_lab(275, 4, H, W))
    torch.cuda.synchronize()
    # S outside [1, 8], a null K, a count below 1, more than 8 rows: DVC_ERR_ARG
    for S, K in ((0, [1]), (9, [1] * 9), (2, None), (2, [0, 4]), (2, [3, -1]), (2, [5, 4])):
        for call in (videos, clips_call, frames_call):
            refused(lambda: call(S, K), -1)
    refused(lambda: videos(2, [2, 2], [(86, 144, 3, 0), (80, 128, 0, 0)], (80, 128)), -2)  # frame size other than the exemplars'
    refused(lambda: clips_call(2, [2, 2], 64), -2)
    refused(lambda: frames_call(2, [2, 2], 64), -2)
    refused(lambda: videos(2, [2, 2], [geoms[0], (70, 96, 7, 0)]), -2)  # clip 1's window leaves its image
    refused(lambda: videos(2, [2, 2], [(50, 80, 1, 0), geoms[1]]), -2)  # clip 0's pad window not around it
    refused(lambda: videos(2, [2, 2], null_at=1), -1)                   # a null frame pointer
    with pytest.raises(dvc.DvcError):
        ctx.colorize_videos_exemplars_rgb8(clips, [2, 2], size, T, first_last_lab=torch.zeros(3, 3, 32, 48))
    with pytest.raises(dvc.DvcError):
        ctx.colorize_videos_exemplars_rgb8(clips, [4], size, T)  # one count per clip
    # the context still works after the refusals
    assert ctx.colorize_videos_exemplars_rgb8(clips, [1, 3], size, T).shape == (4, 2, 64, 96, 3)


# ------------------------------------------------------------------------------------------ the folder tool
def test_colorize_folder_clips_with_reference_folders(ctx, tmp_path):
    """Two clips of different lengths and source sizes with --ref folders of one and of three images: the PNGs are the bytes
    of the call sequence tools/colorize_folder.py documents, restated here."""
    import io

    from PIL import Image

    size, C = (64, 96), 3
    lens, shapes, nref = (7, 4), ((60, 110), (50, 80)), (1, 3)
    dirs, clips, refdirs, refs = [], [], [], []
    for s in range(2):
        d = tmp_path / f"clip{s}"
        d.mkdir()
        fr = _frames(280 + s, lens[s], *shapes[s])
        for t in range(lens[s]):
            Image.fromarray(fr[t].numpy()).save(d / f"f{t + 1}.png")
        rd = tmp_path / f"ref{s}"
        rd.mkdir()
        names = [f"r{chr(ord('c') - k)}.png" for k in range(nref[s])]  # written in reverse name order: the tool sorts them
        for k, n in enumerate(names):
            Image.fromarray(_frames(290 + 3 * s + k, 1, 70, 100)[0].numpy()).save(rd / n)
        dirs.append(d), clips.append(fr), refdirs.append(rd), refs.append(sorted(rd / n for n in names))
    out_dir = tmp_path / "out"
    cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", *map(str, dirs), "--ref", *map(str, refdirs),
           "--out", str(out_dir), "--seeded-weights", "--chunk", str(C), "--image-size", str(size[0]), str(size[1])]
    subprocess.run(cmd, check=True, cwd=str(tmp_path))
    # the documented sequence: rows in clip order, each clip's exemplars sorted by name; each call takes n = min(chunk, frames
    # left) frames of every clip that has frames left; a clip that runs out leaves with its rows, and the others continue
    # with their exemplars re-cached and their rows of last_lab_out
    ref_lab = [ctx.resize_half(ctx.rgb8_to_lab(torch.stack([ctx.centerpad_rgb8(
        torch.from_numpy(np.asarray(Image.open(r).convert("RGB")).copy()).cuda(), size) for r in rs]))) for rs in refs]
    want = {(s, k): [] for s in range(2) for k in range(nref[s])}
    pos, active, last = [0, 0], [0, 1], None
    ctx.set_exemplars(torch.cat([ref_lab[s] for s in active]))
    while active:
        n = min(C, *(lens[s] - pos[s] for s in active))
        out, last = ctx.colorize_videos_exemplars_rgb8([clips[s][pos[s]:pos[s] + n] for s in active], [nref[s] for s in active], size, T,
                                                       first_last_lab=last, return_last=True)
        rows = [(s, k) for s in active for k in range(nref[s])]
        for j, sk in enumerate(rows):
            want[sk] += list(out[j])
        for s in active:
            pos[s] += n
        keep = [s for s in active if pos[s] < lens[s]]
        if len(keep) < len(active):
            last = last[[j for j, (s, _) in enumerate(rows) if s in keep]]
            active = keep
            if active:
                ctx.set_exemplars(torch.cat([ref_lab[s] for s in active]))
    for (s, k), imgs in want.items():
        d = out_dir / dirs[s].name
        if nref[s] > 1:
            d = d / os.path.splitext(refs[s][k].name)[0]
        assert sorted(os.listdir(d)) == sorted(f"f{t + 1}.png" for t in range(lens[s])), (s, k)
        for t in range(lens[s]):
            buf = io.BytesIO()
            Image.fromarray(imgs[t].numpy()).save(buf, format="PNG")
            assert (d / f"f{t + 1}.png").read_bytes() == buf.getvalue(), (s, k, t)
