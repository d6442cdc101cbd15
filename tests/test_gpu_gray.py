"""Greyscale sources (include/dvc.h: dvc_colorize_videos_gray8).  A grey frame g has one correct output: the bytes the sRGB calls
return for g with each byte repeated into R, G and B (PIL's "L" -> "RGB").  Every check below compares with that call by
torch.equal: output bytes, last_lab_out, JPEG sizes, and the kernel launches per call."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu
T = 1e-10
WLS = (500.0, 4.0)
SIZE = (64, 96)  # networks at 32 x 48
CANARY = 0xA5


def _gray(seed, F, Hs, Ws):
    """Blocks with noise that reach 0 and 255: every byte value goes through the L table somewhere."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, Hs // 8 + 1, Ws // 8 + 1)) * 255).astype(np.int32)
    img = np.kron(coarse, np.ones((1, 8, 8), np.int32))[:, :Hs, :Ws]
    return torch.from_numpy(np.clip(img + rng.integers(-40, 41, img.shape), 0, 255).astype(np.uint8))


def _rgb(g):
    return g[..., None].repeat(1, 1, 1, 3)


def _side(on_device):
    return (lambda t: t.cuda()) if on_device else (lambda t: t.pin_memory())


def _counted(ctx, fn):
    torch.cuda.synchronize()
    ctx.launch_count(reset=True)
    res = fn()
    torch.cuda.synchronize()
    return res, ctx.launch_count()


def _check(ctx, clips, K, size=SIZE, source=False, q=None, on_device=False, wls=WLS, first_last=None):
    """The grey call against the sRGB call on the replicated frames; returns the grey call's last state."""
    import dvc

    side = _side(on_device)
    g = [side(c) for c in clips]
    rgb = [side(_rgb(c)) for c in clips]
    fl = None if first_last is None else side(first_last)
    kw = dict(first_last_lab=fl, wls=wls, return_last=True)
    ctx.colorize_videos_gray8(g, K, size, T, first_last_lab=fl, wls=wls, source_resolution=source, quality=q)  # one-off launches
    if q is not None:
        (ref, ref_sizes, ref_last), n_ref = _counted(ctx, lambda: ctx.colorize_videos_jpeg(rgb, K, size, q, source, T, **kw))
        (got, sizes, last), n_got = _counted(ctx, lambda: ctx.colorize_videos_gray8(g, K, size, T, source_resolution=source, quality=q, **kw))
        assert torch.equal(sizes.cpu(), ref_sizes.cpu())
        assert dvc.jpeg_files(got, sizes) == dvc.jpeg_files(ref, ref_sizes)
    elif source:
        (ref, ref_last), n_ref = _counted(ctx, lambda: ctx.colorize_videos_source_rgb8(rgb, K, size, T, **kw))
        (got, last), n_got = _counted(ctx, lambda: ctx.colorize_videos_gray8(g, K, size, T, source_resolution=True, **kw))
        assert len(got) == len(ref) and all(a.is_cuda == on_device for a in got)
        for a, b in zip(got, ref):
            assert torch.equal(a.cpu(), b.cpu())
    else:
        (ref, ref_last), n_ref = _counted(ctx, lambda: ctx.colorize_videos_exemplars_rgb8(rgb, K, size, T, **kw))
        (got, last), n_got = _counted(ctx, lambda: ctx.colorize_videos_gray8(g, K, size, T, **kw))
        assert got.is_cuda == on_device
        assert torch.equal(got.cpu(), ref.cpu())
    assert torch.equal(last.cpu(), ref_last.cpu())
    assert n_got == n_ref
    return got, last


# ------------------------------------------------------------------------------------------ output kinds and counts
KINDS = [(False, None), (True, None), (False, 75), (False, 95), (True, 75), (True, 95)]


@pytest.mark.parametrize("kind", KINDS, ids=lambda k: ("source" if k[0] else "window") + (f"-q{k[1]}" if k[1] else "-srgb"))
@pytest.mark.parametrize("K", [[1], [3], [1, 2, 1]], ids=lambda K: "K" + "-".join(map(str, K)))
def test_output_kinds(ctx, kind, K):
    source, q = kind
    R = sum(K)
    shapes = ((90, 150), (48, 80), (100, 90))
    if R == 1:
        ctx.set_exemplar(make_lab(500, 1, 32, 48))
    else:
        ctx.set_exemplars(make_lab(500, R, 32, 48))
    clips = [_gray(501 + s, 3, *shapes[s]) for s in range(len(K))]
    _check(ctx, clips, K, source=source, q=q, on_device=R % 2 == 0)


def test_one_clip_equals_colorize_video_rgb8(ctx):
    ctx.set_exemplar(make_lab(510, 1, 32, 48))
    g = _gray(511, 4, 90, 150)
    ref, ref_last = ctx.colorize_video_rgb8(_rgb(g).pin_memory(), SIZE, T, return_last=True)
    got, last = ctx.colorize_videos_gray8([g.pin_memory()], [1], SIZE, T, return_last=True)
    assert torch.equal(got, ref) and torch.equal(last, ref_last)


# ------------------------------------------------------------------------------------------ geometries
GEOMETRIES = {
    "window-size": ((64, 96), SIZE),
    "crop-4to3-into-16to9": ((480, 640), (144, 256)),
    "zero-pad": ((40, 50), SIZE),
    "tiny-upscale": ((17, 23), SIZE),
    "odd-width": ((61, 95), SIZE),
}


@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_geometries(ctx, geom, source):
    (Hs, Ws), size = GEOMETRIES[geom]
    ctx.set_exemplar(make_lab(520, 1, size[0] // 2, size[1] // 2))
    _check(ctx, [_gray(521, 3, Hs, Ws)], [1], size=size, source=source, on_device=source)


# ------------------------------------------------------------------------------------------ call options
@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
def test_wls_off_first_last(ctx, source):
    K = [2, 1]
    ctx.set_exemplars(make_lab(530, 3, 32, 48))
    clips = [_gray(531, 3, 70, 120), _gray(532, 3, 33, 47)]
    _check(ctx, clips, K, source=source, wls=None, first_last=make_lab(533, 3, 32, 48))
    _check(ctx, clips, K, source=source, q=80, on_device=True, first_last=make_lab(534, 3, 32, 48))


@pytest.mark.parametrize("source", [False, True], ids=["window", "source"])
def test_chunks_continue_exactly(ctx, source):
    F_, a, K = 6, 4, [2, 1]
    ctx.set_exemplars(make_lab(540, 3, 32, 48))
    clips = [_gray(541, F_, 72, 120).pin_memory(), _gray(542, F_, 100, 90).pin_memory()]
    whole, last = ctx.colorize_videos_gray8(clips, K, SIZE, T, source_resolution=source, return_last=True)
    head, l1 = ctx.colorize_videos_gray8([f[:a] for f in clips], K, SIZE, T, source_resolution=source, return_last=True)
    tail, l2 = ctx.colorize_videos_gray8([f[a:] for f in clips], K, SIZE, T, source_resolution=source, first_last_lab=l1,
                                         return_last=True)
    if source:
        for w, h, t in zip(whole, head, tail):
            assert torch.equal(torch.cat([h, t], 1), w)
    else:
        assert torch.equal(torch.cat([head, tail], 1), whole)
    assert torch.equal(l2, last)


def test_device_memory_does_not_grow_with_F(ctx):
    K = [1, 2]
    ctx.set_exemplars(make_lab(550, 3, 32, 48))
    shapes = ((120, 200), (91, 91))

    def run(F_):
        clips = [_gray(551 + s, F_, *shapes[s]).pin_memory() for s in range(2)]
        ctx.colorize_videos_gray8(clips, K, SIZE, T)
        ctx.colorize_videos_gray8(clips, K, SIZE, T, source_resolution=True)
        ctx.colorize_videos_gray8(clips, K, SIZE, T, quality=75)
        torch.cuda.synchronize()

    run(4)
    free0, _ = torch.cuda.mem_get_info()
    run(12)
    free1, _ = torch.cuda.mem_get_info()
    assert free1 >= free0, (free0, free1)


# ------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(ctx):
    import dvc

    K, F_ = [1, 2], 2
    clips = [_gray(560, F_, 48, 80).pin_memory(), _gray(561, F_, 64, 96).pin_memory()]
    geoms = [(48, 80, 57, 96, 0, 0), (64, 96, 64, 96, 0, 0)]
    ctx.set_exemplars(make_lab(562, 3, 32, 48))
    stride = dvc.jpeg_max_bytes(*SIZE)
    pad = 64
    # sRGB outputs and JPEG slots, each with canary bytes after it
    srgb = [torch.full((k * F_ * SIZE[0] * SIZE[1] * 3 + pad,), CANARY, dtype=torch.uint8).pin_memory() for k in K]
    slots = [torch.full((k * F_ * stride + pad,), CANARY, dtype=torch.uint8).pin_memory() for k in K]
    sizes = torch.full((3 * F_,), -1, dtype=torch.int64).pin_memory()
    torch.cuda.synchronize()
    vp = ctypes.c_void_p

    def call(S=2, Kc=K, frames="clips", gm=geoms, q=0, source=0, out="auto", st=None, sz="auto", rows=None):
        o = (srgb if q == 0 else slots) if out == "auto" else out
        optrs = None if o is None else (vp * 2)(*[t.data_ptr() if t is not None else 0 for t in o])
        fr = None if frames is None else (vp * 2)(*[f.data_ptr() for f in clips])
        g = (ctypes.c_int * 12)(*[v for gg in gm for v in gg])
        st = (0 if q == 0 else stride) if st is None else st
        szp = (None if q == 0 else sizes) if sz == "auto" else sz
        return ctx.lib.dvc_colorize_videos_gray8(ctx.h, S, (ctypes.c_int * 2)(*Kc), fr, F_, g, SIZE[0], SIZE[1], T, vp(0), 1, 500.0, 4.0,
                                                 source, q, optrs, st, vp(szp.data_ptr() if szp is not None else 0), vp(0),
                                                 vp(torch.cuda.current_stream().cuda_stream))

    cases = [
        ({"frames": None}, -1), ({"out": None}, -1), ({"out": [srgb[0], None]}, -1), ({"gm": [geoms[0], (64, 96, 70, 96, 7, 0)]}, -2),
        ({"S": 0}, -1), ({"S": 9}, -1), ({"Kc": [2, 2]}, -2), ({"q": -1}, -1), ({"q": 101}, -1), ({"q": 75, "st": stride - 1}, -2),
        ({"q": 0, "st": stride}, -1), ({"q": 0, "sz": sizes}, -1), ({"q": 75, "sz": None}, -1),
        ({"q": 75, "out": [slots[0], None]}, -1),
    ]
    for kw, want in cases:
        for source in (0, 1):
            n = ctx.launch_count()
            assert call(source=source, **kw) == want, (kw, source)
            assert ctx.launch_count() == n, (kw, source)
    torch.cuda.synchronize()
    for t in srgb + slots:
        assert (t == CANARY).all()  # nothing was written
    assert (sizes == -1).all()
    # the context still works after the refusals, and writes nothing past its outputs
    assert call() == 0 and call(q=75, source=1) == 0
    for k, t in zip(K, srgb):
        assert (t[k * F_ * SIZE[0] * SIZE[1] * 3:] == CANARY).all()
    for k, t in zip(K, slots):
        assert (t[k * F_ * stride:] == CANARY).all()


# ------------------------------------------------------------------------------------------ Python
def test_python_shapes_and_types(ctx):
    import dvc

    ctx.set_exemplar(make_lab(570, 1, 32, 48))
    g = _gray(571, 2, 50, 70).cuda()
    a = ctx.colorize_videos_gray8([g], [1], SIZE, T)
    b = ctx.colorize_videos_gray8([g[..., None]], [1], SIZE, T)
    assert torch.equal(a, b)
    for bad in (g.to(torch.int16), _rgb(g), g[..., None].repeat(1, 1, 1, 4), g.float()):
        with pytest.raises(dvc.DvcError):
            ctx.colorize_videos_gray8([bad], [1], SIZE, T)


# ------------------------------------------------------------------------------------------ the folder tool
def _run_folder(tmp_path, name, dirs, refs, fmt, extra=()):
    out = tmp_path / name
    cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", *map(str, dirs), "--ref", *map(str, refs),
           "--out", str(out), "--seeded-weights", "--chunk", "3", "--image-size", str(SIZE[0]), str(SIZE[1]), "--format", fmt,
           "--jpeg-quality", "85", *extra]
    subprocess.run(cmd, check=True, cwd=str(tmp_path))
    return out


def _tree(root):
    files = {}
    for d, _, names in os.walk(root):
        for n in names:
            p = os.path.join(d, n)
            files[os.path.relpath(p, root)] = open(p, "rb").read()
    return files


def test_colorize_folder_gray_pngs_equal_rgb_pngs(tmp_path):
    """A folder of mode-"L" PNGs (grey path) and the same frames saved as RGB PNGs (colour path) give identical files; so does a
    two-clip run that mixes a grey folder with a colour folder (the grey chunks expanded on the host)."""
    from PIL import Image

    lens, shapes = (5, 4), ((90, 100), (64, 96))
    gdirs, cdirs = [], []
    for s in range(2):
        fr = _gray(580 + s, lens[s], *shapes[s]).numpy()
        gd, cd = tmp_path / "gray" / f"clip{s}", tmp_path / "rgb" / f"clip{s}"
        gd.mkdir(parents=True), cd.mkdir(parents=True)
        for t in range(lens[s]):
            img = Image.fromarray(fr[t])  # a 2-D uint8 array: mode "L"
            assert img.mode == "L"
            img.save(gd / f"f{t + 1}.png")
            img.convert("RGB").save(cd / f"f{t + 1}.png")
        gdirs.append(gd), cdirs.append(cd)
    ref = tmp_path / "ref.png"
    Image.fromarray(np.random.default_rng(590).integers(0, 256, (70, 100, 3), dtype=np.uint8)).save(ref)
    colour = tmp_path / "colour"  # a colour clip for the mixed run
    colour.mkdir()
    rng = np.random.default_rng(591)
    for t in range(3):
        Image.fromarray(rng.integers(0, 256, (80, 120, 3), dtype=np.uint8)).save(colour / f"f{t + 1}.png")
    for fmt, extra in (("png", []), ("jpg", []), ("png", ["--source-resolution"]), ("jpg", ["--source-resolution"])):
        tag = fmt + str(len(extra))
        a = _tree(_run_folder(tmp_path, "g" + tag, [gdirs[0]], [ref], fmt, extra))
        b = _tree(_run_folder(tmp_path, "c" + tag, [cdirs[0]], [ref], fmt, extra))
        assert len(a) == lens[0] and a == b, tag
    for fmt in ("png", "jpg"):
        a = _tree(_run_folder(tmp_path, "gm" + fmt, [gdirs[1], colour], [ref, ref], fmt))
        b = _tree(_run_folder(tmp_path, "cm" + fmt, [cdirs[1], colour], [ref, ref], fmt))
        assert len(a) == lens[1] + 3 and a == b, fmt
