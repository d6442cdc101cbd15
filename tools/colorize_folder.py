"""The reference's test.py:29-125 data flow on the device, using only libdvc entry points (no reference code):

    decoded uint8 frames -> CenterPad + CenterCrop to --image_size -> Lab -> 1/2 resolution -> exemplar features once
    (dvc_set_exemplar) -> per frame VGG19 / WarpNet / correlation / ColorVidNet with the recurrence kept on the device
    -> ab x2 * 1.25 -> WLS filter guided by the full-resolution luminance (test.py:105-112) -> sRGB uint8 -> PNG files

    python tools/colorize_folder.py --clip frames/ --ref exemplar.png --out out/ \
        --vgg vgg19_conv.pth --warp nonlocal_net_iter_76000.pth --color colornet_iter_76000.pth

The frames stream through dvc_colorize_video_rgb8 in chunks of --chunk frames (one call per chunk, the recurrence state
carried from chunk to chunk, so the result is that of one call over the whole clip): a thread pool decodes ahead into a
ring of pinned chunk buffers and another encodes the PNGs while the next chunk runs, so device and host memory are bounded
by the chunk size, not by the clip length.  Consecutive frames of one source size share a chunk.

Several --ref images (test.py:168-181 colorizes the clip once per reference) take one pass: dvc_set_exemplars and the
exemplar-independent half of every frame computed once; each exemplar's frames go to --out/<exemplar file name>/.

An entry of --ref may be a folder: its images, sorted by name (test.py's listing of ref_path), are that entry's exemplars.
A single --clip with a --ref folder is the several-reference pass above.

Several --clip folders (at most 8) take one pass too, with one --ref entry per clip, a file or a folder: clip s against the
K_s exemplars of --ref s, at most 8 exemplars in all.  A clip with one exemplar writes to --out/<clip folder name>/, a clip
with several to --out/<clip folder name>/<exemplar name>/.  Every call (dvc_colorize_videos_exemplars_rgb8 with the per-clip
counts K_s, after dvc_set_exemplars of the clips' exemplars in clip order) takes the same number of frames n from each clip
that has frames left: n = min(--chunk, the run of frames of one source size each such clip has next).  When a clip runs
out, it leaves with its rows: the others continue with dvc_set_exemplars of their exemplars and their rows of the previous
call's last_lab_out.

--source-resolution writes every frame at its source resolution instead of --image-size: the networks still run at
--image-size, and every call is dvc_colorize_videos_source_rgb8 (same chunks, exemplars and recurrence), which resamples the
network's colour onto the source frame, WLS-filters it against the source frame's own luminance and keeps that luminance.
The PNGs cover the part of the frame the window covers (dvc_source_footprint): the whole frame unless CenterPad crops it.

--format jpg writes <frame>.jpg files instead of PNGs, encoded on the device: every call is dvc_colorize_videos_jpeg (window or,
with --source-resolution, source output; same chunks, exemplars and recurrence), whose files are byte-equal to Pillow's
save(f, "JPEG", quality=--jpeg-quality) of the frames the PNG path writes.  Only the compressed files cross PCIe, into a ring of
pinned slots of dvc_jpeg_max_bytes each (bounded by the chunk size), and the writer threads only write bytes.

Grey frames (mode "L" images) are decoded as one byte per pixel.  A call whose clips are all grey is
dvc_colorize_videos_gray8 (every --format, with or without --source-resolution), which uploads and resizes a third of the
bytes and writes what the sRGB calls write for the frames converted to RGB; a call that mixes grey and colour clips expands
the grey frames to RGB on the host.  A folder that changes between grey and colour splits its chunks there, like a change of
size.  Output names and bytes do not depend on which path a frame took.

What the reference does and this script does not: the AVI writer (folder2vid); tools/colorize_y4m.py colorizes a YUV4MPEG2
stream instead, which ffmpeg decodes from and encodes to any container.  Image decode stays on the host (PIL), as in
the reference, and so does PNG encoding.  Without checkpoints (none ship with the reference tree) pass --seeded-weights to run the
pipeline on the seeded random weights of dvc/synth.py (useful as a smoke run only).
"""
import argparse
import collections
import os
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))

import numpy as np
import torch


def load_rgb8(path):
    from PIL import Image

    return np.asarray(Image.open(path).convert("RGB"), dtype=np.uint8)


def load_frame(path):
    """A mode-"L" (8-bit grey) image as [H,W], anything else converted to sRGB [H,W,3]."""
    from PIL import Image

    img = Image.open(path)
    return np.asarray(img if img.mode == "L" else img.convert("RGB"), dtype=np.uint8)


def save_png(img, path):
    from PIL import Image

    Image.fromarray(img).save(path)


def save_bytes(data, path):
    with open(path, "wb") as f:
        f.write(data)


def set_weights(ctx, vgg, warp, color, seeded):
    """The three networks' weights from checkpoint files, or the seeded random weights of dvc/synth.py where a path is missing and
    `seeded` is set."""
    import dvc
    from dvc.synth import make_state_dict

    for net, key, path in ((dvc.NET_VGG, "vgg", vgg), (dvc.NET_WARP, "warp", warp), (dvc.NET_COLOR, "color", color)):
        if path:
            ctx.set_weights(net, torch.load(path, map_location="cpu"))
        elif seeded:
            ctx.set_weights(net, make_state_dict(key, seed=0))
        else:
            raise SystemExit(f"--{key} checkpoint missing (or pass --seeded-weights)")


def exemplars_lab(ctx, paths, size):
    """test.py:44-46 + 57-66: CenterPad(size) + CenterCrop(size) of the exemplar image files, Lab, 1/2 resolution:
    [K,3,size[0]/2,size[1]/2] on the device, ready for dvc_set_exemplar(s)."""
    refs = torch.stack([ctx.centerpad_rgb8(torch.from_numpy(load_rgb8(r).copy()).cuda(), tuple(size)) for r in paths])  # [K,H,W,3]
    return ctx.resize_half(ctx.rgb8_to_lab(refs))


class Source:
    """One clip folder: its frame names in order and a queue of decodes running ahead of the device."""

    def __init__(self, folder, decode, chunk):
        self.folder, self.decode, self.chunk = folder, decode, chunk
        names = sorted(os.listdir(folder), key=lambda f: int("".join(filter(str.isdigit, f)) or -1))
        self.todo = iter(names)
        self.pending = collections.deque()  # (name, decode future), at most two chunks ahead of the device

    def read_ahead(self):
        for n in self.todo:
            self.pending.append((n, self.decode.submit(load_frame, os.path.join(self.folder, n))))
            if len(self.pending) >= 2 * self.chunk:
                break

    def run(self):
        """Number of decoded frames of one source shape (size and grey / colour) at the front, up to the chunk size (0: the clip
        is done)."""
        self.read_ahead()
        n = 0
        while n < min(self.chunk, len(self.pending)):
            if n and self.pending[n][1].result().shape != self.pending[0][1].result().shape:
                break
            n += 1
        return n

    def take(self, n):
        chunk = [(name, f.result()) for name, f in (self.pending.popleft() for _ in range(n))]
        self.read_ahead()
        return chunk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clip", required=True, nargs="+",
                    help="folder(s) of frames (sorted by the digits in the file names, test.py:41); with several (at most 8), "
                         "one pass colorizes them all, each against its own --ref, into --out/<clip folder name>/")
    ap.add_argument("--ref", required=True, nargs="+",
                    help="exemplar image(s) or folder(s) of them (sorted by name); with several images (at most 8), one pass "
                         "colorizes the clip against each and writes --out/<exemplar name>/ (test.py:168-181 loops over a folder "
                         "of references); with several --clip folders, one entry (a file or a folder) per clip, and a clip with "
                         "several exemplars writes --out/<clip folder name>/<exemplar name>/")
    ap.add_argument("--out", required=True)
    ap.add_argument("--vgg"), ap.add_argument("--warp"), ap.add_argument("--color")
    ap.add_argument("--seeded-weights", action="store_true")
    ap.add_argument("--temperature", type=float, default=1e-10)  # test.py:94
    ap.add_argument("--image-size", type=int, nargs=2, default=[216 * 2, 384 * 2], help="test.py:132")
    ap.add_argument("--no-wls", action="store_true", help="skip the Fast Global Smoother (test.py:31 wls_filter_on)")
    ap.add_argument("--lambda-value", type=float, default=500.0)  # test.py:32
    ap.add_argument("--sigma-color", type=float, default=4.0)    # test.py:33
    ap.add_argument("--chunk", type=int, default=32, help="frames per clip and device call (bounds device and host memory)")
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1), help="decode / encode threads each")
    ap.add_argument("--fast", action="store_true",
                    help="one MMA per convolution product (dvc.MATH_FP16X1: 11-bit conv operands, the precision of the "
                         "reference's cuDNN convolutions on a GPU) instead of the fp32-class default")
    ap.add_argument("--source-resolution", action="store_true",
                    help="write every frame at its source resolution (the part of the frame the --image-size window covers): the "
                         "network's colour resampled onto the source frame and WLS-filtered against its own luminance")
    ap.add_argument("--format", choices=("png", "jpg"), default="png",
                    help="png: Pillow on the host; jpg: baseline JPEG encoded on the device (Pillow's bytes at --jpeg-quality)")
    ap.add_argument("--jpeg-quality", type=int, default=75, help="JPEG quality in [1, 100] (75: Pillow's default)")
    args = ap.parse_args()
    if not 1 <= args.jpeg_quality <= 100:
        raise SystemExit("--jpeg-quality must be in [1, 100]")
    if args.chunk < 1:
        raise SystemExit("--chunk must be >= 1")
    S = len(args.clip)
    if S > 8:
        raise SystemExit("--clip: at most 8 folders in one pass")
    if S > 1 and len(args.ref) != S:
        raise SystemExit("--ref: with several --clip folders, give one entry (an image or a folder of images) per clip")
    # each --ref entry: an image, or a folder whose images, sorted by name, are the entry's exemplars
    ref_paths = [sorted(os.path.join(r, f) for f in os.listdir(r) if os.path.isfile(os.path.join(r, f))) if os.path.isdir(r) else [r]
                 for r in args.ref]
    if any(not p for p in ref_paths):
        raise SystemExit("--ref: an empty folder")
    if S == 1:
        ref_paths = [[p for ps in ref_paths for p in ps]]  # one clip: every image is one of its exemplars
    counts = [len(p) for p in ref_paths]
    if sum(counts) > 8:
        raise SystemExit(f"--ref: at most 8 exemplars in one pass, got {sum(counts)}")

    import dvc
    from dvc.prepost import centerpad_geometry

    ctx = dvc.get_context(0)
    if args.fast:
        ctx.set_math(conv=dvc.MATH_FP16X1)
    set_weights(ctx, args.vgg, args.warp, args.color, args.seeded_weights)

    H, W = args.image_size
    if H % 16 or W % 32:
        raise SystemExit("--image-size must have H % 16 == 0 and W % 32 == 0 (the networks run at half of it)")
    ref_lab = [exemplars_lab(ctx, p, (H, W)) for p in ref_paths]  # per clip; the exemplar features are computed once

    def stem(path):
        return os.path.splitext(os.path.basename(path))[0]

    if S > 1:  # clip s against its K_s exemplars, every row's recurrence in one pass
        ctx.set_exemplars(torch.cat(ref_lab))
        outs = []  # per clip: the output folder of each of its exemplars
        for d, paths in zip(args.clip, ref_paths):
            base = os.path.join(args.out, os.path.basename(os.path.normpath(d)))
            outs.append([base] if len(paths) == 1 else [os.path.join(base, stem(p)) for p in paths])
        flat = [d for ds in outs for d in ds]
        if len(set(flat)) != len(flat):
            raise SystemExit("--clip / --ref: the output folders must differ (clip folder names, and the exemplar file names of a clip)")
    elif counts[0] == 1:
        ctx.set_exemplar(ref_lab[0])
        outs = [[args.out]]
    else:  # every exemplar's recurrence in one pass over the clip
        ctx.set_exemplars(ref_lab[0])
        outs = [[os.path.join(args.out, stem(r)) for r in ref_paths[0]]]
        if len(set(outs[0])) != len(outs[0]):
            raise SystemExit("--ref: the exemplar file names must differ (they name the output folders)")
    for ds in outs:
        for d in ds:
            os.makedirs(d, exist_ok=True)
    wls = None if args.no_wls else (args.lambda_value, args.sigma_color)
    C = args.chunk

    decode, encode = ThreadPoolExecutor(args.workers), ThreadPoolExecutor(args.workers)
    sources = [Source(d, decode, C) for d in args.clip]
    active = list(range(S))  # clips with frames left; a call's output and last_lab_out hold their rows, clip by clip
    ring_in = [[None] * S, [None] * S]  # pinned [C,Hs,Ws,3] frame chunks per clip
    ring_out = [None, None]  # pinned [rows,n,H,W,3] result chunks and the encodes still reading them
    writes = [[], []]
    last, done, i = None, [0] * S, 0
    while True:
        runs = [sources[s].run() for s in active]
        keep = [j for j, r in enumerate(runs) if r > 0]
        if not keep:
            break
        if len(keep) < len(active):  # a clip ran out of frames: the others continue with their exemplars and states
            stay = [active[j] for j in keep]
            if last is not None:  # the rows of the clips that stay
                last = last[[r for r, s in enumerate(s for s in active for _ in range(counts[s])) if s in stay]]
            active, runs = stay, [runs[j] for j in keep]
            ctx.set_exemplars(torch.cat([ref_lab[s] for s in active]))
        n, slot = min(runs), i & 1
        chunks = [sources[s].take(n) for s in active]
        # grey frames ([H,W], mode "L") go up one byte per pixel when every clip of the call is grey; beside colour clips they
        # are expanded to (g, g, g) here, which is what the grey call computes anyway
        gray = all(chunk[0][1].ndim == 2 for chunk in chunks)
        for s, chunk in zip(active, chunks):
            shape = chunk[0][1].shape[:2] + (() if gray else (3,))
            if ring_in[slot][s] is None or tuple(ring_in[slot][s].shape[1:]) != shape:
                ring_in[slot][s] = torch.empty((C,) + shape, dtype=torch.uint8).pin_memory()
            for t, (_, img) in enumerate(chunk):
                src = torch.from_numpy(img)
                ring_in[slot][s][t].copy_(src if src.dim() == len(shape) else src[..., None])  # [H,W,1] broadcasts to [H,W,3]
        for f in writes[slot]:  # the encodes of chunk i-2 still read this output slot
            f.result()
        rows = sum(counts[s] for s in active)
        ins, ks = [ring_in[slot][s][:n] for s in active], [counts[s] for s in active]
        if args.format == "jpg":  # the device encodes: one [K_s,n,stride] slot buffer per clip, stride = the largest frame's bound
            sizes_ = [(H, W)]
            if args.source_resolution:
                for chunk in chunks:
                    Hs, Ws = chunk[0][1].shape[:2]
                    sizes_.append(dvc.source_footprint(Hs, Ws, *centerpad_geometry(Hs, Ws, (H, W)), H, W)[2:])
            stride = max(dvc.jpeg_max_bytes(h, w) for h, w in sizes_)
            shapes = [(counts[s], n, stride) for s in active]
            if ring_out[slot] is None or [tuple(o.shape) for o in ring_out[slot][0]] != shapes:
                ring_out[slot] = ([torch.empty(shp, dtype=torch.uint8).pin_memory() for shp in shapes],
                                  torch.empty(rows, n, dtype=torch.int64).pin_memory())
            kw = dict(first_last_lab=last, wls=wls, out=ring_out[slot][0], sizes=ring_out[slot][1], return_last=True)
            if gray:
                slots, sizes, last = ctx.colorize_videos_gray8(ins, ks, (H, W), args.temperature, source_resolution=args.source_resolution,
                                                               quality=args.jpeg_quality, **kw)
            else:
                slots, sizes, last = ctx.colorize_videos_jpeg(ins, ks, (H, W), args.jpeg_quality, args.source_resolution, args.temperature,
                                                              **kw)
            files = dvc.jpeg_files(slots, sizes)
            dests = [(d, chunk) for s, chunk in zip(active, chunks) for d in outs[s]]
            writes[slot] = [encode.submit(save_bytes, files[r][t], os.path.join(d, os.path.splitext(name)[0] + ".jpg"))
                            for r, (d, chunk) in enumerate(dests) for t, (name, _) in enumerate(chunk)]
        elif args.source_resolution:  # every clip's frames at its footprint, one [K_s,n,h,w,3] buffer per clip
            shapes = []
            for chunk in chunks:
                Hs, Ws = chunk[0][1].shape[:2]
                _, _, h, w = dvc.source_footprint(Hs, Ws, *centerpad_geometry(Hs, Ws, (H, W)), H, W)
                shapes.append((h, w))
            shapes = [(counts[s], n, h, w, 3) for s, (h, w) in zip(active, shapes)]
            if ring_out[slot] is None or [tuple(o.shape) for o in ring_out[slot]] != shapes:
                ring_out[slot] = [torch.empty(shp, dtype=torch.uint8).pin_memory() for shp in shapes]
            kw = dict(first_last_lab=last, wls=wls, out=ring_out[slot], return_last=True)
            if gray:
                res, last = ctx.colorize_videos_gray8(ins, ks, (H, W), args.temperature, source_resolution=True, **kw)
            else:
                res, last = ctx.colorize_videos_source_rgb8(ins, ks, (H, W), args.temperature, **kw)
            arr = [row for o in res for row in o.numpy()]
            dests = [(d, chunk) for s, chunk in zip(active, chunks) for d in outs[s]]
        elif gray:  # window output of grey clips, one or several
            if ring_out[slot] is None or tuple(ring_out[slot].shape[:2]) != (rows, n):
                ring_out[slot] = torch.empty(rows, n, H, W, 3, dtype=torch.uint8).pin_memory()
            out, last = ctx.colorize_videos_gray8(ins, ks, (H, W), args.temperature, first_last_lab=last, wls=wls, out=ring_out[slot],
                                                  return_last=True)
            dests = [(d, chunk) for s, chunk in zip(active, chunks) for d in outs[s]]
            arr = out.numpy()
        elif S == 1:
            if ring_out[slot] is None or tuple(ring_out[slot].shape[:2]) != (rows, n):
                ring_out[slot] = torch.empty(rows, n, H, W, 3, dtype=torch.uint8).pin_memory()
            out, last = ctx.colorize_video_rgb8(ring_in[slot][0][:n], (H, W), args.temperature, first_last_lab=last, wls=wls,
                                                out=ring_out[slot], return_last=True)
            dests = [(d, chunks[0]) for d in outs[0]]
            arr = out.numpy()
        else:
            if ring_out[slot] is None or tuple(ring_out[slot].shape[:2]) != (rows, n):
                ring_out[slot] = torch.empty(rows, n, H, W, 3, dtype=torch.uint8).pin_memory()
            out, last = ctx.colorize_videos_exemplars_rgb8([ring_in[slot][s][:n] for s in active], [counts[s] for s in active], (H, W),
                                                           args.temperature, first_last_lab=last, wls=wls, out=ring_out[slot],
                                                           return_last=True)
            dests = [(d, chunk) for s, chunk in zip(active, chunks) for d in outs[s]]
            arr = out.numpy()
        if args.format == "png":
            writes[slot] = [encode.submit(save_png, arr[r][t],os.path.join(d, os.path.splitext(name)[0] + ".png"))
                            for r, (d, chunk) in enumerate(dests) for t, (name, _) in enumerate(chunk)]
        for s in active:
            done[s] += n
        i += 1
    for ws in writes:
        for f in ws:
            f.result()
    decode.shutdown(), encode.shutdown()
    for s, ds in enumerate(outs):
        for d in ds:
            print(f"{done[s]} frames -> {d}")


if __name__ == "__main__":
    main()
