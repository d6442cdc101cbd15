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

What the reference does and this script does not: the AVI writer (folder2vid).  Image decode / encode stays on the host
(PIL), as in the reference.  Without checkpoints (none ship with the reference tree) pass --seeded-weights to run the
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


def save_png(img, path):
    from PIL import Image

    Image.fromarray(img).save(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clip", required=True, help="folder of frames (sorted by the digits in the file names, test.py:41)")
    ap.add_argument("--ref", required=True, nargs="+",
                    help="exemplar image(s); with several (at most 8), one pass colorizes the clip against each and writes "
                         "--out/<exemplar name>/ (test.py:168-181 loops over a folder of references)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--vgg"), ap.add_argument("--warp"), ap.add_argument("--color")
    ap.add_argument("--seeded-weights", action="store_true")
    ap.add_argument("--temperature", type=float, default=1e-10)  # test.py:94
    ap.add_argument("--image-size", type=int, nargs=2, default=[216 * 2, 384 * 2], help="test.py:132")
    ap.add_argument("--no-wls", action="store_true", help="skip the Fast Global Smoother (test.py:31 wls_filter_on)")
    ap.add_argument("--lambda-value", type=float, default=500.0)  # test.py:32
    ap.add_argument("--sigma-color", type=float, default=4.0)    # test.py:33
    ap.add_argument("--chunk", type=int, default=32, help="frames per device call (bounds device and host memory)")
    ap.add_argument("--workers", type=int, default=min(8, os.cpu_count() or 1), help="decode / encode threads each")
    ap.add_argument("--fast", action="store_true",
                    help="one MMA per convolution product (dvc.MATH_FP16X1: 11-bit conv operands, the precision of the "
                         "reference's cuDNN convolutions on a GPU) instead of the fp32-class default")
    args = ap.parse_args()
    if args.chunk < 1:
        raise SystemExit("--chunk must be >= 1")

    import dvc
    from dvc.synth import make_state_dict

    ctx = dvc.get_context(0)
    if args.fast:
        ctx.set_math(conv=dvc.MATH_FP16X1)
    for net, key, path in ((dvc.NET_VGG, "vgg", args.vgg), (dvc.NET_WARP, "warp", args.warp), (dvc.NET_COLOR, "color", args.color)):
        if path:
            ctx.set_weights(net, torch.load(path, map_location="cpu"))
        elif args.seeded_weights:
            ctx.set_weights(net, make_state_dict(key, seed=0))
        else:
            raise SystemExit(f"--{key} checkpoint missing (or pass --seeded-weights)")

    names = sorted(os.listdir(args.clip), key=lambda f: int("".join(filter(str.isdigit, f)) or -1))
    H, W = args.image_size
    if H % 16 or W % 32:
        raise SystemExit("--image-size must have H % 16 == 0 and W % 32 == 0 (the networks run at half of it)")
    # test.py:44-46 + 57-66: CenterPad(image_size) + CenterCrop(image_size) of the exemplar(s), Lab, 1/2, features once
    refs = torch.stack([ctx.centerpad_rgb8(torch.from_numpy(load_rgb8(r).copy()).cuda(), (H, W)) for r in args.ref])  # [K,H,W,3]
    if len(args.ref) == 1:
        ctx.set_exemplar(ctx.resize_half(ctx.rgb8_to_lab(refs)))
        outs = [args.out]
    else:  # every exemplar's recurrence in one pass over the clip
        ctx.set_exemplars(ctx.resize_half(ctx.rgb8_to_lab(refs)))
        outs = [os.path.join(args.out, os.path.splitext(os.path.basename(r))[0]) for r in args.ref]
        if len(set(outs)) != len(outs):
            raise SystemExit("--ref: the exemplar file names must differ (they name the output folders)")
    for d in outs:
        os.makedirs(d, exist_ok=True)
    wls = None if args.no_wls else (args.lambda_value, args.sigma_color)
    K, C = len(outs), args.chunk

    decode, encode = ThreadPoolExecutor(args.workers), ThreadPoolExecutor(args.workers)
    pending = collections.deque()  # (name, decode future), at most two chunks ahead of the device
    todo = iter(names)

    def read_ahead():
        for n in todo:
            pending.append((n, decode.submit(load_rgb8, os.path.join(args.clip, n))))
            if len(pending) >= 2 * C:
                break

    def next_chunk():
        """Up to C consecutive decoded frames of one source size: [(name, array)]."""
        read_ahead()
        chunk = []
        while pending and len(chunk) < C:
            img = pending[0][1].result()
            if chunk and img.shape != chunk[0][1].shape:
                break
            chunk.append((pending.popleft()[0], img))
            read_ahead()
        return chunk

    ring_in = [None, None]   # pinned [C,Hs,Ws,3] frame chunks
    ring_out = [None, None]  # pinned [K,C,H,W,3] result chunks and the encodes still reading them
    writes = [[], []]
    last, done, i = None, 0, 0
    while True:
        chunk = next_chunk()
        if not chunk:
            break
        n, shape, slot = len(chunk), chunk[0][1].shape, i & 1
        if ring_in[slot] is None or tuple(ring_in[slot].shape[1:]) != shape:
            ring_in[slot] = torch.empty((C,) + shape, dtype=torch.uint8).pin_memory()
        for t, (_, img) in enumerate(chunk):
            ring_in[slot][t].copy_(torch.from_numpy(img))
        for f in writes[slot]:  # the encodes of chunk i-2 still read this output slot
            f.result()
        if ring_out[slot] is None or ring_out[slot].shape[1] != n:
            ring_out[slot] = torch.empty(K, n, H, W, 3, dtype=torch.uint8).pin_memory()
        out, last = ctx.colorize_video_rgb8(ring_in[slot][:n], (H, W), args.temperature, first_last_lab=last, wls=wls,
                                            out=ring_out[slot], return_last=True)
        arr = out.numpy()
        writes[slot] = [encode.submit(save_png, arr[k, t], os.path.join(outs[k], os.path.splitext(name)[0] + ".png"))
                        for k in range(K) for t, (name, _) in enumerate(chunk)]
        done += n
        i += 1
    for ws in writes:
        for f in ws:
            f.result()
    decode.shutdown(), encode.shutdown()
    for d in outs:
        print(f"{done} frames -> {d}")


if __name__ == "__main__":
    main()
