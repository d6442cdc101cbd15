"""The reference's test.py:29-125 data flow on the device, using only libdvc entry points (no reference code):

    decoded uint8 frames -> CenterPad + CenterCrop to --image_size (dvc_resize_antialias_crop_rgb8) -> Lab
    (dvc_rgb8_to_lab) -> 1/2 resolution (dvc_resize_half) -> exemplar features once (dvc_set_exemplar) -> per frame
    VGG19 / WarpNet / correlation / ColorVidNet with the recurrence kept on the device (dvc_colorize_clip) -> ab x2 * 1.25
    (dvc_upsample2_scaled) -> WLS filter guided by the full-resolution luminance (dvc_l_to_guide8 + dvc_fgs_filter,
    test.py:105-112) -> sRGB uint8 (dvc_lab_to_rgb8) -> PNG files

    python tools/colorize_folder.py --clip frames/ --ref exemplar.png --out out/ \
        --vgg vgg19_conv.pth --warp nonlocal_net_iter_76000.pth --color colornet_iter_76000.pth

Several --ref images (test.py:168-181 colorizes the clip once per reference) take one pass: dvc_set_exemplars +
dvc_colorize_clip_exemplars run the exemplar-independent half of every frame once, and each exemplar's frames go to
--out/<exemplar file name>/.

What the reference does and this script does not: the AVI writer (folder2vid).  Image decode / encode stays on the host
(PIL), as in the reference.  Without checkpoints (none ship with the reference tree) pass --seeded-weights to run the
pipeline on the seeded random weights of dvc/synth.py (useful as a smoke run only).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))

import numpy as np
import torch


def load_rgb8(path):
    from PIL import Image

    return torch.from_numpy(np.asarray(Image.open(path).convert("RGB"), dtype=np.uint8).copy())


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
    args = ap.parse_args()

    import dvc
    from dvc.synth import make_state_dict

    ctx = dvc.get_context(0)
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
    # test.py:44-46: CenterPad(image_size) + CenterCrop(image_size), anti-aliased resize on the device
    frames = torch.stack([ctx.centerpad_rgb8(load_rgb8(os.path.join(args.clip, n)).cuda(), (H, W)) for n in names])  # [F,H,W,3]
    refs = torch.stack([ctx.centerpad_rgb8(load_rgb8(r).cuda(), (H, W)) for r in args.ref])  # [K,H,W,3]
    F_ = frames.shape[0]

    lab_large = ctx.rgb8_to_lab(frames)                      # [F,3,H,W], centred L   (test.py:44-45)
    lab = ctx.resize_half(lab_large)                         # test.py:71
    L = lab[:, 0:1].contiguous()
    if len(args.ref) == 1:
        ctx.set_exemplar(ctx.resize_half(ctx.rgb8_to_lab(refs)))  # test.py:57-66
        abs_ = [ctx.colorize_clip(L, args.temperature)]           # test.py:68-96, recurrence on the device
        outs = [args.out]
    else:  # every exemplar's recurrence in one pass over the clip
        ctx.set_exemplars(ctx.resize_half(ctx.rgb8_to_lab(refs)))
        abs_ = list(ctx.colorize_clip_exemplars(L, args.temperature))
        outs = [os.path.join(args.out, os.path.splitext(os.path.basename(r))[0]) for r in args.ref]
        if len(set(outs)) != len(outs):
            raise SystemExit("--ref: the exemplar file names must differ (they name the output folders)")

    from PIL import Image

    guide_l = lab_large[:, 0:1].contiguous()                 # the full-resolution luminance guides every exemplar's result
    for ab, out_dir in zip(abs_, outs):
        ab_large = ctx.upsample2_scaled(ab, 1.25)            # test.py:100-102
        if not args.no_wls:                                  # test.py:105-112
            for t in range(F_):
                guide = ctx.l_to_guide8(lab_large[t, 0])
                ab_large[t] = ctx.fgs_filter(guide, ab_large[t], args.lambda_value, args.sigma_color)
        rgb = ctx.lab_to_rgb8(guide_l, ab_large).cpu().numpy()  # test.py:116-119
        os.makedirs(out_dir, exist_ok=True)
        for n, img in zip(names, rgb):
            Image.fromarray(img).save(os.path.join(out_dir, os.path.splitext(n)[0] + ".png"))
        print(f"{F_} frames -> {out_dir}")


if __name__ == "__main__":
    main()
