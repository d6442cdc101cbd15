"""Frames per second of test.py's whole inference path (ingest, networks, post-processing) on the GPU, two ways:

  (a) compose  the stand-alone entry points phase after phase over the clip, as tools/colorize_folder.py did before it
               streamed: every frame uploaded and CenterPad-resized, Lab and 1/2 for the whole clip, dvc_colorize_clip(_exemplars)
               on device-resident L, ab x2 * 1.25, one FGS call per frame and exemplar, lab_to_rgb8, one download
  (b) video    one dvc_colorize_video_rgb8 call over the clip

Workload: synthetic 720x1280 uint8 sources resident in pinned host memory, CenterPad'ed to 432x768 (test.py's default
image size; the networks run at 216x384), seeded weights, WLS on (lambda 500, sigma 4), K = 1 and K = 3 exemplars.
Method: after a warm-up, windows of at least --window seconds alternate between (a) and (b); each window runs whole clips
of --frames frames and ends with a device synchronisation; the rate is the median over --reps windows.  Device memory:
the drop of torch.cuda.mem_get_info's free memory over a method's first clip (library workspaces, and for (a) the
clip-sized tensors the caching allocator keeps), measured for (b) first.  Bytes over PCIe per frame are counted from the
shapes (the uint8 source up, K sRGB frames down), not measured.

    python tools/video_bench.py [--frames 16] [--window 1.0] [--reps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))

import numpy as np
import torch

HS, WS, SIZE = 720, 1280, (432, 768)
T = 1e-10


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl or "unknown"


def synthetic_frames(F):
    rng = np.random.default_rng(0)
    coarse = (rng.random((F, HS // 16 + 1, WS // 16 + 1, 3)) * 255).astype(np.int16)
    img = np.kron(coarse, np.ones((1, 16, 16, 1), np.int16))[:, :HS, :WS]
    img = np.clip(img + rng.integers(-12, 13, img.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    return torch.from_numpy(img).pin_memory()


def compose(ctx, frames, K):
    """(a): the stand-alone entry points, phase after phase over the whole clip (device memory O(F))."""
    crops = torch.stack([ctx.centerpad_rgb8(f.cuda(non_blocking=True), SIZE) for f in frames])
    lab_large = ctx.rgb8_to_lab(crops)
    L = ctx.resize_half(lab_large)[:, 0:1].contiguous()
    abs_ = ctx.colorize_clip(L, T)[None] if K == 1 else ctx.colorize_clip_exemplars(L, T)
    l_large = lab_large[:, 0:1].contiguous()
    outs = []
    for ab in abs_:
        ab_large = ctx.upsample2_scaled(ab, 1.25)
        for t in range(frames.shape[0]):
            ab_large[t] = ctx.fgs_filter(ctx.l_to_guide8(lab_large[t, 0]), ab_large[t], 500.0, 4.0)
        outs.append(ctx.lab_to_rgb8(l_large, ab_large).cpu())
    return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("video_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    F_ = args.frames
    frames = synthetic_frames(F_)
    rows = []
    for K in (1, 3):
        IB = make_lab(40, K, SIZE[0] // 2, SIZE[1] // 2)
        ctx.set_exemplar(IB) if K == 1 else ctx.set_exemplars(IB)
        out = torch.empty(K, F_, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory()
        methods = {"video": lambda: ctx.colorize_video_rgb8(frames, SIZE, T, out=out), "compose": lambda: compose(ctx, frames, K)}
        mem = {}
        for m in ("video", "compose"):  # first clip of each: the memory it takes, and the warm-up
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            free0 = torch.cuda.mem_get_info()[0]
            methods[m]()
            torch.cuda.synchronize()
            mem[m] = free0 - torch.cuda.mem_get_info()[0]
        # the two agree byte for byte (tests/test_gpu_video.py); checked here on the timed workload too
        ref = compose(ctx, frames, K)
        methods["video"]()
        same = all(torch.equal(out[k], ref[k]) for k in range(K))
        rates = {"compose": [], "video": []}
        for _ in range(args.reps):
            for m in ("compose", "video"):
                n, t0 = 0, time.perf_counter()
                while True:
                    methods[m]()
                    torch.cuda.synchronize()
                    n += F_
                    dt = time.perf_counter() - t0
                    if dt >= args.window:
                        break
                rates[m].append(n / dt)
        for m in ("compose", "video"):
            rows.append({"K": K, "method": m, "frames_per_s": statistics.median(rates[m]), "windows_fps": rates[m],
                         "device_mem_MB": mem[m] / 2**20, "h2d_bytes_per_frame": HS * WS * 3,
                         "d2h_bytes_per_frame": K * SIZE[0] * SIZE[1] * 3, "byte_identical": same})
    print(f"card: {name}, power limit {power}; {HS}x{WS} -> {SIZE[0]}x{SIZE[1]}, clips of {F_} frames, WLS on, "
          f"median of {args.reps} windows >= {args.window} s")
    print("| K | method | frames/s | device memory growth over the first clip (MB) | H2D B/frame | D2H B/frame |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['K']} | {r['method']} | {r['frames_per_s']:.1f} | {r['device_mem_MB']:.0f} | {r['h2d_bytes_per_frame']} "
              f"| {r['d2h_bytes_per_frame']} |")
    print(json.dumps({"card": name, "power_limit": power, "frames": F_, "rows": rows}))


if __name__ == "__main__":
    main()
