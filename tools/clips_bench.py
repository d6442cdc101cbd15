"""Aggregate frames per second of test.py's whole inference path for S independent clips, two ways:

  (a) one by one  S back-to-back dvc_set_exemplar + dvc_colorize_video_rgb8 calls, one per clip
  (b) batched     dvc_set_exemplars with the S exemplars + one dvc_colorize_videos_rgb8 call over the S clips

Both pay the same S exemplar prologues.  Workload: S in {1, 2, 4, 8} synthetic 720x1280 uint8 clips of --frames frames
resident in pinned host memory, CenterPad'ed to 432x768 (test.py's default image size; the networks run at 216x384), seeded
weights, WLS on (lambda 500, sigma 4), the default conv arithmetic and MATH_FP16X1.  At this size one clip leaves the H100
underfilled (the 1/8-resolution ColorVidNet layers are ~50 output tiles for 132 SMs, and ColorVidNet is recurrent, so only
frames of other clips can fill them), which is what the batched call is for.
Method: after a warm-up, windows of at least --window seconds alternate between (a) and (b); each window runs whole calls
and ends with a device synchronisation; the rate is the median over --reps windows.  Algorithmic TFLOP/s = frames/s x the
networks' FLOPs per frame, counted from the layer shapes below (VGG19 through r52, the WarpNet query side with theta, the
correlation with its softmax-weighted warp, ColorVidNet; ingest, up-sampling and WLS not counted).  Launches per frame
step: dvc_launch_count over the video calls (not the exemplar prologues) / F.

    python tools/clips_bench.py [--frames 16] [--window 1.0] [--reps 3] [--clips 1 2 4 8] [--trace DIR]

--trace DIR also writes a torch.profiler trace of one batched call at the largest S and prints, per CUDA stream, the summed
kernel time against the call's wall time (the post-processing stream must not be the pipeline's critical path).
"""
import argparse
import collections
import json
import os
import re
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200")):
    sys.path.insert(0, p)

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


def synthetic_frames(seed, F):
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, HS // 16 + 1, WS // 16 + 1, 3)) * 255).astype(np.int16)
    img = np.kron(coarse, np.ones((1, 16, 16, 1), np.int16))[:, :HS, :WS]
    img = np.clip(img + rng.integers(-12, 13, img.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    return torch.from_numpy(img).pin_memory()


def frame_gflop(h, w):
    """Algorithmic GFLOP of one frame's networks at h x w, from the layer shapes: VGG19's convolutions through r52 from the
    weight shapes, the rest by counting the fp64 oracle's convolutions and matmuls on shape-only (meta) tensors."""
    from torch.utils.flop_counter import FlopCounterMode

    from oracle import dvc_oracle as O
    from oracle.weights import make_state_dict

    sds = {k: {n: t.to("meta") for n, t in make_state_dict(k, seed=0).items()} for k in ("vgg", "warp", "color")}
    parts, hh, ww, vgg = {}, h, w, 0.0
    for name in O.VGG_ORDER:  # 3x3 convolutions, pools halve the map; the library stops at r52 (conv5_2)
        if name == "P":
            hh, ww = hh // 2, ww // 2
            continue
        cout, cin = sds["vgg"][name + ".weight"].shape[:2]
        vgg += 2.0 * hh * ww * 9 * cin * cout
        if name == "conv5_2":
            break
    parts["vgg_r52"] = vgg / 1e9
    m = lambda *s: torch.empty(*s, device="meta")  # noqa: E731
    n = (h // 4) * (w // 4)
    counted = {
        "warp_query": lambda: O.project_normalize(sds["warp"], "theta", O.warp_features(
            sds["warp"], m(1, 128, h // 2, w // 2), m(1, 256, h // 4, w // 4), m(1, 512, h // 8, w // 8), m(1, 512, h // 16, w // 16))),
        "correlation": lambda: O.corr_softmax_warp(m(1, 256, n), m(1, 256, n), m(1, n, 3), 1.0),
        "colorvidnet": lambda: O.colorvidnet_forward(sds["color"], m(1, 7, h, w)),
    }
    with torch.no_grad():
        for name, fn in counted.items():
            with FlopCounterMode(display=False) as fc:
                fn()
            parts[name] = fc.get_total_flops() / 1e9
    return parts


def post_stream_share(ctx, clips, S, out, trace_dir):
    """One profiled batched call: summed kernel time per CUDA stream against the call's wall time."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        ctx.colorize_videos_rgb8(clips[:S], SIZE, T, out=out)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    os.makedirs(trace_dir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(trace_dir, f"clips_S{S}.json"))
    busy, names = collections.defaultdict(float), collections.defaultdict(set)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
            kname = e.name
            if kname.startswith("Memcpy") or kname.startswith("Memset"):
                continue
            busy[e.device_resource_id] += e.device_time_total / 1e3  # ms
            short = re.search(r"(\w+)[(<]", kname)  # "void dvc::(anonymous namespace)::fgs_horizontal_kernel(float*, ...)"
            names[e.device_resource_id].add(short.group(1) if short else kname[:40])
    rows = [{"stream": sid, "kernel_ms": ms, "kernels": sorted(names[sid])[:6]} for sid, ms in sorted(busy.items(), key=lambda kv: -kv[1])]
    return wall * 1e3, rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--clips", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--trace", default=None, help="directory for a torch.profiler trace of one batched call at the largest S")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clips_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    F_, Smax = args.frames, max(args.clips)
    gflop = frame_gflop(SIZE[0] // 2, SIZE[1] // 2)
    per_frame = sum(gflop.values())
    clips = [synthetic_frames(s, F_) for s in range(Smax)]
    IB = make_lab(40, Smax, SIZE[0] // 2, SIZE[1] // 2)
    rows, post = [], None
    for math_name, conv in (("default", dvc.MATH_TF32X3), ("fp16x1", dvc.MATH_FP16X1)):
        ctx.set_math(conv=conv)
        for S in args.clips:
            outs = [torch.empty(1, F_, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory() for _ in range(S)]
            out_b = torch.empty(S, F_, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory()
            launches = {"one_by_one": 0, "batched": 0}

            def one_by_one(count=False):
                for s in range(S):
                    ctx.set_exemplar(IB[s:s + 1])
                    n0 = ctx.launch_count()
                    ctx.colorize_video_rgb8(clips[s], SIZE, T, out=outs[s])
                    if count:
                        launches["one_by_one"] += ctx.launch_count() - n0

            def batched(count=False):
                ctx.set_exemplars(IB[:S])
                n0 = ctx.launch_count()
                ctx.colorize_videos_rgb8(clips[:S], SIZE, T, out=out_b)
                if count:
                    launches["batched"] += ctx.launch_count() - n0

            methods = {"one_by_one": one_by_one, "batched": batched}
            for m in methods.values():  # warm-up, and the launches of one call sequence
                m()
                m(count=True)
            torch.cuda.synchronize()
            rates = {m: [] for m in methods}
            for _ in range(args.reps):
                for m, fn in methods.items():
                    n, t0 = 0, time.perf_counter()
                    while True:
                        fn()
                        torch.cuda.synchronize()
                        n += S * F_
                        dt = time.perf_counter() - t0
                        if dt >= args.window:
                            break
                    rates[m].append(n / dt)
            for m in methods:
                fps = statistics.median(rates[m])
                rows.append({"math": math_name, "S": S, "method": m, "frames_per_s": fps, "windows_fps": rates[m],
                             "algorithmic_tflops": fps * per_frame / 1e3, "launches_per_frame_step": launches[m] / F_})
            if args.trace and S == Smax and math_name == "default":
                ctx.set_exemplars(IB[:S])
                post = post_stream_share(ctx, clips, S, out_b, args.trace)
    ctx.set_math(conv=dvc.MATH_TF32X3)
    print(f"card: {name}, power limit {power}; {Smax} synthetic {HS}x{WS} clips max -> {SIZE[0]}x{SIZE[1]}, {F_} frames per clip, "
          f"WLS on, median of {args.reps} alternating windows >= {args.window} s")
    print("networks' algorithmic GFLOP per frame at 216x384: " + ", ".join(f"{k} {v:.1f}" for k, v in gflop.items())
          + f"; total {per_frame:.1f}")
    print("| conv math | S | one by one: frames/s | TFLOP/s | launches / frame step | batched: frames/s | TFLOP/s | "
          "launches / frame step | speed-up |")
    print("|---|---|---|---|---|---|---|---|---|")
    for i in range(0, len(rows), 2):
        a, b = rows[i], rows[i + 1]
        print(f"| {a['math']} | {a['S']} | {a['frames_per_s']:.1f} | {a['algorithmic_tflops']:.1f} | {a['launches_per_frame_step']:.0f} "
              f"| {b['frames_per_s']:.1f} | {b['algorithmic_tflops']:.1f} | {b['launches_per_frame_step']:.0f} "
              f"| {b['frames_per_s'] / a['frames_per_s']:.2f}x |")
    if post:
        wall, streams = post
        print(f"profiled batched call, S = {Smax}: wall {wall:.1f} ms; summed kernel time per stream:")
        for r in streams:
            print(f"  stream {r['stream']}: {r['kernel_ms']:.1f} ms ({', '.join(r['kernels'])})")
    print(json.dumps({"card": name, "power_limit": power, "frames": F_, "gflop_per_frame": gflop, "rows": rows,
                      "post_profile": None if not post else {"wall_ms": post[0], "streams": post[1]}}))


if __name__ == "__main__":
    main()
