"""Cost of source-resolution output: aggregate frames/s of dvc_colorize_videos_exemplars_rgb8 (output at the 432x768 window)
against dvc_colorize_videos_source_rgb8 (output at each frame's source resolution, here the whole 1080x1920 frame) on the same
clips.  Workload: S = 1 and S = 8 synthetic 1080x1920 uint8 clips of --frames frames in pinned host memory, one exemplar each,
CenterPad'ed to 432x768 (test.py's default size; the networks run at 216x384), seeded weights, WLS on (lambda 500, sigma 4),
the default conv arithmetic.

Method: after a warm-up, windows of at least --window seconds alternate between the two calls; each window runs whole calls
and ends with a device synchronisation; the rate is the median over --reps windows.  PCIe bytes per frame are counted from the
shapes (frame upload plus image download).  Kernel launches per frame step are dvc_launch_count over a call of 2F frames minus
one of F frames, divided by F.  The card's name and power limit are read in the same run.

    python tools/source_resolution_bench.py [--frames 16] [--window 1.0] [--reps 3] [--trace DIR]

--trace DIR additionally profiles one S = 8 call of each kind with torch.profiler (a separate run after the timed windows),
writes the traces there and prints the summed kernel time of the post-processing stream (the one running lab_to_rgb8) and of
the ColorVidNet stream (the one running make_last).
"""
import argparse
import collections
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"), os.path.dirname(os.path.abspath(__file__))):
    sys.path.insert(0, p)

import numpy as np
import torch

from clips_bench import card

HS, WS, SIZE, T, WLS = 1080, 1920, (432, 768), 1e-10, (500.0, 4.0)


def synthetic_frames(seed, F):
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, HS // 16 + 1, WS // 16 + 1, 3)) * 255).astype(np.int16)
    img = np.kron(coarse, np.ones((1, 16, 16, 1), np.int16))[:, :HS, :WS]
    img = np.clip(img + rng.integers(-12, 13, img.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    return torch.from_numpy(img).pin_memory()


def calls(ctx, clips, F_):
    import dvc
    from dvc.prepost import centerpad_geometry

    S = len(clips)
    _, _, h, w = dvc.source_footprint(HS, WS, *centerpad_geometry(HS, WS, SIZE), *SIZE)
    win_out = torch.empty(S, F_, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory()
    src_out = [torch.empty(1, F_, h, w, 3, dtype=torch.uint8).pin_memory() for _ in range(S)]
    K = [1] * S
    return {"window": lambda: ctx.colorize_videos_exemplars_rgb8(clips, K, SIZE, T, wls=WLS, out=win_out),
            "source": lambda: ctx.colorize_videos_source_rgb8(clips, K, SIZE, T, wls=WLS, out=src_out)}, (h, w)


def launches_per_step(ctx, clips, F_, kind):
    S, counts = len(clips), []
    for n in (F_, 2 * F_):
        cl = [torch.cat([c] * (n // F_)) for c in clips]
        fn = calls(ctx, cl, n)[0][kind]
        fn()
        torch.cuda.synchronize()
        ctx.launch_count(reset=True)
        fn()
        torch.cuda.synchronize()
        counts.append(ctx.launch_count())
    return (counts[1] - counts[0]) / F_, S


def profile_streams(ctx, fns, trace_dir):
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(trace_dir, exist_ok=True)
    res = {}
    for name, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
        prof.export_chrome_trace(os.path.join(trace_dir, f"source_resolution_S8_{name}.json"))
        busy, marks = collections.defaultdict(float), collections.defaultdict(set)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
                if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
                    continue
                busy[e.device_resource_id] += e.device_time_total / 1e3
                for k in ("lab_to_rgb8_kernel", "make_last_kernel"):
                    if k in e.name:
                        marks[k].add(e.device_resource_id)
        post = sum(busy[s] for s in marks["lab_to_rgb8_kernel"])
        color = sum(busy[s] for s in marks["make_last_kernel"])
        res[name] = {"wall_ms": wall, "post_stream_kernel_ms": post, "colorvidnet_stream_kernel_ms": color}
        print(f"S = 8, {name}: wall {wall:.1f} ms, post stream kernels {post:.1f} ms, ColorVidNet stream kernels {color:.1f} ms")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trace", default=None, help="directory: also profile one S = 8 call of each kind")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("source_resolution_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    print(f"card: {name}, power limit {power}")
    F_ = args.frames
    all_clips = [synthetic_frames(s, F_) for s in range(8)]
    IB = make_lab(40, 8, SIZE[0] // 2, SIZE[1] // 2)
    rows = []
    for S in (1, 8):
        clips = all_clips[:S]
        if S == 1:
            ctx.set_exemplar(IB[:1])
        else:
            ctx.set_exemplars(IB[:S])
        fns, (h, w) = calls(ctx, clips, F_)
        for fn in fns.values():  # warm-up
            fn()
        torch.cuda.synchronize()
        rates = {m: [] for m in fns}
        for _ in range(args.reps):
            for m, fn in fns.items():
                n, t0 = 0, time.perf_counter()
                while True:
                    fn()
                    torch.cuda.synchronize()
                    n += 1
                    dt = time.perf_counter() - t0
                    if dt >= args.window:
                        break
                rates[m].append(n * S * F_ / dt)
        up = HS * WS * 3
        row = {"S": S, "footprint": [h, w]}
        for m in fns:
            down = (SIZE[0] * SIZE[1] if m == "window" else h * w) * 3
            per_step, _ = launches_per_step(ctx, clips, F_, m)
            row[m] = {"frames_per_s": statistics.median(rates[m]), "windows": rates[m], "pcie_up_bytes_per_frame": up,
                      "pcie_down_bytes_per_frame": down, "launches_per_frame_step": per_step}
        rows.append(row)
        if S == 8 and args.trace:
            row["profile"] = profile_streams(ctx, fns, args.trace)
    print(f"{HS}x{WS} synthetic pinned clips -> {SIZE[0]}x{SIZE[1]}, {F_} frames per clip, one exemplar each, WLS on, default conv "
          f"math; median of {args.reps} alternating windows >= {args.window} s")
    print("| S | window: frames/s | source: frames/s | source / window | PCIe down per frame (window / source) | launches per "
          "frame step (window / source) |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        a, b = r["window"], r["source"]
        print(f"| {r['S']} | {a['frames_per_s']:.1f} | {b['frames_per_s']:.1f} | {b['frames_per_s'] / a['frames_per_s']:.2f}x | "
              f"{a['pcie_down_bytes_per_frame']} / {b['pcie_down_bytes_per_frame']} | {a['launches_per_frame_step']:.0f} / "
              f"{b['launches_per_frame_step']:.0f} |")
    print(json.dumps({"card": name, "power_limit": power, "frames": F_, "rows": rows}))


if __name__ == "__main__":
    main()
