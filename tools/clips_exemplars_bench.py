"""Aggregate output images per second of test.py's whole inference path for S clips with K_s exemplars each (the reference's
data layout: a folder of reference images per clip, each colorizing the whole clip), R = sum K_s output rows, three ways:

  (1) per clip        for each clip: dvc_set_exemplars with its K_s exemplars + one dvc_colorize_video_rgb8 call
  (2) per reference   for each reference index k: dvc_set_exemplars with exemplar k of every clip that has one + one
                      dvc_colorize_videos_rgb8 call over those clips (clips with fewer references drop out of later calls)
  (3) one pass        dvc_set_exemplars with all R exemplars + one dvc_colorize_videos_exemplars_rgb8 call

Every arm pays the same R exemplar prologues and writes R x F images.  Workload: per-clip counts (2,2), (4,4), (2,2,2,2),
(1,3,4) and (1,2,2,3); synthetic 720x1280 uint8 clips of --frames frames in pinned host memory, CenterPad'ed to 432x768
(test.py's default size; the networks run at 216x384), seeded weights, WLS on (lambda 500, sigma 4); the default conv
arithmetic and MATH_FP16X1.  Arm (1) runs ColorVidNet at batch K_s only; arm (2) recomputes VGG19 and the WarpNet query side
of every frame once per reference index; arm (3) does neither.
Method: after a warm-up, windows of at least --window seconds alternate between the arms; each window runs whole call
sequences and ends with a device synchronisation; the rate is the median over --reps windows.  Algorithmic TFLOP/s = the
networks' FLOPs of the one-pass decomposition (VGG19 through r52 and the WarpNet query side once per clip frame, the
correlation and ColorVidNet once per row and frame, counted from the layer shapes as tools/clips_bench.py does) over the
time of the arm, the same work for every arm, so it ranks the arms like images/s.

    python tools/clips_exemplars_bench.py [--frames 16] [--window 1.0] [--reps 3] [--trace DIR --trace-counts 1 3 4]

--trace DIR instead profiles one call sequence of each arm for --trace-counts (default math) with torch.profiler, writes the
traces there and prints, per arm, the wall time, the summed kernel time per CUDA stream and the kernels that take the most.
"""
import argparse
import collections
import json
import os
import re
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"), os.path.dirname(os.path.abspath(__file__))):
    sys.path.insert(0, p)

import torch

from clips_bench import HS, SIZE, T, WS, card, frame_gflop, synthetic_frames

COUNTS = [(2, 2), (4, 4), (2, 2, 2, 2), (1, 3, 4), (1, 2, 2, 3)]


def arms(ctx, clips, IB, K, outs):
    """The three call sequences for per-clip counts K; IB holds the R exemplars in row order."""
    S = len(K)
    first = [sum(K[:s]) for s in range(S)]

    def per_clip():
        for s in range(S):
            ctx.set_exemplars(IB[first[s]:first[s] + K[s]])
            ctx.colorize_video_rgb8(clips[s], SIZE, T, out=outs["per_clip"][s])

    def per_reference():
        for k in range(max(K)):
            have = [s for s in range(S) if K[s] > k]
            ctx.set_exemplars(IB[[first[s] + k for s in have]])
            ctx.colorize_videos_rgb8([clips[s] for s in have], SIZE, T, out=outs["per_reference"][k])

    def one_pass():
        ctx.set_exemplars(IB)
        ctx.colorize_videos_exemplars_rgb8(clips[:S], list(K), SIZE, T, out=outs["one_pass"])

    return {"per_clip": per_clip, "per_reference": per_reference, "one_pass": one_pass}


def outputs(K, F_):
    def pinned(*shape):
        return torch.empty(*shape, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory()

    return {"per_clip": [pinned(k, F_) for k in K],
            "per_reference": [pinned(sum(1 for k in K if k > i), F_) for i in range(max(K))],
            "one_pass": pinned(sum(K), F_)}


def profile_arms(ctx, clips, IB, K, F_, trace_dir):
    """One profiled call sequence per arm: wall time, summed kernel time per CUDA stream, the largest kernels."""
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(trace_dir, exist_ok=True)
    fns = arms(ctx, clips, IB, K, outputs(K, F_))
    for fn in fns.values():
        fn()
    tag = "_".join(map(str, K))
    for name, fn in fns.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
        prof.export_chrome_trace(os.path.join(trace_dir, f"clips_exemplars_{tag}_{name}.json"))
        busy, kern = collections.defaultdict(float), collections.defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
                if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
                    continue
                busy[e.device_resource_id] += e.device_time_total / 1e3
                short = re.search(r"(\w+)[(<]", e.name)
                kern[short.group(1) if short else e.name[:40]] += e.device_time_total / 1e3
        print(f"K = {K}, {name}: wall {wall:.1f} ms; kernel ms per stream: "
              + ", ".join(f"{sid}: {ms:.1f}" for sid, ms in sorted(busy.items(), key=lambda kv: -kv[1])))
        print("  largest kernels (ms): " + ", ".join(f"{k} {v:.1f}" for k, v in sorted(kern.items(), key=lambda kv: -kv[1])[:8]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trace", default=None, help="directory: profile one call sequence per arm for --trace-counts instead")
    ap.add_argument("--trace-counts", type=int, nargs="+", default=[1, 3, 4])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clips_exemplars_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    F_ = args.frames
    Smax = max(len(K) for K in COUNTS + [tuple(args.trace_counts)])
    clips = [synthetic_frames(s, F_) for s in range(Smax)]
    IB = make_lab(40, 8, SIZE[0] // 2, SIZE[1] // 2)
    print(f"card: {name}, power limit {power}")
    if args.trace:
        K = tuple(args.trace_counts)
        profile_arms(ctx, clips, IB[:sum(K)], K, F_, args.trace)
        return
    gflop = frame_gflop(SIZE[0] // 2, SIZE[1] // 2)
    per_clip_frame = gflop["vgg_r52"] + gflop["warp_query"]
    per_row_frame = gflop["correlation"] + gflop["colorvidnet"]
    rows = []
    for math_name, conv in (("default", dvc.MATH_TF32X3), ("fp16x1", dvc.MATH_FP16X1)):
        ctx.set_math(conv=conv)
        for K in COUNTS:
            R = sum(K)
            fns = arms(ctx, clips, IB[:R], K, outputs(K, F_))
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
                    rates[m].append(n * R * F_ / dt)
            gflop_seq = F_ * (len(K) * per_clip_frame + R * per_row_frame)
            row = {"math": math_name, "K": list(K), "R": R}
            for m in fns:
                ips = statistics.median(rates[m])
                row[m] = {"images_per_s": ips, "windows": rates[m], "algorithmic_tflops": ips / (R * F_) * gflop_seq / 1e3}
            rows.append(row)
    ctx.set_math(conv=dvc.MATH_TF32X3)
    print(f"{HS}x{WS} synthetic clips -> {SIZE[0]}x{SIZE[1]}, {F_} frames per clip, WLS on, median of {args.reps} alternating windows "
          f">= {args.window} s; algorithmic GFLOP per clip frame (VGG19 + WarpNet query side) {per_clip_frame:.1f}, per row and "
          f"frame (correlation + ColorVidNet) {per_row_frame:.1f}")
    print("| conv math | K | per clip: images/s | TFLOP/s | per reference: images/s | TFLOP/s | one pass: images/s | TFLOP/s "
          "| one pass / better of the two |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        a, b, c = r["per_clip"], r["per_reference"], r["one_pass"]
        best = max(a["images_per_s"], b["images_per_s"])
        print(f"| {r['math']} | {tuple(r['K'])} | {a['images_per_s']:.1f} | {a['algorithmic_tflops']:.1f} | {b['images_per_s']:.1f} "
              f"| {b['algorithmic_tflops']:.1f} | {c['images_per_s']:.1f} | {c['algorithmic_tflops']:.1f} | {c['images_per_s'] / best:.2f}x |")
    print(json.dumps({"card": name, "power_limit": power, "frames": F_, "gflop": gflop, "rows": rows}))


if __name__ == "__main__":
    main()
