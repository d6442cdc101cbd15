"""I420 video: aggregate frames/s of dvc_colorize_videos_i420 with I420 output against the sRGB calls wrapped in host conversions.
Workload (tools/gray_bench.py's): S = 1 and S = 8 synthetic 1080x1920 clips of --frames frames in pinned host memory, one
exemplar each, CenterPad'ed to 432x768 (test.py's default size; the networks run at 216x384), seeded weights, WLS on (lambda
500, sigma 4), the default conv arithmetic; window output and source-resolution output.

  (a) "host": cv2.cvtColor(COLOR_YUV2RGB_I420) of every frame into a pinned RGB clip on the host, the sRGB call
      (dvc_colorize_videos_exemplars_rgb8 or dvc_colorize_videos_source_rgb8), then cv2.cvtColor(COLOR_RGB2YUV_I420) of every
      output frame: what a user with a yuv420p decoder and encoder had to do.
  (b) "device": dvc_colorize_videos_i420 with out_i420 = 1 on the same I420 clips: the same bytes (include/dvc.h).

Method: after a warm-up, windows of at least --window seconds alternate between (a) and (b); each runs whole iterations that end
with a device synchronisation; the rate is the median over --reps windows.  Host core-seconds in cv2 per frame are the process
CPU time across the cv2 calls of (a).  Bytes up and down per frame are counted from the shapes.  Kernel launches per frame step
are dvc_launch_count over a call of 2F frames minus one of F frames, divided by F.  --trace DIR profiles one call of each per S
and output with torch.profiler (after the timed windows), writes the traces there and reports the summed kernel time per frame
step of the ingest stream (the one running zoom_crop_kernel) and of the post-processing stream (the one running
lab_to_rgb8_kernel).  --tool times tools/colorize_y4m.py end to end (process start and weight loading included) on a
--tool-frames 1080p Y4M file, median of 3 runs, and its streaming rate after start-up (the tool's own report).  The card's
name and power limit are read in the same run.

    python tools/yuv_bench.py [--frames 16] [--window 1.0] [--reps 3] [--trace DIR] [--tool] [--tool-frames 96]
"""
import argparse
import collections
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"), os.path.dirname(os.path.abspath(__file__))):
    sys.path.insert(0, p)

import cv2
import numpy as np
import torch

from clips_bench import card

HS, WS, SIZE, T, WLS = 1080, 1920, (432, 768), 1e-10, (500.0, 4.0)


def i420_frames(seed, F):
    """Blocky 1080p content (gray_bench's luma) with smooth chroma, as I420 [F,1620,1920]."""
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, HS // 16 + 1, WS // 16 + 1)) * 219 + 16).astype(np.int16)
    y = np.kron(coarse, np.ones((1, 16, 16), np.int16))[:, :HS, :WS]
    y = np.clip(y + rng.integers(-12, 13, y.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    c = (rng.random((F, 2, HS // 32 + 1, WS // 32 + 1)) * 160 + 48).astype(np.uint8)
    c = np.kron(c, np.ones((1, 1, 16, 16), np.uint8))[:, :, :HS // 2, :WS // 2]
    return torch.from_numpy(np.concatenate([y.reshape(F, -1), c.reshape(F, -1)], axis=1).reshape(F, HS * 3 // 2, WS))


def out_size(source):
    import dvc
    from dvc.prepost import centerpad_geometry

    return tuple(dvc.source_footprint(HS, WS, *centerpad_geometry(HS, WS, SIZE), *SIZE)[2:]) if source else SIZE


class Host:
    """(a): host conversions around the sRGB call, into preallocated pinned buffers; cpu accumulates the cv2 core-seconds."""

    def __init__(self, ctx, yuv, source):
        self.ctx, self.yuv, self.source = ctx, yuv, source
        S, F_ = len(yuv), yuv[0].shape[0]
        h, w = out_size(source)
        self.rgb = [torch.empty(F_, HS, WS, 3, dtype=torch.uint8).pin_memory() for _ in range(S)]
        self.out = [torch.empty(1, F_, h, w, 3, dtype=torch.uint8).pin_memory() for _ in range(S)]
        self.win = torch.empty(S, F_, h, w, 3, dtype=torch.uint8).pin_memory()
        self.res = [np.empty((F_, h * 3 // 2, w), np.uint8) for _ in range(S)]
        self.cpu = 0.0

    def __call__(self):
        S, F_ = len(self.yuv), self.yuv[0].shape[0]
        c0 = time.process_time()
        for s in range(S):
            src, dst = self.yuv[s].numpy(), self.rgb[s].numpy()
            for t in range(F_):
                cv2.cvtColor(src[t], cv2.COLOR_YUV2RGB_I420, dst=dst[t])
        self.cpu += time.process_time() - c0
        if self.source:
            out = self.ctx.colorize_videos_source_rgb8(self.rgb, [1] * S, SIZE, T, wls=WLS, out=self.out)
            frames = [o[0].numpy() for o in out]
        else:
            out = self.ctx.colorize_videos_exemplars_rgb8(self.rgb, [1] * S, SIZE, T, wls=WLS, out=self.win)
            frames = [o.numpy() for o in out]
        c0 = time.process_time()
        for s in range(S):
            for t in range(F_):
                cv2.cvtColor(frames[s][t], cv2.COLOR_RGB2YUV_I420, dst=self.res[s][t])
        self.cpu += time.process_time() - c0
        return self.res


def device_call(ctx, yuv, source):
    S, F_ = len(yuv), yuv[0].shape[0]
    h, w = out_size(source)
    out = [torch.empty(1, F_, h * 3 // 2, w, dtype=torch.uint8).pin_memory() for _ in range(S)]
    return lambda: ctx.colorize_videos_i420(yuv, [1] * S, SIZE, T, wls=WLS, source_resolution=source, out_format="i420", out=out)


def launches_per_step(ctx, yuv, source, kind):
    counts = []
    for n in (1, 2):
        clips = [torch.cat([c] * n).pin_memory() for c in yuv]
        fn = device_call(ctx, clips, source) if kind == "device" else Host(ctx, clips, source)
        fn()
        torch.cuda.synchronize()
        ctx.launch_count(reset=True)
        fn()
        torch.cuda.synchronize()
        counts.append(ctx.launch_count())
    return (counts[1] - counts[0]) / yuv[0].shape[0]


def stream_ms(fns, F_, trace_dir, tag):
    """Summed kernel time per frame step of the ingest stream (zoom_crop_kernel) and the post stream (lab_to_rgb8_kernel)."""
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(trace_dir, exist_ok=True)
    res = {}
    for name, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        prof.export_chrome_trace(os.path.join(trace_dir, f"yuv_{tag}_{name}.json"))
        busy, ingest, post = collections.defaultdict(float), set(), set()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
                if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
                    continue
                busy[e.device_resource_id] += e.device_time_total / 1e3
                if "zoom_crop_kernel" in e.name:
                    ingest.add(e.device_resource_id)
                if "lab_to_rgb8_kernel" in e.name:
                    post.add(e.device_resource_id)
        res[name] = {"ingest": sum(busy[s] for s in ingest) / F_, "post": sum(busy[s] for s in post) / F_}
        print(f"{tag}, {name}: ingest stream {res[name]['ingest']:.3f} ms, post stream {res[name]['post']:.3f} ms per frame step")
    return res


def tool_rate(n_frames, reps):
    from PIL import Image

    res = {"frames": n_frames, "runs": [], "streaming_runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "in.y4m")
        with open(src, "wb") as f:
            f.write(f"YUV4MPEG2 W{WS} H{HS} F25:1 Ip A1:1 C420jpeg\n".encode())
            for c in range(0, n_frames, 16):
                fr = i420_frames(100 + c, min(16, n_frames - c)).numpy()
                for t in range(fr.shape[0]):
                    f.write(b"FRAME\n")
                    f.write(fr[t].tobytes())
        ref = os.path.join(tmp, "ref.png")
        Image.fromarray(np.random.default_rng(22).integers(0, 256, (HS, WS, 3), dtype=np.uint8)).save(ref)
        for _ in range(reps):
            cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_y4m.py"), "-i", src, "-o", os.path.join(tmp, "out.y4m"),
                   "--ref", ref, "--seeded-weights"]
            t0 = time.perf_counter()
            err = subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True).stderr
            res["runs"].append(n_frames / (time.perf_counter() - t0))
            res["streaming_runs"].append(float(re.search(r"\(([0-9.]+) frames/s after start-up\)", err).group(1)))
    res["frames_per_s"] = statistics.median(res["runs"])  # process start, weights and exemplar included
    res["streaming_frames_per_s"] = statistics.median(res["streaming_runs"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trace", default=None, help="directory: also profile one call of each kind")
    ap.add_argument("--tool", action="store_true", help="also time tools/colorize_y4m.py end to end")
    ap.add_argument("--tool-frames", type=int, default=96)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("yuv_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    print(f"card: {name}, power limit {power}, cv2 {cv2.__version__} with {cv2.getNumThreads()} threads, {os.cpu_count()} host cores")
    F_ = args.frames
    all_yuv = [i420_frames(s, F_).pin_memory() for s in range(8)]
    IB = make_lab(40, 8, SIZE[0] // 2, SIZE[1] // 2)
    rows = []
    for S in (1, 8):
        yuv = all_yuv[:S]
        if S == 1:
            ctx.set_exemplar(IB[:1])
        else:
            ctx.set_exemplars(IB[:S])
        for source in (False, True):
            output = "source" if source else "window"
            host = Host(ctx, yuv, source)
            fns = {"host": host, "device": device_call(ctx, yuv, source)}
            got = [o[0].numpy() for o in fns["device"]()]  # warm-up, and the same bytes
            ref = fns["host"]()
            assert all(np.array_equal(a, b) for a, b in zip(got, ref)), "the I420 call and the host pipeline disagree"
            torch.cuda.synchronize()
            rates, frames_host = {m: [] for m in fns}, 0
            host.cpu = 0.0
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
                    if m == "host":
                        frames_host += n * S * F_
            h, w = out_size(source)
            row = {"S": S, "output": output, "out_size": [h, w]}
            for m in fns:
                row[m] = {"frames_per_s": statistics.median(rates[m]), "windows": rates[m],
                          "pcie_up_bytes_per_frame": HS * WS * 3 // (1 if m == "host" else 2),
                          "pcie_down_bytes_per_frame": h * w * 3 // (1 if m == "host" else 2),
                          "launches_per_frame_step": launches_per_step(ctx, yuv, source, m)}
            row["host"]["cv2_core_ms_per_frame"] = 1e3 * host.cpu / frames_host
            if args.trace:
                row["stream_ms_per_step"] = stream_ms(fns, F_, args.trace, f"S{S}_{output}")
            rows.append(row)
    print(f"{HS}x{WS} synthetic I420 pinned clips -> {SIZE[0]}x{SIZE[1]}, {F_} frames per clip, one exemplar each, WLS on, default "
          f"conv math; (a) host cv2 I420 -> RGB, sRGB call, host RGB -> I420 against (b) colorize_videos_i420 with I420 output; "
          f"median of {args.reps} alternating windows >= {args.window} s")
    print("| S | output | (a) host: frames/s | (b) device: frames/s | (b) / (a) | cv2 core-ms per frame (a) | bytes up per frame (a / b) "
          "| bytes down per frame (a / b) | launches per frame step (a / b) |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        a, b = r["host"], r["device"]
        print(f"| {r['S']} | {r['output']} | {a['frames_per_s']:.1f} | {b['frames_per_s']:.1f} | {b['frames_per_s'] / a['frames_per_s']:.3f}x | "
              f"{a['cv2_core_ms_per_frame']:.2f} | {a['pcie_up_bytes_per_frame']} / {b['pcie_up_bytes_per_frame']} | "
              f"{a['pcie_down_bytes_per_frame']} / {b['pcie_down_bytes_per_frame']} | "
              f"{a['launches_per_frame_step']:.0f} / {b['launches_per_frame_step']:.0f} |")
    result = {"card": name, "power_limit": power, "frames": F_, "rows": rows}
    if args.tool:
        result["tool_y4m"] = tool_rate(args.tool_frames, 3)
        print("colorize_y4m.py:", json.dumps(result["tool_y4m"]))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
