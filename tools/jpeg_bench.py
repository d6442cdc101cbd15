"""Device JPEG output: what it costs and what it saves (include/dvc.h: dvc_encode_jpeg, dvc_colorize_videos_jpeg).

  1. the stand-alone encoder: frames/s of dvc_encode_jpeg on batches of 8 frames at 432x768 and 1080x1920, q75 and q95, device
     destination (CUDA events around --iters calls after a warm-up);
  2. video calls: aggregate frames/s of dvc_colorize_videos_jpeg against the rgb8 call it encodes (window output:
     dvc_colorize_videos_exemplars_rgb8; 1080p source output: dvc_colorize_videos_source_rgb8) at S = 1 and 8, q75, on
     source_resolution_bench.py's workload (synthetic 1080x1920 pinned clips -> 432x768, one exemplar each, WLS on); median of
     --reps alternating windows >= --window s, each ending with a device synchronisation.  Bytes down per frame: the rgb8 frame,
     or the mean of the JPEG call's sizes.  Launches per frame step: dvc_launch_count of a 2F-frame call minus an F-frame one,
     over F;
  3. with --trace DIR, one S = 8 source-output call of each kind under torch.profiler (a separate run): summed kernel time of the
     post-processing stream (the one running lab_to_rgb8) and of the encoder's kernels;
  4. with --folder, end-to-end tools/colorize_folder.py frames/s on --folder-frames 1080x1920 PNG frames written first (window
     output): --format png, --format jpg, and the host Pillow JPEG encode of the same output frames on the tool's writer pool
     (the host part a host-JPEG writer would add), with the host core count.

The card's name and power limit are read in the same run.

    python tools/jpeg_bench.py [--frames 16] [--window 1.0] [--reps 3] [--iters 50] [--trace DIR] [--folder]
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"), os.path.dirname(os.path.abspath(__file__))):
    sys.path.insert(0, p)

import numpy as np
import torch

from clips_bench import card
from source_resolution_bench import HS, SIZE, T, WLS, WS, synthetic_frames


def encoder_rate(ctx, H, W, q, iters):
    import dvc

    rgb = synthetic_frames(7, 8)
    if (H, W) != (HS, WS):
        rgb = rgb[:, :H, :W]
    rgb = rgb.contiguous().cuda()
    out = torch.empty(8, dvc.jpeg_max_bytes(H, W), dtype=torch.uint8, device="cuda")
    sizes = torch.empty(8, dtype=torch.int64, device="cuda")
    for _ in range(3):
        ctx.encode_jpeg_into(rgb, out, sizes, q)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ctx.encode_jpeg_into(rgb, out, sizes, q)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return {"H": H, "W": W, "q": q, "frames_per_s": 8e3 / ms, "ms_per_batch_of_8": ms, "mean_bytes": float(sizes.float().mean())}


def video_calls(ctx, clips, F_, source):
    import dvc
    from dvc.prepost import centerpad_geometry

    S, K = len(clips), [1] * len(clips)
    if source:
        _, _, h, w = dvc.source_footprint(HS, WS, *centerpad_geometry(HS, WS, SIZE), *SIZE)
        rgb_out = [torch.empty(1, F_, h, w, 3, dtype=torch.uint8).pin_memory() for _ in range(S)]
        rgb = lambda: ctx.colorize_videos_source_rgb8(clips, K, SIZE, T, wls=WLS, out=rgb_out)  # noqa: E731
    else:
        h, w = SIZE
        rgb_out = torch.empty(S, F_, h, w, 3, dtype=torch.uint8).pin_memory()
        rgb = lambda: ctx.colorize_videos_exemplars_rgb8(clips, K, SIZE, T, wls=WLS, out=rgb_out)  # noqa: E731
    stride = dvc.jpeg_max_bytes(h, w)
    slots = [torch.empty(1, F_, stride, dtype=torch.uint8).pin_memory() for _ in range(S)]
    sizes = torch.empty(S, F_, dtype=torch.int64).pin_memory()
    jpg = lambda: ctx.colorize_videos_jpeg(clips, K, SIZE, 75, source, T, wls=WLS, out=slots, sizes=sizes)  # noqa: E731
    return {"rgb8": rgb, "jpeg": jpg}, (h, w), sizes


def launches_per_step(ctx, clips, F_, source, kind):
    counts = []
    for n in (F_, 2 * F_):
        fn = video_calls(ctx, [torch.cat([c] * (n // F_)) for c in clips], n, source)[0][kind]
        fn()
        torch.cuda.synchronize()
        ctx.launch_count(reset=True)
        fn()
        torch.cuda.synchronize()
        counts.append(ctx.launch_count())
    return (counts[1] - counts[0]) / F_


def profile_post(ctx, fns, trace_dir):
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
        prof.export_chrome_trace(os.path.join(trace_dir, f"jpeg_S8_source_{name}.json"))
        busy, post_streams, jpeg_ms = {}, set(), 0.0
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
                if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
                    continue
                busy[e.device_resource_id] = busy.get(e.device_resource_id, 0.0) + e.device_time_total / 1e3
                if "lab_to_rgb8_kernel" in e.name:
                    post_streams.add(e.device_resource_id)
                if "jpeg_" in e.name:
                    jpeg_ms += e.device_time_total / 1e3
        post = sum(busy[s] for s in post_streams)
        res[name] = {"wall_ms": wall, "post_stream_kernel_ms": post, "jpeg_kernel_ms": jpeg_ms}
        print(f"S = 8 source output, {name}: wall {wall:.1f} ms, post stream kernels {post:.1f} ms (JPEG kernels {jpeg_ms:.1f} ms)")
    return res


def folder_rates(n_frames, workers):
    """End-to-end colorize_folder.py on n_frames 1080x1920 PNGs (window output), PNG and device JPEG, and the host Pillow JPEG
    encode of the PNG run's output frames on a pool of the tool's writer count."""
    from PIL import Image

    res = {"host_cores": os.cpu_count(), "workers": workers, "frames": n_frames}
    with tempfile.TemporaryDirectory() as tmp:
        clip, ref = os.path.join(tmp, "clip"), os.path.join(tmp, "ref.png")
        os.makedirs(clip)
        fr = synthetic_frames(11, n_frames).numpy()
        for t in range(n_frames):
            Image.fromarray(fr[t]).save(os.path.join(clip, f"f{t + 1}.png"))
        Image.fromarray(fr[0]).save(ref)
        for fmt in ("png", "jpg"):
            out = os.path.join(tmp, fmt)
            cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", clip, "--ref", ref, "--out", out,
                   "--seeded-weights", "--format", fmt, "--workers", str(workers)]
            t0 = time.perf_counter()
            subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL)
            res[f"folder_{fmt}_frames_per_s"] = n_frames / (time.perf_counter() - t0)
        imgs = [np.asarray(Image.open(os.path.join(tmp, "png", f"f{t + 1}.png")).convert("RGB")) for t in range(n_frames)]

        def enc(x):
            buf = io.BytesIO()
            Image.fromarray(x).save(buf, "JPEG", quality=75)
            return len(buf.getvalue())

        with ThreadPoolExecutor(workers) as pool:
            list(pool.map(enc, imgs[:2]))
            t0 = time.perf_counter()
            list(pool.map(enc, imgs))
            res["host_pillow_jpeg_encode_frames_per_s"] = n_frames / (time.perf_counter() - t0)
    res["note"] = "end to end, including process start, weight upload and PNG decode of the input frames"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--trace", default=None, help="directory: also profile one S = 8 source-output call of each kind")
    ap.add_argument("--folder", action="store_true", help="also time tools/colorize_folder.py end to end")
    ap.add_argument("--folder-frames", type=int, default=48)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    print(f"card: {name}, power limit {power}")
    result = {"card": name, "power_limit": power, "frames": args.frames, "encoder": [], "video": []}
    for (H, W) in ((432, 768), (1080, 1920)):
        for q in (75, 95):
            r = encoder_rate(ctx, H, W, q, args.iters)
            result["encoder"].append(r)
            print(f"encode_jpeg {H}x{W} q{q}: {r['frames_per_s']:.0f} frames/s ({r['ms_per_batch_of_8']:.3f} ms per 8), "
                  f"{r['mean_bytes'] / 1e3:.1f} KB per frame")
    F_ = args.frames
    all_clips = [synthetic_frames(s, F_) for s in range(8)]
    IB = make_lab(40, 8, SIZE[0] // 2, SIZE[1] // 2)
    for S in (1, 8):
        clips = all_clips[:S]
        if S == 1:
            ctx.set_exemplar(IB[:1])
        else:
            ctx.set_exemplars(IB[:S])
        for source in (False, True):
            fns, (h, w), sizes = video_calls(ctx, clips, F_, source)
            for fn in fns.values():
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
            row = {"S": S, "output": f"source {h}x{w}" if source else f"window {h}x{w}"}
            for m in fns:
                down = h * w * 3 if m == "rgb8" else float(sizes.double().mean())
                row[m] = {"frames_per_s": statistics.median(rates[m]), "windows": rates[m], "bytes_down_per_frame": down,
                          "launches_per_frame_step": launches_per_step(ctx, clips, F_, source, m)}
            result["video"].append(row)
            if S == 8 and source and args.trace:
                row["profile"] = profile_post(ctx, fns, args.trace)
    print(f"{HS}x{WS} synthetic pinned clips -> {SIZE[0]}x{SIZE[1]}, {F_} frames per clip, one exemplar each, WLS on, q75; median "
          f"of {args.reps} alternating windows >= {args.window} s")
    print("| S | output | rgb8: frames/s | JPEG: frames/s | JPEG / rgb8 | bytes down per frame (rgb8 / JPEG) | launches per frame "
          "step (rgb8 / JPEG) |")
    print("|---|---|---|---|---|---|---|")
    for r in result["video"]:
        a, b = r["rgb8"], r["jpeg"]
        print(f"| {r['S']} | {r['output']} | {a['frames_per_s']:.1f} | {b['frames_per_s']:.1f} | "
              f"{b['frames_per_s'] / a['frames_per_s']:.3f}x | {a['bytes_down_per_frame']:.0f} / {b['bytes_down_per_frame']:.0f} | "
              f"{a['launches_per_frame_step']:.0f} / {b['launches_per_frame_step']:.0f} |")
    if args.folder:
        result["folder"] = folder_rates(args.folder_frames, min(8, os.cpu_count() or 1))
        print("colorize_folder.py:", json.dumps(result["folder"]))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
