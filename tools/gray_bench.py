"""Greyscale sources: aggregate frames/s of dvc_colorize_videos_gray8 on grey clips against the sRGB calls on the same frames with
each byte repeated into R, G and B (the bytes of both are equal, include/dvc.h).  Workload: S = 1 and S = 8 synthetic 1080x1920
grey clips of --frames frames in pinned host memory, one exemplar each, CenterPad'ed to 432x768 (test.py's default size; the
networks run at 216x384), seeded weights, WLS on (lambda 500, sigma 4), the default conv arithmetic; window output
(dvc_colorize_videos_exemplars_rgb8) and source-resolution output (dvc_colorize_videos_source_rgb8).

Method (tools/source_resolution_bench.py's): after a warm-up, windows of at least --window seconds alternate between the sRGB
call and the grey call; each window runs whole calls and ends with a device synchronisation; the rate is the median over --reps
windows.  Bytes up per frame and the ingest workspaces (vid.src: two upload slots, vid.f0 / vid.f1: the float64 resize planes)
are counted from the shapes.  Kernel launches per frame step are dvc_launch_count over a call of 2F frames minus one of F
frames, divided by F.  The card's name and power limit are read in the same run.

    python tools/gray_bench.py [--frames 16] [--window 1.0] [--reps 3] [--trace DIR] [--folder] [--folder-frames 48]

--trace DIR additionally profiles one call of each input per S and output with torch.profiler (a separate run after the timed
windows), writes the traces there and prints the summed kernel time per frame of the ingest stream (the one running
zoom_crop_kernel).  --folder times tools/colorize_folder.py --format jpg end to end on --folder-frames 1080x1920 mode-"L" PNGs
against the same frames saved as RGB PNGs (alternating, median of 3 runs each; process start and weight loading included).
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"), os.path.dirname(os.path.abspath(__file__))):
    sys.path.insert(0, p)

import numpy as np
import torch

from clips_bench import card

HS, WS, SIZE, T, WLS = 1080, 1920, (432, 768), 1e-10, (500.0, 4.0)


def gray_frames(seed, F):
    rng = np.random.default_rng(seed)
    coarse = (rng.random((F, HS // 16 + 1, WS // 16 + 1)) * 255).astype(np.int16)
    img = np.kron(coarse, np.ones((1, 16, 16), np.int16))[:, :HS, :WS]
    return torch.from_numpy(np.clip(img + rng.integers(-12, 13, img.shape, dtype=np.int16), 0, 255).astype(np.uint8))


def calls(ctx, gray, rgb, F_, output):
    """{"rgb": the sRGB call on the replicated frames, "gray": the grey call}, both writing into pinned outputs."""
    import dvc
    from dvc.prepost import centerpad_geometry

    S, K = len(gray), [1] * len(gray)
    if output == "window":
        out = torch.empty(S, F_, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory()
        return {"rgb": lambda: ctx.colorize_videos_exemplars_rgb8(rgb, K, SIZE, T, wls=WLS, out=out),
                "gray": lambda: ctx.colorize_videos_gray8(gray, K, SIZE, T, wls=WLS, out=out)}
    _, _, h, w = dvc.source_footprint(HS, WS, *centerpad_geometry(HS, WS, SIZE), *SIZE)
    out = [torch.empty(1, F_, h, w, 3, dtype=torch.uint8).pin_memory() for _ in range(S)]
    return {"rgb": lambda: ctx.colorize_videos_source_rgb8(rgb, K, SIZE, T, wls=WLS, out=out),
            "gray": lambda: ctx.colorize_videos_gray8(gray, K, SIZE, T, wls=WLS, source_resolution=True, out=out)}


def launches_per_step(ctx, gray, rgb, F_, output, kind):
    counts = []
    for n in (F_, 2 * F_):
        g, r = [torch.cat([c] * (n // F_)).pin_memory() for c in gray], [torch.cat([c] * (n // F_)).pin_memory() for c in rgb]
        fn = calls(ctx, g, r, n, output)[kind]
        fn()
        torch.cuda.synchronize()
        ctx.launch_count(reset=True)
        fn()
        torch.cuda.synchronize()
        counts.append(ctx.launch_count())
    return (counts[1] - counts[0]) / F_


def ingest_stream_ms(ctx, fns, F_, S, trace_dir, tag):
    """Summed kernel time per frame step of the stream that runs zoom_crop_kernel, per input kind."""
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(trace_dir, exist_ok=True)
    res = {}
    for name, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        prof.export_chrome_trace(os.path.join(trace_dir, f"gray_{tag}_{name}.json"))
        busy, ingest = collections.defaultdict(float), set()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
                if e.name.startswith("Memcpy") or e.name.startswith("Memset"):
                    continue
                busy[e.device_resource_id] += e.device_time_total / 1e3
                if "zoom_crop_kernel" in e.name:
                    ingest.add(e.device_resource_id)
        res[name] = sum(busy[s] for s in ingest) / F_
        print(f"{tag}, {name}: ingest stream kernels {res[name]:.3f} ms per frame step ({S} clip frames)")
    return res


def folder_rates(n_frames, reps):
    from PIL import Image

    res = {"frames": n_frames, "gray": [], "rgb": []}
    with tempfile.TemporaryDirectory() as tmp:
        fr = gray_frames(21, n_frames).numpy()
        for kind in ("gray", "rgb"):
            d = os.path.join(tmp, kind)
            os.makedirs(d)
            for t in range(n_frames):
                img = Image.fromarray(fr[t])
                (img if kind == "gray" else img.convert("RGB")).save(os.path.join(d, f"f{t + 1}.png"))
        ref = os.path.join(tmp, "ref.png")
        Image.fromarray(np.random.default_rng(22).integers(0, 256, (HS, WS, 3), dtype=np.uint8)).save(ref)
        for _ in range(reps):
            for kind in ("rgb", "gray"):
                cmd = [sys.executable, os.path.join(ROOT, "tools", "colorize_folder.py"), "--clip", os.path.join(tmp, kind), "--ref", ref,
                       "--out", os.path.join(tmp, "out_" + kind), "--seeded-weights", "--format", "jpg"]
                t0 = time.perf_counter()
                subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL)
                res[kind].append(n_frames / (time.perf_counter() - t0))
    res["gray_frames_per_s"], res["rgb_frames_per_s"] = statistics.median(res["gray"]), statistics.median(res["rgb"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--trace", default=None, help="directory: also profile one call of each kind")
    ap.add_argument("--folder", action="store_true", help="also time tools/colorize_folder.py --format jpg end to end")
    ap.add_argument("--folder-frames", type=int, default=48)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gray_bench: needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = card()
    print(f"card: {name}, power limit {power}")
    F_ = args.frames
    all_gray = [gray_frames(s, F_) for s in range(8)]
    all_rgb = [g[..., None].repeat(1, 1, 1, 3).pin_memory() for g in all_gray]
    all_gray = [g.pin_memory() for g in all_gray]
    IB = make_lab(40, 8, SIZE[0] // 2, SIZE[1] // 2)
    rows = []
    for S in (1, 8):
        gray, rgb = all_gray[:S], all_rgb[:S]
        if S == 1:
            ctx.set_exemplar(IB[:1])
        else:
            ctx.set_exemplars(IB[:S])
        for output in ("window", "source"):
            fns = calls(ctx, gray, rgb, F_, output)
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
            row = {"S": S, "output": output}
            for m in fns:
                C = 1 if m == "gray" else 3
                ns = HS * WS * C
                row[m] = {"frames_per_s": statistics.median(rates[m]), "windows": rates[m], "pcie_up_bytes_per_frame": ns,
                          "launches_per_frame_step": launches_per_step(ctx, gray, rgb, F_, output, m),
                          "ingest_workspace_bytes": {"src": 2 * S * ns, "f0": 8 * ns, "f1": 8 * ns}}
            if args.trace:
                row["ingest_stream_ms_per_step"] = ingest_stream_ms(ctx, fns, F_, S, args.trace, f"S{S}_{output}")
            rows.append(row)
    print(f"{HS}x{WS} synthetic grey pinned clips -> {SIZE[0]}x{SIZE[1]}, {F_} frames per clip, one exemplar each, WLS on, default "
          f"conv math; sRGB call on the frames repeated into R, G, B against the grey call; median of {args.reps} alternating "
          f"windows >= {args.window} s")
    print("| S | output | sRGB: frames/s | grey: frames/s | grey / sRGB | bytes up per frame (sRGB / grey) | launches per frame step "
          "(sRGB / grey) |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        a, b = r["rgb"], r["gray"]
        print(f"| {r['S']} | {r['output']} | {a['frames_per_s']:.1f} | {b['frames_per_s']:.1f} | "
              f"{b['frames_per_s'] / a['frames_per_s']:.3f}x | {a['pcie_up_bytes_per_frame']} / {b['pcie_up_bytes_per_frame']} | "
              f"{a['launches_per_frame_step']:.0f} / {b['launches_per_frame_step']:.0f} |")
    result = {"card": name, "power_limit": power, "frames": F_, "rows": rows}
    if args.folder:
        result["folder_jpg"] = folder_rates(args.folder_frames, 3)
        print("colorize_folder.py --format jpg:", json.dumps(result["folder_jpg"]))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
