"""Several exemplars for one clip: one colorize_clip_exemplars call against K back-to-back colorize_clip calls.

test.py:168-181 colorizes the whole clip once per reference image; the multi-exemplar path computes the exemplar-independent
half of every frame (VGG19, feature_normalize, the WarpNet query side) once and runs the correlation and ColorVidNet at
batch K.  Both arms include their exemplar prologues (set_exemplars vs K set_exemplar calls), as a user of either pays
them once per clip.  Frames are resident in HBM and seeded (dvc.synth), so PCIe is out of the picture.

    python tools/exemplars_bench.py [--frames 16] [--min-window 1.0]

One JSON line per (size, K): ms per frame step (one frame for all K exemplars) of each arm, their ratio, library kernel
launches per frame step, max |ab difference| between the arms on frame 0 (ColorVidNet runs at batch K in one arm and at
batch 1 in the other: fp32 InstanceNorm summation order and device-derived fp16 scales), and the GPU's name and power limit
read in the same run.  Each arm is timed over windows of at least --min-window seconds with CUDA events, the arms
alternating, three times; the median window is reported.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))

import torch


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        power = out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--min-window", type=float, default=1.0, help="seconds per timed window")
    ap.add_argument("--sizes", default="216x384,480x864")
    ap.add_argument("--ks", default="1,2,4")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("exemplars_bench needs a CUDA device")

    import dvc
    from dvc.synth import make_lab, make_state_dict

    ctx = dvc.get_context(0)
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, make_state_dict(key, seed=0))
    name, power = gpu_info()
    F_ = args.frames

    for size in args.sizes.split(","):
        H, W = (int(v) for v in size.split("x"))
        L = make_lab(500, F_, H, W)[:, 0:1].contiguous().cuda()
        for K in (int(v) for v in args.ks.split(",")):
            IB = make_lab(600 + K, K, H, W).cuda()
            seq_out = [torch.empty(F_, 2, H, W, device="cuda") for _ in range(K)]
            multi_out = torch.empty(K, F_, 2, H, W, device="cuda")

            def multi():
                ctx.set_exemplars(IB)
                ctx.colorize_clip_exemplars(L, out=multi_out)

            def sequential():
                for k in range(K):
                    ctx.set_exemplar(IB[k:k + 1])
                    ctx.colorize_clip(L, out=seq_out[k])

            arms = {"multi": multi, "sequential": sequential}
            for fn in arms.values():  # warm-up: every shape, workspace and kernel attribute of both arms
                fn()
            torch.cuda.synchronize()
            launches = {}
            for arm, fn in arms.items():
                ctx.launch_count(reset=True)
                fn()
                launches[arm] = ctx.launch_count() / F_
            dab = max(float((multi_out[k, 0] - seq_out[k][0]).abs().max()) for k in range(K))
            reps = {}
            for arm, fn in arms.items():  # calls per window from one timed call
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                reps[arm] = max(1, int(args.min_window * 1000.0 / e0.elapsed_time(e1)) + 1)
            ms = {arm: [] for arm in arms}
            for _ in range(3):
                for arm, fn in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps[arm]):
                        fn()
                    e1.record()
                    e1.synchronize()
                    ms[arm].append(e0.elapsed_time(e1) / (reps[arm] * F_))
            med = {arm: sorted(v)[1] for arm, v in ms.items()}
            print(json.dumps({
                "H": H, "W": W, "K": K, "frames": F_,
                "multi_ms_per_frame_step": round(med["multi"], 3), "sequential_ms_per_frame_step": round(med["sequential"], 3),
                "speedup": round(med["sequential"] / med["multi"], 3),
                "multi_runs_ms": [round(v, 3) for v in ms["multi"]], "sequential_runs_ms": [round(v, 3) for v in ms["sequential"]],
                "launches_per_frame_step": {k: round(v, 1) for k, v in launches.items()},
                "max_abs_dab_frame0": dab, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
