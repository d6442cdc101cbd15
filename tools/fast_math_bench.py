"""The opt-in one-pass convolution mode (DVC_MATH_FP16X1) against the default three-pass mode (TF32X3), on the GPU:

  fused frame  colorize_frames at 480x864, frames resident in HBM, one cached exemplar; windows of at least --window
               seconds alternate between the two modes, the rate is the median over --reps windows
  video        colorize_video_rgb8 over synthetic 720x1280 uint8 sources -> 432x768 (the networks run at 216x384), WLS
               on, K = 1 and 3 exemplars, same alternating windows
  per layer    CUDA-event time of each tensor-core convolution launch (dvc_profile_conv) at the 480x864 frame's geometry,
               through dvc_debug_conv2d, and its TFLOP/s (algorithmic FLOPs: 2 x output pixels x taps x Cin x Cout)
  accuracy     the fused frame at the default 216x384 / 480x864 goldens against fp64: mean |ab - ab64| and the query rows
               whose warped colour differs from fp64's, for both modes and for the fp64 oracle with every convolution
               operand rounded to TF32 (the reference on a GPU, where cuDNN convolutions use TF32 by default)

The card's name and power limit are read in the same run.

    python tools/fast_math_bench.py [--window 1.0] [--reps 3] [--no-accuracy] [--out results/fast_math.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))

import torch  # noqa: E402

T = 1e-10


def set_mode(ctx, mode):
    import dvc

    ctx.set_math(conv={"default": dvc.MATH_TF32X3, "fp16x1": dvc.MATH_FP16X1}[mode], corr=dvc.MATH_FP16X3)


def alternate(run, prepare, window, reps):
    """{mode: [rate per window]}: `prepare(mode)` untimed, then `run()` -> units of work, until the window is full."""
    rates = {"default": [], "fp16x1": []}
    for _ in range(reps):
        for mode in rates:
            prepare(mode)
            run()  # warm-up of the mode's kernels (and its exemplar)
            torch.cuda.synchronize()
            n, t0 = 0, time.perf_counter()
            while True:
                n += run()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                if dt >= window:
                    break
            rates[mode].append(n / dt)
    return rates


def fused_frame(ctx, window, reps):
    from dvc.synth import make_lab

    H, W = 480, 864
    IB, IA, last = make_lab(1, 1, H, W), make_lab(2, 1, H, W), make_lab(3, 1, H, W)
    L, last = IA[:, 0:1].cuda(), last.cuda()

    def prepare(mode):
        set_mode(ctx, mode)
        ctx.set_exemplar(IB)  # a mode change invalidates the cached exemplar

    def run():
        ctx.colorize_frames(L, last, T)
        return 1

    return alternate(run, prepare, window, reps)


def video(ctx, window, reps, K):
    from dvc.synth import make_lab
    from video_bench import HS, SIZE, WS, synthetic_frames

    F_ = 8
    frames = synthetic_frames(F_)
    IB = make_lab(40, K, SIZE[0] // 2, SIZE[1] // 2)
    out = torch.empty(K, F_, SIZE[0], SIZE[1], 3, dtype=torch.uint8).pin_memory()

    def prepare(mode):
        set_mode(ctx, mode)
        ctx.set_exemplar(IB) if K == 1 else ctx.set_exemplars(IB)

    def run():
        ctx.colorize_video_rgb8(frames, SIZE, T, out=out)
        return F_

    assert (HS, WS) == (720, 1280)
    return alternate(run, prepare, window, reps)


# (label, net, name, cin, cout, H, W, kwargs) at the 480x864 frame's geometry
LAYERS = [
    ("full 64->64 (vgg conv1_2)", 0, "conv1_2", 64, 64, 480, 864, dict(act=1)),
    ("full 128->128 (conv10_2 + tail)", 2, "conv10_2", 128, 128, 480, 864, dict(act=2, slope=0.2, fuse_tail=True)),
    ("half 128->128 (vgg conv2_2)", 0, "conv2_2", 128, 128, 240, 432, dict(act=1)),
    ("quarter 256->256 (vgg conv3_2)", 0, "conv3_2", 256, 256, 120, 216, dict(act=1)),
    ("quarter 256->256 reflect+stats (res block)", 1, "layer.0.conv1", 256, 256, 120, 216, dict(reflect=True, want_stats=True)),
    ("eighth 512->512 (vgg conv4_2)", 0, "conv4_2", 512, 512, 60, 108, dict(act=1)),
    ("eighth 512->512 dil 2 (conv5_2)", 2, "conv5_2", 512, 512, 60, 108, dict(act=1, dil=2)),
    ("eighth->quarter upconv 512->256 (conv8_1)", 2, "conv8_1.1", 512, 256, 60, 108, dict(act=1, upconv=True)),
    ("half->full upconv 128->128 (conv10_1)", 2, "conv10_1.1", 128, 128, 240, 432, dict(act=1, upconv=True)),
]


def per_layer(ctx, reps=20):
    rows = []
    for label, net, name, cin, cout, H, W, kw in LAYERS:
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(1, cin, H, W, device="cuda", generator=g).abs()
        row = {"layer": label}
        for mode in ("default", "fp16x1"):
            set_mode(ctx, mode)
            ctx.debug_conv2d(net, name, x, cout, **kw)
            ctx.profile_conv(True)
            ctx.conv_profile(0, reset=True)
            for _ in range(reps):
                ctx.debug_conv2d(net, name, x, cout, **kw)
            torch.cuda.synchronize()
            n, ms, fl = ctx.conv_profile(0, reset=True)
            ctx.profile_conv(False)
            row[mode] = {"us": 1e3 * ms / reps, "tflops": fl / (ms * 1e-3) / 1e12 if ms > 0 else float("nan")}
        row["speedup"] = row["default"]["us"] / row["fp16x1"]["us"]
        rows.append(row)
    return rows


def golden_inputs(g):
    """(IA, IB, last) of a golden: stored, or regenerated from its seed (tests/test_gpu_headline.py)."""
    from dvc.synth import make_lab

    if "IA_lab" in g:
        return tuple(torch.from_numpy(g[k]) for k in ("IA_lab", "IB_lab", "IA_last_lab"))
    seed, (H, W) = int(g["seed"]), g["ab64"].shape[2:]
    return make_lab(seed, 1, H, W), make_lab(seed + 1, 1, H, W), make_lab(seed + 2, 1, H, W) * 0.5


def accuracy(ctx, sds):
    from conftest import load_golden
    from oracle import dvc_oracle as O
    from tf32_reference import tf32_conv_operands

    out = []
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    for name in ("default_216x384", "default_480x864"):
        g = load_golden(name)
        IA, IB, last = golden_inputs(g)
        ab64 = torch.from_numpy(g["ab64"]).double()
        ex, ex_e = {}, {}
        with torch.no_grad():
            O.frame_colorization(sds64, IA.double(), IB.double(), last.double(), O.exemplar_features(sds64["vgg"], IB.double()),
                                 extras=ex)
            with tf32_conv_operands():
                ab_e, _, _, _ = O.frame_colorization(sds64, IA.double(), IB.double(), last.double(),
                                                     O.exemplar_features(sds64["vgg"], IB.double()), extras=ex_e)
        V, am64 = ex["V"][0], ex["argmax"][0]

        def rows_off(colours):  # query rows whose warped colour is not fp64's (indices of equal colours are ambiguous)
            return int(((colours - V[am64]).abs().max(-1).values > 1e-4).sum())

        row = {"frame": name, "emulated_tf32": {"mean_abs_ab": float((ab_e - ab64).abs().mean()),
                                                "rows_off": rows_off(V[ex_e["argmax"][0]])}}
        for mode in ("default", "fp16x1"):
            set_mode(ctx, mode)
            ctx.set_exemplar(IB)
            ab, warp, _ = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T, want_warp=True)
            # at T -> 0 the warp of a query row is the pooled exemplar colour of its argmax
            wd = warp.cpu().double()[0, :, ::4, ::4].reshape(3, -1).t()
            row[mode] = {"mean_abs_ab": float((ab.cpu().double() - ab64).abs().mean()), "rows_off": rows_off(wd)}
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-accuracy", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fast_math_bench: needs a CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dvc
    from video_bench import card
    from oracle.weights import make_state_dict

    ctx = dvc.get_context(0)
    sds = {k: make_state_dict(k, seed=0) for k in ("vgg", "warp", "color")}
    for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
        ctx.set_weights(net, sds[key])
    name, power = card()
    res = {"card": name, "power_limit": power}
    print(f"card: {name}, power limit {power}; median of {args.reps} alternating windows >= {args.window} s", flush=True)
    r = fused_frame(ctx, args.window, args.reps)
    res["fused_480x864_fps"] = {m: {"median": statistics.median(v), "windows": v} for m, v in r.items()}
    print(f"fused frame 480x864: default {statistics.median(r['default']):.2f} frames/s, "
          f"fp16x1 {statistics.median(r['fp16x1']):.2f} frames/s", flush=True)
    for K in (1, 3):
        r = video(ctx, args.window, args.reps, K)
        res[f"video_K{K}_fps"] = {m: {"median": statistics.median(v), "windows": v} for m, v in r.items()}
        print(f"video 720x1280 -> 432x768, K = {K}: default {statistics.median(r['default']):.2f} frames/s, "
              f"fp16x1 {statistics.median(r['fp16x1']):.2f} frames/s", flush=True)
    res["layers"] = per_layer(ctx)
    print("| layer (480x864 frame) | default us | TFLOP/s | fp16x1 us | TFLOP/s | speed-up |")
    print("|---|---|---|---|---|---|")
    for row in res["layers"]:
        d, f = row["default"], row["fp16x1"]
        print(f"| {row['layer']} | {d['us']:.1f} | {d['tflops']:.0f} | {f['us']:.1f} | {f['tflops']:.0f} | {row['speedup']:.2f}x |")
    if not args.no_accuracy:
        res["accuracy"] = accuracy(ctx, sds)
        print("| frame | mode | mean abs(ab - ab64) | query rows whose warped colour differs from fp64 |")
        print("|---|---|---|---|")
        for row in res["accuracy"]:
            for m in ("default", "fp16x1", "emulated_tf32"):
                print(f"| {row['frame']} | {m} | {row[m]['mean_abs_ab']:.3e} | {row[m]['rows_off']} |")
    set_mode(ctx, "default")
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
