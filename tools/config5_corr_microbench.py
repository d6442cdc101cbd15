"""BASELINE.json configs[4]: the correlation-only microbench at feature maps 128^2, 256^2, 512^2 (C = 256), both
temperatures -- this library's fused K7 against the reference's own formulation (NonlocalNet.py:477-497:
torch.matmul -> max -> softmax(f / T) -> torch.matmul) run (a) on the same GPU through cuBLAS fp32 (TF32 off) in query-row
chunks that fit HBM, and (b) on this box's CPU cores (a sub-sample of the query rows, scaled; stated in the line).

    python tools/config5_corr_microbench.py [--out gpurun_out/config5_r2.jsonl] [--cpu-rows 2048]

The torch path is the comparison target the survey names (SURVEY.md §8d), not part of the product."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))
import torch

import dvc

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
ap.add_argument("--cpu-rows", type=int, default=2048)
ap.add_argument("--sides", default="128,256,512")
args = ap.parse_args()
torch.backends.cuda.matmul.allow_tf32 = False
ctx = dvc.get_context(0)


def torch_reference(th_rows, ph, V, T, chunk):
    """NonlocalNet.py:477-497 on [rows, C] x [C, N]: returns (y, sim); rows processed `chunk` at a time."""
    ys, sims = [], []
    for r0 in range(0, th_rows.shape[0], chunk):
        f = torch.matmul(th_rows[r0:r0 + chunk], ph)       # 477: f = theta^T phi
        sims.append(f.max(-1).values)                       # 481-483: similarity_map
        p = torch.softmax(f / T, dim=-1)                    # 486-489
        ys.append(torch.matmul(p, V))                       # 496-497
    return torch.cat(ys), torch.cat(sims)


def timed_gpu(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


lines = []
for side in [int(x) for x in args.sides.split(",")]:
    N = side * side
    g = torch.Generator(device="cuda").manual_seed(7)
    th = torch.nn.functional.normalize(torch.randn(1, 256, N, device="cuda", generator=g), dim=1)
    ph = torch.nn.functional.normalize(torch.randn(1, 256, N, device="cuda", generator=g), dim=1)
    V = torch.randn(1, N, 3, device="cuda", generator=g) * 30
    th_rows = th[0].t().contiguous()
    flop = 2.0 * N * N * 259
    chunk = max(256, min(N, (1 << 31) // (4 * N)))  # <= 2 GiB of fp32 scores per chunk (x3 live copies)
    reps = 5 if side <= 256 else 1
    for T in (1e-10, 0.01):
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        ms_ours = timed_gpu(lambda: ctx.corr_softmax_warp(th, ph, V, T), reps)
        y, sim = ctx.corr_softmax_warp(th, ph, V, T)
        ms_torch = timed_gpu(lambda: torch_reference(th_rows, ph[0], V[0], T, chunk), 1 if side == 512 else 3)
        yt, simt = torch_reference(th_rows, ph[0], V[0], T, chunk)
        # CPU: a sub-sample of query rows against the full reference side, scaled to N rows
        rows = min(N, args.cpu_rows)
        thc, phc, Vc = th_rows[:rows].cpu(), ph[0].cpu(), V[0].cpu()
        torch_reference(thc[:256], phc, Vc, T, 256)
        t0 = time.perf_counter()
        torch_reference(thc, phc, Vc, T, 512)
        cpu_ms = (time.perf_counter() - t0) * 1e3 * N / rows
        line = {"config": "BASELINE configs[4] correlation-only", "features": f"{side}x{side}", "N": N, "C": 256, "T": T,
                "ours_ms": ms_ours, "ours_tflops_algorithmic": flop / ms_ours / 1e9, "ours_math": "fp16x3 (T<=2e-10: screened one pass + exact re-scoring)",
                "torch_gpu_ms": ms_torch, "torch_gpu_tflops": flop / ms_torch / 1e9, "torch_gpu_note": f"cuBLAS fp32 (TF32 off), {chunk}-row chunks",
                "speedup_vs_torch_gpu": ms_torch / ms_ours,
                "torch_cpu_ms_scaled": cpu_ms, "torch_cpu_note": f"{rows} of {N} query rows timed on {torch.get_num_threads()} threads, scaled by N/rows",
                "speedup_vs_torch_cpu": cpu_ms / ms_ours,
                "max_abs_sim_diff_vs_torch_gpu": float((sim[0] - simt).abs().max()),
                "max_abs_y_diff_vs_torch_gpu": float((y[0] - yt).abs().max())}
        lines.append(line)
        print(json.dumps(line), flush=True)
    del th, ph, V, th_rows
    torch.cuda.empty_cache()
if args.out:
    with open(args.out, "w") as f:
        for l in lines:
            f.write(json.dumps(l) + "\n")
