"""Scratch: first-light check of the tensor-core correlation kernel against the CUDA-core one + timing."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))
import torch
import dvc
ctx = dvc.get_context(0)
names = {dvc.MATH_TF32X3: "tf32x3", dvc.MATH_BF16X3: "bf16x3", dvc.MATH_FP16X3: "fp16x3"}
only = sys.argv[1:]
for math in (dvc.MATH_TF32X3, dvc.MATH_BF16X3, dvc.MATH_FP16X3):
    if only and names[math] not in only: continue
    for (NA, NB) in ((128, 256), (300, 517), (1000, 130), (5184, 5184), (25920, 25920)):
        g = torch.Generator().manual_seed(NA + NB)
        th = torch.nn.functional.normalize(torch.randn(1, 256, NA, generator=g), dim=1).cuda()
        ph = torch.nn.functional.normalize(torch.randn(1, 256, NB, generator=g), dim=1).cuda()
        V = (torch.randn(1, NB, 3, generator=g) * 30).cuda()
        f64 = th[0].double().t() @ ph[0].double() if NA * NB <= 5184 * 5184 else None
        for T in (1e-10, 0.01):
            ctx.set_math(corr=dvc.MATH_FP32)
            y0, s0, a0 = ctx.corr_softmax_warp(th, ph, V, T, want_argmax=True)
            ctx.set_math(corr=math)
            y1, s1, a1 = ctx.corr_softmax_warp(th, ph, V, T, want_argmax=True)
            torch.cuda.synchronize()
            msg = f"{names[math]} NA={NA} NB={NB} T={T:g}: |sim-simt| {float((s1-s0).abs().max()):.2e} |y-simt| {float((y1-y0).abs().max()):.2e}"
            if T < 1e-9: msg += f" argmax!=simt {int((a1!=a0).sum())}"
            if f64 is not None:
                m64, i64 = f64.max(1)
                msg += f" |sim-f64| tc {float((s1[0].double()-m64).abs().max()):.2e} simt {float((s0[0].double()-m64).abs().max()):.2e}"
                if T < 1e-9: msg += f" argmax!=f64 tc {int((a1[0]!=i64).sum())} simt {int((a0[0]!=i64).sum())}"
            print(msg, flush=True)
    N = 25920
    th = torch.nn.functional.normalize(torch.randn(1, 256, N, device="cuda"), dim=1); ph = torch.nn.functional.normalize(torch.randn(1, 256, N, device="cuda"), dim=1)
    V = torch.randn(1, N, 3, device="cuda")
    ctx.profile_corr(True)
    for T in (1e-10, 0.01):
        ctx.set_math(corr=math)
        ctx.corr_softmax_warp(th, ph, V, T); ctx.corr_mean_ms(True)
        for _ in range(5): ctx.corr_softmax_warp(th, ph, V, T)
        ms = ctx.corr_mean_ms(True)
        print(f"{names[math]} N=25920 T={T:g}: {ms:.3f} ms (incl. operand split + merge) -> {2*N*N*259/ms/1e9:.1f} TFLOP/s algorithmic", flush=True)
    th8 = torch.nn.functional.normalize(torch.randn(8, 256, N, device="cuda"), dim=1)
    ctx.corr_softmax_warp(th8, ph, V, 1e-10); ctx.corr_mean_ms(True)
    for _ in range(3): ctx.corr_softmax_warp(th8, ph, V, 1e-10)
    ms = ctx.corr_mean_ms(True)
    print(f"{names[math]} B=8 frames vs 1 exemplar N=25920: {ms:.3f} ms -> {8*2*N*N*259/ms/1e9:.1f} TFLOP/s", flush=True)
print("tc check done")
