"""Scratch: precision budget of the fp32 CUDA path (plain vs two-level accumulation) against the fp64 oracle."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))
import numpy as np, torch
import dvc
from oracle import dvc_oracle as O
from oracle.weights import make_lab, make_state_dict

sds = {k: make_state_dict(k, seed=0) for k in ("vgg", "warp", "color")}
sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
ctx = dvc.get_context(0)
for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
    ctx.set_weights(net, sds[key])
G = lambda n: dict(np.load(os.path.join(ROOT, "tests", "golden", n + ".npz")))

def run(H, W, seed, tl):
    if tl >= 20:
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_TF32X3); ctx.debug_flag("tc_kc", tl - 20)
    else:
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32)
        ctx.debug_flag("two_level", tl)
    IA, IB, last = make_lab(seed, 1, H, W), make_lab(seed + 1, 1, H, W), make_lab(seed + 2, 1, H, W)
    ex64, ex32 = {}, {}
    with torch.no_grad():
        fB = O.exemplar_features(sds64["vgg"], IB.double())
        ab64, w64, s64, fA64 = O.frame_colorization(sds64, IA.double(), IB.double(), last.double(), fB, extras=ex64)
        fB32 = O.exemplar_features(sds["vgg"], IB)
        ab32, w32, s32, fA32 = O.frame_colorization(sds, IA, IB, last, fB32, extras=ex32)
    gap = O.top2_gap(ex64["theta_hat"], ex64["phi_hat"])[0]
    ctx.set_exemplar(IB)
    ab, warp, sim = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), 1e-10, want_warp=True)
    N = (H // 4) * (W // 4)
    print(f"  (mode {tl}: 0 plain fp32, 1 two-level fp32, 2x wgmma tf32x3 with kc = x)")
    th = ctx.debug_buffer("fr.theta", act=False)[: N * 256].view(N, 256).t().cpu().double()
    ph = ctx.debug_buffer("ex.phi", act=False)[: N * 256].view(N, 256).t().cpu().double()
    e_th = (th - ex64["theta_hat"][0]).abs().max().item(); e_th32 = (ex32["theta_hat"][0].double() - ex64["theta_hat"][0]).abs().max().item()
    e_ph = (ph - ex64["phi_hat"][0]).abs().max().item(); e_ph32 = (ex32["phi_hat"][0].double() - ex64["phi_hat"][0]).abs().max().item()
    # argmax of our operands in fp64 vs oracle
    f_ours = th.t() @ ph
    am_ours = f_ours.argmax(1); am64 = ex64["argmax"][0]
    flips = (am_ours != am64)
    wr = warp.cpu()[0, :, ::4, ::4].reshape(3, -1).t()
    w64r = w64.float()[0, :, ::4, ::4].reshape(3, -1).t()
    kflips = (wr != w64r).any(1)
    print(f"[{H}x{W} two_level={tl}] theta err ours {e_th:.2e} (cpu32 {e_th32:.2e})  phi err ours {e_ph:.2e} (cpu32 {e_ph32:.2e})")
    print(f"    argmax flips from operand error: {int(flips.sum())} (min gap among flips {gap[flips].min().item() if flips.any() else float('nan'):.2e}); kernel-output flips {int(kflips.sum())} max gap {gap[kflips].max().item() if kflips.any() else float('nan'):.2e}; cpu32 flips {int((ex32['argmax'][0]!=am64).sum())}")
    print(f"    sim err {float((sim.cpu().double()-s64).abs().max()):.2e}  |ab-ab64| ours {float((ab.cpu().double()-ab64).abs().max()):.2e}  cpu32 {float((ab32.double()-ab64).abs().max()):.2e}")
    # stage maps
    for nm, ref in (("fr.r22", fA64[1]), ("fr.r52", fA64[4])):
        t = ctx.debug_buffer(nm).cpu().double()
        print(f"    {nm} rel err ours {float((t-ref).abs().max()/ref.abs().max()):.2e}  cpu32 {float((fA32[int(nm[-2])-1].double()-ref).abs().max()/ref.abs().max()):.2e}")

MODES = [int(a) for a in sys.argv[1:]] or [1, 2]
for tl in MODES:
    for name in ("small_32x48", "padbranch_40x64"):
        g = G(name)
        if tl >= 20:
            ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_TF32X3); ctx.debug_flag("tc_kc", tl - 20)
        else:
            ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32); ctx.debug_flag("two_level", tl)
        IA, last = torch.from_numpy(g["IA_lab"]), torch.from_numpy(g["IA_last_lab"])
        up = lambda a: torch.nn.functional.interpolate(torch.from_numpy(a), scale_factor=4, mode="nearest")
        x = torch.cat((IA[:, 0:1], up(g["warped32"])[:, 1:3], up(g["sim32"]), last), 1)
        out = ctx.colorvidnet_forward(x.cuda()).cpu().numpy()
        print(f"[{name} two_level={tl}] colorvidnet(golden input) |out-ab64| {np.abs(out-g['ab64']).max():.3e} floor {np.abs(g['ab32']-g['ab64']).max():.3e}")
    run(64, 64, 70, tl)
    run(216, 384, 606, tl)
# timing impact
H, W = 480, 864
ctx.set_exemplar(make_lab(60, 1, H, W)); L = make_lab(61, 1, H, W)[:, 0:1].cuda(); last = torch.zeros(1, 3, H, W, device="cuda")
for tl in MODES:
    if tl >= 20:
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_TF32X3); ctx.debug_flag("tc_kc", tl - 20)
    else:
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32); ctx.debug_flag("two_level", tl)
    ctx.set_exemplar(make_lab(60, 1, H, W))
    for _ in range(2): ctx.colorize_frames(L, last)
    torch.cuda.synchronize(); e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True); e0.record()
    for _ in range(3): ctx.colorize_frames(L, last)
    e1.record(); torch.cuda.synchronize(); print(f"480x864 two_level={tl}: {e0.elapsed_time(e1)/3:.2f} ms/frame")
