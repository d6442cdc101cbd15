"""Precision table: |ab - ab_fp64| of the fused frame path per engine configuration, next to the
reference's own fp32-vs-fp64 distance on the same inputs (tests/golden).  Run on a GPU box:
    python tools/precision_table.py > gpurun_out/precision_table.md
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "deep-exemplar-based-video-colorization_b200"))
import numpy as np, torch
import dvc
from dvc.synth import make_state_dict

ctx = dvc.get_context(0)
for net, key in ((dvc.NET_VGG, "vgg"), (dvc.NET_WARP, "warp"), (dvc.NET_COLOR, "color")):
    ctx.set_weights(net, make_state_dict(key, seed=0))
G = lambda n: dict(np.load(os.path.join(ROOT, "tests", "golden", n + ".npz")))
NAMES = ["small_32x48", "padbranch_40x64", "softmax_32x64", "softmax5_48x48", "default_216x384"]
MODES = [  # label, conv math, f16 planes, kc, cluster, (unused)
    ("CUDA cores, exact fp32 (two-level sums)", dvc.MATH_FP32, 0, 1, 1, 0),
    ("wgmma 3xTF32, chunk 1", dvc.MATH_TF32X3, 0, 1, 2, 0),
    ("wgmma 3xFP16 scaled planes, chunk 1", dvc.MATH_TF32X3, 1, 1, 2, 0),
    ("wgmma 3xFP16 scaled planes, chunk 2", dvc.MATH_TF32X3, 1, 2, 2, 0),
    ("wgmma 3xFP16 scaled planes, chunk 4", dvc.MATH_TF32X3, 1, 4, 2, 0),
]
MODES.append(("wgmma 3xFP16 scaled planes, chunk 8", dvc.MATH_TF32X3, 1, 8, 2, 0))
gs = {n: G(n) for n in NAMES}
print("| engine | " + " | ".join(NAMES) + " | 480x864 ms/frame (one stream) |")
print("|---|" + "---:|" * (len(NAMES) + 1))
floor = [np.abs(gs[n]["ab32"].astype(np.float64) - gs[n]["ab64"]).max() for n in NAMES]
print("| reference fp32 vs fp64 (the noise floor) | " + " | ".join("%.2e" % f for f in floor) + " | |")
from dvc.synth import make_lab
Hb, Wb = 480, 864
IBb = make_lab(60, 1, Hb, Wb); Lb = make_lab(61, 4, Hb, Wb)[:, 0:1].cuda(); lastb = torch.zeros(1, 3, Hb, Wb, device="cuda")
def frame_ms():
    ctx.set_exemplar(IBb)
    for t in range(2): ctx.colorize_frames(Lb[t:t + 1], lastb)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for t in range(4): ctx.colorize_frames(Lb[t:t + 1], lastb)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 4
for label, cm, f16, kc, cl, mb in MODES:
    ctx.set_math(conv=cm, corr=dvc.MATH_FP32 if cm == dvc.MATH_FP32 else dvc.MATH_FP16X3)
    ctx.debug_flag("tc_f16", f16); ctx.debug_flag("tc_kc", kc); ctx.debug_flag("tc_cluster", cl)
    cells = []
    for n, fl in zip(NAMES, floor):
        g = gs[n]
        IA, IB, last = (torch.from_numpy(g[k]) for k in ("IA_lab", "IB_lab", "IA_last_lab"))
        ctx.set_exemplar(IB)
        ab = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), float(g["temperature"]))
        err = np.abs(ab.cpu().numpy().astype(np.float64) - g["ab64"]).max()
        cells.append("%.2e (%.2fx)" % (err, err / fl))
    ms = frame_ms() if cm != dvc.MATH_FP32 else float("nan")
    print("| " + label + " | " + " | ".join(cells) + f" | {ms:.2f} |", flush=True)
