"""Oracle parity AT the headline configuration (run with -m gpu on an H100).

BASELINE.json configs[1] (480x854 padded to 480x864, N = 25920 positions -- the size bench.py measures) and configs[0]
(256x256), against golden outputs of the UNMODIFIED reference run in fp32 and fp64 by oracle/make_golden.py
(tests/golden/default_480x864.npz, cfg1_256x256.npz; the inputs are regenerated from the stored seed).  At this size the
launcher runs the 512-channel layers on 128-channel tiles over more than one round of 2-CTA clusters and the correlation
on a multi-split grid, neither of which the small goldens reach.

Gates (SURVEY.md §8c): similarity |d| < 2e-5; tie-aware argmax (rows whose fp64 top-2 gap > 1e-5 must warp to the
fp64 colour); ab within max(1e-3, 1.25 x floor) of the fp64 reference, where floor = |ab32_tf - ab64| is the reference's
own fp32 ColorVidNet on the same (fp64) warp -- at N = 25920 a single near-tie row whose fp32 / fp64 argmax differ moves
the reference's own ab32 by O(10), so the raw |ab32 - ab64| is not a noise floor there (PIN_REPORT.txt).
"""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu

CASES = [("default_480x864", 480, 864), ("cfg1_256x256", 256, 256)]


def inputs(g, H, W):
    seed = int(g["seed"])
    return make_lab(seed, 1, H, W), make_lab(seed + 1, 1, H, W), make_lab(seed + 2, 1, H, W) * 0.5


@pytest.fixture(params=["fp32", "tf32x3"])
def engine(request, ctx):
    """The exact-fp32 CUDA-core engines and the default tensor-core engines (3xFP16 CTA pairs, launcher's own tiles)."""
    import dvc

    if request.param == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32)
    else:
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    yield request.param
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)


@pytest.mark.parametrize("name,H,W", CASES)
def test_fused_frame_vs_reference_at_full_size(ctx, engine, name, H, W):
    g = load_golden(name)
    IA, IB, last = inputs(g, H, W)
    T = float(g["temperature"])
    ctx.set_exemplar(IB)
    if engine == "tf32x3":
        ctx.profile_conv(True)
        ctx.conv_profile(0, reset=True)
    ab, warp, sim = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), T, want_warp=True)
    torch.cuda.synchronize()
    if engine == "tf32x3":
        n128 = ctx.conv_profile(128)[0]
        ctx.conv_profile(0, reset=True)
        ctx.profile_conv(False)
        if H == 480:  # the 1/8-resolution 512-channel layers among them
            assert n128 >= 12, f"only {n128} launches ran on the 128-channel tile: this test must cover the bench's engine"
    ss = sim.cpu().numpy()[:, :, ::4, ::4]
    ys = warp.cpu().numpy()[:, :, ::4, ::4].reshape(1, 3, -1)
    e_sim = np.abs(ss - g["sim64"]).max()
    assert e_sim < 2e-5, e_sim
    w64, w32 = g["warped64"].reshape(1, 3, -1), g["warped32"].reshape(1, 3, -1)
    clear = g["gap64"] > 1e-5
    m = np.broadcast_to(clear[:, None, :], ys.shape)
    nbad = int((np.abs(ys[m] - w64[m]) > 1e-4).sum())
    assert nbad == 0, f"{nbad} warped values differ from the fp64 reference on rows with a clear argmax"
    # ab: against whichever reference run chose the same near-tie rows as we did
    floor = np.abs(g["ab32_tf"].astype(np.float64) - g["ab64"]).max()
    ours = ab.cpu().numpy().astype(np.float64)
    same64 = np.abs(ys - w64).max() < 1e-4
    same32 = np.abs(ys - w32).max() < 1e-4
    e64, e32 = np.abs(ours - g["ab64"]).max(), np.abs(ours - g["ab32"].astype(np.float64)).max()
    print(f"{name}/{engine}: |sim-ref64| {e_sim:.2e}; rows equal to fp64 run: {same64}, to fp32 run: {same32}; "
          f"|ab-ab64| {e64:.3e} |ab-ab32| {e32:.3e} floor {floor:.3e}; near-tie rows {int((~clear).sum())}")
    if same64:
        assert e64 <= max(1e-3, 1.25 * floor), (e64, floor)
    elif same32:  # ours and the fp32 reference are each within the band of the (unavailable) fp64 run on these rows
        assert e32 <= max(2e-3, 2.25 * floor), (e32, floor)
    # else: a near-tie row resolved differently from both reference runs -- legal under the tie-aware metric; the
    # colour network is then checked by the teacher-forced test below


@pytest.mark.parametrize("name,H,W", CASES)
def test_colorvidnet_teacher_forced_at_full_size(ctx, engine, name, H, W):
    """ColorVidNet.forward on the reference's own fp64 warp / similarity (FrameColor.py:63-65) at full size."""
    g = load_golden(name)
    IA, _, last = inputs(g, H, W)
    up = lambda a: torch.nn.functional.interpolate(torch.from_numpy(a).float(), scale_factor=4, mode="nearest")
    x = torch.cat((IA[:, 0:1], up(g["warped64"])[:, 1:3], up(g["sim64"]), last), 1)
    out = ctx.colorvidnet_forward(x.cuda()).cpu().numpy().astype(np.float64)
    floor = np.abs(g["ab32_tf"].astype(np.float64) - g["ab64"]).max()
    err = np.abs(out - g["ab64"]).max()
    print(f"{name}/{engine}: teacher-forced |ab-ab64| {err:.3e} floor {floor:.3e} ({err / floor:.2f}x)")
    assert err <= max(1e-3, 1.25 * floor), (err, floor)


# ------------------------------------------------------------------------------------------ K7 at N = 25920
@pytest.fixture(scope="module")
def corr_oracle_25920():
    """fp64 scores of 25920 x 25920 unit vectors in row chunks (never materialised whole): sim, argmax, top-2 gap and
    the softmax-weighted colours at T = 0.01 (NonlocalNet.py:477-498)."""
    N, T = 25920, 0.01
    gen = torch.Generator().manual_seed(77)
    th = torch.nn.functional.normalize(torch.randn(1, 256, N, generator=gen), dim=1)
    ph = torch.nn.functional.normalize(torch.randn(1, 256, N, generator=gen), dim=1)
    # correlated content: every query is a noisy copy of some reference position (like a frame and its exemplar)
    perm = torch.randperm(N, generator=gen)
    th = torch.nn.functional.normalize(0.6 * ph[:, :, perm] + 0.8 * th, dim=1)
    V = torch.randn(1, N, 3, generator=gen) * 30
    th64, ph64, V64 = th.double(), ph.double(), V.double()
    sims, idxs, gaps, ys = [], [], [], []
    for r0 in range(0, N, 2160):
        f = torch.matmul(th64[0, :, r0:r0 + 2160].t(), ph64[0])
        t2 = torch.topk(f, 2, dim=-1)
        sims.append(t2.values[:, 0]), idxs.append(t2.indices[:, 0]), gaps.append(t2.values[:, 0] - t2.values[:, 1])
        ys.append(torch.softmax(f / T, dim=-1) @ V64[0])
    return dict(th=th, ph=ph, V=V, T=T, sim=torch.cat(sims), idx=torch.cat(idxs), gap=torch.cat(gaps), y=torch.cat(ys))


@pytest.mark.parametrize("mode", ["fp16x3", "fp16x3-single", "fp16x3-noscreen", "tf32x3", "bf16x3", "fp32"])
def test_corr_kernel_vs_oracle_25920(ctx, corr_oracle_25920, mode):
    """The 204 row blocks x 5 column splits of the bench's correlation launch, against the chunked fp64 oracle."""
    import dvc

    o = corr_oracle_25920
    name = mode.replace("-single", "").replace("-noscreen", "")
    ctx.debug_flag("corr_screen", 0 if "noscreen" in mode else 1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr={"fp32": dvc.MATH_FP32, "tf32x3": dvc.MATH_TF32X3, "bf16x3": dvc.MATH_BF16X3,
                                              "fp16x3": dvc.MATH_FP16X3}[name])
    ctx.debug_flag("corr_cluster", 1 if mode.endswith("-single") else 2)
    try:
        th, ph, V = o["th"].cuda(), o["ph"].cuda(), o["V"].cuda()
        y, sim, am = ctx.corr_softmax_warp(th, ph, V, 1e-10, want_argmax=True)
        tol = 8e-6 if name == "bf16x3" else 2e-6
        e_sim = (sim.cpu().double()[0] - o["sim"]).abs().max().item()
        assert e_sim < tol, e_sim
        clear = o["gap"] > 4 * tol
        assert clear.float().mean() > 0.99
        assert (am.cpu()[0][clear].long() == o["idx"][clear]).all()
        assert torch.equal(y.cpu()[0][clear], o["V"][0][o["idx"][clear]])
        y2, sim2 = ctx.corr_softmax_warp(th, ph, V, o["T"])
        e_y = (y2.cpu().double()[0] - o["y"]).abs().max().item()
        print(f"N=25920 {mode}: |sim-f64| {e_sim:.2e}, softmax(T=0.01) |y-f64| {e_y:.2e}")
        assert (sim2.cpu().double()[0] - o["sim"]).abs().max().item() < tol
        assert e_y < (2e-2 if name == "bf16x3" else 2e-3)
    finally:
        ctx.debug_flag("corr_cluster", 2)
        ctx.debug_flag("corr_screen", 1)
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
