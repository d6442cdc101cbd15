"""Several exemplars for one clip (include/dvc.h: dvc_set_exemplars and the *_exemplars entry points), the capability
behind test.py:168-181, which colorizes the whole clip once per reference image.  Exemplar k's results must be those of
frame_colorization(IA_t, IB_k, last_k) with last_k = cat(L_t, ab_k,t-1) (test.py:96): checked against the
single-exemplar path (bit for bit wherever the arithmetic is the same) and against the fp64 oracle."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import dvc_oracle as O
from oracle.weights import make_lab

pytestmark = pytest.mark.gpu
nrm = torch.nn.functional.normalize


@pytest.fixture(params=["fp32", "tf32x3", "tf32x3-nof16"])
def conv_math(request, ctx):
    """The exact CUDA-core engines, and the tensor-core convolutions with and without the fp16 planes of bounded layers."""
    import dvc

    if request.param == "fp32":
        ctx.set_math(conv=dvc.MATH_FP32, corr=dvc.MATH_FP32)
    else:
        ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
        ctx.debug_flag("tc_f16", 0 if request.param.endswith("nof16") else 1)
    yield request.param
    ctx.debug_flag("tc_f16", 1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)


@pytest.fixture(params=["fp32", "tf32x3", "bf16x3", "fp16x3", "tf32x3-single", "fp16x3-single", "fp16x3-noscreen",
                        "fp16x3-noscreen-single"])
def corr_math(request, ctx):
    """Every correlation arithmetic, as 2-CTA clusters and single CTAs; fp16x3 at T -> 0 screens unless "-noscreen"."""
    import dvc

    name = request.param.replace("-single", "").replace("-noscreen", "")
    mode = {"fp32": dvc.MATH_FP32, "tf32x3": dvc.MATH_TF32X3, "bf16x3": dvc.MATH_BF16X3, "fp16x3": dvc.MATH_FP16X3}[name]
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=mode)
    ctx.debug_flag("corr_cluster", 1 if request.param.endswith("-single") else 2)
    ctx.debug_flag("corr_screen", 0 if "noscreen" in request.param else 1)
    yield name
    ctx.debug_flag("corr_cluster", 2)
    ctx.debug_flag("corr_screen", 1)
    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)


def _rc(err):
    """dvc_status of a DvcError ("... failed (rc): text")."""
    return int(str(err).split("(")[1].split(")")[0])


# ------------------------------------------------------------------------------------------ K = 1
def test_one_exemplar_is_the_single_path(ctx, conv_math):
    g = load_golden("clip3_32x48")
    frames, IB = torch.from_numpy(g["frames_lab"]), torch.from_numpy(g["IB_lab"])
    L = frames[:, 0:1].contiguous()
    last = torch.from_numpy(g["frames_lab"][:1]).cuda() * 0.5
    ctx.set_exemplar(IB)
    ref = ctx.colorize_clip(L.pin_memory())
    ref_ab, ref_warp, ref_sim = ctx.colorize_frames(L[:1].cuda(), last, want_warp=True)
    for setter in (ctx.set_exemplar, ctx.set_exemplars):
        setter(IB)
        out = ctx.colorize_clip_exemplars(L.pin_memory())
        assert out.shape == (1,) + tuple(ref.shape) and torch.equal(out[0], ref)
        ab, warp, sim = ctx.colorize_frames_exemplars(L[:1].cuda(), last, want_warp=True)
        assert torch.equal(ab, ref_ab) and torch.equal(warp, ref_warp) and torch.equal(sim, ref_sim)


# ------------------------------------------------------------------------------------------ correlation
@pytest.mark.parametrize("NA,NB,K,T", [(96, 96, 3, 1e-10), (300, 517, 2, 1e-10), (300, 517, 3, 0.01), (1000, 130, 5, 0.005),
                                       (5184, 5184, 2, 1e-10)])
def test_corr_exemplars_vs_single_and_oracle(ctx, corr_math, NA, NB, K, T):
    gen = torch.Generator().manual_seed(NA + 7 * K)
    th = nrm(torch.randn(1, 256, NA, generator=gen), dim=1)
    ph = nrm(torch.randn(K, 256, NB, generator=gen), dim=1)
    V = torch.randn(K, NB, 3, generator=gen) * 30
    y, sim, am = ctx.corr_softmax_warp_exemplars(th.cuda(), ph.cuda(), V.cuda(), T, want_argmax=True)
    assert y.shape == (K, NA, 3) and sim.shape == (K, NA) and am.shape == (K, NA)
    tol = 8e-6 if corr_math == "bf16x3" else 2e-6  # as test_corr_kernel_vs_oracle
    for k in range(K):
        y1, s1, a1 = ctx.corr_softmax_warp(th.cuda(), ph[k:k + 1].cuda(), V[k:k + 1].cuda(), T, want_argmax=True)
        # the scores are the same products in the same order whatever the batch: the row maxima are bit-equal
        assert torch.equal(sim[k], s1[0])
        yo, so, io = O.corr_softmax_warp(th.double(), ph[k:k + 1].double(), V[k:k + 1].double(), T, return_argmax=True)
        gap = O.top2_gap(th.double(), ph[k:k + 1].double())[0]
        assert (sim[k].cpu().double() - so[0]).abs().max() < tol
        if T < 1e-9:
            assert torch.equal(am[k], a1[0])
            unique = gap > 1e-6  # a unique maximum: y is that V row exactly in both calls
            assert torch.equal(y[k][unique.cuda()], y1[0][unique.cuda()])
            clear = gap > 4 * tol
            assert (am.cpu()[k][clear] == io[0][clear]).all()
            assert torch.equal(y.cpu()[k][clear], V[k][io[0][clear]])
        else:
            # a different column-split count is a different summation order of the softmax weights
            assert (y[k] - y1[0]).abs().max() < 1e-4
            assert (y.cpu()[k].double() - yo[0]).abs().max() < (2e-2 if corr_math == "bf16x3" else 2e-3)


def test_corr_exemplars_duplicated_columns_in_one_slot(ctx, corr_math):
    """Bit-equal maxima in slot 1 only (duplicated exemplar columns): averaged there as the reference's softmax(f / 1e-10)
    does (test_corr_duplicated_exemplar_columns_average); slot 0 is unaffected."""
    gen = torch.Generator().manual_seed(19)
    NA, NB = 300, 700
    ph = nrm(torch.randn(2, 256, NB, generator=gen), dim=1)
    dup = [3, 150, 151, 400, 699]
    ph[1:, :, dup] = ph[1:, :, 3:4]
    ph[1:, :, [20, 21]] = ph[1:, :, 20:21]
    th = nrm(torch.randn(1, 256, NA, generator=gen), dim=1)
    th[:, :, :40] = nrm(ph[1:, :, 3:4] + 0.05 * th[:, :, :40], dim=1)
    th[:, :, 40:60] = nrm(ph[1:, :, 20:21] + 0.05 * th[:, :, 40:60], dim=1)
    V = torch.randn(2, NB, 3, generator=gen) * 30
    y, sim, am = ctx.corr_softmax_warp_exemplars(th.cuda(), ph.cuda(), V.cuda(), 1e-10, want_argmax=True)
    yc = y.cpu().double()
    assert (yc[1, :40] - V[1, dup].double().mean(0)).abs().max() < 1e-4
    assert (yc[1, 40:60] - V[1, [20, 21]].double().mean(0)).abs().max() < 1e-4
    assert (am.cpu()[1, :40] == 3).all() and (am.cpu()[1, 40:60] == 20).all()
    tol = {"bf16x3": 8e-6, "tf32x3": 4e-6}.get(corr_math, 2e-6)
    for k in range(2):
        yo, so, io = O.corr_softmax_warp(th.double(), ph[k:k + 1].double(), V[k:k + 1].double(), 1e-10, return_argmax=True)
        gap = O.top2_gap(th.double(), ph[k:k + 1].double())[0]
        ok = (gap == 0) | (gap > 4 * tol)
        assert (yc[k][ok] - yo[0][ok]).abs().max() < 1e-3
        assert (sim.cpu().double()[k] - so[0]).abs().max() < tol
    y0, s0, a0 = ctx.corr_softmax_warp(th.cuda(), ph[:1].cuda(), V[:1].cuda(), 1e-10, want_argmax=True)
    assert torch.equal(sim[0], s0[0]) and torch.equal(am[0], a0[0])


# ------------------------------------------------------------------------------------------ frames
@pytest.mark.parametrize("H,W", [(32, 64), (40, 64)])
@pytest.mark.parametrize("T", [1e-10, 0.01])
def test_frame_slots_equal_single_exemplar_frames(ctx, conv_math, H, W, T):
    IB = make_lab(80, 3, H, W)
    L = make_lab(81, 1, H, W)[:, 0:1].cuda()
    last = make_lab(82, 3, H, W).cuda()
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_exemplars(L, last, T, want_warp=True)
    assert ab.shape == (3, 2, H, W) and warp.shape == (3, 3, H, W) and sim.shape == (3, 1, H, W)
    for k in range(3):
        ctx.set_exemplar(IB[k:k + 1])
        ab1, warp1, sim1 = ctx.colorize_frames(L, last[k:k + 1], T, want_warp=True)
        assert torch.equal(sim[k:k + 1], sim1)
        if T < 1e-9:
            assert torch.equal(warp[k:k + 1], warp1)
        else:
            assert (warp[k:k + 1] - warp1).abs().max() < 1e-4
        # ColorVidNet at batch K: InstanceNorm sums and device-derived scales differ from batch 1 (test_fused_batch_equals_single)
        assert (ab[k:k + 1] - ab1).abs().max() < 5e-3


def test_frame_exemplars_vs_oracle_64x64(ctx, conv_math, sds):
    IA, IB, last = make_lab(120, 1, 64, 64), make_lab(121, 2, 64, 64), make_lab(122, 2, 64, 64)
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_exemplars(IA[:, 0:1].cuda(), last.cuda(), want_warp=True)
    sds64 = {k: O._cast(v, torch.float64) for k, v in sds.items()}
    for k in range(2):
        IBk, lastk = IB[k:k + 1], last[k:k + 1]
        ex = {}
        with torch.no_grad():
            fB = O.exemplar_features(sds64["vgg"], IBk.double())
            ab64, warped64, sim64, _ = O.frame_colorization(sds64, IA.double(), IBk.double(), lastk.double(), fB, extras=ex)
            ab32, _, _, _ = O.frame_colorization(sds, IA, IBk, lastk, O.exemplar_features(sds["vgg"], IBk))
        gap = O.top2_gap(ex["theta_hat"], ex["phi_hat"])
        assert (sim[k:k + 1].cpu().double() - sim64).abs().max() < 2e-5
        clear = (gap > 1e-5).view(1, 1, 16, 16).expand(1, 3, 16, 16)
        assert (warp[k:k + 1].cpu()[:, :, ::4, ::4][clear].double() - warped64[:, :, ::4, ::4][clear]).abs().max() < 1e-4
        floor = (ab32.double() - ab64).abs().max().item()
        assert (ab[k:k + 1].cpu().double() - ab64).abs().max().item() <= max(1e-3, 2 * floor)


# ------------------------------------------------------------------------------------------ clip
def test_clip_exemplars_equals_chained_frames(ctx, conv_math):
    """K recurrences in one clip call == chaining colorize_frames_exemplars with last_k = cat(L, ab_k), bit for bit, from
    pinned host memory and from device memory, on one and on two phase-A streams, and with --frame_propagate."""
    g = load_golden("clip3_32x48")
    L = torch.from_numpy(g["frames_lab"])[:, 0:1].contiguous()
    F_, _, H, W = L.shape
    IB = make_lab(90, 3, H, W)
    ctx.set_exemplars(IB)
    out = ctx.colorize_clip_exemplars(L.pin_memory())
    assert out.shape == (3, F_, 2, H, W) and not out.is_cuda
    assert torch.equal(ctx.colorize_clip_exemplars(L.cuda()).cpu(), out)
    ctx.debug_flag("clip_astreams", 2)
    try:
        out2 = ctx.colorize_clip_exemplars(L.pin_memory())
    finally:
        ctx.debug_flag("clip_astreams", 1)
    assert torch.equal(out, out2)
    for first, res in ((None, out), (IB, ctx.colorize_clip_exemplars(L.cuda(), first_last_lab=IB.cuda()).cpu())):
        last = torch.zeros(3, 3, H, W, device="cuda") if first is None else first.cuda()
        for t in range(F_):
            Lt = L[t:t + 1].cuda()
            ab = ctx.colorize_frames_exemplars(Lt, last)
            assert torch.equal(ab.cpu(), res[:, t]), (first is None, t)
            last = torch.cat((Lt.expand(3, 1, H, W), ab), 1)
    assert not torch.equal(res, out)


# ------------------------------------------------------------------------------------------ state and errors
def test_exemplar_slots_state_and_errors(ctx):
    import dvc

    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    H, W = 32, 64
    IB = make_lab(100, 3, H, W)
    L, last1 = make_lab(101, 1, H, W)[:, 0:1].cuda(), make_lab(102, 1, H, W).cuda()
    ctx.set_exemplar(IB[:1])
    ref = ctx.colorize_frames(L, last1)
    ctx.set_exemplars(IB)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    # the single-exemplar entry points never fall back to slot 0
    for call in (lambda: ctx.colorize_frames(L, last1), lambda: ctx.colorize_clip(L.cpu().pin_memory()),
                 lambda: ctx.exemplar_export(H, W)):
        with pytest.raises(dvc.DvcError) as e:
            call()
        assert _rc(e.value) == -4 and "exemplars" in str(e.value)
    with pytest.raises(dvc.DvcError) as e:  # K = 0
        ctx.set_exemplars(torch.zeros(0, 3, H, W))
    assert _rc(e.value) == -1
    with pytest.raises(dvc.DvcError) as e:  # K = 9
        ctx.set_exemplars(make_lab(103, 9, H, W))
    assert _rc(e.value) == -1
    with pytest.raises(dvc.DvcError) as e:  # K differs from the cached count
        ctx.colorize_frames_exemplars(L, make_lab(104, 2, H, W).cuda())
    assert _rc(e.value) == -2
    with pytest.raises(dvc.DvcError) as e:  # frame size differs from the exemplars'
        ctx.colorize_frames_exemplars(make_lab(105, 1, H, 48)[:, 0:1].cuda(), make_lab(106, 3, H, 48).cuda())
    assert _rc(e.value) == -2
    out = torch.empty(2, 1, 2, H, W, device="cuda")
    rc = ctx.lib.dvc_colorize_clip_exemplars(ctx.h, dvc._ptr(L), 1, H, W, 1e-10, None, 2, dvc._ptr(out), dvc._stream(ctx.device))
    assert rc == -2
    rc = ctx.lib.dvc_colorize_clip_exemplars(ctx.h, dvc._ptr(L), 1, H, W, 1e-10, None, 9, dvc._ptr(out), dvc._stream(ctx.device))
    assert rc == -1
    # peer outputs of the row-sharded correlation are not combined with several exemplars
    y4, s4 = torch.zeros(16, 4, device="cuda"), torch.zeros(16, device="cuda")
    ctx.corr_set_peer_outputs([y4.data_ptr()], [s4.data_ptr()], 0)
    try:
        with pytest.raises(dvc.DvcError) as e:
            ctx.corr_softmax_warp_exemplars(nrm(torch.randn(1, 256, 16), dim=1).cuda(), nrm(torch.randn(2, 256, 16), dim=1).cuda(),
                                            torch.randn(2, 16, 3).cuda(), 1e-10)
        assert _rc(e.value) == -4
    finally:
        ctx.corr_set_peer_outputs()
    assert ctx.launch_count() == n0  # every refusal came before any launch
    assert torch.equal(y4, torch.zeros_like(y4))
    # the failed calls left the K = 3 cache usable, and one exemplar again restores the single path's bits
    ctx.colorize_frames_exemplars(L, make_lab(107, 3, H, W).cuda())
    ctx.set_exemplar(IB[:1])
    assert torch.equal(ctx.colorize_frames(L, last1), ref)


# ------------------------------------------------------------------------------------------ full size
def test_full_size_480x864_three_exemplars(ctx, conv_math):
    H, W = 480, 864
    IB = make_lab(110, 3, H, W)
    L = make_lab(111, 1, H, W)[:, 0:1].cuda()
    last = torch.zeros(3, 3, H, W, device="cuda")
    ctx.set_exemplars(IB)
    ab, warp, sim = ctx.colorize_frames_exemplars(L, last, want_warp=True)
    ab2, warp2, sim2 = ctx.colorize_frames_exemplars(L, last, want_warp=True)
    assert torch.equal(ab, ab2) and torch.equal(warp, warp2) and torch.equal(sim, sim2)
    assert torch.isfinite(ab).all() and ab.abs().max() <= 128.0
    for k in range(3):
        # one-hot warp: every warped colour of slot k is a row of ITS OWN 4x4-pooled exemplar
        V = torch.nn.functional.avg_pool2d(IB[k:k + 1], 4).view(3, -1).t().contiguous()
        rows = warp[k, :, ::4, ::4].reshape(3, -1).t().cpu()
        assert torch.cdist(rows[::97].double(), V.double()).min(dim=1).values.max() < 1e-4
    for k in range(3):
        ctx.set_exemplar(IB[k:k + 1])
        _, warp1, sim1 = ctx.colorize_frames(L, last[k:k + 1], want_warp=True)
        assert torch.equal(warp[k:k + 1], warp1) and torch.equal(sim[k:k + 1], sim1)
