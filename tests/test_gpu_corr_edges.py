"""Edge cases of the correlation K7 (corr_tc.cu, corr_simt.cu) against its fp64 evaluation (run with -m gpu on an H100).

Gates (as in test_gpu_parity.py): sim within 2e-6 of fp64 (8e-6 for bf16x3); at T -> 0 the argmax is exact on every row
whose fp64 top-2 gap exceeds 4 x that tolerance, and y on those rows is the V row of the argmax bit for bit; softmax y
within 2e-3 (2e-2 for bf16x3).  Every case runs through all correlation modes of the corr_math fixture.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import dvc_oracle as O
from oracle import screen_adversary as S
from oracle.weights import make_lab
from test_gpu_parity import corr_math  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
BM, BN = 128, 256  # query rows per CTA, reference positions per score tile (corr_tc.cu)


def unit(*shape, gen):
    return torch.nn.functional.normalize(torch.randn(*shape, generator=gen), dim=1)


def score_tol(mode):
    return 8e-6 if mode == "bf16x3" else 2e-6


def split_plan(NA, NB, B, cl, num_sms):
    """(column tiles, column-range splits, tiles per split) exactly as launch_corr_tc chooses them."""
    row_blocks = ((NA + BM - 1) // BM + cl - 1) // cl * cl
    ntiles = (NB + BN - 1) // BN
    nsplit, best = 1, -1.0
    for sp in range(1, min(16, ntiles) + 1):
        tps = (ntiles + sp - 1) // sp
        eff_sp = (ntiles + tps - 1) // tps
        total = row_blocks * B * eff_sp
        waves = (total + num_sms - 1) // num_sms
        eff = total / (waves * num_sms) * (ntiles / (tps * eff_sp)) - 0.01 * sp
        if eff > best:
            best, nsplit = eff, eff_sp
    tps = (ntiles + nsplit - 1) // nsplit
    return ntiles, (ntiles + tps - 1) // tps, tps


def check_vs_oracle(ctx, mode, th, ph, V, T):
    """th [B,C,NA], ph [Bphi,C,NB], V [Bphi,NB,3] (CPU float32) through the stand-alone entry, gated against fp64.
    Returns the GPU results (y, sim, argmax) on the CPU."""
    y, sim, am = (t.cpu() for t in ctx.corr_softmax_warp(th.cuda(), ph.cuda(), V.cuda(), T, want_argmax=True))
    yo, so, io = O.corr_softmax_warp(th.double(), ph.double(), V.double(), T, return_argmax=True)
    tol = score_tol(mode)
    assert (sim.double() - so).abs().max() < tol
    if T <= 2e-10:
        NB = ph.shape[2]
        gap = O.top2_gap(th.double(), ph.double()) if NB > 1 else torch.full(sim.shape, np.inf, dtype=torch.float64)
        clear = gap > 4 * tol
        assert torch.equal(am[clear].long(), io[clear])
        Vb = V.expand(th.shape[0], -1, -1)
        picked = torch.gather(Vb, 1, am.long().clamp(0, NB - 1).unsqueeze(-1).expand(-1, -1, 3))
        assert torch.equal(y[clear], picked[clear])  # one-hot: exact rows of V
    else:
        assert (y.double() - yo).abs().max() < (2e-2 if mode == "bf16x3" else 2e-3)
    return y, sim, am


# ------------------------------------------------------------------------------------------ tile and cluster edges
@pytest.mark.parametrize("NB", [1, 255, 256, 257, 4096, 4097])
@pytest.mark.parametrize("NA", [1, 127, 128, 129, 257])
def test_corr_tile_edges(ctx, corr_math, NA, NB):
    """Query counts around the 128-row CTA tile (NA = 1 and 129, 257: a 2-CTA cluster whose partner has no valid rows)
    against reference counts around the 256-column score tile (NB = 1: the TMA box is larger than the whole tensor).
    NB = 4096 with few query tiles makes the launcher use its maximum of 16 column splits; NB = 4097 gives 9 splits
    whose last one is a single tile holding a single column."""
    gen = torch.Generator().manual_seed(10007 * NA + NB)
    th, ph = unit(1, 256, NA, gen=gen), unit(1, 256, NB, gen=gen)
    V = torch.randn(1, NB, 3, generator=gen) * 30
    for T in (1e-10, 0.01):
        check_vs_oracle(ctx, corr_math, th, ph, V, T)


@pytest.mark.parametrize("Bphi", [1, 3])
def test_corr_batched_layouts_vs_oracle(ctx, corr_math, Bphi):
    """B = 3 frames of 200 positions: query tiles straddle frames; with per-frame exemplars (Bphi = 3) of 333 positions
    the reference tiles straddle them too.  Every exemplar has its own colours, so a neighbour's columns would show."""
    gen = torch.Generator().manual_seed(31 + Bphi)
    th, ph = unit(3, 256, 200, gen=gen), unit(Bphi, 256, 333, gen=gen)
    V = torch.randn(Bphi, 333, 3, generator=gen) * 30
    for T in (1e-10, 0.01):
        check_vs_oracle(ctx, corr_math, th, ph, V, T)


# ------------------------------------------------------------------------------------------ screening-bound adversary
@functools.lru_cache(maxsize=None)
def adversary(case):
    th, ph, info = S.split_case() if case == "split" else S.stale_case()
    gen = torch.Generator().manual_seed(77)
    V = torch.randn(1, ph.shape[0], 3, generator=gen) * 30
    return torch.from_numpy(th.T.copy())[None], torch.from_numpy(ph.T.copy())[None], V, info


def bf16x3_scores(th, ph):
    """Scores of the 3xBF16 operand split (corr_tc.cu split_planes_kernel: hi = bf16(x), lo = bf16(x - hi), lo.lo dropped)
    in fp64, for th [C, NA], ph [C, NB]."""
    def split(x):
        hi = x.t().bfloat16().float()
        return hi.double(), (x.t() - hi).bfloat16().double()

    ha, la = split(th)
    hb, lb = split(ph)
    return ha @ (hb + lb).t() + la @ hb.t()


def test_corr_screening_adversary(ctx, corr_math):
    """Rows whose screened (fp16 hi-plane) scores rank a rival above the true maximum by > 80 % of the candidate threshold
    (oracle/screen_adversary.py; the margin is checked on the CPU by test_screen_adversary.py), and one such query,
    copied to four rows, whose 28 rivals overflow the candidate lists in the uneven last column split."""
    th, ph, V, info = adversary("split")
    NB = ph.shape[2]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for cl in (1, 2):
        ntiles, nsplit, tps = split_plan(th.shape[2], NB, 1, cl, sms)
        assert nsplit * tps > ntiles and info["crowd_cols"].min() >= (nsplit - 1) * tps * BN  # crowd in a short last split
    if corr_math == "bf16x3":
        # every component has the same significand, so the lo.lo products the 3xBF16 split drops add up coherently
        # (1e-5 here, above the random-data tolerance): gate the scores against an exact model of the split instead
        y, sim, am = (t.cpu() for t in ctx.corr_softmax_warp(th.cuda(), ph.cuda(), V.cuda(), 1e-10, want_argmax=True))
        assert (sim[0].double() - bf16x3_scores(th[0], ph[0]).max(1).values).abs().max() < 2e-6
    else:
        y, sim, am = check_vs_oracle(ctx, corr_math, th, ph, V, 1e-10)
    rows, best = torch.from_numpy(info["rows"]), torch.from_numpy(info["best"])
    assert torch.equal(am[0, rows].long(), best)
    assert torch.equal(y[0, rows], V[0, best])


# ------------------------------------------------------------------------------------------ cached exemplar side
def screen_cells(ctx):
    return ctx.debug_buffer("corr.screen_cells", act=False).view(torch.int32).cpu()


def default_math(ctx):
    import dvc

    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    ctx.debug_flag("corr_cluster", 2)
    ctx.debug_flag("corr_screen", 1)


def test_screen_cells_survive_smaller_batches(ctx):
    """The fused frame path keeps the exemplar's screening norms across calls.  Batches of 2, 1, 3, 1 frames against one
    exemplar must leave its reference-side maxima untouched (a short last batch reads them back) and give the bits of
    the same call made right after a fresh dvc_set_exemplar."""
    default_math(ctx)
    IB = make_lab(80, 1, 32, 64)
    L = make_lab(81, 3, 32, 64)[:, 0:1].cuda()
    last = make_lab(82, 3, 32, 64).cuda()
    fresh = {}
    for B in (1, 2, 3):
        ctx.set_exemplar(IB)
        fresh[B] = ctx.colorize_frames(L[:B], last[:B], want_warp=True)
    ctx.set_exemplar(IB)
    ctx.colorize_frames(L[:1], last[:1])
    ref_cells = screen_cells(ctx)[2:4].clone()
    for B in (2, 1, 3, 1):
        out = ctx.colorize_frames(L[:B], last[:B], want_warp=True)
        assert torch.equal(screen_cells(ctx)[2:4], ref_cells), B
        assert all(torch.equal(a, b) for a, b in zip(out, fresh[B])), B


def test_screen_cells_static_exemplar_fewer_rows(ctx):
    """The stand-alone entry with corr_phi_static: 400 query rows, then 300, then 400 again against one prepared
    exemplar side -- same reference-side maxima and same bits as preparing the exemplar side for every call."""
    default_math(ctx)
    gen = torch.Generator().manual_seed(90)
    ph = unit(1, 256, 600, gen=gen).cuda()
    V = (torch.randn(1, 600, 3, generator=gen) * 30).cuda()
    ths = {NA: unit(1, 256, NA, gen=gen).cuda() for NA in (400, 300)}
    fresh = {NA: ctx.corr_softmax_warp(ths[NA], ph, V, 1e-10, want_argmax=True) for NA in (400, 300)}
    ctx.debug_flag("corr_phi_static", 1)
    try:
        ctx.corr_softmax_warp(ths[400], ph, V, 1e-10)
        ref_cells = screen_cells(ctx)[2:4].clone()
        for NA in (400, 300, 400):
            out = ctx.corr_softmax_warp(ths[NA], ph, V, 1e-10, want_argmax=True)
            assert torch.equal(screen_cells(ctx)[2:4], ref_cells), NA
            assert all(torch.equal(a, b) for a, b in zip(out, fresh[NA])), NA
    finally:
        ctx.debug_flag("corr_phi_static", 0)


def test_screening_adversary_after_a_larger_batch(ctx):
    """The adversarial rows against a cached exemplar side, right after a call with twice the query rows: the threshold
    must still be the full bound (a stale reference-side maximum shrinks it below the adversary's margin)."""
    default_math(ctx)
    th, ph, V, info = adversary("stale")
    rows, best = torch.from_numpy(info["rows"]), torch.from_numpy(info["best"])
    ph, V = ph.cuda(), V.cuda()
    ctx.debug_flag("corr_phi_static", 1)
    try:
        ctx.corr_softmax_warp(th.expand(2, -1, -1).contiguous().cuda(), ph, V, 1e-10)
        y, sim, am = (t.cpu() for t in ctx.corr_softmax_warp(th.cuda(), ph, V, 1e-10, want_argmax=True))
    finally:
        ctx.debug_flag("corr_phi_static", 0)
    wrong = int((am[0, rows].long() != best).sum())
    assert wrong == 0, f"{wrong} of {len(rows)} adversarial rows lost their true maximum"
    assert torch.equal(y[0, rows], V[0, best].cpu())
    assert (sim.double() - O.corr_softmax_warp(th.double(), ph.cpu().double(), V.cpu().double(), 1e-10)[1]).abs().max() < 2e-6


# ------------------------------------------------------------------------------------------ degenerate inputs
def test_corr_zero_query_rows(ctx, corr_math):
    """All-zero query rows: every score is exactly 0, so every column ties -- y is the mean of all V rows, the argmax
    the lowest column, and in the screened path every candidate list overflows into brute force."""
    gen = torch.Generator().manual_seed(91)
    th, ph = unit(1, 256, 300, gen=gen), unit(1, 256, 1000, gen=gen)
    zero = [0, 1, 2, 127, 128, 150, 299]
    th[:, :, zero] = 0
    V = torch.randn(1, 1000, 3, generator=gen) * 30 + 10
    mean = V[0].double().mean(0)
    for T in (1e-10, 0.01):
        y, sim, am = check_vs_oracle(ctx, corr_math, th, ph, V, T)
        assert (sim[0, zero] == 0).all()
        assert (y[0, zero].double() - mean).abs().max() <= 1e-4 * mean.abs().max()
        if T <= 2e-10:
            assert (am[0, zero] == 0).all()


def test_corr_duplicated_query_rows_identical(ctx, corr_math):
    """Copies of one query row in different warps, 128-row tiles and cluster ranks give the same bits."""
    gen = torch.Generator().manual_seed(92)
    th, ph = unit(1, 256, 300, gen=gen), unit(1, 256, 700, gen=gen)
    copies = [5, 13, 77, 130, 255, 299]
    th[:, :, copies] = th[:, :, 5:6]
    V = torch.randn(1, 700, 3, generator=gen) * 30
    for T in (1e-10, 0.01):
        y, sim, am = check_vs_oracle(ctx, corr_math, th, ph, V, T)
        for r in copies[1:]:
            assert torch.equal(y[0, r], y[0, 5]) and torch.equal(sim[0, r], sim[0, 5]) and am[0, r] == am[0, 5], (T, r)


@pytest.mark.parametrize("T", [2e-10, 2.5e-10, 1e-8])
def test_corr_temperature_switch_with_ties(ctx, corr_math, T):
    """Either side of the argmax / softmax switch at T = 2e-10, on duplicated exemplar columns (the data of
    test_corr_duplicated_exemplar_columns_average): clear rows give V[argmax] bit for bit, exact ties the mean."""
    gen = torch.Generator().manual_seed(9)
    NA, NB = 300, 700
    ph = unit(1, 256, NB, gen=gen)
    dup = [3, 150, 151, 400, 699]
    ph[:, :, dup] = ph[:, :, 3:4]
    ph[:, :, [20, 21]] = ph[:, :, 20:21]
    th = unit(1, 256, NA, gen=gen)
    th[:, :, :40] = torch.nn.functional.normalize(ph[:, :, 3:4] + 0.05 * th[:, :, :40], dim=1)
    th[:, :, 40:60] = torch.nn.functional.normalize(ph[:, :, 20:21] + 0.05 * th[:, :, 40:60], dim=1)
    V = torch.randn(1, NB, 3, generator=gen) * 30
    y, sim, am = (t.cpu() for t in ctx.corr_softmax_warp(th.cuda(), ph.cuda(), V.cuda(), T, want_argmax=True))
    _, so, io = O.corr_softmax_warp(th.double(), ph.double(), V.double(), T, return_argmax=True)
    tol = {"bf16x3": 8e-6, "tf32x3": 4e-6}.get(corr_math, 2e-6)  # matched rows score ~1.0
    assert (sim.double() - so).abs().max() < tol
    assert (y[0, :40].double() - V[0, dup].double().mean(0)).abs().max() < 1e-4
    assert (y[0, 40:60].double() - V[0, [20, 21]].double().mean(0)).abs().max() < 1e-4
    clear = O.top2_gap(th.double(), ph.double())[0] > 4 * tol
    assert clear.sum() > 200
    assert torch.equal(y[0][clear], V[0][io[0][clear]])


def test_corr_large_temperature(ctx, corr_math):
    """T = 1e3: near-uniform weights over 5184 reference positions (the softmax path's sums over every column)."""
    gen = torch.Generator().manual_seed(93)
    th, ph = unit(1, 256, 300, gen=gen), unit(1, 256, 5184, gen=gen)
    V = torch.randn(1, 5184, 3, generator=gen) * 30 + 5
    check_vs_oracle(ctx, corr_math, th, ph, V, 1e3)


# ------------------------------------------------------------------------------------------ contextual loss
@pytest.mark.parametrize("C", [64, 256])
def test_contextual_loss_unequal_sizes(ctx, C):
    """ContextualLoss_forward with X and Y of different sizes (24x32 against 16x20 positions), B = 2: per-frame
    exemplars, per-row temperatures, NX != NY."""
    default_math(ctx)
    g = torch.Generator().manual_seed(94 + C)
    X = torch.relu(torch.randn(2, C, 24, 32, generator=g))
    Y = torch.relu(torch.randn(2, C, 16, 20, generator=g) + 0.5 * X[:, :, :16, :20])
    for centering in (True, False):
        with torch.no_grad():
            ref64 = O.contextual_loss_forward(X.double(), Y.double(), 0.1, centering)
            ref32 = O.contextual_loss_forward(X, Y, 0.1, centering)
        out = ctx.contextual_loss_forward(X.cuda(), Y.cuda(), 0.1, centering).cpu().double()
        floor = (ref32.double() - ref64).abs().max().item()
        err = (out - ref64).abs().max().item()
        assert err <= max(2e-4 * ref64.abs().max().item(), 4 * floor), (err, floor, ref64)
