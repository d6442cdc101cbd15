"""Row-shared taps of the tensor-core convolution engine (conv_tc.cu: CfgRS): the three horizontal taps of a 3x3 row read
one activation tile through descriptors that start a few rows apart.  Per-layer parity against an fp64 F.conv2d and the
network goldens, in both descriptor variants (debug flag tc_rowshare = 1: plain shifted start address, 2: shifted start
address + the descriptor's base-offset field).  Run with -m gpu on an H100."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from test_gpu_conv_layers import BENCH, LAYERS, run_layer

pytestmark = pytest.mark.gpu
MODES = [int(m) for m in os.environ.get("DVC_TEST_ROWSHARE", "").split(",") if m]
if not MODES:
    pytest.skip("row-shared taps are exercised with DVC_TEST_ROWSHARE=1[,2]", allow_module_level=True)


@pytest.fixture(params=MODES)
def rowshare(request, ctx):
    import dvc

    ctx.set_math(conv=dvc.MATH_TF32X3, corr=dvc.MATH_FP16X3)
    ctx.debug_flag("tc_rowshare", request.param)
    yield request.param
    ctx.debug_flag("tc_rowshare", 0)
    ctx.debug_flag("tc_force_bn", 0)
    ctx.debug_flag("tc_cluster", 2)


@pytest.mark.parametrize("cluster", [2, 1])
@pytest.mark.parametrize("force_bn", [0, 256, 128, 64])
@pytest.mark.parametrize("layer", [l for l in LAYERS if l[2] not in ("theta", "conv3_3_short")], ids=lambda l: l[0])
def test_layer_rowshare_vs_fp64(ctx, sds, rowshare, layer, force_bn, cluster):
    _, net, name, cin, cout, H, W, kw = layer
    ctx.debug_flag("tc_force_bn", force_bn)
    ctx.debug_flag("tc_cluster", cluster)
    err, floor = run_layer(ctx, sds, net, name, cin, cout, H, W, **kw)
    assert err <= 4e-6, (layer[0], force_bn, cluster, rowshare, err, floor)


@pytest.mark.parametrize("layer", BENCH, ids=[l[0] for l in BENCH])
def test_layer_rowshare_at_bench_geometry(ctx, sds, rowshare, layer):
    _, net, name, cin, cout, H, W, kw, _ = layer
    err, floor = run_layer(ctx, sds, net, name, cin, cout, H, W, **kw)
    assert err <= 4e-6, (layer[0], rowshare, err, floor)


@pytest.mark.parametrize("name", ["small_32x48", "padbranch_40x64", "default_216x384"])
def test_fused_frame_rowshare_vs_golden(ctx, rowshare, name):
    g = load_golden(name)
    IA, IB, last = (torch.from_numpy(g[k]) for k in ("IA_lab", "IB_lab", "IA_last_lab"))
    ctx.set_exemplar(IB)
    ab, warp, sim = ctx.colorize_frames(IA[:, 0:1].cuda(), last.cuda(), float(g["temperature"]), want_warp=True)
    assert np.abs(sim.cpu().numpy()[:, :, ::4, ::4] - g["sim64"]).max() < 2e-5
    floor = np.abs(g["ab32"].astype(np.float64) - g["ab64"]).max()
    err = np.abs(ab.cpu().numpy().astype(np.float64) - g["ab64"]).max()
    assert err <= max(1e-3, 1.25 * floor), (err, floor)
