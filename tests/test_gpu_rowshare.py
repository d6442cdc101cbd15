"""Row-shared taps of the tensor-core convolution engine (conv_tc.cu: CfgRS): the three horizontal taps of a 3x3 row read
one activation tile through descriptors that start a few rows apart.  Per-layer parity against an fp64 F.conv2d and the
network goldens, in both descriptor variants (debug flag tc_rowshare = 1: plain shifted start address, 2: shifted start
address + the descriptor's base-offset field).  Run with -m gpu on an H100."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from test_gpu_conv_layers import BENCH, COLOR, LAYERS, run_layer

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


# dilation 3 and 4 shift the taps of a row by 3 / 6 and 4 / 8 rows of the shared tile (the nets only use 1 and 2);
# synthetic layers of test_gpu_conv_edges.py, (cin, cout, H, W, B, kwargs)
DILATED = [
    ("d3_c64_o72", 64, 72, 7, 17, 1, dict(dil=3, act=1)),
    ("d4_c256_o200_b2_stats", 256, 200, 5, 13, 2, dict(dil=4, want_stats=True)),
    ("d3_c64_o320_lrelu", 64, 320, 11, 29, 1, dict(dil=3, act=2, slope=0.2)),
    ("d4_c256_o264_b3_relu", 256, 264, 3, 3, 3, dict(dil=4, act=1)),
    ("d2_c64_o40_reflect_w3", 64, 40, 5, 3, 3, dict(dil=2, reflect=True, want_stats=True)),
]


@pytest.mark.parametrize("cluster", [2, 1])
@pytest.mark.parametrize("force_bn", [0, 256, 128, 64])
@pytest.mark.parametrize("layer", DILATED, ids=lambda l: l[0])
def test_dilated_rowshare_vs_fp64(request, ctx, sds, rowshare, layer, force_bn, cluster):
    from test_gpu_conv_edges import cout_pad_tc, load_synthetic

    if rowshare == 2:  # strict: a fix of the base-offset variant must turn these into passes
        request.node.add_marker(pytest.mark.xfail(strict=True, reason="the descriptor base-offset variant (tc_rowshare = 2, off "
                                                  "by default) computes dilated layers wrongly on sm_90a (error ~0.9 of max |y|)"))

    _, cin, cout, H, W, B, kw = layer
    if force_bn and cout_pad_tc(cout) % force_bn:
        pytest.skip("the channel tile does not divide the padded Cout")
    name, sd = load_synthetic(ctx, cin, cout)
    ctx.debug_flag("tc_force_bn", force_bn)
    ctx.debug_flag("tc_cluster", cluster)
    err, floor = run_layer(ctx, sds, COLOR, name, cin, cout, H, W, B=B, sd=sd, **kw)
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
