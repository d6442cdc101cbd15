"""CPU check of the scale-bound adversaries (oracle/conv_adversary.py) that the GPU tests feed the device-scaled fp16
store: in float64, the target output of every case must reach at least 99 % of the bound dyn_out_exponent computes from
the same weight L1 norm, bias and addend maxima, and never exceed it."""
import math

import numpy as np
import pytest
import torch

from oracle import conv_adversary as ADV


def test_e16_from_bound_keeps_one_binade_of_headroom():
    assert ADV.e16_from_bound(1.0) == 14  # an exact power of two lands at 2^14
    assert ADV.e16_from_bound(32768.0) == -1
    assert ADV.e16_from_bound(32767.0) == 0
    assert ADV.e16_from_bound(0.0) == 24
    for b in (0.37, 3.0, 1000.0, 65504.0):
        e = ADV.e16_from_bound(b)
        assert b * 2.0 ** e <= 32768.0 < b * 2.0 ** (e + 1)


def test_phase_weights_reproduce_the_upconvolution():
    g = torch.Generator().manual_seed(5)
    w = torch.randn(6, 4, 3, 3, generator=g, dtype=torch.float64)
    x = torch.randn(1, 4, 3, 5, generator=g, dtype=torch.float64)
    up = torch.nn.functional.conv2d(torch.nn.functional.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1)
    pw = ADV.phase_weights(w).double()
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
    for ph in range(4):
        a, b = ph >> 1, ph & 1
        # phase (a, b) reads low-resolution rows i-1+a .. i+a and columns j-1+b .. j+b
        y = torch.nn.functional.conv2d(xp[:, :, a:a + 4, b:b + 6], pw[ph])
        assert torch.allclose(y, up[:, :, a::2, b::2], atol=1e-5), ph


@pytest.mark.parametrize("case", list(ADV.CASES))
def test_adversary_attains_the_bound(case):
    adv = ADV.build(case)
    y = ADV.forward64(adv)
    o, py, px = adv["target"]
    attained, bound = abs(y[0, o, py, px].item()), adv["bound"]
    e = ADV.e16_from_bound(bound)
    print(f"{case}: |y*| / bound = {attained / bound:.5f}, exponent {e}, |y*| * 2^e = {attained * 2.0 ** e:.1f}")
    assert adv["x"].abs().max().item() == adv["A"] and math.log2(adv["A"]) == int(math.log2(adv["A"]))
    assert attained >= 0.99 * bound
    assert y.abs().max().item() <= bound  # the bound holds
    assert attained * 2.0 ** e <= 32768.0


@pytest.mark.parametrize("case,term", [("color_conv8_1_upconv_add", "aadd"), ("synthetic_lrelu3_bias", "bmax"),
                                       ("synthetic_lrelu3_bias", "gain")])
def test_dropping_a_bound_term_would_saturate(case, term):
    """The tuned cases carry >= 3/4 of their bound in one term: a bound without it picks an exponent at least two
    higher, and the attained output then exceeds the fp16 maximum."""
    adv = ADV.build(case)
    t = dict(adv["terms"])
    t[term] = 1.0 if term == "gain" else 0.0
    wrong = ADV.device_bound(adv["A"], t["l1max"], t["bmax"], t["aadd"], t["gain"])
    e, e_wrong = ADV.e16_from_bound(adv["bound"]), ADV.e16_from_bound(wrong)
    y = ADV.forward64(adv)
    o, py, px = adv["target"]
    assert e_wrong >= e + 2
    assert abs(y[0, o, py, px].item()) * 2.0 ** e_wrong > 65504.0  # the fp16 maximum
