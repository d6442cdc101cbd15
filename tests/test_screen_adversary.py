"""CPU check of the screening-bound adversary (oracle/screen_adversary.py) that the GPU tests feed the screened T -> 0
correlation: in a float64 model of the fp16 screening pass, with the kernel's own threshold formula, the true maximum
of every adversarial row must rank below another column by at least 80 % of the candidate threshold."""
import numpy as np
import pytest

from oracle import screen_adversary as S

SCREEN_K = 16  # corr_tc.cu: candidates kept per (row, column split, quad thread)


def test_planes_match_fp16_round_to_nearest_even():
    x = np.array([[1028.4921875, -1028.5078125, 1027.5, 1028.5, 3.0, 0.0]], dtype=np.float32) * np.float32(2.0 ** -14)
    hi, nd, nh = S.screen_planes(x)
    assert np.array_equal(hi[0] * 2.0 ** 14, [1028.0, -1029.0, 1028.0, 1028.0, 3.0, 0.0])  # ties to even
    assert np.isclose(nd[0], np.sqrt(2 * 0.4921875 ** 2 + 2 * 0.5 ** 2) * 2.0 ** -14 * 1.0001 + 1e-12)


@pytest.mark.parametrize("case", ["split", "stale"])
def test_adversary_inverts_screened_order_by_80_percent_of_the_bound(case):
    theta, phi, info = S.split_case() if case == "split" else S.stale_case()
    rows, best = info["rows"], info["best"]
    f = theta.astype(np.float64) @ phi.T.astype(np.float64)
    # the planted column is the true maximum, clear by more than 4 x the loosest score tolerance of the GPU tests
    assert np.array_equal(f[rows].argmax(1), best)
    top2 = np.sort(f[rows], 1)[:, -2:]
    assert (top2[:, 1] - top2[:, 0]).min() > 4 * 8e-6
    margin = S.screening_margin(theta, phi, rows, best)
    print(f"{case}: screened inversion / threshold over {len(rows)} rows: min {margin.min():.4f}, max {margin.max():.4f}")
    assert margin.min() >= 0.8
    # and the bound itself holds: no screened score is off by more than half the threshold
    fs, thr = S.screen_emulate(theta, phi)
    assert (np.abs(fs - f) <= thr[:, None] / 2).all()


def test_crowd_overflows_one_candidate_list_in_the_last_split():
    theta, phi, info = S.split_case()
    fs, thr = S.screen_emulate(theta, phi)
    for r in info["crowd_rows"]:
        cand = np.nonzero(fs[r] >= fs[r].max() - thr[r])[0]
        part = cand[(cand >= 5120) & ((cand // 2) % 4 == 0)]
        assert len(part) > SCREEN_K and info["best"][list(info["rows"]).index(r)] in part
