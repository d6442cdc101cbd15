"""Worst-case inputs for the screened T -> 0 correlation (corr_tc.cu: screen_planes_kernel, corr_screen_kernel).

The screening pass scores every (query, reference) pair with the fp16 hi planes of x * 2^14 only and keeps the columns
within screen_threshold() of the row's screened maximum.  The threshold is a Cauchy-Schwarz bound on what the dropped
parts d = x - hi * 2^-14 can change, |d_a . b| + |a_hi . d_b|.  Random unit vectors come nowhere near that bound, so a
threshold that were too small by half would still pass tests on them.  The rows built here do come near it:

  every component has magnitude ~1/16 (x * 2^14 ~ 1028.5, where the fp16 spacing is 1) and sits 2^-7 inside a rounding
  midpoint, so each dropped component is +-0.4921875 fp16 ulp with a sign chosen per component;
  the query's dropped part points along its true-best column (on the dimensions where the rival differs) and that
  column's dropped part along the query's hi part, both with the sign that LOWERS the best column's screened score;
  a rival column, true score lower by delta ~ 4e-5, gets the opposite alignment, which RAISES its screened score.

The screened scores then rank the rival above the true maximum by more than 80 % of the threshold, so a bound that
were 20 % too small would drop the true maximum.  screen_emulate() is a float64 model of the screening pass and the
kernel's threshold formula, used to check that margin without a GPU.
"""
import numpy as np

U = 2.0 ** -14          # the planes hold x * 2^14: one fp16 ulp at 1024..2048 is U in true units
BASE = 1028             # integer part of |x| * 2^14 (inside [1024, 2048), where the fp16 spacing is exactly 1)
FRAC = 0.5 - 2.0 ** -7  # |dropped part| in fp16 ulps: 2^-7 inside the rounding midpoint, exact in fp32
Q_DIFF = 184            # dimensions where best and rival columns differ in sign (the rest agree with the query)
DELTA = 4e-5            # true-score gap best - rival: above 4 x the bf16x3 score tolerance, far below the threshold


def screen_planes(x):
    """fp16 hi plane of x * 2^14 (round to nearest even) in true units and the norms screen_planes_kernel stores:
    nd = ||x - hi|| and nh = ||hi||, both rounded up as the kernel does.  x: float32 [R, C]."""
    x = np.asarray(x, dtype=np.float32)
    hi = (x * np.float32(16384.0)).astype(np.float16).astype(np.float64) * U
    d = x.astype(np.float64) - hi
    nd = np.sqrt((d * d).sum(1)) * 1.0001 + 1e-12
    nh = np.sqrt((hi * hi).sum(1)) * 1.0001
    return hi, nd, nh


def screen_threshold(nd_a, nh_a, nd_b, nh_b):
    """corr_tc.cu screen_threshold(): 2 eps_i, in true-score units."""
    return 2.0 * (nd_a * (nh_b + nd_b) + nh_a * nd_b + 4e-6) * 1.001


def screen_emulate(theta, phi):
    """float64 model of the screening pass for theta [NA, C], phi [NB, C] (rows = positions):
    (screened scores [NA, NB], candidate threshold per query row [NA])."""
    ha, nda, nha = screen_planes(theta)
    hb, ndb, nhb = screen_planes(phi)
    return ha @ hb.T, screen_threshold(nda, nha, ndb.max(), nhb.max())


def _vec(signs, resid, mag):
    """Components signs * mag * 2^-14 whose dropped parts are resid * FRAC ulp (mag: integer parts)."""
    m = mag + 0.5 - resid * signs * 2.0 ** -7
    return (signs * m * U).astype(np.float32)


def _balanced(rng, n):
    z = np.ones(n)
    z[rng.permutation(n)[: n // 2]] = -1.0
    return z


def _triple(rng, n_rivals, C=256):
    """(query, best column, rival columns): rival k scores DELTA + ~k * 4e-6 below best in exact arithmetic."""
    s_a = rng.choice([-1.0, 1.0], C)
    perm = rng.permutation(C)
    P, Q = perm[: C - Q_DIFF], perm[C - Q_DIFF:]
    s_b = s_a.copy()
    s_b[Q] = s_a[Q] * _balanced(rng, Q_DIFF)        # best . query gets nothing from Q ...
    s_r = s_b.copy()
    s_r[Q] = -s_b[Q]                                # ... and neither does the rival, which differs from best on all of Q
    r_a = np.empty(C)
    r_a[Q] = s_b[Q]                                 # query residual: + along best, - along the rival (on Q)
    r_a[P] = s_b[P] * _balanced(rng, C - Q_DIFF)    # no net effect on P, where best and rival agree
    mag = np.full(C, float(BASE))
    a, b = _vec(s_a, r_a, mag), _vec(s_b, s_a, mag)  # best's residual along the query's hi part
    fa = a.astype(np.float64)
    f_b = fa @ b.astype(np.float64)
    rivals = []
    for k in range(n_rivals):
        mag_r = mag.copy()
        r = _vec(s_r, -s_a, mag_r)                  # the rival's residual against it
        # one unit of |x| * 2^14 on a dimension of P moves the rival's true score by ~1028.5 * 2^-28 = 3.8e-6
        target = DELTA + 4e-6 * k
        order = rng.permutation(P)
        for d in order:
            gap = f_b - fa @ r.astype(np.float64)
            step = abs(fa[d]) * U * 16384.0 * U
            if abs(gap - target) <= step / 2:
                break
            mag_r[d] += 1.0 if gap > target else -1.0
            r = _vec(s_r, -s_a, mag_r)
        assert abs(f_b - fa @ r.astype(np.float64) - target) < 4e-6
        rivals.append(r)
    return a, b, rivals


def make_adversary(NA, NB, n_adv, crowd_cols=(), crowd_rows=(), seed=0, C=256):
    """theta [NA, C], phi [NB, C] float32 (rows = positions) and a dict of what was placed where.

    Query rows 0 .. n_adv-1 are adversarial, each with its best column at 2 i and its rival at 2 i + 1.  If crowd_cols
    is given, its first entry is the best column of one more adversarial query and the others are all its rivals: that
    query is written to every row of crowd_rows.  All other rows and columns are random unit vectors; a filler column
    that happens to come within 1e-3 of an adversarial row's maximum is redrawn."""
    rng = np.random.default_rng(seed)
    crowd_cols, crowd_rows = list(crowd_cols), list(crowd_rows)
    assert 2 * n_adv <= NB and n_adv <= NA and not set(crowd_cols) & set(range(2 * n_adv))
    assert not set(crowd_rows) & set(range(n_adv))

    def rand_rows(n):
        g = rng.standard_normal((n, C))
        return (g / np.linalg.norm(g, axis=1, keepdims=True)).astype(np.float32)

    theta, phi = rand_rows(NA), rand_rows(NB)
    best, own = {}, {}  # query row -> its best column, and every column of its own triple

    def place_triple(i):
        a, b, (r,) = _triple(rng, 1, C)
        theta[i], phi[2 * i], phi[2 * i + 1] = a, b, r

    for i in range(n_adv):
        place_triple(i)
        best[i], own[i] = 2 * i, {2 * i, 2 * i + 1}
    if crowd_cols:
        a, b, rivals = _triple(rng, len(crowd_cols) - 1, C)
        phi[crowd_cols[0]] = b
        for c, r in zip(crowd_cols[1:], rivals):
            phi[c] = r
        for i in crowd_rows:
            theta[i] = a
            best[i], own[i] = crowd_cols[0], set(crowd_cols)
    placed = set(range(2 * n_adv)) | set(crowd_cols)
    filler = np.array([j for j in range(NB) if j not in placed], dtype=np.int64)
    rows = np.array(sorted(best), dtype=np.int64)
    want = np.array([best[i] for i in rows], dtype=np.int64)
    # random columns, and the columns of other triples, score ~N(0, 1/256) against a query; its true maximum is ~0.28:
    # redraw whatever comes within 1e-3 of it
    for _ in range(100):
        f = theta[rows].astype(np.float64) @ phi.T.astype(np.float64)
        close = f > f[np.arange(len(rows)), want][:, None] - 1e-3
        for k, i in enumerate(rows):
            close[k, list(own[i])] = False
        if not close.any():
            break
        cols = np.nonzero(close.any(0))[0]
        phi[np.intersect1d(cols, filler)] = rand_rows(len(np.intersect1d(cols, filler)))
        for j in np.setdiff1d(cols, filler):
            if j < 2 * n_adv:
                place_triple(j // 2)
            else:
                raise RuntimeError("a crowd column competes with another query")
    else:
        raise RuntimeError("could not separate the adversarial rows")
    return theta, phi, {"rows": rows, "best": want, "crowd_rows": np.array(crowd_rows, dtype=np.int64),
                        "crowd_cols": np.array(crowd_cols, dtype=np.int64)}


# The two data sets the GPU tests run (tests/test_gpu_corr_edges.py) and the CPU test checks.
#
# split_case: 256 query rows against 5220 reference positions = 21 column tiles of 256, which the launcher splits into
# 11 ranges of 2 tiles on an H100 (132 or 114 SMs, with or without clusters): the last range holds only the 100
# columns 5120..5219.  One more adversarial query, copied to four rows in both 128-row tiles, has its best column and
# 28 rivals there, 26 of them among the columns of one quad thread of the score tile ((col / 2) % 4 == 0): more than
# SCREEN_K = 16 candidates for one list, so that part of the row takes the brute-force re-scoring.
SPLIT_NA, SPLIT_NB = 256, 5220
SPLIT_CROWD_COLS = tuple([c for c in range(5120, 5220) if (c // 2) % 4 == 0][:26] + [5122, 5124, 5219])
SPLIT_CROWD_ROWS = (130, 131, 200, 255)


def split_case():
    return make_adversary(SPLIT_NA, SPLIT_NB, 120, SPLIT_CROWD_COLS, SPLIT_CROWD_ROWS, seed=1)


# stale_case: 200 query rows (150 adversarial) against 333 positions: sized so that a call with twice the query rows
# followed by one with these would have read the reference-side maxima from the earlier call's per-row norms when the
# screening workspace kept the query-side norms in front of them.
def stale_case():
    return make_adversary(200, 333, 150, seed=2)


def screening_margin(theta, phi, rows, best):
    """(screened maximum - screened score of the true best column) / threshold, per listed row: > 0 means the
    screened scores rank another column above the true maximum by that fraction of the candidate threshold."""
    fs, thr = screen_emulate(theta[rows], phi)
    return (fs.max(1) - fs[np.arange(len(rows)), best]) / thr
