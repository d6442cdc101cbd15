"""CPU oracle of the pre / post-processing the reference runs around the networks (SURVEY.md §8f rows 2-3).
TEST INFRASTRUCTURE ONLY: imported by tests/ (and never by the product).

* fgs_filter: cv2.ximgproc.createFastGlobalSmootherFilter(guide, lambda, sigma_color).filter(src) as test.py:105-112 uses
  it.  opencv-contrib is NOT installed in this image (cv2 here is the headless build without ximgproc) and the reference
  ships no vectors for it: PARITY UNPINNED.  The restatement follows Min et al., "Fast Global Image Smoothing Based on
  Weighted Least Squares", IEEE TIP 2014 (separable 1-D WLS, Thomas algorithm, Alg. 1) with the OpenCV-contrib
  parameterisation (weights_LUT[d^2] = -exp(-sqrt(d^2) / sigma_color) in fp32, lambda_attenuation = 0.25, num_iter = 3,
  lambda multiplied by the attenuation after every horizontal + vertical iteration, fp32 work type), and
  `fgs_reference_f64` checks it against what it must compute: the float64 sparse solve of (I + lambda_n L) u = f per line.

* centerpad_transform: utils/util_distortion.py:217-258 (CenterPad) followed by torchvision CenterCrop (test.py:45).
  skimage is not installed either; its resize() is restated over the two scipy.ndimage functions it calls
  (scikit-image >= 0.19: gaussian_filter + zoom(grid_mode=True)), which ARE installed here -- so the arithmetic is pinned to
  scipy, the thin wrapper around it is restated (requirements.txt:8 leaves the skimage version open).
"""
import numpy as np


# ------------------------------------------------------------------------------------------------ FGS
def _thomas_lines(u, C, lam):
    """Solve (I + lam L) x = u for every row of u [R, n] in float32; C [R, n] holds -w_{j,j+1} (0 in the last column).
    Every operation is a separately rounded float32 operation, in the order of csrc/prepost.cu."""
    f32 = np.float32
    R, n = u.shape
    u = u.astype(f32).copy()
    D = np.zeros((R, n), f32)
    lam = f32(lam)
    cprev = lam * C[:, 0]
    denom = f32(1) - cprev
    D[:, 0] = cprev / denom
    u[:, 0] = u[:, 0] / denom
    for j in range(1, n):
        cj = lam * C[:, j]
        denom = ((f32(1) - cprev) - cj) - cprev * D[:, j - 1]
        D[:, j] = cj / denom
        u[:, j] = (u[:, j] - cprev * u[:, j - 1]) / denom
        cprev = cj
    for j in range(n - 2, -1, -1):
        u[:, j] = u[:, j] - D[:, j] * u[:, j + 1]
    return u


def fgs_weights(guide_u8, sigma_color):
    g = guide_u8.astype(np.int32)
    import math

    # evaluated in double and rounded once to the fp32 work type (csrc/dvc_api.cu does the same with libm's exp)
    lut = np.array([-math.exp(-d / float(np.float32(sigma_color))) for d in range(256)], dtype=np.float64).astype(np.float32)
    Ch = np.zeros(g.shape, np.float32)
    Cv = np.zeros(g.shape, np.float32)
    Ch[:, :-1] = lut[np.abs(g[:, :-1] - g[:, 1:])]
    Cv[:-1, :] = lut[np.abs(g[:-1, :] - g[1:, :])]
    return Ch, Cv


def fgs_filter(guide_u8, src, lam, sigma_color, lambda_attenuation=0.25, num_iter=3):
    """guide_u8 [H, W] uint8, src [P, H, W] float32 -> [P, H, W] float32."""
    Ch, Cv = fgs_weights(guide_u8, sigma_color)
    out = []
    for plane in np.asarray(src, np.float32):
        cur = plane.copy()
        l = np.float32(lam)
        for _ in range(num_iter):
            cur = _thomas_lines(cur, Ch, l)
            cur = _thomas_lines(cur.T.copy(), Cv.T.copy(), l).T.copy()
            l = np.float32(l * np.float32(lambda_attenuation))
        out.append(cur)
    return np.stack(out)


def fgs_reference_f64(guide_u8, src, lam, sigma_color, lambda_attenuation=0.25, num_iter=3):
    """What the filter must compute, in float64 with a sparse direct solver: per line (I + lam_n L) u = f."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spl

    g = guide_u8.astype(np.float64)
    wh = np.exp(-np.abs(g[:, :-1] - g[:, 1:]) / sigma_color)
    wv = np.exp(-np.abs(g[:-1, :] - g[1:, :]) / sigma_color)

    def solve_lines(u, w, l):
        out = np.empty_like(u)
        for r in range(u.shape[0]):
            n = u.shape[1]
            off = -l * w[r]
            diag = np.ones(n)
            diag[:-1] -= off
            diag[1:] -= off
            A = sp.diags([off, diag, off], [-1, 0, 1], format="csc")
            out[r] = spl.spsolve(A, u[r])
        return out

    res = []
    for plane in np.asarray(src, np.float64):
        cur, l = plane.copy(), float(lam)
        for _ in range(num_iter):
            cur = solve_lines(cur, wh, l)
            cur = solve_lines(cur.T.copy(), wv.T.copy(), l).T.copy()
            l *= lambda_attenuation
        res.append(cur)
    return np.stack(res)


def l_to_guide8(l_centred):
    """test.py:106: guide_image = uncenter_l(curr_bs_l) * 255 / 100, .astype(np.uint8) (float32 tensor arithmetic)."""
    v = (np.asarray(l_centred, np.float32) + np.float32(50)) * np.float32(255) / np.float32(100)
    return np.clip(np.trunc(v), 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ fp32 resampling
def fma_f32(a, b, c):
    """fmaf(a, b, c) on float32 arrays: a * b + c rounded once.  The product of two float32 is exact in float64; the float64
    sum is rounded to odd (when inexact, to the neighbour with an odd last bit), after which the rounding to float32 is the
    rounding of the exact value (53 >= 24 + 2 bits), subnormal results included."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    p, c = np.broadcast_arrays(p, c)
    s = p + c
    t = s - p
    err = (p - (s - t)) + (c - t)                            # TwoSum: p + c = s + err exactly
    even = (s.view(np.int64) & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def resize_half_f32(x):
    """resize_half_kernel (csrc/elementwise.cu) operation by operation: x [..., H, W] float32, H and W even ->
    [..., H/2, W/2].  Per 2 x 2 block (a = upper row, b = lower row): r = fma(r.x, 0.5, r.y * 0.5) for both rows, then
    fma(ra, 0.5, rb * 0.5).  Halving is exact except on subnormals, so on normal values this is the plain block mean."""
    x = np.asarray(x, np.float32)
    h = np.float32(0.5)
    ax, ay, bx, by = x[..., 0::2, 0::2], x[..., 0::2, 1::2], x[..., 1::2, 0::2], x[..., 1::2, 1::2]
    ra, rb = fma_f32(ax, h, ay * h), fma_f32(bx, h, by * h)
    return fma_f32(ra, h, rb * h)


def upsample2_scaled_f32(x, scale=1.25):
    """upsample2_kernel (csrc/elementwise.cu) operation by operation: x [..., h, w] float32 -> [..., 2h, 2w].  Output I samples
    source max(0, (I + 0.5) * 0.5 - 0.5) with the upper neighbour clamped to the last row; with l the fractional part,
    top = fma(lx, v01, (1 - lx) * v00), bot = fma(1 - lx, v10, lx * v11), out = fma(1 - ly, top, ly * bot) * scale."""
    x = np.asarray(x, np.float32)
    f32 = np.float32

    def axis(n):
        s = np.maximum((np.arange(2 * n, dtype=f32) + f32(0.5)) * f32(0.5) - f32(0.5), f32(0))
        i0 = s.astype(np.int64)
        return i0, np.minimum(i0 + 1, n - 1), (s - i0.astype(f32)).astype(f32)

    y0, y1, ly = axis(x.shape[-2])
    x0, x1, lx = axis(x.shape[-1])
    ly = ly[:, None]
    wy, wx = f32(1) - ly, f32(1) - lx
    v00, v01 = x[..., y0, :][..., x0], x[..., y0, :][..., x1]
    v10, v11 = x[..., y1, :][..., x0], x[..., y1, :][..., x1]
    top, bot = fma_f32(lx, v01, wx * v00), fma_f32(wx, v10, lx * v11)
    return fma_f32(wy, top, ly * bot) * f32(scale)


# ------------------------------------------------------------------------------------------------ CenterPad
def resize_taps_twin(in_len, out_len):
    """Twin of the host function that feeds the resize kernel its Gaussian taps (csrc/dvc_api.cu: resize_taps for one axis):
    scipy.ndimage._gaussian_kernel1d with libm's exp (math.exp) per tap and numpy's sum.  [] when the axis needs no filter."""
    import math

    sigma = max(0.0, (in_len / out_len - 1.0) / 2.0)
    if not sigma > 1e-15:
        return np.zeros(0)
    r = int(4.0 * sigma + 0.5)
    phi = np.array([math.exp(-0.5 / (sigma * sigma) * float(x * x)) for x in range(-r, r + 1)])
    return phi / phi.sum()


def skimage_resize(image, new_size):
    """skimage.transform.resize(I, new_size, mode="reflect", preserve_range=True, clip=False, anti_aliasing=True) for an
    [H, W, C] array (scikit-image >= 0.19 code path), through the scipy.ndimage calls skimage makes."""
    import scipy.ndimage as ndi

    image = np.asarray(image).astype(np.float64)
    out_shape = (int(new_size[0]), int(new_size[1]), image.shape[2])
    factors = np.divide(image.shape, out_shape)
    sigma = np.maximum(0, (factors - 1) / 2)
    filtered = ndi.gaussian_filter(image, sigma, cval=0, mode="mirror")
    zoom = [1 / f for f in factors]
    return ndi.zoom(filtered, zoom, order=1, mode="mirror", cval=0, grid_mode=True)


def resize_restated(image, new_size):
    """The same resize written out (what csrc/prepost.cu evaluates): separable Gaussian with mirrored borders (centre tap,
    then the symmetric pairs from the outside in), then bilinear sampling at (o + 0.5) * in / out - 0.5."""
    img = np.asarray(image).astype(np.float64)
    Hs, Ws, C = img.shape
    Hr, Wr = int(new_size[0]), int(new_size[1])

    def mirror(i, n):
        if n == 1:
            return np.zeros_like(i)
        p = 2 * (n - 1)
        i = np.mod(i, p)
        return np.where(i < n, i, p - i)

    def gauss(a, axis, sigma):
        if sigma <= 1e-15:
            return a
        r = int(4.0 * sigma + 0.5)
        x = np.arange(-r, r + 1)
        w = np.exp(-0.5 / (sigma * sigma) * x ** 2)
        w = w / w.sum()
        n = a.shape[axis]
        pos = np.arange(n)
        acc = np.take(a, pos, axis=axis) * w[r]
        for k in range(r, 0, -1):
            acc = acc + (np.take(a, mirror(pos - k, n), axis=axis) + np.take(a, mirror(pos + k, n), axis=axis)) * w[r + k]
        return acc

    f = gauss(img, 0, max(0.0, (Hs / Hr - 1) / 2))
    f = gauss(f, 1, max(0.0, (Ws / Wr - 1) / 2))
    cy = (np.arange(Hr) + 0.5) * (Hs / Hr) - 0.5
    cx = (np.arange(Wr) + 0.5) * (Ws / Wr) - 0.5
    fy, fx = np.floor(cy), np.floor(cx)
    ty, tx = (cy - fy)[:, None, None], (cx - fx)[None, :, None]
    y0, y1 = mirror(fy.astype(int), Hs), mirror(fy.astype(int) + 1, Hs)
    x0, x1 = mirror(fx.astype(int), Ws), mirror(fx.astype(int) + 1, Ws)
    v00, v01 = f[y0][:, x0], f[y0][:, x1]
    v10, v11 = f[y1][:, x0], f[y1][:, x1]
    out = (v00 * (1.0 - ty)) * (1.0 - tx)
    out = out + (v01 * (1.0 - ty)) * tx
    out = out + (v10 * ty) * (1.0 - tx)
    out = out + (v11 * ty) * tx
    return out


def centerpad(image_u8, size, resize=skimage_resize):
    """utils/util_distortion.py:217-258, line by line (returns the uint8 array Image.fromarray would wrap)."""
    I = np.array(image_u8)
    height_old, width_old = np.size(I, 0), np.size(I, 1)
    old_size = [height_old, width_old]
    height, width = size
    I_pad = np.zeros((height, width, np.size(I, 2)))
    ratio = height / width
    if height_old / width_old == ratio:
        if height_old == height:
            return I.astype(np.uint8)
        new_size = [int(x * height / height_old) for x in old_size]
        return resize(I, new_size).astype(np.uint8)
    if height_old / width_old > ratio:
        new_size = [int(x * width / width_old) for x in old_size]
        I_resize = resize(I, new_size)
        start_height = (np.size(I_resize, 0) - height) // 2
        I_pad[:, :, :] = I_resize[start_height:(start_height + height), :, :]
    else:
        new_size = [int(x * height / height_old) for x in old_size]
        I_resize = resize(I, new_size)
        start_width = (np.size(I_resize, 1) - width) // 2
        I_pad[:, :, :] = I_resize[:, start_width:(start_width + width), :]
    return I_pad.astype(np.uint8)


def center_crop(img, size):
    """torchvision.transforms.CenterCrop on an [H, W, C] array (test.py:45): zero pad when smaller, then the centred crop."""
    th, tw = size
    h, w = img.shape[:2]
    if tw > w or th > h:
        pl, pt = (tw - w) // 2 if tw > w else 0, (th - h) // 2 if th > h else 0
        pr, pb = (tw - w + 1) // 2 if tw > w else 0, (th - h + 1) // 2 if th > h else 0
        img = np.pad(img, ((pt, pb), (pl, pr), (0, 0)))
        h, w = img.shape[:2]
        if tw == w and th == h:
            return img
    top, left = int(round((h - th) / 2.0)), int(round((w - tw) / 2.0))
    return img[top:top + th, left:left + tw]


def centerpad_transform(image_u8, size, resize=skimage_resize):
    """CenterPad(size) then CenterCrop(size): the uint8 [size] image that enters RGB2Lab (test.py:44-46)."""
    return center_crop(centerpad(image_u8, size, resize), size)
