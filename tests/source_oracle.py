"""Float32 oracle of the source-resolution resampling (include/dvc.h: dvc_source_footprint, dvc_ab_to_source).
TEST INFRASTRUCTURE ONLY: imported by tests/ (and never by the product)."""
import numpy as np


def source_footprint(geometry, size):
    """(y0, x0, h, w): the source pixels of geometry (Hs, Ws, Hr, Wr, oy, ox) whose centres fall inside the window's extent
    [-0.5, Ho - 0.5] x [-0.5, Wo - 0.5], size = (Ho, Wo): row ys iff 2 oy Hs <= (2 ys + 1) Hr <= 2 (oy + Ho) Hs."""
    Hs, Ws, Hr, Wr, oy, ox = (int(v) for v in geometry)

    def axis(n_src, n_res, off, n_win):
        i = np.arange(n_src, dtype=np.int64)
        p = (2 * i + 1) * n_res
        inside = i[(p >= 2 * off * n_src) & (p <= 2 * (off + n_win) * n_src)]
        return int(inside[0]), len(inside)

    y0, h = axis(Hs, Hr, oy, size[0])
    x0, w = axis(Ws, Wr, ox, size[1])
    return y0, x0, h, w


def ab_to_source(ab, geometry, size):
    """The window's planes ab [P, Ho, Wo] float32 resampled onto the source footprint -> [P, h, w] float32, as csrc/prepost.cu
    computes it: window coordinate cy = ((2 ys + 1) Hr - (2 oy + 1) Hs) / (2 Hs) (int64 numerator, one float64 division),
    clamped to [0, Ho - 1], then upsample2's bilinear expression with every float32 operation separately rounded."""
    Hs, Ws, Hr, Wr, oy, ox = (int(v) for v in geometry)
    Ho, Wo = int(size[0]), int(size[1])
    y0, x0, h, w = source_footprint(geometry, size)
    f32 = np.float32

    def axis(first, n, n_src, n_res, off, n_win):
        i = np.arange(first, first + n, dtype=np.int64)
        c = np.clip(((2 * i + 1) * n_res - (2 * off + 1) * n_src) / (2.0 * n_src), 0.0, n_win - 1.0)
        i0 = np.floor(c).astype(np.int64)
        return i0, np.minimum(i0 + 1, n_win - 1), (c - i0).astype(f32)

    ya, yb, ly = axis(y0, h, Hs, Hr, oy, Ho)
    xa, xb, lx = axis(x0, w, Ws, Wr, ox, Wo)
    ly, lx = ly[:, None], lx[None, :]
    a = np.asarray(ab, f32)
    v00, v01 = a[:, ya][:, :, xa], a[:, ya][:, :, xb]
    v10, v11 = a[:, yb][:, :, xa], a[:, yb][:, :, xb]
    wy, wx = f32(1) - ly, f32(1) - lx
    return (wy * (wx * v00 + lx * v01) + ly * (wx * v10 + lx * v11)).astype(f32)
