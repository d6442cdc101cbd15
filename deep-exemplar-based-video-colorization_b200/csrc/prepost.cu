// Pre / post-processing around the networks that the reference runs on the CPU (SURVEY.md §8f rows 2-3):
//
//  * Fast Global Smoother (the "WLS filter" of test.py:105-112: cv2.ximgproc.createFastGlobalSmootherFilter(guide,
//    lambda, sigma_color).filter(plane)).  Restated from Min, Choi, Lu, Ham, Sohn, Do, "Fast Global Image Smoothing Based
//    on Weighted Least Squares", IEEE TIP 2014 and the documented parameters of the OpenCV-contrib implementation
//    (lambda_attenuation = 0.25, num_iter = 3): per iteration one horizontal and one vertical sweep, each solving the
//    tridiagonal system  (I + lambda_n L) u = f  of every line with the Thomas algorithm in fp32, where L is the 1-D
//    graph Laplacian with weights exp(-|g_p - g_q| / sigma_color) between neighbours of the uint8 guide, and
//    lambda_{n+1} = lambda_n * lambda_attenuation.  opencv-contrib is not in this image: parity unpinned
//    (oracle/prepost_oracle.py restates the same algorithm and is validated against a float64 sparse solve).
//    HBM/latency-bound: the recurrences are sequential along a line, parallel across lines and planes.
//
//  * CenterPad (utils/util_distortion.py:217-258): aspect-preserving skimage.transform.resize(order=1, mode="reflect",
//    anti_aliasing=True, preserve_range=True, clip=False) -- i.e. scipy.ndimage.gaussian_filter(sigma = (factor-1)/2,
//    mode="mirror", truncate=4) followed by scipy.ndimage.zoom(order=1, mode="mirror", grid_mode=True), both float64 --
//    truncation to uint8 and the centred crop / zero pad to the target size.  The taps come from the host (dvc_api.cu:
//    gaussian_taps): summed as numpy sums them (pairwise), each exp from libm.  Reproducing numpy's own vectorised float64
//    exp, which CPUs with AVX-512 use and which misses libm's by the last bit on some arguments, was not attempted: scipy's
//    bytes are then not the same on every machine either.  The guarantee is therefore: scipy's bytes exactly whenever the
//    taps agree (on the x86-64 hosts measured: every down-scale below 5x) and the source is down-scaled; else at most one level, and only where
//    scipy's float64 value lies on an integer (flat areas).  When up-scaling, sample points before the first / after the last
//    source pixel are split into floor and fraction and the index is mirrored, where scipy mirrors the coordinate first: the
//    same two neighbours with weights one rounding apart (tests/test_gpu_prepost_edges.py asserts both cases).
#include <math.h>
#include <stdint.h>

#include "dvc_internal.cuh"

namespace dvc {

namespace {

// ------------------------------------------------------------------------------------------------ FGS
// C_h(i, j) = -w(g(i, j), g(i, j+1)), 0 in the last column; C_v(i, j) = -w(g(i, j), g(i+1, j)), 0 in the last row.
// Guide blockIdx.y of [G][H][W] -> its Ch / Cv planes of [G][H][W].
__global__ void __launch_bounds__(256) fgs_weights_kernel(const unsigned char* __restrict__ g, const float* __restrict__ lut,
                                                          float* __restrict__ Ch, float* __restrict__ Cv, int H, int W) {
  const int n = H * W;
  const size_t base = (size_t)blockIdx.y * n;
  g += base, Ch += base, Cv += base;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const int i = p / W, j = p - i * W;
    const int c = g[p];
    Ch[p] = (j + 1 < W) ? __ldg(lut + abs(c - (int)g[p + 1])) : 0.f;
    Cv[p] = (i + 1 < H) ? __ldg(lut + abs(c - (int)g[p + W])) : 0.f;
  }
}

// One line of the Thomas algorithm, element j of a line lives at base + j * stride.  Every operation is a separately
// rounded fp32 operation (no FMA contraction), in the order of the oracle.
//   forward : denom_j = (1 - lam C_{j-1} - lam C_j) - lam C_{j-1} * D_{j-1};  D_j = lam C_j / denom_j;
//             u_j = (u_j - lam C_{j-1} u_{j-1}) / denom_j
//   backward: u_j = u_j - D_j u_{j+1}
// Plane pl is smoothed with the coefficients of guide gsrc.at(pl / 2): the a and b planes of one row share their guide.
// Vertical sweep: thread = (plane, column), adjacent threads touch adjacent addresses (coalesced).
__global__ void __launch_bounds__(128) fgs_vertical_kernel(float* __restrict__ cur, const float* __restrict__ Cv, float* __restrict__ D,
                                                           int planes, const PlaneSrc gsrc, int H, int W, float lam) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= planes * W) return;
  const int pl = t / W, x = t - pl * W;
  float* u = cur + (size_t)pl * H * W + x;
  float* d = D + (size_t)pl * H * W + x;
  const float* c = Cv + (size_t)gsrc.at(pl / 2) * H * W + x;
  float cprev = __fmul_rn(lam, c[0]);
  float denom = __fsub_rn(1.f, cprev);
  float dprev = __fdiv_rn(cprev, denom);
  float uprev = __fdiv_rn(u[0], denom);
  d[0] = dprev, u[0] = uprev;
  for (int i = 1; i < H; ++i) {
    const float ci = __fmul_rn(lam, c[(size_t)i * W]);
    denom = __fsub_rn(__fsub_rn(__fsub_rn(1.f, cprev), ci), __fmul_rn(cprev, dprev));
    dprev = __fdiv_rn(ci, denom);
    uprev = __fdiv_rn(__fsub_rn(u[(size_t)i * W], __fmul_rn(cprev, uprev)), denom);
    d[(size_t)i * W] = dprev, u[(size_t)i * W] = uprev;
    cprev = ci;
  }
  for (int i = H - 2; i >= 0; --i) {
    uprev = __fsub_rn(u[(size_t)i * W], __fmul_rn(d[(size_t)i * W], uprev));
    u[(size_t)i * W] = uprev;
  }
}

// Horizontal sweep: one warp owns 32 consecutive rows of one plane (lane = row) and walks along x in 32-column tiles
// that are moved between global and shared memory with coalesced row accesses (a thread per row reading its own row
// directly would touch one sector per element).
__global__ void __launch_bounds__(32) fgs_horizontal_kernel(float* __restrict__ cur, const float* __restrict__ Ch, float* __restrict__ D,
                                                            int planes, const PlaneSrc gsrc, int H, int W, float lam) {
  __shared__ float su[32][33], sc[32][33], sd[32][33];
  const int lane = threadIdx.x;
  const int groups = (H + 31) / 32;
  const int pl = blockIdx.x / groups, r0 = (blockIdx.x - pl * groups) * 32;
  const int nrows = min(32, H - r0);
  float* ub = cur + ((size_t)pl * H + r0) * W;
  float* db = D + ((size_t)pl * H + r0) * W;
  const float* cb = Ch + ((size_t)gsrc.at(pl / 2) * H + r0) * W;
  float cprev = 0.f, dprev = 0.f, uprev = 0.f;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int nx = min(32, W - x0);
    for (int k = 0; k < nrows; ++k)
      if (lane < nx) su[k][lane] = ub[(size_t)k * W + x0 + lane], sc[k][lane] = __ldg(cb + (size_t)k * W + x0 + lane);
    __syncwarp();
    if (lane < nrows) {
      for (int j = 0; j < nx; ++j) {
        const float cj = __fmul_rn(lam, sc[lane][j]);
        float denom;
        if (x0 + j == 0)
          denom = __fsub_rn(1.f, cj);
        else
          denom = __fsub_rn(__fsub_rn(__fsub_rn(1.f, cprev), cj), __fmul_rn(cprev, dprev));
        dprev = __fdiv_rn(cj, denom);
        uprev = (x0 + j == 0) ? __fdiv_rn(su[lane][j], denom) : __fdiv_rn(__fsub_rn(su[lane][j], __fmul_rn(cprev, uprev)), denom);
        sd[lane][j] = dprev, su[lane][j] = uprev;
        cprev = cj;
      }
    }
    __syncwarp();
    for (int k = 0; k < nrows; ++k)
      if (lane < nx) ub[(size_t)k * W + x0 + lane] = su[k][lane], db[(size_t)k * W + x0 + lane] = sd[k][lane];
    __syncwarp();
  }
  // backward substitution, tiles right to left; uprev holds u_{W-1}
  const int last_tile = ((W - 1) / 32) * 32;
  for (int x0 = last_tile; x0 >= 0; x0 -= 32) {
    const int nx = min(32, W - x0);
    for (int k = 0; k < nrows; ++k)
      if (lane < nx) su[k][lane] = ub[(size_t)k * W + x0 + lane], sd[k][lane] = db[(size_t)k * W + x0 + lane];
    __syncwarp();
    if (lane < nrows) {
      for (int j = nx - 1; j >= 0; --j) {
        if (x0 + j == W - 1) continue;  // u_{W-1} is final after the forward sweep
        uprev = __fsub_rn(su[lane][j], __fmul_rn(sd[lane][j], uprev));
        su[lane][j] = uprev;
      }
    }
    __syncwarp();
    for (int k = 0; k < nrows; ++k)
      if (lane < nx) ub[(size_t)k * W + x0 + lane] = su[k][lane];
    __syncwarp();
  }
}

// test.py:106: guide = uint8(uncenter_l(L) * 255 / 100), fp32 arithmetic, truncation toward zero
__global__ void __launch_bounds__(256) l_to_guide8_kernel(const float* __restrict__ l, unsigned char* __restrict__ g, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    g[i] = guide8_of_l(__ldg(l + i));
}

// Centred L of a grey byte g, i.e. of the pixel (g, g, g): rgb8_to_lab_kernel's plane 0 with the same float64 operations
// (rgb8_lab_f), one entry per byte value, built by each block of the C = 1 ingest kernels before they read it.
__device__ __forceinline__ void gray_l_table(float* __restrict__ lut) {
  for (int g = threadIdx.x; g < 256; g += blockDim.x) {
    const unsigned char px[3] = {(unsigned char)g, (unsigned char)g, (unsigned char)g};
    double f[3];
    rgb8_lab_f(px, f);
    lut[g] = (float)(116.0 * f[1] - 16.0) - 50.0f;
  }
  __syncthreads();
}

// Video ingest (test.py:44-46,71,106 for the luminance only -- the frames' a / b are never used).  A warp owns a 2 x 16
// pixel tile (lane = row * 16 + column) of the centred uint8 frame [H][W][C], one thread per pixel; the 2 x 2 neighbourhoods
// of the half-resolution plane are gathered with shuffles.  L is rgb8_to_lab_kernel's plane 0 (the same float64 operations,
// rgb8_lab_f; for a grey frame, C = 1, looked up in gray_l_table), the half-resolution value resize_half_kernel's arithmetic on
// those four floats, the guide l_to_guide8's.
template <int C>
__global__ void __launch_bounds__(256) rgb8_to_l_half_kernel(const unsigned char* __restrict__ rgb, float* __restrict__ l,
                                                             float* __restrict__ l_half, unsigned char* __restrict__ guide, int H,
                                                             int W) {
  __shared__ float gray_l[C == 1 ? 256 : 1];
  if constexpr (C == 1) gray_l_table(gray_l);
  const int lane = threadIdx.x & 31;
  const int tw = (W + 15) / 16, ntiles = (H / 2) * tw, nwarps = gridDim.x * (blockDim.x >> 5);
  for (int tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); tile < ntiles; tile += nwarps) {  // warp-uniform
    const int i = tile / tw, x = (tile - i * tw) * 16 + (lane & 15), y = 2 * i + (lane >> 4);
    float v = 0.f;
    if (x < W) {
      const size_t pix = (size_t)y * W + x;
      if constexpr (C == 1) {
        v = gray_l[rgb[pix]];
      } else {
        double f[3];
        rgb8_lab_f(rgb + pix * 3, f);
        v = (float)(116.0 * f[1] - 16.0) - 50.0f;
      }
      l[pix] = v;
      if (guide) guide[pix] = guide8_of_l(v);
    }
    // resize_half: 0.5 * (0.5 * a.x + 0.5 * a.y) + 0.5 * (0.5 * b.x + 0.5 * b.y), a = row 2i, b = row 2i + 1
    const float nb = __shfl_xor_sync(0xffffffffu, v, 1);
    const float r = (lane & 1) ? 0.5f * nb + 0.5f * v : 0.5f * v + 0.5f * nb;
    const float r1 = __shfl_xor_sync(0xffffffffu, r, 16);
    if (lane < 16 && !(lane & 1) && x < W) l_half[(size_t)i * (W / 2) + x / 2] = 0.5f * r + 0.5f * r1;
  }
}

// Source-resolution luminance of the video path: over the footprint rectangle (y0, x0, h, w) of a uint8 source frame
// [Hs][Ws][C], the centred L [h][w] (rgb8_to_lab_kernel's plane 0: rgb8_lab_f, the same float64 operations; gray_l_table for
// C = 1) and, when guide != nullptr, the WLS guide [h][w] (l_to_guide8's).
template <int C>
__global__ void __launch_bounds__(256) rgb8_to_l_guide_kernel(const unsigned char* __restrict__ rgb, int Ws, int y0, int x0, int h, int w,
                                                              float* __restrict__ l, unsigned char* __restrict__ guide) {
  __shared__ float gray_l[C == 1 ? 256 : 1];
  if constexpr (C == 1) gray_l_table(gray_l);
  const size_t n = (size_t)h * w;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(i / w), x = (int)(i - (size_t)y * w);
    float v;
    if constexpr (C == 1) {
      v = gray_l[rgb[(size_t)(y0 + y) * Ws + x0 + x]];
    } else {
      double f[3];
      rgb8_lab_f(rgb + ((size_t)(y0 + y) * Ws + x0 + x) * 3, f);
      v = (float)(116.0 * f[1] - 16.0) - 50.0f;
    }
    l[i] = v;
    if (guide) guide[i] = guide8_of_l(v);
  }
}

// The window's ab [planes][Ho][Wo] resampled onto the footprint (fy, fx, h, w) of the source grid: source pixel (ys, xs) sits at
// window coordinate cy = ((2 ys + 1) Hr - (2 oy + 1) Hs) / (2 Hs) (an exact integer numerator, one float64 division; cx the
// same), clamped to the window, and takes upsample2_kernel's bilinear expression with every operation separately rounded.
__global__ void __launch_bounds__(256) ab_to_source_kernel(const float* __restrict__ ab, int planes, int Ho, int Wo, int Hs, int Ws, int Hr,
                                                           int Wr, int oy, int ox, int fy, int fx, int h, int w, float* __restrict__ dst) {
  const size_t n = (size_t)planes * h * w;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(idx % w);
    const size_t t = idx / w;
    const int y = (int)(t % h);
    const size_t pl = t / h;
    const long long ny = (2LL * (fy + y) + 1) * Hr - (2LL * oy + 1) * Hs, nx = (2LL * (fx + x) + 1) * Wr - (2LL * ox + 1) * Ws;
    const double cy = fmin(fmax(__ddiv_rn((double)ny, 2.0 * Hs), 0.0), (double)(Ho - 1));
    const double cx = fmin(fmax(__ddiv_rn((double)nx, 2.0 * Ws), 0.0), (double)(Wo - 1));
    const int y0 = (int)floor(cy), x0 = (int)floor(cx);
    const int y1 = min(y0 + 1, Ho - 1), x1 = min(x0 + 1, Wo - 1);
    const float ly = (float)(cy - y0), lx = (float)(cx - x0);
    const float* sp = ab + pl * Ho * Wo;
    const float v00 = __ldg(sp + (size_t)y0 * Wo + x0), v01 = __ldg(sp + (size_t)y0 * Wo + x1);
    const float v10 = __ldg(sp + (size_t)y1 * Wo + x0), v11 = __ldg(sp + (size_t)y1 * Wo + x1);
    const float wy = __fsub_rn(1.f, ly), wx = __fsub_rn(1.f, lx);
    const float top = __fadd_rn(__fmul_rn(wx, v00), __fmul_rn(lx, v01)), bot = __fadd_rn(__fmul_rn(wx, v10), __fmul_rn(lx, v11));
    dst[idx] = __fadd_rn(__fmul_rn(wy, top), __fmul_rn(ly, bot));
  }
}

// ------------------------------------------------------------------------------------------------ CenterPad resize
__device__ __forceinline__ int mirror_idx(int i, int n) {  // scipy.ndimage mode="mirror": d c b | a b c d | c b a
  if (n == 1) return 0;
  const int period = 2 * (n - 1);
  i = i % period;
  if (i < 0) i += period;
  return i < n ? i : period - i;
}

// Gaussian along one axis in float64 (scipy.ndimage.gaussian_filter1d: weights exp(-0.5 k^2 / sigma^2) / sum, radius
// int(4 sigma + 0.5), correlate with mode="mirror").  src [n_outer][len][inner] -> dst, taps in `w` (2 r + 1 doubles).
template <typename TIn>
__global__ void __launch_bounds__(256) gauss_axis_kernel(const TIn* __restrict__ src, double* __restrict__ dst, const double* __restrict__ w,
                                                         int radius, size_t n_outer, int len, int inner) {
  const size_t total = n_outer * (size_t)len * inner;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int in_i = (int)(idx % inner);
    const size_t t = idx / inner;
    const int pos = (int)(t % len);
    const size_t outer = t / len;
    const TIn* base = src + outer * (size_t)len * inner + in_i;
    // scipy's correlate1d for symmetric weights: centre tap first, then the pairs (left + right) * w from the OUTSIDE in.
    // Separately rounded multiplies and adds (no FMA contraction): with sigma = 0.125 (a 1.25x down-scale) the taps are
    // (1.3e-14, 1, 1.3e-14), the filtered values sit within 1e-12 of integers and the final truncation to uint8 sees
    // the last bit -- scipy's C code is compiled without FMA.
    double acc = __dmul_rn((double)base[(size_t)pos * inner], w[radius]);
    for (int k = radius; k >= 1; --k) {
      const double l = (double)base[(size_t)mirror_idx(pos - k, len) * inner], r = (double)base[(size_t)mirror_idx(pos + k, len) * inner];
      acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(l, r), w[radius + k]));
    }
    dst[idx] = acc;
  }
}

// scipy.ndimage.zoom(order=1, mode="mirror", grid_mode=True) of a [Hs][Ws][C] float64 image to [Hr][Wr], truncated to
// uint8 (ndarray.astype(np.uint8) of in-range values), then CenterPad's centred crop (offset oy, ox) / zero pad into
// the [Ho][Wo][C] output.  Channels are independent: a grey frame (C = 1) gives each channel of its (g, g, g) expansion.
template <int C>
__global__ void __launch_bounds__(256) zoom_crop_kernel(const double* __restrict__ src, int Hs, int Ws, int Hr, int Wr, int oy, int ox,
                                                        unsigned char* __restrict__ dst, int Ho, int Wo) {
  const size_t total = (size_t)Ho * Wo * C;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % C);
    const size_t t = idx / C;
    const int xo = (int)(t % Wo), yo = (int)(t / Wo);
    const int yr = yo + oy, xr = xo + ox;  // position in the resized image
    unsigned char out = 0;
    if (yr >= 0 && yr < Hr && xr >= 0 && xr < Wr) {
      // grid_mode: pixel centres align, in = (out + 0.5) * (in_len / out_len) - 0.5
      // (separately rounded operations throughout: see gauss_axis_kernel)
      const double cy = __dsub_rn(__dmul_rn(__dadd_rn((double)yr, 0.5), __ddiv_rn((double)Hs, (double)Hr)), 0.5);
      const double cx = __dsub_rn(__dmul_rn(__dadd_rn((double)xr, 0.5), __ddiv_rn((double)Ws, (double)Wr)), 0.5);
      const double fy = floor(cy), fx = floor(cx);
      const double ty = __dsub_rn(cy, fy), tx = __dsub_rn(cx, fx);
      const int y0 = mirror_idx((int)fy, Hs), y1 = mirror_idx((int)fy + 1, Hs);
      const int x0 = mirror_idx((int)fx, Ws), x1 = mirror_idx((int)fx + 1, Ws);
      const double v00 = src[((size_t)y0 * Ws + x0) * C + ch], v01 = src[((size_t)y0 * Ws + x1) * C + ch];
      const double v10 = src[((size_t)y1 * Ws + x0) * C + ch], v11 = src[((size_t)y1 * Ws + x1) * C + ch];
      // scipy (ni_interpolation.c) sums the 2 x 2 neighbourhood, row-major, each term ((value * wy) * wx)
      const double wy0 = __dsub_rn(1.0, ty), wx0 = __dsub_rn(1.0, tx);
      double v = __dmul_rn(__dmul_rn(v00, wy0), wx0);
      v = __dadd_rn(v, __dmul_rn(__dmul_rn(v01, wy0), tx));
      v = __dadd_rn(v, __dmul_rn(__dmul_rn(v10, ty), wx0));
      v = __dadd_rn(v, __dmul_rn(__dmul_rn(v11, ty), tx));
      out = (unsigned char)fmin(fmax(trunc(v), 0.0), 255.0);
    }
    dst[idx] = out;
  }
}

// ------------------------------------------------------------------------------------------------ contextual loss
// mean over the N positions of every (image, channel): one block per (b, c), double accumulation
__global__ void __launch_bounds__(256) chan_mean_kernel(const float* __restrict__ x, float* __restrict__ mean, int N) {
  __shared__ double red[256];
  const float* p = x + (size_t)blockIdx.x * N;
  double acc = 0.0;
  for (int i = threadIdx.x; i < N; i += 256) acc += (double)__ldg(p + i);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o >= 1; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean[blockIdx.x] = (float)(red[0] / N);
}

// NCHW [B][C][N] -> position-major rows [B][N][C] of (x - mean_c) / (||x - mean||_2 over C + eps)  (ContextualLoss.py:99-111,
// feature_normalize util.py:155-158).  One block = 32 positions: first the norms (reads coalesced over positions), then a
// 32 x 32 shared-memory transpose per channel group so that the row stores are contiguous.
__global__ void __launch_bounds__(256) center_norm_rows_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                                               float* __restrict__ rows, int C, int N, float eps) {
  __shared__ float tile[32][33];
  __shared__ float s_inv[32];
  __shared__ float s_part[8][32];
  const int b = blockIdx.y, n0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float* xb = x + (size_t)b * C * N;
  const float* mb = mean ? mean + (size_t)b * C : nullptr;
  const int n = n0 + tx;
  float ss = 0.f;
  for (int c = ty; c < C; c += 8) {
    const float v = (n < N ? __ldg(xb + (size_t)c * N + n) : 0.f) - (mb ? __ldg(mb + c) : 0.f);
    ss = fmaf(v, v, ss);
  }
  s_part[ty][tx] = ss;
  __syncthreads();
  if (ty == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += s_part[k][tx];
    s_inv[tx] = 1.f / (sqrtf(t) + eps);
  }
  __syncthreads();
  for (int c0 = 0; c0 < C; c0 += 32) {
    for (int k = ty; k < 32; k += 8) {  // channel c0 + k, position n0 + tx
      const int c = c0 + k;
      tile[k][tx] = (c < C && n < N) ? (__ldg(xb + (size_t)c * N + n) - (mb ? __ldg(mb + c) : 0.f)) * s_inv[tx] : 0.f;
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {  // position n0 + k, channel c0 + tx
      if (n0 + k < N && c0 + tx < C) rows[((size_t)b * N + n0 + k) * C + c0 + tx] = tile[tx][k];
    }
    __syncthreads();
  }
}

// log2(e) / T_i with T_i = h * (min_j d_ij + 1e-5) = h * (1 - max_j f_ij + 1e-5)   (ContextualLoss.py:118-122)
__global__ void __launch_bounds__(256) ctx_row_scale_kernel(const float* __restrict__ rowmax, float* __restrict__ row_sc, size_t n, float h) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    row_sc[i] = 1.4426950408889634f / (h * ((1.f - __ldg(rowmax + i)) + 1e-5f));
}

// loss_b = -log(mean_i max_j A_ij) with max_j A_ij = 1 / sum_j exp((f_ij - m_i) / T_i)   (ContextualLoss.py:123-126)
__global__ void __launch_bounds__(256) ctx_loss_kernel(const float* __restrict__ denom, float* __restrict__ loss, int N) {
  __shared__ double red[256];
  const float* p = denom + (size_t)blockIdx.x * N;
  double acc = 0.0;
  for (int i = threadIdx.x; i < N; i += 256) acc += 1.0 / (double)__ldg(p + i);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o >= 1; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[blockIdx.x] = (float)(-log(red[0] / N));
}

// ------------------------------------------------------------------------------------------------ I420 <-> sRGB
// OpenCV's BT.601 limited-range 4:2:0 conversions (cv2.cvtColor COLOR_YUV2RGB_I420 / COLOR_RGB2YUV_I420, modules/imgproc
// color_yuv.simd.hpp): fixed point with 20 fraction bits, rounding by + 2^19, arithmetic >> 20, saturation to [0, 255].  Every
// intermediate fits in int32, so the bytes do not depend on the compiler's contraction choices.  An I420 frame [3H/2][W] is the Y
// plane [H][W], then U [H/2][W/2], then V [H/2][W/2]; H and W are even.  One thread per 2 x 2 block of pixels, which shares one
// (u, v): nearest-neighbour chroma in both directions (the chroma siting is not modelled).
constexpr int kYuvShift = 20, kYuvHalf = 1 << (kYuvShift - 1);
constexpr int kY2Rgb = 1220542, kV2R = 1673527, kV2G = -852492, kU2G = -409993, kU2B = 2116026;
constexpr int kR2Y = 269484, kG2Y = 528482, kB2Y = 102760;
constexpr int kR2U = -155188, kG2U = -305135, kB2U = 460324, kR2V = 460324, kG2V = -385875, kB2V = -74448;

__device__ __forceinline__ unsigned char sat_u8(int v) { return (unsigned char)min(max(v, 0), 255); }

// yuv [B][3H/2][W] -> rgb [B][H][W][3]
__global__ void __launch_bounds__(256) i420_to_rgb8_kernel(const unsigned char* __restrict__ yuv, unsigned char* __restrict__ rgb, int B,
                                                           int H, int W) {
  const int h2 = H / 2, w2 = W / 2;
  const size_t nb = (size_t)h2 * w2, frame = (size_t)H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B * nb; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / nb, q = i - b * nb;
    const int by = (int)(q / w2), bx = (int)(q - (size_t)by * w2);
    const unsigned char* Y = yuv + b * (frame * 3 / 2);
    const int d = (int)__ldg(Y + frame + q) - 128, e = (int)__ldg(Y + frame + nb + q) - 128;
    const int r = kYuvHalf + kV2R * e, g = kYuvHalf + kV2G * e + kU2G * d, bl = kYuvHalf + kU2B * d;
    unsigned char* out = rgb + (b * frame + (size_t)2 * by * W + 2 * bx) * 3;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int y = max(0, (int)__ldg(Y + (size_t)(2 * by + dy) * W + 2 * bx + dx) - 16) * kY2Rgb;
        unsigned char* px = out + ((size_t)dy * W + dx) * 3;
        px[0] = sat_u8((y + r) >> kYuvShift);
        px[1] = sat_u8((y + g) >> kYuvShift);
        px[2] = sat_u8((y + bl) >> kYuvShift);
      }
  }
}

// rgb [B][H][W][3] -> yuv [B][3H/2][W]: Y of every pixel, U and V of the top-left pixel of each 2 x 2 block (no averaging)
__global__ void __launch_bounds__(256) rgb8_to_i420_kernel(const unsigned char* __restrict__ rgb, unsigned char* __restrict__ yuv, int B,
                                                           int H, int W) {
  const int h2 = H / 2, w2 = W / 2;
  const size_t nb = (size_t)h2 * w2, frame = (size_t)H * W;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B * nb; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / nb, q = i - b * nb;
    const int by = (int)(q / w2), bx = (int)(q - (size_t)by * w2);
    const unsigned char* in = rgb + (b * frame + (size_t)2 * by * W + 2 * bx) * 3;
    unsigned char* Y = yuv + b * (frame * 3 / 2);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const unsigned char* px = in + ((size_t)dy * W + dx) * 3;
        const int v = kR2Y * __ldg(px) + kG2Y * __ldg(px + 1) + kB2Y * __ldg(px + 2) + kYuvHalf + (16 << kYuvShift);
        Y[(size_t)(2 * by + dy) * W + 2 * bx + dx] = sat_u8(v >> kYuvShift);
      }
    const int r = __ldg(in), g = __ldg(in + 1), bl = __ldg(in + 2);
    Y[frame + q] = sat_u8((kR2U * r + kG2U * g + kB2U * bl + kYuvHalf + (128 << kYuvShift)) >> kYuvShift);
    Y[frame + nb + q] = sat_u8((kR2V * r + kG2V * g + kB2V * bl + kYuvHalf + (128 << kYuvShift)) >> kYuvShift);
  }
}

inline int grid_for(size_t total, int threads, int cap = 132 * 16) {
  const size_t g = (total + threads - 1) / threads;
  return (int)(g < (size_t)cap ? (g ? g : 1) : cap);
}

}  // namespace

void launch_chan_mean(const float* x, float* mean, int B, int C, int N, cudaStream_t s) {
  chan_mean_kernel<<<B * C, 256, 0, s>>>(x, mean, N);
  launch_counter_add(1);
}
void launch_center_norm_rows(const float* x, const float* mean, float* rows, int B, int C, int N, float eps, cudaStream_t s) {
  center_norm_rows_kernel<<<dim3((N + 31) / 32, B), 256, 0, s>>>(x, mean, rows, C, N, eps);
  launch_counter_add(1);
}
void launch_ctx_row_scale(const float* rowmax, float* row_sc, size_t n, float h, cudaStream_t s) {
  ctx_row_scale_kernel<<<grid_for(n, 256), 256, 0, s>>>(rowmax, row_sc, n, h);
  launch_counter_add(1);
}
void launch_ctx_loss(const float* denom, float* loss, int B, int N, cudaStream_t s) {
  ctx_loss_kernel<<<B, 256, 0, s>>>(denom, loss, N);
  launch_counter_add(1);
}
void launch_fgs_weights(const unsigned char* guide, const float* lut, float* Ch, float* Cv, int G, int H, int W, cudaStream_t s) {
  fgs_weights_kernel<<<dim3(grid_for((size_t)H * W, 256), G), 256, 0, s>>>(guide, lut, Ch, Cv, H, W);
  launch_counter_add(1);
}
void launch_fgs_horizontal(float* cur, const float* Ch, float* D, int planes, const PlaneSrc& gsrc, int H, int W, float lam,
                           cudaStream_t s) {
  fgs_horizontal_kernel<<<planes * ((H + 31) / 32), 32, 0, s>>>(cur, Ch, D, planes, gsrc, H, W, lam);
  launch_counter_add(1);
}
void launch_fgs_vertical(float* cur, const float* Cv, float* D, int planes, const PlaneSrc& gsrc, int H, int W, float lam,
                         cudaStream_t s) {
  fgs_vertical_kernel<<<(planes * W + 127) / 128, 128, 0, s>>>(cur, Cv, D, planes, gsrc, H, W, lam);
  launch_counter_add(1);
}
void launch_l_to_guide8(const float* l, unsigned char* g, size_t n, cudaStream_t s) {
  l_to_guide8_kernel<<<grid_for(n, 256), 256, 0, s>>>(l, g, n);
  launch_counter_add(1);
}
void launch_rgb8_to_l_half(const unsigned char* rgb, int C, float* l, float* l_half, unsigned char* guide, int H, int W, cudaStream_t s) {
  const int grid = grid_for((size_t)(H / 2) * ((W + 15) / 16) * 32, 256);
  if (C == 1)
    rgb8_to_l_half_kernel<1><<<grid, 256, 0, s>>>(rgb, l, l_half, guide, H, W);
  else
    rgb8_to_l_half_kernel<3><<<grid, 256, 0, s>>>(rgb, l, l_half, guide, H, W);
  launch_counter_add(1);
}
void launch_rgb8_to_l_guide(const unsigned char* rgb, int C, int Ws, int y0, int x0, int h, int w, float* l, unsigned char* guide,
                            cudaStream_t s) {
  if (C == 1)
    rgb8_to_l_guide_kernel<1><<<grid_for((size_t)h * w, 256), 256, 0, s>>>(rgb, Ws, y0, x0, h, w, l, guide);
  else
    rgb8_to_l_guide_kernel<3><<<grid_for((size_t)h * w, 256), 256, 0, s>>>(rgb, Ws, y0, x0, h, w, l, guide);
  launch_counter_add(1);
}
void launch_ab_to_source(const float* ab, int planes, int Ho, int Wo, const int g[6], const int fp[4], float* dst, cudaStream_t s) {
  ab_to_source_kernel<<<grid_for((size_t)planes * fp[2] * fp[3], 256), 256, 0, s>>>(ab, planes, Ho, Wo, g[0], g[1], g[2], g[3], g[4], g[5],
                                                                                    fp[0], fp[1], fp[2], fp[3], dst);
  launch_counter_add(1);
}
void launch_gauss_axis_u8(const unsigned char* src, double* dst, const double* w, int radius, size_t n_outer, int len, int inner,
                          cudaStream_t s) {
  gauss_axis_kernel<unsigned char><<<grid_for(n_outer * len * inner, 256), 256, 0, s>>>(src, dst, w, radius, n_outer, len, inner);
  launch_counter_add(1);
}
void launch_gauss_axis_f64(const double* src, double* dst, const double* w, int radius, size_t n_outer, int len, int inner,
                           cudaStream_t s) {
  gauss_axis_kernel<double><<<grid_for(n_outer * len * inner, 256), 256, 0, s>>>(src, dst, w, radius, n_outer, len, inner);
  launch_counter_add(1);
}
void launch_zoom_crop(const double* src, int C, int Hs, int Ws, int Hr, int Wr, int oy, int ox, unsigned char* dst, int Ho, int Wo,
                      cudaStream_t s) {
  if (C == 1)
    zoom_crop_kernel<1><<<grid_for((size_t)Ho * Wo, 256), 256, 0, s>>>(src, Hs, Ws, Hr, Wr, oy, ox, dst, Ho, Wo);
  else
    zoom_crop_kernel<3><<<grid_for((size_t)Ho * Wo * 3, 256), 256, 0, s>>>(src, Hs, Ws, Hr, Wr, oy, ox, dst, Ho, Wo);
  launch_counter_add(1);
}
void launch_i420_to_rgb8(const unsigned char* yuv, unsigned char* rgb, int B, int H, int W, cudaStream_t s) {
  i420_to_rgb8_kernel<<<grid_for((size_t)B * (H / 2) * (W / 2), 256), 256, 0, s>>>(yuv, rgb, B, H, W);
  launch_counter_add(1);
}
void launch_rgb8_to_i420(const unsigned char* rgb, unsigned char* yuv, int B, int H, int W, cudaStream_t s) {
  rgb8_to_i420_kernel<<<grid_for((size_t)B * (H / 2) * (W / 2), 256), 256, 0, s>>>(rgb, yuv, B, H, W);
  launch_counter_add(1);
}

}  // namespace dvc
