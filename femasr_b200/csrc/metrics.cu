// PSNR and SSIM, the training configs' other two validation metrics, as pyiqa's `psnr` / `ssim` define them (recalled,
// not verified offline: DESIGN.md section 6, "PSNR / SSIM").  Inputs x, y [B,3,H,W] fp32 NCHW in [0, 1]; one score per
// image.  Both kernels end in the fixed-order per-image reduction of common.cuh (image_sum_last_block), so an image's
// score depends neither on the other images of the batch nor on the block schedule, and every per-pixel formula treats
// x and y symmetrically, so metric(x, y) == metric(y, x) bit for bit.
#include <cmath>

#include "common.cuh"

namespace femasr {

constexpr int MET_THREADS = 256, MET_WARPS = MET_THREADS / 32;
constexpr int PSNR_PIX_PER_THREAD = 8, PSNR_PIX = MET_THREADS * PSNR_PIX_PER_THREAD;   // pixels per PSNR block
constexpr int SSIM_WIN = 11, SSIM_HALO = SSIM_WIN - 1;
constexpr int SSIM_TW = 32, SSIM_TH = 16;                                               // output tile per SSIM block
constexpr int SSIM_IW = SSIM_TW + SSIM_HALO, SSIM_IH = SSIM_TH + SSIM_HALO;

// The Y channel of one pixel, in a fixed operation order without contraction (the CPU oracle reproduces it bit for bit):
// yiq ((0.299 R + 0.587 G) + 0.114 B); ycbcr (((65.481 R + 128.553 G) + 24.966 B) + 16) / 255.
__device__ __forceinline__ float y_of(float r, float g, float b, int mode) {
  if (mode == FEMASR_METRIC_Y_YIQ)
    return __fadd_rn(__fadd_rn(__fmul_rn(0.299f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
  const float t = __fadd_rn(__fadd_rn(__fmul_rn(65.481f, r), __fmul_rn(128.553f, g)), __fmul_rn(24.966f, b));
  return __fdiv_rn(__fadd_rn(t, 16.f), 255.f);
}

// Block sum of one fp64 value per thread: the fixed xor tree per warp, then the warps in order by thread 0 (the only
// thread whose result is meaningful).
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum_d(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < MET_WARPS; ++i) t += red[i];
  return t;
}

// grid (ceil(Hc*Wc / PSNR_PIX), B).  Thread t of block k owns the cropped pixels k*PSNR_PIX + j*256 + t (j < 8) in
// row-major order: coalesced 4-byte loads, all 48 issued before the first is used.  x - y in fp32, its square summed in fp64.
__global__ void __launch_bounds__(MET_THREADS) psnr_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                           int H, int W, int crop, int mode, float* __restrict__ out,
                                                           double* __restrict__ partial,
                                                           unsigned int* __restrict__ count) {
  __shared__ double red[MET_THREADS];
  const int b = blockIdx.y, Wc = W - 2 * crop, n = (H - 2 * crop) * Wc;      // n < 2^31: metric_blocks
  const long plane = (long)H * W;
  const float* xb = x + (long)b * 3 * plane;
  const float* yb = y + (long)b * 3 * plane;
  const int first = blockIdx.x * PSNR_PIX + threadIdx.x;
  float xv[PSNR_PIX_PER_THREAD][3], yv[PSNR_PIX_PER_THREAD][3];
#pragma unroll
  for (int j = 0; j < PSNR_PIX_PER_THREAD; ++j) {    // every load first (a pixel past the end reads pixel 0, unused)
    const int i = first + j * MET_THREADS;
    const long off = i < n ? (long)(i / Wc + crop) * W + i % Wc + crop : 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      xv[j][c] = __ldg(xb + c * plane + off);
      yv[j][c] = __ldg(yb + c * plane + off);
    }
  }
  double acc = 0.0;
#pragma unroll
  for (int j = 0; j < PSNR_PIX_PER_THREAD; ++j) {
    if (first + j * MET_THREADS >= n) break;
    if (mode == FEMASR_METRIC_RGB) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double d = __fsub_rn(xv[j][c], yv[j][c]);
        acc += d * d;                              // exact: a float squared fits a double
      }
    } else {
      const double d = __fsub_rn(y_of(xv[j][0], xv[j][1], xv[j][2], mode), y_of(yv[j][0], yv[j][1], yv[j][2], mode));
      acc += d * d;
    }
  }
  double total = 0.0;
  if (!image_sum_last_block<MET_THREADS>(block_sum(acc, red), partial, count, red, total)) return;
  if (threadIdx.x == 0) {
    const double mse = total / ((mode == FEMASR_METRIC_RGB ? 3.0 : 1.0) * (double)n);
    out[b] = (float)(10.0 * log10(1.0 / (mse + 1e-8)));
  }
}

struct Gauss11 {
  double w[SSIM_WIN];
};

// One SSIM map value from the five window moments.  Explicit roundings (no contraction), so that swapping x and y swaps
// operands of commutative operations only, and so that x == y gives l == cs == 1 exactly (2a and a + a are both exact).
__device__ __forceinline__ double ssim_map(double mx, double my, double exx, double eyy, double exy) {
  const double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
  const double mxx = __dmul_rn(mx, mx), myy = __dmul_rn(my, my), mxy = __dmul_rn(mx, my);
  const double vx = __dsub_rn(exx, mxx), vy = __dsub_rn(eyy, myy), cxy = __dsub_rn(exy, mxy);
  const double cs = fmax(__ddiv_rn(__dadd_rn(__dmul_rn(2.0, cxy), C2), __dadd_rn(__dadd_rn(vx, vy), C2)), 0.0);
  const double l = __ddiv_rn(__dadd_rn(__dmul_rn(2.0, mxy), C1), __dadd_rn(__dadd_rn(mxx, myy), C1));
  return __dmul_rn(l, cs);
}

// grid (tiles_y * tiles_x, B), a 32x16 output tile per block ('valid' filtering: output (Hc-10) x (Wc-10)).  Per channel
// (one for Y, three for RGB): stage the tile plus its 10-pixel halo of both images into shared memory at data range 255
// (Y rounded half to even, RGB channels unrounded), the horizontal 11-tap pass into the five moments mu_x, mu_y, E[x^2],
// E[y^2], E[xy] in fp64, the vertical pass and the map in fp64.
__global__ void __launch_bounds__(MET_THREADS) ssim_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                           int H, int W, int crop, int mode, Gauss11 g,
                                                           float* __restrict__ out, double* __restrict__ partial,
                                                           unsigned int* __restrict__ count) {
  __shared__ float sx[SSIM_IH][SSIM_IW], sy[SSIM_IH][SSIM_IW];
  __shared__ double hm[5][SSIM_IH][SSIM_TW];
  __shared__ double red[MET_THREADS];
  const int b = blockIdx.y;
  const int Hc = H - 2 * crop, Wc = W - 2 * crop, Ho = Hc - SSIM_HALO, Wo = Wc - SSIM_HALO;
  const int tiles_x = (Wo + SSIM_TW - 1) / SSIM_TW;
  const int ty0 = (blockIdx.x / tiles_x) * SSIM_TH, tx0 = (blockIdx.x % tiles_x) * SSIM_TW;
  const long plane = (long)H * W;
  const float* xb = x + (long)b * 3 * plane;
  const float* yb = y + (long)b * 3 * plane;
  const int nch = mode == FEMASR_METRIC_RGB ? 3 : 1;
  double acc = 0.0;
  for (int c = 0; c < nch; ++c) {
    for (int i = threadIdx.x; i < SSIM_IH * SSIM_IW; i += MET_THREADS) {
      const int r = i / SSIM_IW, q = i % SSIM_IW;
      float vx = 0.f, vy = 0.f;                    // outside the image: feeds no valid output
      if (ty0 + r < Hc && tx0 + q < Wc) {
        const long off = (long)(ty0 + r + crop) * W + tx0 + q + crop;
        if (mode == FEMASR_METRIC_RGB) {
          vx = __fmul_rn(__ldg(xb + c * plane + off), 255.f);
          vy = __fmul_rn(__ldg(yb + c * plane + off), 255.f);
        } else {
          vx = rintf(__fmul_rn(y_of(__ldg(xb + off), __ldg(xb + plane + off), __ldg(xb + 2 * plane + off), mode), 255.f));
          vy = rintf(__fmul_rn(y_of(__ldg(yb + off), __ldg(yb + plane + off), __ldg(yb + 2 * plane + off), mode), 255.f));
        }
      }
      sx[r][q] = vx;
      sy[r][q] = vy;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SSIM_IH * SSIM_TW; i += MET_THREADS) {
      const int r = i / SSIM_TW, q = i % SSIM_TW;
      double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0, m4 = 0.0;
#pragma unroll
      for (int j = 0; j < SSIM_WIN; ++j) {
        const double a = sx[r][q + j], e = sy[r][q + j], w = g.w[j];
        m0 = fma(w, a, m0);
        m1 = fma(w, e, m1);
        m2 = fma(w, a * a, m2);                    // products of two floats are exact in fp64
        m3 = fma(w, e * e, m3);
        m4 = fma(w, a * e, m4);
      }
      hm[0][r][q] = m0; hm[1][r][q] = m1; hm[2][r][q] = m2; hm[3][r][q] = m3; hm[4][r][q] = m4;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SSIM_TH * SSIM_TW; i += MET_THREADS) {
      const int r = i / SSIM_TW, q = i % SSIM_TW;
      if (ty0 + r >= Ho || tx0 + q >= Wo) continue;
      double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int j = 0; j < SSIM_WIN; ++j) {
        const double w = g.w[j];
#pragma unroll
        for (int k = 0; k < 5; ++k) m[k] = fma(w, hm[k][r + j][q], m[k]);
      }
      acc += ssim_map(m[0], m[1], m[2], m[3], m[4]);
    }
    __syncthreads();
  }
  double total = 0.0;
  if (!image_sum_last_block<MET_THREADS>(block_sum(acc, red), partial, count, red, total)) return;
  if (threadIdx.x == 0) out[b] = (float)(total / ((double)nch * Ho * Wo));
}

// The normalised 11-tap Gaussian, sigma 1.5, in fp64 (the 2-D window is its outer product).
const Gauss11& gauss11() {
  static const Gauss11 g = [] {
    Gauss11 t;
    double s = 0.0;
    for (int i = 0; i < SSIM_WIN; ++i) s += t.w[i] = std::exp(-(double)((i - 5) * (i - 5)) / (2.0 * 1.5 * 1.5));
    for (int i = 0; i < SSIM_WIN; ++i) t.w[i] /= s;
    return t;
  }();
  return g;
}

// Blocks per image of `kind`, or -1 with the error set when the geometry is refused.
long metric_blocks(const char* name, int kind, int B, int H, int W, int crop, int mode) {
  const std::string n(name);
  if (B <= 0 || B > 65535) return fail(FEMASR_ERR_ARG, n + ": B must be in [1, 65535]"), -1;
  if (H <= 0 || W <= 0 || crop < 0 || 2l * crop >= H || 2l * crop >= W)
    return fail(FEMASR_ERR_ARG, n + ": crop_border must be >= 0 and leave at least one pixel (2*crop < H and W)"), -1;
  if (mode != FEMASR_METRIC_RGB && mode != FEMASR_METRIC_Y_YIQ && mode != FEMASR_METRIC_Y_YCBCR)
    return fail(FEMASR_ERR_ARG, n + ": mode must be FEMASR_METRIC_RGB, _Y_YIQ or _Y_YCBCR"), -1;
  const long Hc = H - 2l * crop, Wc = W - 2l * crop;
  long nblk;
  if (kind == FEMASR_METRIC_PSNR) {
    nblk = cdiv(Hc * Wc, PSNR_PIX);
  } else if (kind == FEMASR_METRIC_SSIM) {
    if (Hc < SSIM_WIN || Wc < SSIM_WIN)
      return fail(FEMASR_ERR_ARG, n + ": the cropped image must be at least 11x11 (the Gaussian window)"), -1;
    nblk = cdiv(Hc - SSIM_HALO, SSIM_TH) * cdiv(Wc - SSIM_HALO, SSIM_TW);
  } else {
    return fail(FEMASR_ERR_ARG, n + ": kind must be FEMASR_METRIC_PSNR or FEMASR_METRIC_SSIM"), -1;
  }
  if (Hc * Wc + PSNR_PIX >= (1l << 31)) return fail(FEMASR_ERR_ARG, n + ": image too large (2^31 pixels)"), -1;
  return nblk;
}

int metric_launch(int kind, const float* x, const float* y, int B, int H, int W, int crop, int mode, float* out,
                  void* scratch, void* stream) {
  const char* name = kind == FEMASR_METRIC_PSNR ? "psnr" : "ssim";
  FEMASR_CHECK_ARG(x && y && out && scratch, std::string(name) + ": null pointer");
  const long nblk = metric_blocks(name, kind, B, H, W, crop, mode);
  if (nblk < 0) return FEMASR_ERR_ARG;
  double* partial = reinterpret_cast<double*>(scratch);
  unsigned int* count = reinterpret_cast<unsigned int*>(partial + (size_t)B * nblk);
  cudaStream_t st = as_stream(stream);
  FEMASR_CUDA(cudaMemsetAsync(count, 0, (size_t)B * sizeof(unsigned int), st));
  const dim3 grid((unsigned)nblk, (unsigned)B);
  if (kind == FEMASR_METRIC_PSNR) {
    psnr_kernel<<<grid, MET_THREADS, 0, st>>>(x, y, H, W, crop, mode, out, partial, count);
    return launch_status("psnr_kernel");
  }
  ssim_kernel<<<grid, MET_THREADS, 0, st>>>(x, y, H, W, crop, mode, gauss11(), out, partial, count);
  return launch_status("ssim_kernel");
}

}  // namespace femasr

using namespace femasr;

// [B][nblk] fp64 partials, then B uint32 arrival counters
extern "C" size_t femasr_metric_scratch_bytes(int kind, int B, int H, int W, int crop) {
  const long nblk = metric_blocks(kind == FEMASR_METRIC_PSNR ? "psnr" : "ssim", kind, B, H, W, crop, FEMASR_METRIC_RGB);
  if (nblk < 0) return 0;
  return (size_t)B * nblk * sizeof(double) + (size_t)B * sizeof(unsigned int);
}

extern "C" int femasr_psnr(const float* x, const float* y, int B, int H, int W, int crop, int mode, float* out,
                           void* scratch, void* stream) {
  return metric_launch(FEMASR_METRIC_PSNR, x, y, B, H, W, crop, mode, out, scratch, stream);
}

extern "C" int femasr_ssim(const float* x, const float* y, int B, int H, int W, int crop, int mode, float* out,
                           void* scratch, void* stream) {
  return metric_launch(FEMASR_METRIC_SSIM, x, y, B, H, W, crop, mode, out, scratch, stream);
}
