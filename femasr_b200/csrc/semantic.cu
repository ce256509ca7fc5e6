// The small kernels of the HQ stage's semantic loss (femasr_arch.py:301-309, 318-320, 344-347): the normalising
// im2col of VGG19's conv1_1, the fp32 max-pool of the SIMT path and the squared-difference rows of the MSE.  The
// twelve VGG convs and conv_semantic themselves run on femasr_tc_igemm / femasr_igemm_simt with the ReLU epilogue,
// and the pool of the tensor-core path is femasr_tc_prepare's FEMASR_PRO_MAXPOOL2 mode.
#include <cuda_fp16.h>

#include "common.cuh"

namespace femasr {

// conv1_1's operand: per output pixel the 3x3x3 window of (x - mean) / std (vgg_arch.py forward: division, not a
// multiply by 1/std), k = (kh * 3 + kw) * 3 + ci, zero padded to K = 64.  Thread = (pixel, 8-wide k chunk).
// mean == NULL: the window of x itself (the discriminator's conv0).
__global__ void __launch_bounds__(256) vgg_im2col_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                                         const float* __restrict__ stdv, uint4* __restrict__ hi,
                                                         uint4* __restrict__ lo, float4* __restrict__ f32, int H, int W,
                                                         long total) {
  const long i = (long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const int j = (int)(i & 7);
  const long m = i >> 3;
  const int ox = (int)(m % W);
  const long t = m / W;
  const int oy = (int)(t % H);
  const long b = t / H;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = j * 8 + e;
    v[e] = 0.f;
    if (k < 27) {
      const int tap = k / 3, ci = k - tap * 3;
      const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        const float px = __ldg(x + ((b * 3 + ci) * H + iy) * W + ix);
        v[e] = mean ? __fdiv_rn(__fsub_rn(px, __ldg(mean + ci)), __ldg(stdv + ci)) : px;   // NULL mean/std: raw image
      }
    }
  }
  if (f32) {
    f32[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
    f32[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
    return;
  }
  __align__(16) __half h[8], l[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float cl = fminf(fmaxf(v[e], -65504.f), 65504.f);
    h[e] = __float2half_rn(cl);
    l[e] = __float2half_rn(cl - __half2float(h[e]));
  }
  hi[i] = *reinterpret_cast<const uint4*>(h);
  lo[i] = *reinterpret_cast<const uint4*>(l);
}

// OIHW [Cout,3,3,3] -> [Cout][64] fp32 in the im2col K order, zero padded
__global__ void vgg_weight_pad_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cout * 64) return;
  const int co = i >> 6, k = i & 63;
  float v = 0.f;
  if (k < 27) { const int tap = k / 3, ci = k - tap * 3; v = w[((co * 3 + ci) * 3 + tap / 3) * 3 + tap % 3]; }
  out[i] = v;
}

__global__ void __launch_bounds__(256) maxpool2_kernel(const float* __restrict__ x, float4* __restrict__ y, int H, int W,
                                                       int C, long total8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  float v[8];
  const long o = pool2_max8(x, i, H, W, C, v) / 4;
  y[o] = make_float4(v[0], v[1], v[2], v[3]);
  y[o + 1] = make_float4(v[4], v[5], v[6], v[7]);
}

// one warp per row: lane-strided fp32 FMA chain, then the fixed xor-tree - the same order on every run
__global__ void __launch_bounds__(256) sq_diff_rows_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                           float* __restrict__ rows, int N, int C) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= N) return;
  const int lane = threadIdx.x & 31;
  const float* pa = a + (long)r * C;
  const float* pb = b + (long)r * C;
  float s = 0.f;
  for (int k = lane; k < C; k += 32) {
    const float d = __fsub_rn(__ldg(pa + k), __ldg(pb + k));
    s = fmaf(d, d, s);
  }
  s = warp_sum(s);
  if (lane == 0) rows[r] = s;
}

}  // namespace femasr

using namespace femasr;

extern "C" int femasr_vgg_im2col(const float* x, const float* mean, const float* std_, void* a_hi, void* a_lo, float* a_f32,
                                 int B, int H, int W, void* stream) {
  FEMASR_CHECK_ARG(x && B > 0 && H > 0 && W > 0, "vgg_im2col: bad argument");
  FEMASR_CHECK_ARG(!mean == !std_, "vgg_im2col: give both mean and std, or neither (no normalisation)");
  FEMASR_CHECK_ARG(a_f32 ? (!a_hi && !a_lo) : (a_hi && a_lo), "vgg_im2col: give either a_hi/a_lo or a_f32");
  const long total = (long)B * H * W * 8;
  vgg_im2col_kernel<<<(unsigned)cdiv(total, 256), 256, 0, as_stream(stream)>>>(
      x, mean, std_, reinterpret_cast<uint4*>(a_hi), reinterpret_cast<uint4*>(a_lo), reinterpret_cast<float4*>(a_f32), H, W,
      total);
  return launch_status("vgg_im2col_kernel");
}

extern "C" int femasr_vgg_pad_weight(const float* w_oihw, float* w_padded, int Cout, void* stream) {
  FEMASR_CHECK_ARG(w_oihw && w_padded && Cout > 0, "vgg_pad_weight: bad argument");
  vgg_weight_pad_kernel<<<(unsigned)cdiv((long)Cout * 64, 256), 256, 0, as_stream(stream)>>>(w_oihw, w_padded, Cout);
  return launch_status("vgg_weight_pad_kernel");
}

extern "C" int femasr_maxpool2(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  FEMASR_CHECK_ARG(x && y && B > 0 && H >= 2 && W >= 2, "maxpool2: bad argument");
  FEMASR_CHECK_ARG(C % 8 == 0, "maxpool2: C must be a multiple of 8");
  const long total8 = (long)B * (H / 2) * (W / 2) * (C / 8);
  maxpool2_kernel<<<(unsigned)cdiv(total8, 256), 256, 0, as_stream(stream)>>>(x, reinterpret_cast<float4*>(y), H, W, C, total8);
  return launch_status("maxpool2_kernel");
}

extern "C" int femasr_sq_diff_rows(const float* a, const float* b, float* rows, int N, int C, void* stream) {
  FEMASR_CHECK_ARG(a && b && rows && N > 0 && C > 0, "sq_diff_rows: bad argument");
  sq_diff_rows_kernel<<<(unsigned)cdiv(N, 8), 256, 0, as_stream(stream)>>>(a, b, rows, N, C);
  return launch_status("sq_diff_rows_kernel");
}
