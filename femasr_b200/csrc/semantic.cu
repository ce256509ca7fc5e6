// The small kernels of the HQ stage's semantic loss (femasr_arch.py:301-309, 318-320, 344-347): the normalising
// im2col of VGG19's conv1_1 (also LPIPS' first conv and the discriminator's conv0), the fp32 max-pools of the SIMT path
// and the squared-difference rows of the MSE.  The
// twelve VGG convs and conv_semantic themselves run on femasr_tc_igemm / femasr_igemm_simt with the ReLU epilogue,
// and the pool of the tensor-core path is femasr_tc_prepare's FEMASR_PRO_MAXPOOL2 mode.
#include <cuda_fp16.h>

#include "common.cuh"

namespace femasr {

// The operand of a 3-channel first conv as a 1x1 GEMM: per output pixel the ks x ks window (stride, pad) of the
// transformed image, k = (kh * ks + kw) * 3 + ci, zero padded to kpad (a multiple of 64).  Thread = (pixel, 8-wide k
// chunk).  The transform is x' = 2x - 1 when two_x_minus_1 (LPIPS normalize=True), then (x' - mean) / std as a true
// division (vgg_arch.py forward, LPIPS' ScalingLayer); mean == NULL: the window of x itself (the discriminator's conv0).
// Images [0, B0) come from x0, the rest from x1 (the two inputs of a pair without a concatenated copy).
__global__ void __launch_bounds__(256) vgg_im2col_kernel(const float* __restrict__ x0, const float* __restrict__ x1,
                                                         int B0, const float* __restrict__ mean,
                                                         const float* __restrict__ stdv, int two_x_minus_1,
                                                         uint4* __restrict__ hi, uint4* __restrict__ lo,
                                                         float4* __restrict__ f32, int H, int W, int Ho, int Wo, int ks,
                                                         int stride, int pad, int kc8, long total) {
  const long i = (long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const int j = (int)(i % kc8);
  const long m = i / kc8;
  const int ox = (int)(m % Wo);
  const long t = m / Wo;
  const int oy = (int)(t % Ho);
  const long b = t / Ho;
  const float* x = b < B0 ? x0 + b * 3 * H * W : x1 + (b - B0) * 3 * H * W;
  const int kk = ks * ks * 3;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = j * 8 + e;
    v[e] = 0.f;
    if (k < kk) {
      const int tap = k / 3, ci = k - tap * 3;
      const int iy = oy * stride + tap / ks - pad, ix = ox * stride + tap % ks - pad;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
        float px = __ldg(x + ((long)ci * H + iy) * W + ix);
        if (two_x_minus_1) px = __fsub_rn(__fmul_rn(2.f, px), 1.f);
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

// OIHW [Cout,3,ks,ks] -> [Cout][kpad] fp32 in the im2col K order, zero padded
__global__ void vgg_weight_pad_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int ks, int kpad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cout * kpad) return;
  const int co = i / kpad, k = i - co * kpad;
  float v = 0.f;
  if (k < ks * ks * 3) { const int tap = k / 3, ci = k - tap * 3; v = w[((co * 3 + ci) * ks + tap / ks) * ks + tap % ks]; }
  out[i] = v;
}

template <int K>
__global__ void __launch_bounds__(256) maxpool_kernel(const float* __restrict__ x, float4* __restrict__ y, int H, int W,
                                                      int C, long total8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  float v[8];
  const long o = pool_max8<K>(x, i, H, W, C, v) / 4;
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

extern "C" int femasr_vgg_im2col_ex(const float* x0, const float* x1, int B, int H, int W, int ksize, int stride, int pad,
                                    int kpad, const float* mean, const float* std_, int two_x_minus_1, void* a_hi,
                                    void* a_lo, float* a_f32, void* stream) {
  FEMASR_CHECK_ARG(x0 && B > 0 && H > 0 && W > 0, "vgg_im2col: bad argument");
  FEMASR_CHECK_ARG(!mean == !std_, "vgg_im2col: give both mean and std, or neither (no normalisation)");
  FEMASR_CHECK_ARG(a_f32 ? (!a_hi && !a_lo) : (a_hi && a_lo), "vgg_im2col: give either a_hi/a_lo or a_f32");
  FEMASR_CHECK_ARG(ksize > 0 && stride > 0 && pad >= 0 && kpad % 64 == 0 && kpad >= 3 * ksize * ksize,
                   "vgg_im2col: need ksize, stride > 0, pad >= 0 and kpad a multiple of 64 holding 3 * ksize^2 taps");
  const int Ho = (H + 2 * pad - ksize) / stride + 1, Wo = (W + 2 * pad - ksize) / stride + 1;
  FEMASR_CHECK_ARG(H + 2 * pad >= ksize && W + 2 * pad >= ksize, "vgg_im2col: input smaller than the window");
  const long total = (long)(x1 ? 2 * B : B) * Ho * Wo * (kpad / 8);
  vgg_im2col_kernel<<<(unsigned)cdiv(total, 256), 256, 0, as_stream(stream)>>>(
      x0, x1, B, mean, std_, two_x_minus_1 ? 1 : 0, reinterpret_cast<uint4*>(a_hi), reinterpret_cast<uint4*>(a_lo),
      reinterpret_cast<float4*>(a_f32), H, W, Ho, Wo, ksize, stride, pad, kpad / 8, total);
  return launch_status("vgg_im2col_kernel");
}

extern "C" int femasr_vgg_im2col(const float* x, const float* mean, const float* std_, void* a_hi, void* a_lo, float* a_f32,
                                 int B, int H, int W, void* stream) {
  return femasr_vgg_im2col_ex(x, nullptr, B, H, W, 3, 1, 1, 64, mean, std_, 0, a_hi, a_lo, a_f32, stream);
}

extern "C" int femasr_vgg_pad_weight_ex(const float* w_oihw, float* w_padded, int Cout, int ksize, int kpad, void* stream) {
  FEMASR_CHECK_ARG(w_oihw && w_padded && Cout > 0, "vgg_pad_weight: bad argument");
  FEMASR_CHECK_ARG(ksize > 0 && kpad % 64 == 0 && kpad >= 3 * ksize * ksize, "vgg_pad_weight: kpad must hold 3 * ksize^2");
  vgg_weight_pad_kernel<<<(unsigned)cdiv((long)Cout * kpad, 256), 256, 0, as_stream(stream)>>>(w_oihw, w_padded, Cout, ksize, kpad);
  return launch_status("vgg_weight_pad_kernel");
}

extern "C" int femasr_vgg_pad_weight(const float* w_oihw, float* w_padded, int Cout, void* stream) {
  return femasr_vgg_pad_weight_ex(w_oihw, w_padded, Cout, 3, 64, stream);
}

template <int K>
static int maxpool_impl(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  FEMASR_CHECK_ARG(x && y && B > 0 && H >= K && W >= K, "maxpool: bad argument (H, W must be at least the window)");
  FEMASR_CHECK_ARG(C % 8 == 0, "maxpool: C must be a multiple of 8");
  const long total8 = (long)B * ((H - K) / 2 + 1) * ((W - K) / 2 + 1) * (C / 8);
  maxpool_kernel<K><<<(unsigned)cdiv(total8, 256), 256, 0, as_stream(stream)>>>(x, reinterpret_cast<float4*>(y), H, W, C, total8);
  return launch_status("maxpool_kernel");
}
extern "C" int femasr_maxpool2(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  return maxpool_impl<2>(x, y, B, H, W, C, stream);
}
extern "C" int femasr_maxpool3s2(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  return maxpool_impl<3>(x, y, B, H, W, C, stream);
}

extern "C" int femasr_sq_diff_rows(const float* a, const float* b, float* rows, int N, int C, void* stream) {
  FEMASR_CHECK_ARG(a && b && rows && N > 0 && C > 0, "sq_diff_rows: bad argument");
  sq_diff_rows_kernel<<<(unsigned)cdiv(N, 8), 256, 0, as_stream(stream)>>>(a, b, rows, N, C);
  return launch_status("sq_diff_rows_kernel");
}
