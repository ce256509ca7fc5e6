// The small kernels of UNetDiscriminatorSN (discriminator_arch.py): the eval-mode spectral-norm sigma of a weight and the
// division by it, and the fp32 bilinear x2 upsample of the SIMT path.  The convs themselves run on femasr_tc_igemm /
// femasr_igemm_simt with the LeakyReLU epilogue, conv0 on femasr_vgg_im2col's rows, conv9 on femasr_out_conv3x3_n, and
// the upsample of the tensor-core path is femasr_tc_prepare's FEMASR_PRO_BILINEAR2 mode.
#include "common.cuh"

namespace femasr {

constexpr int SN_THREADS = 1024;

// One block.  t_i = sum_k W[i][k] v[k] per row (one warp per row, lane-strided fp64 sums, fixed xor tree), kept in shared
// memory; then thread 0 forms u . t and |t|^2 in row order.  The same order on every run.
__global__ void __launch_bounds__(SN_THREADS) spectral_sigma_kernel(const float* __restrict__ w, const float* __restrict__ u,
                                                                    const float* __restrict__ v, int Cout, int K,
                                                                    float* __restrict__ out) {
  extern __shared__ double t[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < Cout; r += SN_THREADS / 32) {
    const float* row = w + (long)r * K;
    double s = 0.0;
    for (int k = lane; k < K; k += 32) s = fma((double)__ldg(row + k), (double)__ldg(v + k), s);
    s = warp_sum_d(s);
    if (lane == 0) t[r] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double dot = 0.0, sq = 0.0;
    for (int r = 0; r < Cout; ++r) {
      dot = fma((double)__ldg(u + r), t[r], dot);
      sq = fma(t[r], t[r], sq);
    }
    out[0] = (float)dot;
    out[1] = (float)sqrt(sq);
  }
}

__global__ void spectral_normalize_kernel(const float* __restrict__ w, const float* __restrict__ sigma, float* __restrict__ y,
                                          long n) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __fdiv_rn(__ldg(w + i), __ldg(sigma));
}

__global__ void __launch_bounds__(256) bilinear_up2_kernel(const float* __restrict__ x, float4* __restrict__ y, int H, int W,
                                                           int C, long total8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  float v[8];
  const long o = bilinear2_8(x, i, H, W, C, v) / 4;
  y[o] = make_float4(v[0], v[1], v[2], v[3]);
  y[o + 1] = make_float4(v[4], v[5], v[6], v[7]);
}

}  // namespace femasr

using namespace femasr;

extern "C" int femasr_spectral_sigma(const float* w, const float* u, const float* v, int Cout, int K, float* out,
                                     void* stream) {
  FEMASR_CHECK_ARG(w && u && v && out && Cout > 0 && K > 0, "spectral_sigma: bad argument");
  FEMASR_CHECK_ARG(Cout <= 4096, "spectral_sigma: Cout must be <= 4096");
  spectral_sigma_kernel<<<1, SN_THREADS, (size_t)Cout * sizeof(double), as_stream(stream)>>>(w, u, v, Cout, K, out);
  return launch_status("spectral_sigma_kernel");
}

extern "C" int femasr_spectral_normalize(const float* w, const float* sigma, float* w_sn, size_t n, void* stream) {
  FEMASR_CHECK_ARG(w && sigma && w_sn && n > 0, "spectral_normalize: bad argument");
  spectral_normalize_kernel<<<(unsigned)cdiv((long)n, 256), 256, 0, as_stream(stream)>>>(w, sigma, w_sn, (long)n);
  return launch_status("spectral_normalize_kernel");
}

extern "C" int femasr_bilinear_up2(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  FEMASR_CHECK_ARG(x && y && B > 0 && H > 0 && W > 0, "bilinear_up2: bad argument");
  FEMASR_CHECK_ARG(C % 8 == 0, "bilinear_up2: C must be a multiple of 8");
  const long total8 = (long)B * 2 * H * 2 * W * (C / 8);
  bilinear_up2_kernel<<<(unsigned)cdiv(total8, 256), 256, 0, as_stream(stream)>>>(x, reinterpret_cast<float4*>(y), H, W, C,
                                                                                 total8);
  return launch_status("bilinear_up2_kernel");
}
