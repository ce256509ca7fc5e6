// The LPIPS head (lpips package, v0.1: normalize_tensor, the lin layers' 1x1 no-bias conv, spatial_average): for one
// tap, per pixel the channel norms of both images' features, the weighted squared difference of the unit vectors, and
// the per-image spatial mean.  The backbones run on femasr_igemm_simt / femasr_tc_igemm; this is the only new reduction.
#include "common.cuh"

namespace femasr {

constexpr int HEAD_WARPS = 8, HEAD_PIX_PER_WARP = 8, HEAD_PIX = HEAD_WARPS * HEAD_PIX_PER_WARP;   // pixels per block

// grid (ceil(HW / HEAD_PIX), B).  One warp per pixel: lane-strided fp32 FMA chains over the channels, then the fixed
// xor-tree (all lanes end with the same value).  Each block sums its pixels in fp64 in pixel order into partial[b][blk];
// the block that finishes last for image b sums those partials in a fixed order, so the result does not depend on the
// block schedule.  The arithmetic of a pixel does not depend on its position or on which image of the pair is first:
// (n0 - n1)^2 == (n1 - n0)^2 exactly.
__global__ void __launch_bounds__(256) lpips_head_kernel(const float* __restrict__ f, const float* __restrict__ w, int B,
                                                         int HW, int C, float* __restrict__ r, int k,
                                                         float* __restrict__ dist, double* __restrict__ partial,
                                                         unsigned int* __restrict__ count) {
  __shared__ double red[256];
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c2 = C / 2;
  const float2* w2 = reinterpret_cast<const float2*>(w);
  double acc = 0.0;
  for (int t = 0; t < HEAD_PIX_PER_WARP; ++t) {
    const long pix = (long)blockIdx.x * HEAD_PIX + warp * HEAD_PIX_PER_WARP + t;
    if (pix >= HW) break;
    const float2* a = reinterpret_cast<const float2*>(f + ((long)b * HW + pix) * C);
    const float2* c = reinterpret_cast<const float2*>(f + ((long)(B + b) * HW + pix) * C);
    float s0 = 0.f, s1 = 0.f;
    for (int j = lane; j < c2; j += 32) {
      const float2 u = __ldg(a + j), v = __ldg(c + j);
      s0 = fmaf(u.x, u.x, s0); s0 = fmaf(u.y, u.y, s0);
      s1 = fmaf(v.x, v.x, s1); s1 = fmaf(v.y, v.y, s1);
    }
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    const float d0 = __fadd_rn(__fsqrt_rn(s0), 1e-10f), d1 = __fadd_rn(__fsqrt_rn(s1), 1e-10f);
    float s = 0.f;
    for (int j = lane; j < c2; j += 32) {
      const float2 u = __ldg(a + j), v = __ldg(c + j), ww = __ldg(w2 + j);
      const float ex = __fsub_rn(__fdiv_rn(u.x, d0), __fdiv_rn(v.x, d1));
      const float ey = __fsub_rn(__fdiv_rn(u.y, d0), __fdiv_rn(v.y, d1));
      s = fmaf(ww.x, __fmul_rn(ex, ex), s);
      s = fmaf(ww.y, __fmul_rn(ey, ey), s);
    }
    acc += (double)warp_sum(s);
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  double blk = 0.0, total = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < HEAD_WARPS; ++i) blk += red[i];
  if (!image_sum_last_block<256>(blk, partial, count, red, total)) return;
  if (threadIdx.x == 0) {
    const float rk = (float)(total / (double)HW);
    r[(long)k * B + b] = rk;
    if (dist) {
      float d = k == 0 ? rk : __ldcg(r + b);
      for (int j = 1; j <= k; ++j) d = __fadd_rn(d, j == k ? rk : __ldcg(r + (long)j * B + b));
      dist[b] = d;
    }
  }
}

}  // namespace femasr

using namespace femasr;

// [B][nblk] fp64 partials, then B uint32 arrival counters
extern "C" size_t femasr_lpips_head_scratch_bytes(int B, int HW) {
  if (B <= 0 || HW <= 0) return 0;
  return (size_t)B * cdiv(HW, HEAD_PIX) * sizeof(double) + (size_t)B * sizeof(unsigned int);
}

extern "C" int femasr_lpips_head(const float* feat, const float* w, int B, int HW, int C, float* r, int k, float* dist,
                                 void* scratch, void* stream) {
  FEMASR_CHECK_ARG(feat && w && r && scratch && B > 0 && HW > 0, "lpips_head: bad argument");
  FEMASR_CHECK_ARG(C > 0 && C % 64 == 0, "lpips_head: C must be a positive multiple of 64");
  FEMASR_CHECK_ARG(k >= 0 && k < 5, "lpips_head: tap index k must be in [0, 5)");
  const long nblk = cdiv(HW, HEAD_PIX);
  FEMASR_CHECK_ARG(nblk < (1l << 31) && B <= 65535, "lpips_head: too many pixels or images");
  double* partial = reinterpret_cast<double*>(scratch);
  unsigned int* count = reinterpret_cast<unsigned int*>(partial + (size_t)B * nblk);
  cudaStream_t st = as_stream(stream);
  FEMASR_CUDA(cudaMemsetAsync(count, 0, (size_t)B * sizeof(unsigned int), st));
  lpips_head_kernel<<<dim3((unsigned)nblk, (unsigned)B), 256, 0, st>>>(feat, w, B, HW, C, r, k, dist, partial, count);
  return launch_status("lpips_head_kernel");
}
