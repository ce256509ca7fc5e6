// Shared host/device helpers for libfemasr_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "femasr_b200.h"

namespace femasr {

void set_error(const std::string& msg);
int fail(int code, const std::string& msg);
// global launch counter (incremented by every kernel launch helper); read by the engine
extern thread_local long g_launches;

#define FEMASR_CHECK_ARG(cond, msg)                                           \
  do {                                                                        \
    if (!(cond)) return ::femasr::fail(FEMASR_ERR_ARG, std::string(msg));     \
  } while (0)

#define FEMASR_CUDA(call)                                                                       \
  do {                                                                                          \
    cudaError_t _e = (call);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      return ::femasr::fail(FEMASR_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)

inline int launch_status(const char* what) {
  cudaError_t e = cudaGetLastError();
  ++g_launches;
  if (e != cudaSuccess) return fail(FEMASR_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
  return FEMASR_OK;
}

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Per-device one-time state.  cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count belong to a DEVICE, not
// to the process: engines on several GPUs may live in one process (the reference surface is `.to(any device)`).
constexpr int MAX_DEVICES = 64;
inline int current_device() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= MAX_DEVICES) d = 0;
  return d;
}
struct PerDeviceFlag {
  bool set[MAX_DEVICES] = {};
  bool& cur() { return set[current_device()]; }
};
inline int sm_count() {
  static int counts[MAX_DEVICES] = {};
  const int d = current_device();
  if (!counts[d]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d);
    counts[d] = n > 0 ? n : 132;
  }
  return counts[d];
}

__host__ __device__ inline long cdiv(long a, long b) { return (a + b - 1) / b; }

__device__ __forceinline__ float silu_f(float v) { return v / (1.0f + expf(-v)); }
// exact-erf GELU (nn.GELU default; SURVEY 7.3-7: tanh approximation breaks parity)
__device__ __forceinline__ float gelu_erf_f(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f)); }

// Branch-free exact-erf GELU for hot epilogues: erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7); max abs error
// of the whole GELU vs fp64 on [-8,8]: 3.3e-7 (fp32 emulation of the formula below; ATen's own fp32 GELU: 1.2e-6).
// erff() has a two-branch implementation that diverges inside a warp and costs ~3x as many instructions.
// single-instruction MUFU forms (the __expf / __fdividef intrinsics add ~10 instructions of denormal handling each when
// the file is not compiled with -ftz; inputs here are never denormal-sensitive)
__device__ __forceinline__ float ex2_approx_ftz(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx_ftz(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// 15 instructions (2 MUFU):  gelu(v) = max(v,0) - |v|/2 * q,  q = 1 - erf(|v|/sqrt2) = poly(t) * t * exp(-z^2)
__device__ __forceinline__ float gelu_erf_fast_f(float v) {
  const float az = fabsf(v) * 0.70710678118654752440f;
  const float t = rcp_approx_ftz(fmaf(0.3275911f, az, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx_ftz(az * az * -1.4426950408889634f);
  const float q = p * t * e;
  return fmaf(-0.5f * fabsf(v), q, fmaxf(v, 0.0f));
}

// KxK stride-2 max-pool of 8 consecutive channels (nn.MaxPool2d(K, 2), floor; K = 2 for VGG, 3 for AlexNet): element i
// of the pooled NHWC tensor [B,(H-K)/2+1,(W-K)/2+1,C] in 8-channel units; returns the pooled tensor's element offset.
// Max in window order (row-major).
template <int K>
__device__ __forceinline__ long pool_max8(const float* __restrict__ x, long i, int H, int W, int C, float (&v)[8]) {
  const int c8 = C / 8, Ho = (H - K) / 2 + 1, Wo = (W - K) / 2 + 1;
  const int cq = (int)(i % c8);
  const long pix = i / c8;
  const int ox = (int)(pix % Wo);
  const long t = pix / Wo;
  const int oy = (int)(t % Ho);
  const long b = t / Ho;
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = -INFINITY;
#pragma unroll
  for (int dy = 0; dy < K; ++dy)
#pragma unroll
    for (int dx = 0; dx < K; ++dx) {
      const float4* s = reinterpret_cast<const float4*>(x + ((b * H + 2 * oy + dy) * W + 2 * ox + dx) * C + cq * 8);
      const float4 a = __ldg(s), c = __ldg(s + 1);
      const float w[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], w[k]);
    }
  return pix * C + cq * 8;
}

// F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) of 8 consecutive channels: element i of the
// upsampled NHWC tensor [B,2H,2W,C] in 8-channel units; returns its element offset.  Source index and weights as ATen
// computes them (src = max(0.5 * (o + 0.5) - 0.5, 0), the far neighbour clamped at the border), then
// h0 * (w0 * x00 + w1 * x01) + h1 * (w0 * x10 + w1 * x11).
__device__ __forceinline__ long bilinear2_8(const float* __restrict__ x, long i, int H, int W, int C, float (&v)[8]) {
  const int c8 = C / 8, Ho = 2 * H, Wo = 2 * W;
  const int cq = (int)(i % c8);
  const long pix = i / c8;
  const int ox = (int)(pix % Wo);
  const long t = pix / Wo;
  const int oy = (int)(t % Ho);
  const long b = t / Ho;
  const float sy = fmaxf(0.5f * (oy + 0.5f) - 0.5f, 0.f), sx = fmaxf(0.5f * (ox + 0.5f) - 0.5f, 0.f);
  const int y0 = (int)sy, x0 = (int)sx;
  const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  const float h1 = sy - y0, h0 = 1.f - h1, w1 = sx - x0, w0 = 1.f - w1;
  float a[4][8];
  const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4* s = reinterpret_cast<const float4*>(x + ((b * H + ys[q >> 1]) * W + xs[q & 1]) * C + cq * 8);
    const float4 p0 = __ldg(s), p1 = __ldg(s + 1);
    a[q][0] = p0.x; a[q][1] = p0.y; a[q][2] = p0.z; a[q][3] = p0.w;
    a[q][4] = p1.x; a[q][5] = p1.y; a[q][6] = p1.z; a[q][7] = p1.w;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = h0 * (w0 * a[0][k] + w1 * a[1][k]) + h1 * (w0 * a[2][k] + w1 * a[3][k]);
  return pix * C + cq * 8;
}

__device__ __forceinline__ float lrelu02_f(float v) { return v > 0.f ? v : v * 0.2f; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The tail of a per-image fixed-order reduction over a grid (nblk, B) of NT-thread blocks (NT a power of two).  Every
// thread of the block calls it; thread 0 passes the block's sum in `block_sum`, which is stored in
// partial[b * nblk + blk].  The block that arrives last for image b sums that image's partials (thread-strided in index
// order, then a tree over `red`, NT doubles of shared memory), resets count[b] for the next launch and returns true,
// with the total in thread 0's `total`; every other block returns false.  The result depends only on the partials, not
// on the block schedule or on the other images of the batch.
template <int NT>
__device__ __forceinline__ bool image_sum_last_block(double block_sum, double* __restrict__ partial,
                                                     unsigned int* __restrict__ count, double* red, double& total) {
  __shared__ bool last;
  const int b = blockIdx.y, nblk = gridDim.x;
  if (threadIdx.x == 0) {
    partial[(long)b * nblk + blockIdx.x] = block_sum;
    __threadfence();
    last = atomicAdd(count + b, 1u) == (unsigned)(nblk - 1);
  }
  __syncthreads();
  if (!last) return false;
  __threadfence();
  double t = 0.0;
  for (int i = threadIdx.x; i < nblk; i += NT) t += __ldcg(partial + (long)b * nblk + i);
  red[threadIdx.x] = t;
  __syncthreads();
  for (int o = NT / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    total = red[0];
    count[b] = 0u;
  }
  return true;
}

}  // namespace femasr
