// GroupNorm / LayerNorm statistics kernels (deterministic, fp32 partials reduced in double).
#include "common.cuh"

namespace femasr {

constexpr int GN_GROUPS = 32;
constexpr int GN_CHUNK = 512;   // pixels per partial block

// The sums are taken about a shift K per (image, group), the group's first channel at the image's first pixel: the fp32
// sum of squares of x itself would round away var / mean^2 of its own precision, so a2 / n - mean^2 loses (mean / std)^2
// ulps; about K it loses ((mean - K) / std)^2 instead, and K is a sample of the group.
__device__ __forceinline__ const float* gn_shift_ptr(const float* x, int b, int HW, int C, int g) {
  return x + (long)b * HW * C + g * (C / GN_GROUPS);
}

// partial[b][chunk][g][2] = (sum, sumsq) of x - K over `GN_CHUNK` pixels x (C/32) channels, fp32 per thread then
// combined in double in a fixed order.
__global__ void __launch_bounds__(256) gn_partial_kernel(const float* __restrict__ x, double* __restrict__ partial,
                                                         int HW, int C, int nchunks) {
  __shared__ float red[256][8];   // per thread: 4 sums + 4 sumsqs
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int quads = C / 4;                 // 64, 32 or 16
  const int lanes = 256 / quads;           // pixel lanes 4, 8 or 16
  const int q = threadIdx.x % quads, lane = threadIdx.x / quads;
  const int p0 = chunk * GN_CHUNK;
  const int p1 = min(p0 + GN_CHUNK, HW);
  // the quad's channels 4q..4q+3 lie in one group for cpg 4 and 8, in two (4q, 4q+2) for cpg 2
  const int cpg = C / GN_GROUPS;
  const float ka = __ldg(gn_shift_ptr(x, b, HW, C, 4 * q / cpg));
  const float kb = cpg == 2 ? __ldg(gn_shift_ptr(x, b, HW, C, 4 * q / 2 + 1)) : ka;
  float s[4] = {0.f, 0.f, 0.f, 0.f}, ss[4] = {0.f, 0.f, 0.f, 0.f};
  const float* base = x + ((long)b * HW) * C + q * 4;
  for (int p = p0 + lane; p < p1; p += lanes) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(base + (long)p * C));
    const float d0 = v.x - ka, d1 = v.y - ka, d2 = v.z - kb, d3 = v.w - kb;
    s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
    ss[0] = fmaf(d0, d0, ss[0]); ss[1] = fmaf(d1, d1, ss[1]);
    ss[2] = fmaf(d2, d2, ss[2]); ss[3] = fmaf(d3, d3, ss[3]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) { red[threadIdx.x][i] = s[i]; red[threadIdx.x][4 + i] = ss[i]; }
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {
    const int g = threadIdx.x;
    const int cpg = C / GN_GROUPS;         // 8, 4 or 2 channels per group
    double a = 0.0, a2 = 0.0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      const int qq = c >> 2, e = c & 3;
      for (int l = 0; l < lanes; ++l) {
        a += (double)red[l * quads + qq][e];
        a2 += (double)red[l * quads + qq][4 + e];
      }
    }
    double* out = partial + (((long)b * nchunks + chunk) * GN_GROUPS + g) * 2;
    out[0] = a; out[1] = a2;
  }
}

// one warp per (b, group): reduce partials, then write the folded scale/shift for its channels.
__global__ void gn_finalize_kernel(const float* __restrict__ x, const double* __restrict__ partial,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* __restrict__ scale, float* __restrict__ shift, int HW, int C, int nchunks,
                                   float eps) {
  const int b = blockIdx.x, g = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double a = 0.0, a2 = 0.0;
  for (int ch = lane; ch < nchunks; ch += 32) {
    const double* in = partial + (((long)b * nchunks + ch) * GN_GROUPS + g) * 2;
    a += in[0]; a2 += in[1];
  }
  a = warp_sum_d(a); a2 = warp_sum_d(a2);
  const int cpg = C / GN_GROUPS;
  const double n = (double)HW * cpg;
  const double dm = a / n;                                    // mean of x - K
  const double mean = (double)__ldg(gn_shift_ptr(x, b, HW, C, g)) + dm;
  double var = a2 / n - dm * dm;
  if (var < 0.0) var = 0.0;
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float meanf = (float)mean;
  if (lane < cpg) {
    const int c = g * cpg + lane;
    const float sc = rstd * gamma[c];
    scale[(long)b * C + c] = sc;
    shift[(long)b * C + c] = fmaf(-sc, meanf, beta[c]);
  }
}

// Same, from the fp32 partial rows the tensor-core conv epilogue wrote: partial[b][row][g][2].
// One CTA per image: lane = group (coalesced 256-byte row reads), 32 row slices reduced through shared memory
// in a fixed order.
__global__ void __launch_bounds__(1024) gn_finalize_rows_kernel(const float* __restrict__ partial,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, float* __restrict__ scale,
                                                                float* __restrict__ shift, int HW, int C, int rows, float eps) {
  __shared__ double red[2][32][33];
  const int b = blockIdx.x, g = threadIdx.x & 31, slice = threadIdx.x >> 5;
  double a = 0.0, a2 = 0.0;
  const float2* base = reinterpret_cast<const float2*>(partial) + (long)b * rows * GN_GROUPS + g;
  // eight row loads in flight per thread (the 512x512 maps have 8192 partial rows = 2 MB per image and only B CTAs
  // run); the adds keep the r = slice, slice + 32, ... order, so the sums are bit-identical to the one-at-a-time loop
  int r = slice;
  for (; r + 7 * 32 < rows; r += 8 * 32) {
    float2 v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldg(base + (long)(r + 32 * u) * GN_GROUPS);
#pragma unroll
    for (int u = 0; u < 8; ++u) { a += (double)v[u].x; a2 += (double)v[u].y; }
  }
  for (; r < rows; r += 32) {
    const float2 v = __ldg(base + (long)r * GN_GROUPS);
    a += (double)v.x; a2 += (double)v.y;
  }
  red[0][slice][g] = a; red[1][slice][g] = a2;
  __syncthreads();
  if (slice == 0) {
    a = 0.0; a2 = 0.0;
    for (int s = 0; s < 32; ++s) { a += red[0][s][g]; a2 += red[1][s][g]; }
    const int cpg = C / GN_GROUPS;
    const double n = (double)HW * cpg;
    const double mean = a / n;
    double var = a2 / n - mean * mean;
    if (var < 0.0) var = 0.0;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float meanf = (float)mean;
    for (int k = 0; k < cpg; ++k) {
      const int c = g * cpg + k;
      const float sc = rstd * gamma[c];
      scale[(long)b * C + c] = sc;
      shift[(long)b * C + c] = fmaf(-sc, meanf, beta[c]);
    }
  }
}

// one warp per row of 256 channels: two-pass mean / variance in registers.
__global__ void __launch_bounds__(256) ln_stats_kernel(const float* __restrict__ x, float* __restrict__ mean,
                                                       float* __restrict__ rstd, long M, float eps) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const float4* r = reinterpret_cast<const float4*>(x + row * 256);
  const float4 a = __ldg(r + lane), b = __ldg(r + 32 + lane);
  float s = ((a.x + a.y) + (a.z + a.w)) + ((b.x + b.y) + (b.z + b.w));
  s = warp_sum(s);
  const float mu = s * (1.0f / 256.0f);
  float d, v = 0.f;
  d = a.x - mu; v = fmaf(d, d, v); d = a.y - mu; v = fmaf(d, d, v);
  d = a.z - mu; v = fmaf(d, d, v); d = a.w - mu; v = fmaf(d, d, v);
  d = b.x - mu; v = fmaf(d, d, v); d = b.y - mu; v = fmaf(d, d, v);
  d = b.z - mu; v = fmaf(d, d, v); d = b.w - mu; v = fmaf(d, d, v);
  v = warp_sum(v) * (1.0f / 256.0f);
  if (lane == 0) { mean[row] = mu; rstd[row] = 1.0f / sqrtf(v + eps); }
}

}  // namespace femasr

using namespace femasr;

extern "C" size_t femasr_gn_scratch_floats(int B, int HW, int C) {
  (void)C;
  const long nchunks = cdiv(HW, GN_CHUNK);
  return (size_t)B * nchunks * GN_GROUPS * 2 * 2;   // doubles stored in a float-typed scratch
}

extern "C" int femasr_gn_stats(const float* x, const float* gamma, const float* beta, float* scale, float* shift,
                               float* scratch, int B, int HW, int C, float eps, void* stream) {
  FEMASR_CHECK_ARG(x && gamma && beta && scale && shift && scratch, "gn_stats: null pointer");
  FEMASR_CHECK_ARG(B > 0 && HW > 0, "gn_stats: empty input");
  FEMASR_CHECK_ARG(C == 64 || C == 128 || C == 256 || C == 512, "gn_stats: C must be 64/128/256/512");
  FEMASR_CHECK_ARG(((uintptr_t)scratch & 7) == 0, "gn_stats: scratch must be 8-byte aligned");
  const int nchunks = (int)cdiv(HW, GN_CHUNK);
  double* partial = reinterpret_cast<double*>(scratch);
  if (C == 512) return fail(FEMASR_ERR_ARG, "gn_stats: C=512 not used on this path");
  gn_partial_kernel<<<dim3(nchunks, B), 256, 0, as_stream(stream)>>>(x, partial, HW, C, nchunks);
  int st = launch_status("gn_partial_kernel");
  if (st) return st;
  gn_finalize_kernel<<<B, GN_GROUPS * 32, 0, as_stream(stream)>>>(x, partial, gamma, beta, scale, shift, HW, C, nchunks, eps);
  return launch_status("gn_finalize_kernel");
}

extern "C" int femasr_gn_finalize_rows(const float* partial, const float* gamma, const float* beta, float* scale,
                                       float* shift, int B, int rows, int HW, int C, float eps, void* stream) {
  FEMASR_CHECK_ARG(partial && gamma && beta && scale && shift, "gn_finalize_rows: null pointer");
  FEMASR_CHECK_ARG(B > 0 && rows > 0 && HW > 0 && (C == 64 || C == 128 || C == 256), "gn_finalize_rows: bad shape");
  gn_finalize_rows_kernel<<<B, GN_GROUPS * 32, 0, as_stream(stream)>>>(partial, gamma, beta, scale, shift, HW, C, rows, eps);
  return launch_status("gn_finalize_rows_kernel");
}

extern "C" int femasr_ln_stats(const float* x, float* mean, float* rstd, int M, int C, float eps, void* stream) {
  FEMASR_CHECK_ARG(x && mean && rstd, "ln_stats: null pointer");
  FEMASR_CHECK_ARG(C == 256, "ln_stats: C must be 256 (Swin embed dim)");
  FEMASR_CHECK_ARG(M > 0, "ln_stats: empty input");
  ln_stats_kernel<<<(unsigned)cdiv(M, 8), 256, 0, as_stream(stream)>>>(x, mean, rstd, M, eps);
  return launch_status("ln_stats_kernel");
}
