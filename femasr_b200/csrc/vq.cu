// VectorQuantizer feature matching (femasr_arch.py:50-100): fp32-exact distance formula + argmin +
// codebook gather + straight-through residual.  The z.e^T products come from the GEMM path; this file
// reproduces the reference's rounding sequence d_j = fl(fl(A + B_j) - 2 C_j) and its tie rule
// (lowest index wins), which is what makes the indices bit-exact (SURVEY 7.3-2).
#include "common.cuh"

namespace femasr {

// out[r] = sum_k x[r][k]^2   (torch.sum(y**2, dim=1), femasr_arch.py:37)
__global__ void row_sumsq_kernel(const float* __restrict__ x, float* __restrict__ out, int rows, int cols) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int k = lane; k < cols; k += 32) { const float v = x[(long)r * cols + k]; s = fmaf(v, v, s); }
  s = warp_sum(s);
  if (lane == 0) out[r] = s;
}

// one warp per feature row
__global__ void __launch_bounds__(256) vq_select_kernel(const float* __restrict__ z, const float* __restrict__ zc,
                                                        const float* __restrict__ codebook,
                                                        const float* __restrict__ esq, int64_t* __restrict__ idx,
                                                        float* __restrict__ zq, float* __restrict__ loss_rows,
                                                        int N, int n_e, int e_dim) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= N) return;
  const int lane = threadIdx.x & 31;
  const float* zr = z + (long)r * e_dim;
  float a = 0.f;
  for (int k = lane; k < e_dim; k += 32) { const float v = zr[k]; a = fmaf(v, v, a); }
  a = warp_sum(a);                                     // A = sum z^2 (all lanes hold the same value)
  const float* cr = zc + (long)r * n_e;
  float best = INFINITY;
  int bj = 0x7fffffff;
  for (int j = lane; j < n_e; j += 32) {
    const float ab = __fadd_rn(a, __ldg(esq + j));     // fl(A + B_j)
    const float d = __fsub_rn(ab, __fmul_rn(2.0f, cr[j]));   // fl(. - 2 C_j); 2*C_j is exact
    if (d < best) { best = d; bj = j; }                // strict <: the lowest j of this lane wins
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float od = __shfl_xor_sync(0xffffffffu, best, o);
    const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
    if (od < best || (od == best && oj < bj)) { best = od; bj = oj; }
  }
  if (bj == 0x7fffffff) bj = 0;                        // all-NaN row: torch.argmin would also return a valid index
  if (lane == 0 && idx) idx[r] = (int64_t)bj;
  const float* er = codebook + (long)bj * e_dim;
  float l = 0.f;
  for (int k = lane; k < e_dim; k += 32) {
    const float zv = zr[k];
    const float diff = __fsub_rn(__ldg(er + k), zv);   // (z_q - z)
    l = fmaf(diff, diff, l);
    if (zq) zq[(long)r * e_dim + k] = __fadd_rn(zv, diff);   // z + (z_q - z).detach(), femasr_arch.py:95
  }
  l = warp_sum(l);
  if (lane == 0 && loss_rows) loss_rows[r] = l;
}

// Second half of the fused VQ (after femasr_vq_match_tc): one warp per feature row.
//   cand[r][0..3]  the four smallest tensor-core distances with their codes, ascending in (d, j)
// A row whose runner-up is more than VQ_MARGIN_ULPS ulps behind the best keeps the best code.  Otherwise every
// candidate inside the margin gets its distance recomputed with an exact dot product (fp64 accumulate, rounded once:
// what "any fp32-accurate z.e" of SURVEY 7.3-2 asks for) through the reference's rounding sequence
// fl(fl(A + B_j) - 2 C_j) and the lowest-index tie rule; if even the fourth candidate is inside the margin the whole
// codebook is rescanned exactly.
// Then: gather, straight-through residual z + (e - z), per-row loss (femasr_arch.py:67-100).
// Margin.  With u = the grid step of the fp32 distance formula (ulp of max(A + B, d): the subtraction may cancel),
// tensor-core and exact distance of code j differ by at most u + |2 dC_j|, so the true argmin (and every exact tie with
// a lower index) lies within 2u + |2 dC_best| + |2 dC_argmin| of the tensor-core best.  The margin is 2.5 u plus two
// bounds of the tensor-core error of 2C:
//   * relative: four times 3 * e_dim / 16 truncating accumulations of <= 1 ulp each of 2C;
//   * absolute: z is split into fp16 hi / lo planes without a scale, so below |z| ~ 2^-3 the lo plane is subnormal and
//     each z_k carries up to 2^-25 of absolute error whatever its size.  By Cauchy-Schwarz that moves 2 C_j by at most
//     2^-24 * sqrt(e_dim * B_j); twice that (the best code and the true argmin), taken at the largest B_j of the four
//     candidates.  A code outside the list escapes this only if its norm exceeds all four candidates' and its exact
//     distance beats them all.
// The grid step u shrinks as |z|^2 while the absolute term does not: for z of std 2^-12 the absolute term is ~2000 u,
// for z of std ~1 it is ~1e-3 u.
constexpr float VQ_MARGIN_ULPS = 2.5f;
__device__ __forceinline__ float ulp_of(float x) {      // spacing of fp32 numbers at |x| (normal range)
  return __uint_as_float(__float_as_uint(x) & 0x7f800000u) * 1.1920929e-7f;
}
__device__ __forceinline__ float vq_exact_distance(const float* __restrict__ zr, const float* __restrict__ er, float a,
                                                    float b, int e_dim, int lane) {
  double s = 0.0;
  for (int k = lane; k < e_dim; k += 32) s = fma((double)zr[k], (double)__ldg(er + k), s);
  s = warp_sum_d(s);
  const float c = (float)s;
  return __fsub_rn(__fadd_rn(a, b), __fmul_rn(2.0f, c));
}

__global__ void __launch_bounds__(256) vq_finish_kernel(const float* __restrict__ z, const float* __restrict__ a,
                                                        const uint2* __restrict__ cand, const float* __restrict__ codebook,
                                                        const float* __restrict__ esq, int64_t* __restrict__ idx,
                                                        float* __restrict__ zq, float* __restrict__ loss_rows,
                                                        unsigned int* __restrict__ stats, int N, int n_e, int e_dim) {
  __shared__ __align__(16) float zs[8][1024];           // z rows of the (rare) whole-codebook rescans; e_dim <= 1024
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= N) return;
  const int lane = threadIdx.x & 31;
  const float* zr = z + (long)r * e_dim;
  const uint2 cv = cand[(long)r * 4 + (lane & 3)];
  float d[4]; int j[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    d[k] = __uint_as_float(__shfl_sync(0xffffffffu, cv.x, k));
    j[k] = (int)__shfl_sync(0xffffffffu, cv.y, k);
  }
  int bj = j[0];
  if (bj == 0x7fffffff) {
    bj = 0;                                            // all-NaN row: torch.argmin also returns a valid index
  } else {
    const float ar0 = a[r];
    const float ab0 = ar0 + __ldg(esq + bj);
    float bmax = __ldg(esq + bj);
#pragma unroll
    for (int k = 1; k < 4; ++k) if (j[k] != 0x7fffffff) bmax = fmaxf(bmax, __ldg(esq + j[k]));
    const float margin = VQ_MARGIN_ULPS * ulp_of(fmaxf(fabsf(ab0), fabsf(d[0]))) +
                         4.0f * 1.1920929e-7f * (float)(3 * e_dim / 16) * fabsf(ab0 - d[0]) +
                         0x1p-23f * sqrtf((float)e_dim * bmax) + 1e-30f;
    int nc = 1;
#pragma unroll
    for (int k = 1; k < 4; ++k) nc += (j[k] != 0x7fffffff && d[k] - d[0] <= margin) ? 1 : 0;   // ascending: a prefix
    if (nc > 1) {
      const float ar = ar0;
      float best = INFINITY;
      int bb = 0x7fffffff;
      if (nc == 4) {
        // candidate list overflowed: exact scan of the whole codebook.  The z row goes to shared memory and every lane
        // walks its own codes (lane, lane + 32, ...: increasing, so '<' keeps the lowest index) with four independent
        // fp64 chains - no shuffles on the critical path; then a lexicographic (d, code) warp reduction.
        float* zw = zs[threadIdx.x >> 5];
        for (int k = lane; k < e_dim; k += 32) zw[k] = zr[k];
        __syncwarp();
        for (int c = lane; c < n_e; c += 32) {
          const float4* er4 = reinterpret_cast<const float4*>(codebook + (long)c * e_dim);
          double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
          for (int k4 = 0; k4 < e_dim / 4; k4 += 8) {          // e_dim % 32 == 0 (multiple of 64): 8 row loads in flight
            float4 ev[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) ev[u] = __ldg(er4 + k4 + u);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const float4 zv = *reinterpret_cast<const float4*>(zw + 4 * (k4 + u));
              s0 = fma((double)zv.x, (double)ev[u].x, s0); s1 = fma((double)zv.y, (double)ev[u].y, s1);
              s2 = fma((double)zv.z, (double)ev[u].z, s2); s3 = fma((double)zv.w, (double)ev[u].w, s3);
            }
          }
          const float cc = (float)((s0 + s1) + (s2 + s3));
          const float dd = __fsub_rn(__fadd_rn(ar, __ldg(esq + c)), __fmul_rn(2.0f, cc));
          if (dd < best) { best = dd; bb = c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float od = __shfl_xor_sync(0xffffffffu, best, o);
          const int oj = __shfl_xor_sync(0xffffffffu, bb, o);
          if (od < best || (od == best && oj < bb)) { best = od; bb = oj; }
        }
      } else {
        for (int k = 0; k < nc; ++k) {
          const float dd = vq_exact_distance(zr, codebook + (long)j[k] * e_dim, ar, __ldg(esq + j[k]), e_dim, lane);
          if (dd < best || (dd == best && j[k] < bb)) { best = dd; bb = j[k]; }
        }
      }
      if (bb != 0x7fffffff) bj = bb;
      if (stats && lane == 0) { atomicAdd(stats, 1u); if (nc == 4) atomicAdd(stats + 1, 1u); if (bb != j[0]) atomicAdd(stats + 2, 1u); }
    }
  }
  if (lane == 0 && idx) idx[r] = (int64_t)bj;
  const float* er = codebook + (long)bj * e_dim;
  float l = 0.f;
  for (int k = lane; k < e_dim; k += 32) {
    const float zv = zr[k];
    const float diff = __fsub_rn(__ldg(er + k), zv);   // (z_q - z)
    l = fmaf(diff, diff, l);
    if (zq) zq[(long)r * e_dim + k] = __fadd_rn(zv, diff);   // z + (z_q - z).detach(), femasr_arch.py:95
  }
  l = warp_sum(l);
  if (lane == 0 && loss_rows) loss_rows[r] = l;
}

// Compact wire format of index maps (femasr_b200/wire.py): `bits` = ceil(log2 n_e) bits per code, little-endian bit
// stream (code i occupies bits [i*bits, (i+1)*bits), least significant bit first).  Eight codes are exactly `bits`
// bytes, so one thread packs / unpacks one group of eight through a 128-bit shift register.  bits <= 16.
__global__ void __launch_bounds__(256) pack_codes_kernel(const int64_t* __restrict__ idx, uint8_t* __restrict__ out,
                                                         long n, int bits, int n_e, int* __restrict__ bad) {
  const long g = (long)blockIdx.x * 256 + threadIdx.x;
  if (g * 8 >= n) return;
  unsigned long long lo = 0ull, hi = 0ull;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long i = g * 8 + k;
    long v = i < n ? idx[i] : 0;
    if (v < 0 || v >= n_e) { atomicExch(bad, 1); v = 0; }
    const int sh = k * bits;
    const unsigned long long u = (unsigned long long)v;
    if (sh < 64) { lo |= u << sh; if (sh + bits > 64) hi |= u >> (64 - sh); }
    else hi |= u << (sh - 64);
  }
  const long total = (n * bits + 7) / 8;
  for (int b = 0; b < bits; ++b) {
    const long o = g * bits + b;
    if (o < total) out[o] = (uint8_t)(b < 8 ? (lo >> (8 * b)) : (hi >> (8 * (b - 8))));
  }
}

__global__ void __launch_bounds__(256) unpack_codes_kernel(const uint8_t* __restrict__ in, int64_t* __restrict__ idx, long n,
                                                           int bits) {
  const long g = (long)blockIdx.x * 256 + threadIdx.x;
  if (g * 8 >= n) return;
  const long total = (n * bits + 7) / 8;
  unsigned long long lo = 0ull, hi = 0ull;
  for (int b = 0; b < bits; ++b) {
    const long o = g * bits + b;
    const unsigned long long v = o < total ? in[o] : 0;
    if (b < 8) lo |= v << (8 * b); else hi |= v << (8 * (b - 8));
  }
  const unsigned long long mask = (1ull << bits) - 1ull;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long i = g * 8 + k;
    if (i >= n) break;
    const int sh = k * bits;
    unsigned long long u;
    if (sh < 64) { u = lo >> sh; if (sh + bits > 64) u |= hi << (64 - sh); }
    else u = hi >> (sh - 64);
    idx[i] = (int64_t)(u & mask);
  }
}

template <bool ACC>
__global__ void __launch_bounds__(1024) sum_scaled_kernel(const float* __restrict__ x, float* __restrict__ out, size_t n,
                                                          double scale) {
  __shared__ double red[32];
  double s = 0.0;
  for (size_t i = threadIdx.x; i < n; i += 1024) s += (double)x[i];
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = warp_sum_d(red[threadIdx.x]);
    if (threadIdx.x == 0) out[0] = ACC ? (float)((double)out[0] + s * scale) : (float)(s * scale);
  }
}

// out[B,H,W,Ca+Cb] = cat(a[B,H,W,Ca], nearest(b[B,Hb,Wb,Cb] -> H x W))  -- torch.cat along channels with
// F.interpolate's default nearest mode (src = floor(dst * in / out)); femasr_arch.py:332-335, fema_utils.py:93-96.
__global__ void __launch_bounds__(256) concat_channels_kernel(const float4* __restrict__ a, const float4* __restrict__ b,
                                                              float4* __restrict__ out, int H, int W, int Hb, int Wb,
                                                              int ca4, int cb4, long total4) {
  const long i = (long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total4) return;
  const int c4 = ca4 + cb4;
  const int c = (int)(i % c4);
  const long pix = i / c4;
  if (c < ca4) { out[i] = __ldg(a + pix * ca4 + c); return; }
  const int x = (int)(pix % W);
  const long t = pix / W;
  const int y = (int)(t % H);
  const long bi = t / H;
  const int ys = min((int)(((long)y * Hb) / H), Hb - 1), xs = min((int)(((long)x * Wb) / W), Wb - 1);
  out[i] = __ldg(b + ((bi * Hb + ys) * Wb + xs) * cb4 + (c - ca4));
}

// gt_indices branch of the VQ loss (femasr_arch.py:70-78, 87-88): zq_gt[r] = codebook[gt[r]],
// rows[r] = sum_k (zq_gt[r][k] - z[r][k])^2.  One warp per row.
__global__ void __launch_bounds__(256) vq_gt_rows_kernel(const float* __restrict__ z, const float* __restrict__ codebook,
                                                         const int64_t* __restrict__ gt, float* __restrict__ zq_gt,
                                                         float* __restrict__ rows, int N, int n_e, int e_dim) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= N) return;
  const int lane = threadIdx.x & 31;
  long j = gt[r];
  j = j < 0 ? 0 : (j >= n_e ? n_e - 1 : j);
  float l = 0.f;
  for (int k = lane; k < e_dim; k += 32) {
    const float e = __ldg(codebook + j * e_dim + k);
    const float d = __fsub_rn(e, z[(long)r * e_dim + k]);
    l = fmaf(d, d, l);
    zq_gt[(long)r * e_dim + k] = e;
  }
  l = warp_sum(l);
  if (lane == 0) rows[r] = l;
}

// Gram-matrix texture loss (femasr_arch.py:40-48): per image G(x) = x^T x / HW over x [HW, C];
// partial[b][tile] = sum over the 32x32 tile of (G(x) - G(y))^2.  256 threads, 2x2 outputs each, fp32 FMA.
__global__ void __launch_bounds__(256) gram_diff_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                        float* __restrict__ partial, int HW, int C) {
  __shared__ float xi[32][33], xj[32][33], yi[32][33], yj[32][33];
  __shared__ float red[8];
  const int tiles = C / 32;
  const int b = blockIdx.y, ti = blockIdx.x / tiles, tj = blockIdx.x % tiles;
  const float* xb = x + (long)b * HW * C;
  const float* yb = y + (long)b * HW * C;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float ax[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, ay[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int k0 = 0; k0 < HW; k0 += 32) {
    for (int e = threadIdx.x; e < 1024; e += 256) {
      const int kk = e >> 5, cc = e & 31;
      const bool in = k0 + kk < HW;
      const long row = (long)(k0 + kk) * C;
      xi[kk][cc] = in ? xb[row + ti * 32 + cc] : 0.f;
      xj[kk][cc] = in ? xb[row + tj * 32 + cc] : 0.f;
      yi[kk][cc] = in ? yb[row + ti * 32 + cc] : 0.f;
      yj[kk][cc] = in ? yb[row + tj * 32 + cc] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < 32; ++kk) {
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          ax[u][v] = fmaf(xi[kk][ty * 2 + u], xj[kk][tx * 2 + v], ax[u][v]);
          ay[u][v] = fmaf(yi[kk][ty * 2 + u], yj[kk][tx * 2 + v], ay[u][v]);
        }
    }
    __syncthreads();
  }
  const float inv = 1.0f / (float)HW;
  float s = 0.f;
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int v = 0; v < 2; ++v) { const float d = ax[u][v] * inv - ay[u][v] * inv; s = fmaf(d, d, s); }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tsum = 0.f;
    for (int w = 0; w < 8; ++w) tsum += red[w];
    partial[(long)b * gridDim.x + blockIdx.x] = tsum;
  }
}

__global__ void codebook_gather_kernel(const int64_t* __restrict__ idx, const float* __restrict__ codebook,
                                       float* __restrict__ zq, int N, int n_e, int e_dim) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= N) return;
  long j = idx[r];
  j = j < 0 ? 0 : (j >= n_e ? n_e - 1 : j);
  for (int k = threadIdx.x & 31; k < e_dim; k += 32) zq[(long)r * e_dim + k] = __ldg(codebook + j * e_dim + k);
}

}  // namespace femasr

using namespace femasr;

extern "C" int femasr_row_sumsq(const float* x, float* out, int rows, int cols, void* stream) {
  FEMASR_CHECK_ARG(x && out && rows > 0 && cols > 0, "row_sumsq: bad argument");
  row_sumsq_kernel<<<(rows + 7) / 8, 256, 0, as_stream(stream)>>>(x, out, rows, cols);
  return launch_status("row_sumsq_kernel");
}

extern "C" int femasr_vq_select(const float* z, const float* zc, const float* codebook, const float* esq,
                                int64_t* idx, float* zq, float* loss_rows, int N, int n_e, int e_dim,
                                int write_zq_passthrough, void* stream) {
  (void)write_zq_passthrough;
  FEMASR_CHECK_ARG(z && zc && codebook && esq, "vq_select: null pointer");
  FEMASR_CHECK_ARG(N > 0 && n_e > 0 && e_dim > 0, "vq_select: empty input");
  vq_select_kernel<<<(N + 7) / 8, 256, 0, as_stream(stream)>>>(z, zc, codebook, esq, idx, zq, loss_rows, N, n_e, e_dim);
  return launch_status("vq_select_kernel");
}

extern "C" int femasr_vq_finish(const float* z, const float* a, const void* cand, const float* codebook, const float* esq,
                                int64_t* idx, float* zq, float* loss_rows, unsigned int* stats, int N, int n_e, int e_dim,
                                void* stream) {
  FEMASR_CHECK_ARG(z && a && cand && codebook && esq, "vq_finish: null pointer");
  FEMASR_CHECK_ARG(N > 0 && n_e > 0 && e_dim > 0 && e_dim <= 1024 && e_dim % 32 == 0, "vq_finish: e_dim must be a multiple of 32, at most 1024");
  vq_finish_kernel<<<(unsigned)cdiv(N, 8), 256, 0, as_stream(stream)>>>(z, a, reinterpret_cast<const uint2*>(cand), codebook, esq,
                                                                        idx, zq, loss_rows, stats, N, n_e, e_dim);
  return launch_status("vq_finish_kernel");
}

static int code_bits_of(int n_e) { int b = 0; while ((1l << b) < n_e) ++b; return b < 1 ? 1 : b; }

extern "C" size_t femasr_packed_code_bytes(size_t numel, int n_e) {
  return n_e < 2 ? 0 : (numel * (size_t)code_bits_of(n_e) + 7) / 8;
}

// status: device int set to 1 when a code lies outside [0, n_e) (the caller checks it; such codes are packed as 0)
extern "C" int femasr_pack_codes(const int64_t* indices, void* packed, size_t numel, int n_e, int* status, void* stream) {
  FEMASR_CHECK_ARG(indices && packed && status && numel > 0, "pack_codes: bad argument");
  FEMASR_CHECK_ARG(n_e >= 2 && n_e <= 65536, "pack_codes: n_e must be in [2, 65536]");
  cudaStream_t st = as_stream(stream);
  FEMASR_CUDA(cudaMemsetAsync(status, 0, sizeof(int), st));
  const long groups = (long)cdiv((long)numel, 8);
  pack_codes_kernel<<<(unsigned)cdiv(groups, 256), 256, 0, st>>>(indices, reinterpret_cast<uint8_t*>(packed), (long)numel,
                                                                code_bits_of(n_e), n_e, status);
  return launch_status("pack_codes_kernel");
}

extern "C" int femasr_unpack_codes(const void* packed, int64_t* indices, size_t numel, int n_e, void* stream) {
  FEMASR_CHECK_ARG(indices && packed && numel > 0, "unpack_codes: bad argument");
  FEMASR_CHECK_ARG(n_e >= 2 && n_e <= 65536, "unpack_codes: n_e must be in [2, 65536]");
  const long groups = (long)cdiv((long)numel, 8);
  unpack_codes_kernel<<<(unsigned)cdiv(groups, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const uint8_t*>(packed),
                                                                                   indices, (long)numel, code_bits_of(n_e));
  return launch_status("unpack_codes_kernel");
}

extern "C" int femasr_sum_scaled(const float* x, float* out, size_t n, double scale, void* stream) {
  FEMASR_CHECK_ARG(x && out && n > 0, "sum_scaled: bad argument");
  sum_scaled_kernel<false><<<1, 1024, 0, as_stream(stream)>>>(x, out, n, scale);
  return launch_status("sum_scaled_kernel");
}

extern "C" int femasr_sum_scaled_add(const float* x, float* out, size_t n, double scale, void* stream) {
  FEMASR_CHECK_ARG(x && out && n > 0, "sum_scaled_add: bad argument");
  sum_scaled_kernel<true><<<1, 1024, 0, as_stream(stream)>>>(x, out, n, scale);
  return launch_status("sum_scaled_kernel");
}

extern "C" int femasr_concat_channels(const float* a, int Ca, const float* b, int Hb, int Wb, int Cb, float* out, int B,
                                      int H, int W, void* stream) {
  FEMASR_CHECK_ARG(a && b && out && B > 0 && H > 0 && W > 0 && Hb > 0 && Wb > 0, "concat_channels: bad argument");
  FEMASR_CHECK_ARG(Ca > 0 && Cb > 0 && Ca % 4 == 0 && Cb % 4 == 0, "concat_channels: channel counts must be multiples of 4");
  const long total4 = (long)B * H * W * ((Ca + Cb) / 4);
  concat_channels_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(b), reinterpret_cast<float4*>(out), H, W, Hb, Wb,
      Ca / 4, Cb / 4, total4);
  return launch_status("concat_channels_kernel");
}

extern "C" int femasr_vq_gt_rows(const float* z, const float* codebook, const int64_t* gt, float* zq_gt, float* rows,
                                 int N, int n_e, int e_dim, void* stream) {
  FEMASR_CHECK_ARG(z && codebook && gt && zq_gt && rows && N > 0 && n_e > 0 && e_dim > 0, "vq_gt_rows: bad argument");
  vq_gt_rows_kernel<<<(N + 7) / 8, 256, 0, as_stream(stream)>>>(z, codebook, gt, zq_gt, rows, N, n_e, e_dim);
  return launch_status("vq_gt_rows_kernel");
}

extern "C" int femasr_gram_diff_tiles(int C) { return C > 0 && C % 32 == 0 ? (C / 32) * (C / 32) : 0; }

extern "C" int femasr_gram_diff(const float* x, const float* y, float* partial, int B, int HW, int C, void* stream) {
  FEMASR_CHECK_ARG(x && y && partial && B > 0 && HW > 0, "gram_diff: bad argument");
  FEMASR_CHECK_ARG(C > 0 && C % 32 == 0 && B <= 65535, "gram_diff: C must be a multiple of 32");
  const dim3 grid((unsigned)femasr_gram_diff_tiles(C), (unsigned)B);
  gram_diff_kernel<<<grid, 256, 0, as_stream(stream)>>>(x, y, partial, HW, C);
  return launch_status("gram_diff_kernel");
}

extern "C" int femasr_codebook_gather(const int64_t* idx, const float* codebook, float* zq, int N, int n_e, int e_dim,
                                      void* stream) {
  FEMASR_CHECK_ARG(idx && codebook && zq && N > 0, "codebook_gather: bad argument");
  codebook_gather_kernel<<<(N + 7) / 8, 256, 0, as_stream(stream)>>>(idx, codebook, zq, N, n_e, e_dim);
  return launch_status("codebook_gather_kernel");
}
