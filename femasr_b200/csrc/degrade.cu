// BSRGAN's degradation steps (degradation_bsrgan, basicsr/data/bsrgan_util.py of the reference) on HWC fp32 RGB images:
// mirror convolution, separable resizes from host tap tables, noise add and the JPEG round trip of add_JPEG_noise.
// include/femasr_b200.h states each entry point's semantics; femasr_b200/degrade.py builds the tables and the draws.
#include <cmath>

#include "common.cuh"

namespace femasr {

constexpr int DG_THREADS = 256;
constexpr int CONV_T = 16;          // output tile side of the mirror convolution (16x16 threads)

// ndimage's 'mirror' boundary: reflect about the edge samples (period 2n - 2), any offset.
__device__ __forceinline__ int mirror_idx(int i, int n) {
  if (n == 1) return 0;
  const int p = 2 * n - 2;
  i %= p;
  if (i < 0) i += p;
  return i >= n ? p - i : i;
}

struct ConvTaps {
  double k[FEMASR_DEGRADE_MAX_KSIZE * FEMASR_DEGRADE_MAX_KSIZE];   // flipped (correlation order), row-major
};

// grid (ceil(Wo/16), ceil(Ho/16)), 16x16 threads.  The input footprint of the output tile ((15 s + kh) x (15 s + kw)
// pixels, mirror-folded) is staged in shared memory; each thread sums its taps row-major in fp64 (products and sums
// rounded separately, the order of the fp64 oracle) and rounds to fp32 once.
__global__ void __launch_bounds__(CONV_T * CONV_T) mirror_conv_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                      int H, int W, int kh, int kw, int stride,
                                                                      int clip, ConvTaps t) {
  extern __shared__ float tile[];
  const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
  const int EH = (CONV_T - 1) * stride + kh, EW = (CONV_T - 1) * stride + kw;
  const int oy0 = blockIdx.y * CONV_T, ox0 = blockIdx.x * CONV_T;
  const int iy0 = oy0 * stride - kh / 2, ix0 = ox0 * stride - kw / 2;
  const int tid = threadIdx.y * CONV_T + threadIdx.x;
  for (int i = tid; i < EH * EW; i += CONV_T * CONV_T) {
    const int r = i / EW, q = i % EW;
    const float* s = x + ((long)mirror_idx(iy0 + r, H) * W + mirror_idx(ix0 + q, W)) * 3;
    tile[i * 3 + 0] = __ldg(s);
    tile[i * 3 + 1] = __ldg(s + 1);
    tile[i * 3 + 2] = __ldg(s + 2);
  }
  __syncthreads();
  const int oy = oy0 + threadIdx.y, ox = ox0 + threadIdx.x;
  if (oy >= Ho || ox >= Wo) return;
  double a0 = 0.0, a1 = 0.0, a2 = 0.0;
  for (int i = 0; i < kh; ++i) {
    const float* row = tile + ((threadIdx.y * stride + i) * EW + threadIdx.x * stride) * 3;
    for (int j = 0; j < kw; ++j) {
      const double w = t.k[i * kw + j];
      a0 = __dadd_rn(a0, __dmul_rn(w, (double)row[j * 3 + 0]));
      a1 = __dadd_rn(a1, __dmul_rn(w, (double)row[j * 3 + 1]));
      a2 = __dadd_rn(a2, __dmul_rn(w, (double)row[j * 3 + 2]));
    }
  }
  float v[3] = {(float)a0, (float)a1, (float)a2};
  float* d = y + ((long)oy * Wo + ox) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) d[c] = clip ? fminf(fmaxf(v[c], 0.f), 1.f) : v[c];
}

// One separable resize pass along rows (axis 0) or columns (axis 1) of an [H, W, 3] image: out[o] = sum_k w[o][k]
// * in[idx[o][k]], accumulated in fp32 in tap order from the first product, without contraction.  One thread per
// output value.
__global__ void __launch_bounds__(DG_THREADS) resize_pass_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                 int H, int W, int axis, int out_n,
                                                                 const int* __restrict__ idx,
                                                                 const float* __restrict__ wt, int K, int clip) {
  const int Ho = axis == 0 ? out_n : H, Wo = axis == 0 ? W : out_n;
  const long n = (long)Ho * Wo * 3;
  const long i = (long)blockIdx.x * DG_THREADS + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % 3);
  const long p = i / 3;
  const int ox = (int)(p % Wo), oy = (int)(p / Wo);
  const int o = axis == 0 ? oy : ox;
  const int* ix = idx + (long)o * K;
  const float* w = wt + (long)o * K;
  const long step = axis == 0 ? (long)W * 3 : 3;
  const float* base = axis == 0 ? x + (long)ox * 3 + c : x + (long)oy * W * 3 + c;
  float acc = __fmul_rn(__ldg(base + __ldg(ix) * step), __ldg(w));
  for (int k = 1; k < K; ++k) acc = __fadd_rn(acc, __fmul_rn(__ldg(base + __ldg(ix + k) * step), __ldg(w + k)));
  y[i] = clip ? fminf(fmaxf(acc, 0.f), 1.f) : acc;
}

// out = clip(x + noise, 0, 1) in fp32; the noise field has 3 channels or 1 (broadcast over the three).
__global__ void __launch_bounds__(DG_THREADS) noise_add_clip_kernel(const float* __restrict__ x,
                                                                    const float* __restrict__ noise, int noise_ch,
                                                                    long n, float* __restrict__ y) {
  const long i = (long)blockIdx.x * DG_THREADS + threadIdx.x;
  if (i >= n) return;
  const float v = __fadd_rn(__ldg(x + i), __ldg(noise + (noise_ch == 3 ? i : i / 3)));
  y[i] = fminf(fmaxf(v, 0.f), 1.f);
}

// ------------------------------------------------------------------------------------------------------------- JPEG
// Baseline JPEG at 4:2:0 as libjpeg-turbo computes it (integer arithmetic throughout, so the result is exact):
// single2uint, RGB -> YCbCr (16-bit fixed point), luma edge-replicated to whole blocks, chroma edge-replicated to whole
// 16-column MCUs and an even height, 2x2-averaged with biases 1, 2, 1, 2, ... and replicated down to whole blocks;
// islow FDCT, quantisation by reciprocal, dequantisation, islow IDCT, range limit; then h2v2 fancy upsampling and
// YCbCr -> RGB, and k / 255 rounded to fp32.  The entropy coder is lossless, so it is left out.
struct JpegTables {
  int q[2][64];        // quantisation tables (natural order): luma, chroma
  int recip[2][64], corr[2][64], shift[2][64];
};

constexpr int F_0_298631336 = 2446, F_0_390180644 = 3196, F_0_541196100 = 4433, F_0_765366865 = 6270,
              F_0_899976223 = 7373, F_1_175875602 = 9633, F_1_501321110 = 12299, F_1_847759065 = 15137,
              F_1_961570560 = 16069, F_2_053119869 = 16819, F_2_562915447 = 20995, F_3_072711026 = 25172;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

__device__ __forceinline__ unsigned char single2uint(float v) {
  return (unsigned char)rintf(__fmul_rn(fminf(fmaxf(v, 0.f), 1.f), 255.f));
}

__device__ __forceinline__ void rgb_ycc(const float* p, int& y, int& cb, int& cr) {
  const int r = single2uint(p[0]), g = single2uint(p[1]), b = single2uint(p[2]);
  y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// One 8-point islow FDCT pass over d[0], d[s], ..., d[7 s]; pass 2 descales by PASS1_BITS + CONST_BITS.
__device__ __forceinline__ void fdct8(int* d, int s, bool pass2) {
  const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
  const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  const int sh = pass2 ? 15 : 11;
  d[0] = pass2 ? descale(t10 + t11, 2) : (t10 + t11) * 4;
  d[4 * s] = pass2 ? descale(t10 - t11, 2) : (t10 - t11) * 4;
  int z1 = (t12 + t13) * F_0_541196100;
  d[2 * s] = descale(z1 + t13 * F_0_765366865, sh);
  d[6 * s] = descale(z1 - t12 * F_1_847759065, sh);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * F_1_175875602;
  const int a4 = t4 * F_0_298631336, a5 = t5 * F_2_053119869, a6 = t6 * F_3_072711026, a7 = t7 * F_1_501321110;
  z1 = -z1 * F_0_899976223;
  z2 = -z2 * F_2_562915447;
  z3 = -z3 * F_1_961570560 + z5;
  z4 = -z4 * F_0_390180644 + z5;
  d[7 * s] = descale(a4 + z1 + z3, sh);
  d[5 * s] = descale(a5 + z2 + z4, sh);
  d[3 * s] = descale(a6 + z2 + z3, sh);
  d[s] = descale(a7 + z1 + z4, sh);
}

// One 8-point islow IDCT pass; pass 1 descales by CONST_BITS - PASS1_BITS, pass 2 by CONST_BITS + PASS1_BITS + 3.
__device__ __forceinline__ void idct8(int* d, int s, bool pass2) {
  int z1 = (d[2 * s] + d[6 * s]) * F_0_541196100;
  const int t2e = z1 - d[6 * s] * F_1_847759065, t3e = z1 + d[2 * s] * F_0_765366865;
  const int t0e = (d[0] + d[4 * s]) * 8192, t1e = (d[0] - d[4 * s]) * 8192;
  const int t10 = t0e + t3e, t13 = t0e - t3e, t11 = t1e + t2e, t12 = t1e - t2e;
  int t0 = d[7 * s], t1 = d[5 * s], t2 = d[3 * s], t3 = d[s];
  z1 = t0 + t3;
  int z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
  const int z5 = (z3 + z4) * F_1_175875602;
  t0 *= F_0_298631336; t1 *= F_2_053119869; t2 *= F_3_072711026; t3 *= F_1_501321110;
  z1 = -z1 * F_0_899976223;
  z2 = -z2 * F_2_562915447;
  z3 = -z3 * F_1_961570560 + z5;
  z4 = -z4 * F_0_390180644 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  const int sh = pass2 ? 18 : 11;
  d[0] = descale(t10 + t3, sh); d[7 * s] = descale(t10 - t3, sh);
  d[s] = descale(t11 + t2, sh); d[6 * s] = descale(t11 - t2, sh);
  d[2 * s] = descale(t12 + t1, sh); d[5 * s] = descale(t12 - t1, sh);
  d[3 * s] = descale(t13 + t0, sh); d[4 * s] = descale(t13 - t0, sh);
}

struct JpegGeom {
  int H, W;
  int lbw, lbh;     // luma blocks per row / column: ceil(W/8), ceil(H/8)
  int cbw, cbh;     // chroma blocks per row / column: ceil(W/16), ceil(ceil(H/2)/8)
  int ch, cw;       // real chroma samples: ceil(H/2), ceil(W/2)
};

__host__ __device__ inline JpegGeom jpeg_geom(int H, int W) {
  JpegGeom g;
  g.H = H; g.W = W;
  g.lbw = (W + 7) / 8; g.lbh = (H + 7) / 8;
  g.ch = (H + 1) / 2; g.cw = (W + 1) / 2;
  g.cbw = (W + 15) / 16; g.cbh = (g.ch + 7) / 8;
  return g;
}

// One thread per 8x8 block (luma blocks, then Cb, then Cr): gather, code and decode the block into its plane of ws:
// luma [lbh*8][lbw*8], then Cb and Cr [cbh*8][cbw*8] each.
__global__ void __launch_bounds__(DG_THREADS) jpeg_block_kernel(const float* __restrict__ x, JpegGeom g,
                                                                JpegTables t, unsigned char* __restrict__ ws) {
  const int nl = g.lbw * g.lbh, nc = g.cbw * g.cbh;
  const int b = blockIdx.x * DG_THREADS + threadIdx.x;
  if (b >= nl + 2 * nc) return;
  const int comp = b < nl ? 0 : (b < nl + nc ? 1 : 2);
  const int bi = comp == 0 ? b : b - nl - (comp - 1) * nc;
  const int bw = comp == 0 ? g.lbw : g.cbw;
  const int by = bi / bw, bx = bi % bw;
  int d[64];
  for (int r = 0; r < 8; ++r)
    for (int c = 0; c < 8; ++c) {
      int v, yy, cb, cr;
      if (comp == 0) {
        const int py = min(by * 8 + r, g.H - 1), px = min(bx * 8 + c, g.W - 1);
        rgb_ycc(x + ((long)py * g.W + px) * 3, v, cb, cr);
      } else {
        const int sr = min(by * 8 + r, g.ch - 1), sc = bx * 8 + c;
        int s = (sc & 1) ? 2 : 1;
        for (int dy = 0; dy < 2; ++dy)
          for (int dx = 0; dx < 2; ++dx) {
            const int py = min(2 * sr + dy, g.H - 1), px = min(2 * sc + dx, g.W - 1);
            rgb_ycc(x + ((long)py * g.W + px) * 3, yy, cb, cr);
            s += comp == 1 ? cb : cr;
          }
        v = s >> 2;
      }
      d[r * 8 + c] = v - 128;
    }
  for (int r = 0; r < 8; ++r) fdct8(d + r * 8, 1, false);
  for (int c = 0; c < 8; ++c) fdct8(d + c, 8, true);
  const int tb = comp == 0 ? 0 : 1;
  for (int i = 0; i < 64; ++i) {
    const int a = d[i] < 0 ? -d[i] : d[i];
    const int m = (int)(((long long)(a + t.corr[tb][i]) * t.recip[tb][i]) >> t.shift[tb][i]);
    d[i] = (d[i] < 0 ? -m : m) * t.q[tb][i];
  }
  for (int c = 0; c < 8; ++c) idct8(d + c, 8, false);
  for (int r = 0; r < 8; ++r) idct8(d + r * 8, 1, true);
  const int pw = bw * 8;
  unsigned char* plane = ws + (comp == 0 ? 0 : (long)g.lbw * g.lbh * 64 + (long)(comp - 1) * nc * 64);
  for (int r = 0; r < 8; ++r)
    for (int c = 0; c < 8; ++c)
      plane[(long)(by * 8 + r) * pw + bx * 8 + c] = (unsigned char)min(max(d[r * 8 + c] + 128, 0), 255);
}

// h2v2 upsampled chroma at output pixel (py, px): the triangle filter (3/4 nearer, 1/4 farther; rows, then columns
// with bias 8 left / 7 right) with replicated edges, or 2x2 replication when the chroma rows are 2 samples or fewer.
__device__ __forceinline__ int upsample_c(const unsigned char* __restrict__ p, int pw, const JpegGeom& g, int py, int px) {
  const int r = py >> 1, c = px >> 1;
  if (g.cw <= 2) return p[(long)r * pw + c];
  const int rn = (py & 1) ? min(r + 1, g.ch - 1) : max(r - 1, 0);
  const int cn = (px & 1) ? min(c + 1, g.cw - 1) : max(c - 1, 0);
  const int s0 = 3 * p[(long)r * pw + c] + p[(long)rn * pw + c];
  const int s1 = 3 * p[(long)r * pw + cn] + p[(long)rn * pw + cn];
  return (3 * s0 + s1 + ((px & 1) ? 7 : 8)) >> 4;
}

__global__ void __launch_bounds__(DG_THREADS) jpeg_output_kernel(const unsigned char* __restrict__ ws, JpegGeom g,
                                                                 float* __restrict__ y) {
  const long i = (long)blockIdx.x * DG_THREADS + threadIdx.x;
  if (i >= (long)g.H * g.W) return;
  const int py = (int)(i / g.W), px = (int)(i % g.W);
  const int cpw = g.cbw * 8;
  const unsigned char* cbp = ws + (long)g.lbw * g.lbh * 64;
  const unsigned char* crp = cbp + (long)g.cbw * g.cbh * 64;
  const int yv = ws[(long)py * g.lbw * 8 + px];
  const int cb = upsample_c(cbp, cpw, g, py, px) - 128, cr = upsample_c(crp, cpw, g, py, px) - 128;
  const int rgb[3] = {yv + ((91881 * cr + 32768) >> 16), yv + ((-22554 * cb + 32768 - 46802 * cr) >> 16),
                      yv + ((116130 * cb + 32768) >> 16)};
#pragma unroll
  for (int c = 0; c < 3; ++c) y[i * 3 + c] = __double2float_rn((double)min(max(rgb[c], 0), 255) / 255.0);
}

// The quantisation tables (natural order) with libjpeg-turbo's reciprocals for the islow FDCT, whose output carries a
// factor 8: |c| / (8 q) rounded = ((|c| + corr) * recip) >> shift.
JpegTables jpeg_tables(const int* qtab) {
  JpegTables t;
  for (int k = 0; k < 2; ++k)
    for (int i = 0; i < 64; ++i) {
      const int q = qtab[k * 64 + i];
      const unsigned d = (unsigned)q << 3;
      int r = 16;
      for (unsigned v = d; v > 1; v >>= 1) ++r;               // 16 + floor(log2 d)
      unsigned long long fq = (1ull << r) / d, fr = (1ull << r) % d;
      int c = (int)(d / 2);
      if (fr == 0) { fq >>= 1; --r; }
      else if (fr <= d / 2) ++c;
      else ++fq;
      t.q[k][i] = q; t.recip[k][i] = (int)fq; t.corr[k][i] = c; t.shift[k][i] = r;
    }
  return t;
}

bool image_ok(int H, int W) { return H > 0 && W > 0 && (long)H * W <= (1l << 28); }

}  // namespace femasr

using namespace femasr;

extern "C" int femasr_degrade_mirror_conv(const float* x, float* y, int H, int W, const double* taps, int kh, int kw,
                                          int stride, int clip, void* stream) {
  FEMASR_CHECK_ARG(x && y && taps, "degrade_mirror_conv: null pointer");
  FEMASR_CHECK_ARG(image_ok(H, W), "degrade_mirror_conv: H and W must be >= 1 and H*W <= 2^28");
  FEMASR_CHECK_ARG(kh >= 1 && kw >= 1 && kh <= FEMASR_DEGRADE_MAX_KSIZE && kw <= FEMASR_DEGRADE_MAX_KSIZE &&
                       (kh & 1) && (kw & 1),
                   "degrade_mirror_conv: kernel sides must be odd and in [1, 25]");
  FEMASR_CHECK_ARG(stride >= 1 && stride <= FEMASR_DEGRADE_MAX_STRIDE, "degrade_mirror_conv: stride must be in [1, 4]");
  FEMASR_CHECK_ARG(clip == 0 || clip == 1, "degrade_mirror_conv: clip must be 0 or 1");
  ConvTaps t;
  for (int i = 0; i < kh * kw; ++i) t.k[i] = taps[kh * kw - 1 - i];          // convolution = correlation, flipped
  const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
  const size_t smem = (size_t)((CONV_T - 1) * stride + kh) * ((CONV_T - 1) * stride + kw) * 3 * sizeof(float);
  static PerDeviceFlag attr_set;
  if (!attr_set.cur()) {
    const int most = (int)((CONV_T - 1) * FEMASR_DEGRADE_MAX_STRIDE + FEMASR_DEGRADE_MAX_KSIZE);
    FEMASR_CUDA(cudaFuncSetAttribute(mirror_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     most * most * 3 * (int)sizeof(float)));
    attr_set.cur() = true;
  }
  const dim3 grid((unsigned)cdiv(Wo, CONV_T), (unsigned)cdiv(Ho, CONV_T)), block(CONV_T, CONV_T);
  mirror_conv_kernel<<<grid, block, smem, as_stream(stream)>>>(x, y, H, W, kh, kw, stride, clip, t);
  return launch_status("mirror_conv_kernel");
}

extern "C" int femasr_degrade_resize_pass(const float* x, float* y, int H, int W, int axis, int out_n, const int* idx,
                                          const float* w, int K, int clip, void* stream) {
  FEMASR_CHECK_ARG(x && y && idx && w, "degrade_resize_pass: null pointer");
  FEMASR_CHECK_ARG(image_ok(H, W), "degrade_resize_pass: H and W must be >= 1 and H*W <= 2^28");
  FEMASR_CHECK_ARG(axis == 0 || axis == 1, "degrade_resize_pass: axis must be 0 (rows) or 1 (columns)");
  FEMASR_CHECK_ARG(out_n >= 1 && image_ok(axis == 0 ? out_n : H, axis == 0 ? W : out_n),
                   "degrade_resize_pass: out_n must be >= 1 and the output at most 2^28 pixels");
  FEMASR_CHECK_ARG(K >= 1 && K <= 64, "degrade_resize_pass: K (taps per output) must be in [1, 64]");
  FEMASR_CHECK_ARG(clip == 0 || clip == 1, "degrade_resize_pass: clip must be 0 or 1");
  const long n = (long)(axis == 0 ? out_n : H) * (axis == 0 ? W : out_n) * 3;
  resize_pass_kernel<<<(unsigned)cdiv(n, DG_THREADS), DG_THREADS, 0, as_stream(stream)>>>(x, y, H, W, axis, out_n, idx,
                                                                                         w, K, clip);
  return launch_status("resize_pass_kernel");
}

extern "C" int femasr_degrade_noise_add(const float* x, const float* noise, int noise_ch, int H, int W, float* y,
                                        void* stream) {
  FEMASR_CHECK_ARG(x && noise && y, "degrade_noise_add: null pointer");
  FEMASR_CHECK_ARG(image_ok(H, W), "degrade_noise_add: H and W must be >= 1 and H*W <= 2^28");
  FEMASR_CHECK_ARG(noise_ch == 1 || noise_ch == 3, "degrade_noise_add: noise_ch must be 1 or 3");
  const long n = (long)H * W * 3;
  noise_add_clip_kernel<<<(unsigned)cdiv(n, DG_THREADS), DG_THREADS, 0, as_stream(stream)>>>(x, noise, noise_ch, n, y);
  return launch_status("noise_add_clip_kernel");
}

extern "C" size_t femasr_degrade_jpeg_workspace_bytes(int H, int W) {
  if (!image_ok(H, W)) return 0;
  const JpegGeom g = jpeg_geom(H, W);
  return (size_t)(g.lbw * g.lbh + 2 * g.cbw * g.cbh) * 64;
}

extern "C" int femasr_degrade_jpeg(const float* x, float* y, int H, int W, const int* qtables, void* workspace,
                                   void* stream) {
  FEMASR_CHECK_ARG(x && y && qtables && workspace, "degrade_jpeg: null pointer");
  FEMASR_CHECK_ARG(image_ok(H, W), "degrade_jpeg: H and W must be >= 1 and H*W <= 2^28");
  for (int i = 0; i < 128; ++i)
    FEMASR_CHECK_ARG(qtables[i] >= 1 && qtables[i] <= 255, "degrade_jpeg: quantisation table entries must be in [1, 255]");
  const JpegGeom g = jpeg_geom(H, W);
  const long nblk = (long)g.lbw * g.lbh + 2l * g.cbw * g.cbh;
  cudaStream_t st = as_stream(stream);
  jpeg_block_kernel<<<(unsigned)cdiv(nblk, DG_THREADS), DG_THREADS, 0, st>>>(x, g, jpeg_tables(qtables),
                                                                            static_cast<unsigned char*>(workspace));
  int rc = launch_status("jpeg_block_kernel");
  if (rc) return rc;
  jpeg_output_kernel<<<(unsigned)cdiv((long)H * W, DG_THREADS), DG_THREADS, 0, st>>>(
      static_cast<const unsigned char*>(workspace), g, y);
  return launch_status("jpeg_output_kernel");
}
