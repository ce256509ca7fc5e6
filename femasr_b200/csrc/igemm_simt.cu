// fp32 SIMT implicit-GEMM convolution / linear (NHWC), the exact-arithmetic path of libfemasr_b200.
//
//   y[m, n] = act( sum_{tap, c} pro(x)[src(m, tap), c] * w[tap*Cin + c, n] + bias[n] ) + res1 + res2
//
// M = B*Ho*Wo output pixels (or tokens), N = Cout, K = ksize^2 * Cin.  128 x BN x 16 tiles, 256
// threads, 8 x (BN/16) register micro-tiles, double-buffered shared memory with register prefetch.
// Replaces nn.Conv2d / nn.Linear on the reference path (see include/femasr_b200.h).
#include "common.cuh"

namespace femasr {

struct IgemmP {
  const float* x; const float* w; const float* bias; const float* res1; const float* res2; float* y;
  const float* pro_a; const float* pro_b; const float* gamma; const float* beta;
  int B, Hin, Win, Cin, Cout, Ho, Wo;
  int ksize, stride, upsample, pad, act;
  long M;
};

constexpr int BM = 128, BK = 16, LDA = BM + 4;

template <int BN, int PRO>
__global__ void __launch_bounds__(256, 2) igemm_simt_kernel(const IgemmP p) {
  constexpr int TN = BN / 16;              // columns per thread (8 or 4)
  constexpr int BV = BK * BN / 4 / 256;    // float4 B loads per thread (2 or 1)
  __shared__ __align__(16) float As[2][BK][LDA];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long m0 = (long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // ---- A loader: this thread fetches channels [kq, kq+4) of rows ra and ra+64
  const int ra = tid >> 2, kq = (tid & 3) * 4;
  int rb[2], roy[2], rox[2];
  bool rvalid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    long m = m0 + ra + i * 64;
    rvalid[i] = m < p.M;
    long mm = rvalid[i] ? m : 0;
    int hw = p.Ho * p.Wo;
    rb[i] = (int)(mm / hw);
    int r = (int)(mm - (long)rb[i] * hw);
    roy[i] = r / p.Wo;
    rox[i] = r - roy[i] * p.Wo;
  }
  const int taps = p.ksize * p.ksize;
  const int cchunks = p.Cin / BK;
  const int nk = taps * cchunks;
  const int HinE = p.upsample ? p.Hin * 2 : p.Hin;   // extent of the (virtually upsampled) conv input
  const int WinE = p.upsample ? p.Win * 2 : p.Win;

  float4 ga[2];
  float4 gb[BV];

  auto load_chunk = [&](int kc) {
    const int tap = kc / cchunks;
    const int c0 = (kc - tap * cchunks) * BK;
    const int kh = tap / p.ksize, kw = tap - kh * p.ksize;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      int iy = roy[i] * p.stride + kh - p.pad;
      int ix = rox[i] * p.stride + kw - p.pad;
      if (rvalid[i] && iy >= 0 && iy < HinE && ix >= 0 && ix < WinE) {
        if (p.upsample) { iy >>= 1; ix >>= 1; }
        const long pix = ((long)rb[i] * p.Hin + iy) * p.Win + ix;
        const int c = c0 + kq;
        v = __ldg(reinterpret_cast<const float4*>(p.x + pix * p.Cin + c));
        if (PRO == FEMASR_PRO_GN_SILU) {
          const float4 s = __ldg(reinterpret_cast<const float4*>(p.pro_a + (long)rb[i] * p.Cin + c));
          const float4 t = __ldg(reinterpret_cast<const float4*>(p.pro_b + (long)rb[i] * p.Cin + c));
          v.x = silu_f(fmaf(v.x, s.x, t.x)); v.y = silu_f(fmaf(v.y, s.y, t.y));
          v.z = silu_f(fmaf(v.z, s.z, t.z)); v.w = silu_f(fmaf(v.w, s.w, t.w));
        } else if (PRO == FEMASR_PRO_LN) {
          const float mu = __ldg(p.pro_a + pix), rs = __ldg(p.pro_b + pix);
          const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma + c));
          const float4 b = __ldg(reinterpret_cast<const float4*>(p.beta + c));
          v.x = (v.x - mu) * rs * g.x + b.x; v.y = (v.y - mu) * rs * g.y + b.y;
          v.z = (v.z - mu) * rs * g.z + b.z; v.w = (v.w - mu) * rs * g.w + b.w;
        }
      }
      ga[i] = v;
    }
    const long krow0 = (long)tap * p.Cin + c0;
#pragma unroll
    for (int i = 0; i < BV; ++i) {
      const int idx = tid + i * 256;
      const int k = idx / (BN / 4), n4 = idx - k * (BN / 4);
      gb[i] = __ldg(reinterpret_cast<const float4*>(p.w + (krow0 + k) * p.Cout + n0 + n4 * 4));
    }
  };
  auto store_chunk = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = ra + i * 64;
      As[buf][kq + 0][r] = ga[i].x; As[buf][kq + 1][r] = ga[i].y;
      As[buf][kq + 2][r] = ga[i].z; As[buf][kq + 3][r] = ga[i].w;
    }
#pragma unroll
    for (int i = 0; i < BV; ++i) {
      const int idx = tid + i * 256;
      const int k = idx / (BN / 4), n4 = idx - k * (BN / 4);
      *reinterpret_cast<float4*>(&Bs[buf][k][n4 * 4]) = gb[i];
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_chunk(0);
  store_chunk(0);
  __syncthreads();
  for (int kc = 0; kc < nk; ++kc) {
    const int buf = kc & 1;
    if (kc + 1 < nk) load_chunk(kc + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[TN];
      *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      if (TN == 8) *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][k][BN / 2 + tx * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kc + 1 < nk) {
      store_chunk(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
#pragma unroll
    for (int jj = 0; jj < TN / 4; ++jj) {
      const int n = n0 + (jj == 0 ? tx * 4 : BN / 2 + tx * 4);
      float4 o = make_float4(acc[i][jj * 4 + 0], acc[i][jj * 4 + 1], acc[i][jj * 4 + 2], acc[i][jj * 4 + 3]);
      if (p.bias) {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + n));
        o.x += bv.x; o.y += bv.y; o.z += bv.z; o.w += bv.w;
      }
      if (p.act == FEMASR_ACT_GELU) { o.x = gelu_erf_f(o.x); o.y = gelu_erf_f(o.y); o.z = gelu_erf_f(o.z); o.w = gelu_erf_f(o.w); }
      else if (p.act == FEMASR_ACT_RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
      else if (p.act == FEMASR_ACT_LRELU) { o.x = lrelu02_f(o.x); o.y = lrelu02_f(o.y); o.z = lrelu02_f(o.z); o.w = lrelu02_f(o.w); }
      const long off = m * p.Cout + n;
      if (p.res1) {
        const float4 r = *reinterpret_cast<const float4*>(p.res1 + off);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      if (p.res2) {
        const float4 r = *reinterpret_cast<const float4*>(p.res2 + off);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      *reinterpret_cast<float4*>(p.y + off) = o;
    }
  }
}

template <int BN>
static int launch_bn(const IgemmP& p, int prologue, cudaStream_t st) {
  dim3 grid((unsigned)cdiv(p.M, BM), p.Cout / BN);
  switch (prologue) {
    case FEMASR_PRO_NONE: igemm_simt_kernel<BN, FEMASR_PRO_NONE><<<grid, 256, 0, st>>>(p); break;
    case FEMASR_PRO_GN_SILU: igemm_simt_kernel<BN, FEMASR_PRO_GN_SILU><<<grid, 256, 0, st>>>(p); break;
    case FEMASR_PRO_LN: igemm_simt_kernel<BN, FEMASR_PRO_LN><<<grid, 256, 0, st>>>(p); break;
    default: return fail(FEMASR_ERR_ARG, "igemm: bad prologue");
  }
  return launch_status("igemm_simt_kernel");
}

int igemm_out_dims(const femasr_igemm_args* a, int* Ho, int* Wo) {
  if (a->ksize == 1) {
    if (a->stride != 1 || a->upsample) return fail(FEMASR_ERR_ARG, "igemm: 1x1 supports stride 1, no upsample");
    *Ho = a->Hin; *Wo = a->Win;
    return FEMASR_OK;
  }
  if (a->ksize == 4) {      // 4x4 pad 1 stride 2 (UNetDiscriminatorSN's down convs)
    if (a->stride != 2 || a->upsample) return fail(FEMASR_ERR_ARG, "igemm: 4x4 supports stride 2, no upsample");
    if (a->Hin < 2 || a->Win < 2) return fail(FEMASR_ERR_ARG, "igemm: a 4x4 stride-2 conv needs Hin, Win >= 2");
    *Ho = (a->Hin + 2 - 4) / 2 + 1; *Wo = (a->Win + 2 - 4) / 2 + 1;
    return FEMASR_OK;
  }
  if (a->ksize == 5) {      // 5x5 pad 2 stride 1 (AlexNet conv2 of LPIPS)
    if (a->stride != 1 || a->upsample) return fail(FEMASR_ERR_ARG, "igemm: 5x5 supports stride 1, no upsample");
    *Ho = a->Hin; *Wo = a->Win;
    return FEMASR_OK;
  }
  if (a->ksize != 3) return fail(FEMASR_ERR_ARG, "igemm: ksize must be 1, 3, 4 or 5");
  const int He = a->upsample ? 2 * a->Hin : a->Hin, We = a->upsample ? 2 * a->Win : a->Win;
  if (a->stride == 1) { *Ho = He; *Wo = We; }
  else if (a->stride == 2) { *Ho = (He + 2 - 3) / 2 + 1; *Wo = (We + 2 - 3) / 2 + 1; }
  else return fail(FEMASR_ERR_ARG, "igemm: stride must be 1 or 2");
  return FEMASR_OK;
}

}  // namespace femasr

using namespace femasr;

extern "C" int femasr_igemm_simt(const femasr_igemm_args* a, void* stream) {
  FEMASR_CHECK_ARG(a && a->x && a->w && a->y, "igemm: null pointer");
  FEMASR_CHECK_ARG(a->B > 0 && a->Hin > 0 && a->Win > 0, "igemm: empty input");
  FEMASR_CHECK_ARG(a->Cin % 16 == 0 && a->Cout % 64 == 0, "igemm: Cin %16 / Cout %64 required");
  FEMASR_CHECK_ARG(a->prologue == FEMASR_PRO_NONE || (a->pro_a && a->pro_b), "igemm: prologue tables missing");
  FEMASR_CHECK_ARG(a->prologue != FEMASR_PRO_LN || (a->gamma && a->beta && a->ksize == 1), "igemm: LN prologue needs gamma/beta, 1x1");
  IgemmP p;
  int st = igemm_out_dims(a, &p.Ho, &p.Wo);
  if (st) return st;
  p.x = a->x; p.w = a->w; p.bias = a->bias; p.res1 = a->res1; p.res2 = a->res2; p.y = a->y;
  p.pro_a = a->pro_a; p.pro_b = a->pro_b; p.gamma = a->gamma; p.beta = a->beta;
  p.B = a->B; p.Hin = a->Hin; p.Win = a->Win; p.Cin = a->Cin; p.Cout = a->Cout;
  p.ksize = a->ksize; p.stride = a->stride; p.upsample = a->upsample; p.pad = a->ksize == 1 ? 0 : (a->ksize == 5 ? 2 : 1);
  p.act = a->act;
  p.M = (long)a->B * p.Ho * p.Wo;
  if (a->Cout % 128 == 0) return launch_bn<128>(p, a->prologue, as_stream(stream));
  return launch_bn<64>(p, a->prologue, as_stream(stream));
}
