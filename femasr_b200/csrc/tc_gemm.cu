// Hopper (sm_90a) tensor-core implicit GEMM (3x3 convolution, stride 1 or 2, 4x4 stride 2, 5x5 stride 1, the fused nearest-x2
// upsample conv, and linear layers) with fp32-grade accuracy from a two-term fp16 operand split:
//
//     a = a_hi + a_lo,  w*2^s = w_hi + w_lo          (fp16, 11-bit significands each)
//     D = a_hi*w_hi + a_hi*w_lo + a_lo*w_hi          (3 wgmma f16 products per k-step, fp32 accumulate in registers)
//
// i.e. ~22 significand bits per operand; the dropped a_lo*w_lo term is ~2^-22 relative (SURVEY 7.3-1:
// the path needs >=18 bits before the VQ and >=13 after it; single-pass fp16/bf16/tf32 fails parity).
//
// Structure (one persistent CTA per SM, 288 threads, warp-specialised):
//   warp 8     TMA producer (one elected lane): activation tile = 4-D box (64 ch x Wt x Ht x 1) of the NHWC fp16 planes
//              at the tap offset (kh-1, kw-1) - out-of-bounds rows/cols are zero-filled by TMA, which IS the conv
//              padding - and the weight tile = 2-D box (64 x BN) of the K-major fp16 planes; 128B swizzle; a ring of
//              full / empty mbarriers.
//   warps 0-7  two consumer warpgroups, each owning 64 rows of the 128 x BN tile: wgmma m64nBNk16 straight from the
//              swizzled shared-memory stages into a register accumulator, then the epilogue from those registers
//              (*2^-s + bias -> GELU -> + residual(s) -> fp32 NHWC or split-fp16 planes, GroupNorm partials, VQ top-4).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>

#include "common.cuh"

namespace femasr {

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok;
}
// Bounded wait: a protocol bug must not hang the GPU; after 4 s the kernel traps (reported as a
// CUDA error by the next API call) instead of spinning forever.
__device__ __forceinline__ uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    // 4 s: far beyond any legitimate wait.  No printf here: a call inside the main loop would make ptxas serialise
    // every wgmma of the kernel.
    if ((++spins & 0xFFFu) == 0 && global_ns() - t0 > 4000000000ull) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// Programmatic dependent launch: a kernel launched with the programmatic-serialisation attribute may start (its CTAs
// become resident as the predecessor's retire, it runs its prologue) before the predecessor has finished;
// griddepcontrol.wait blocks until the predecessor grid has completed and its memory is visible.  Both are no-ops in a
// plain launch.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// One lane of a converged warp (elect.sync): the TMA producer role is entered through this instead of `lane == 0` so
// that ptxas knows a single lane issues the loads (no per-load serialisation loop).
__device__ __forceinline__ bool elect_one() {
  uint32_t p;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}"
      : "=r"(p));
  return p != 0;
}

// wgmma: D (registers of the warpgroup) += A (shared, K-major) x B (shared, K-major).  `accumulate` = 0 overwrites D.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// m64nNk16 (f16) / m64nNk32 (e4m3) with N / 2 fp32 accumulator registers per thread; operands after them: A and B
// descriptors, then the accumulate flag
#define FEMASR_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define FEMASR_ACC32 FEMASR_ACC8(0), FEMASR_ACC8(8), FEMASR_ACC8(16), FEMASR_ACC8(24)
#define FEMASR_ACC64 FEMASR_ACC32, FEMASR_ACC8(32), FEMASR_ACC8(40), FEMASR_ACC8(48), FEMASR_ACC8(56)
#define FEMASR_REGS32 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define FEMASR_REGS64 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define FEMASR_WGMMA(name, NREG, shape, tail, REGS, ACC, IA, IB, IP)                                                   \
  __device__ __forceinline__ void name(float (&d)[NREG], uint64_t da, uint64_t db, uint32_t accumulate) {              \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " IP ", 0;\n\twgmma.mma_async.sync.aligned." shape " {" REGS "}, " \
                 IA ", " IB ", p, 1, 1" tail ";\n\t}"                                                                  \
                 : ACC : "l"(da), "l"(db), "r"(accumulate));                                                           \
  }
FEMASR_WGMMA(wgmma_f16_n64, 32, "m64n64k16.f32.f16.f16", ", 0, 0", FEMASR_REGS32, FEMASR_ACC32, "%32", "%33", "%34")
FEMASR_WGMMA(wgmma_e4m3_n64, 32, "m64n64k32.f32.e4m3.e4m3", "", FEMASR_REGS32, FEMASR_ACC32, "%32", "%33", "%34")
FEMASR_WGMMA(wgmma_f16_n128, 64, "m64n128k16.f32.f16.f16", ", 0, 0", FEMASR_REGS64, FEMASR_ACC64, "%64", "%65", "%66")
FEMASR_WGMMA(wgmma_e4m3_n128, 64, "m64n128k32.f32.e4m3.e4m3", "", FEMASR_REGS64, FEMASR_ACC64, "%64", "%65", "%66")
template <int BN> struct Wgmma;
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void f16(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { wgmma_f16_n64(d, a, b, acc); }
  static __device__ __forceinline__ void e4m3(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { wgmma_e4m3_n64(d, a, b, acc); }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void f16(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_f16_n128(d, a, b, acc); }
  static __device__ __forceinline__ void e4m3(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_e4m3_n128(d, a, b, acc); }
};
// keeps the compiler from moving accumulator reads / writes across a wgmma wait
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// (x, y) -> packed fp16 hi pair and lo pair; the conversion saturates to +-65504 instead of overflowing to inf
__device__ __forceinline__ void split_pack2(float x, float y, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(y), "f"(x));     // d = {hi half: first src, lo half: second}
  const __half2 h = *reinterpret_cast<const __half2*>(&hi);
  const float2 hf = __half22float2(h);
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(y - hf.y), "f"(x - hf.x));
}

// K-major, 128B-swizzled operand tile ([rows][128 B], 8-row atoms of 1024 B) as a wgmma matrix descriptor: start
// address >> 4, leading-dimension offset unused for swizzled K-major (1), stride-dimension offset 1024 B between 8-row
// groups, layout type 1 (SWIZZLE_128B) in bits 62-63.  A k-step inside the 128-byte atom advances the start address by
// its 32 bytes (16 fp16 / 32 e4m3); the hardware applies the swizzle to the absolute address, like the TMA that wrote it.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t saddr) {
  uint64_t d = (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// ------------------------------------------------------------------------------------------------ kernel
struct TcP {
  const float* bias; const float* res1; const float* res2; float* y; const float* inv_scale;
  __half* out_hi; __half* out_lo;   // when set: the result is written as split fp16 planes (next GEMM's A operand)
  float* gn_partial;                // when set: per-(image, tile, 32-row quarter) GroupNorm partial sums of the OUTPUT
  int gn_rows, cpg;                 // partial rows per image; channels per group (Cout / 32)
  int B, H, W, Cin, Cout, taps, act;
  int stride;                    // 1 or 2 (3x3 stride-2: TMA traversal stride 2, tiles run over the output grid)
  int up;                        // 1: nearest-x2 upsample + 3x3 conv evaluated as 4 sub-pixel phases of 2x2 taps
  int Wt, Ht, wt_shift;          // 128-pixel tile = Ht rows x Wt cols (Wt power of two)
  int tiles_x, tiles_y, n_tiles; // per image spatial tiles, Cout / BN
  int num_tiles, cchunks;        // total tiles, Cin / 64
  int kb_begin, kb_end;          // k-block range of this launch (a K-slice; the caller sums slices through res1)
  int slice_kb;                  // >0: in-kernel K slicing - every slice_kb k-blocks the accumulator is folded into an
                                 // fp32 running sum (round-to-nearest adds), so the tensor core's accumulation, which
                                 // does not round to nearest, never runs longer than a slice
  int f8;                        // F8 mode: the "lo" planes of both operands hold interleaved e4m3 bytes per 64-channel chunk
                                 // (A: [a_lo * 2^10 | a_hi * 2^-2], B: [w_hi * 2^-10 | w_lo * 2^2]); one K = 128 fp8 product per k-block
                                 // replaces the two fp16 cross products
  // VQ mode (template VQ): the GEMM is z . E^T and the epilogue keeps, per feature row, the four smallest distances
  // fl(fl(A + B_j) - 2 C_j) over all codes instead of storing the [N, n_e] product (femasr_arch.py:35-38, 63-66)
  const float* vq_a;             // [M]   A = sum z^2 per row
  const float* vq_esq;           // [Cout] B_j = sum e_j^2 per code
  uint2* vq_cand;                // [M][4] {distance bits, code}, ascending (distance, code)
};

constexpr int TC_BM = 128, TC_BK = 64;
constexpr int A_PLANE_BYTES = TC_BM * TC_BK * 2;   // 16 KB
constexpr int TC_CONSUMER_WARPS = 8, TC_THREADS = 32 * TC_CONSUMER_WARPS + 32;
constexpr int TC_SMEM_LIMIT = 232448;              // 227 KB of opt-in shared memory per block on H100

template <int BN>
struct TcCfg {
  static_assert(BN == 64 || BN == 128, "tile width");
  static constexpr int B_PLANE_BYTES = BN * TC_BK * 2;
  static constexpr int STAGE_BYTES = 2 * A_PLANE_BYTES + 2 * B_PLANE_BYTES;        // a_hi, a_lo, w_hi, w_lo
  static constexpr int RED_BYTES = TC_CONSUMER_WARPS * 64 * 2 * 4;                  // per-warp GroupNorm partials
  static constexpr int STAGES = (TC_SMEM_LIMIT - 1024 - 256 - RED_BYTES) / STAGE_BYTES;   // 3 (BN 128) / 4 (BN 64)
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + RED_BYTES;
  static constexpr int NF = BN / 2;                                                  // accumulator floats per thread
  static_assert(SMEM_BYTES <= TC_SMEM_LIMIT, "shared memory budget");
  static_assert(16 * STAGES <= 256, "barrier area");
};

// running top-4 of (d, j), ascending lexicographically; precondition: (d, j) sorts before (td[3], tj[3])
__device__ __forceinline__ void top4_insert(float (&td)[4], int (&tj)[4], float d, int j) {
  td[3] = d; tj[3] = j;
#pragma unroll
  for (int k = 3; k > 0; --k)
    if (td[k] < td[k - 1] || (td[k] == td[k - 1] && tj[k] < tj[k - 1])) {
      const float t = td[k - 1]; td[k - 1] = td[k]; td[k] = t;
      const int u = tj[k - 1]; tj[k - 1] = tj[k]; tj[k] = u;
    }
}

// RES: the layer adds a residual tile (res1) in the epilogue (a template parameter: the load is in the hot loop).
// F8: the F8 cross-term mode (p.f8).  A template parameter because a runtime choice between the two accumulator sets
// inside the k-loop makes ptxas serialise every wgmma of the kernel.
// VQ: the z . E^T product of the VectorQuantizer with the argmin fused into the epilogue (see the VQ epilogue below);
// work is ordered M-major so that one CTA sees ALL code tiles of its 128 feature rows back to back.
// EXT: taps and epilogues beyond the generator's.  1: the discriminator's 4x4 taps and LeakyReLU epilogue; 2: LPIPS'
// 5x5 pad-2 taps (AlexNet conv2).  A template parameter so that the other instantiations keep exactly the instruction
// stream they had without them (measured: 1.3% slower GEMMs otherwise).
template <int BN, bool RES, bool F8, bool VQ = false, int EXT = 0>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_igemm_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo, const TcP p) {
  using Cfg = TcCfg<BN>;
  constexpr int STAGES = Cfg::STAGES, NF = Cfg::NF;
  static_assert(!VQ || (!RES && !F8), "VQ mode: plain linear tiles");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
  float* red = reinterpret_cast<float*>(smem_raw + (bar_base + 256u - smem_u32(smem_raw)));
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int worker = (int)blockIdx.x, nworkers = (int)gridDim.x;
  const int num_m = p.num_tiles / p.n_tiles;
  // it-th work item of this CTA (-1: done).  Default: items strided over the CTAs.  VQ: m-tiles strided over the
  // CTAs, and for each m-tile every n-tile (code tile) in turn.
  auto work_of = [&](int it) -> int {
    if (VQ) {
      const int mt = (it / p.n_tiles) * nworkers + worker;
      return mt < num_m ? mt * p.n_tiles + it % p.n_tiles : -1;
    }
    const int w = worker + it * nworkers;
    return w < p.num_tiles ? w : -1;
  };
  // work item -> (n-tile, m-tile); the m-tile decodes into (phase, image, tile row/col)
  struct TileCoord { int nt, tx, ty, b, ph; };
  auto decode = [&](int work) {
    TileCoord tc;
    tc.nt = work % p.n_tiles;
    int mt = work / p.n_tiles;
    tc.tx = mt % p.tiles_x; mt /= p.tiles_x;
    tc.ty = mt % p.tiles_y; mt /= p.tiles_y;
    tc.b = mt % p.B;
    tc.ph = mt / p.B;                                // sub-pixel phase (0 unless p.up)
    return tc;
  };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_launch_dependents();        // the next kernel of the stream may begin its own prologue as our CTAs retire
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), TC_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                     // barriers initialised: from here on the predecessor's output is read

  if (warp == TC_CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    if (!elect_one()) return;
    const int ksz = EXT == 1 && p.taps == 16 ? 4 : EXT == 2 && p.taps == 25 ? 5 : (p.taps == 9 ? 3 : 1);   // (p.up: taps == 4)
    int stage = 0; uint32_t phase = 0;
    for (int it = 0, work; (work = work_of(it)) >= 0; ++it) {
      const TileCoord tc = decode(work);
      const int n0 = tc.ph * p.Cout + tc.nt * BN;
      for (int kb = p.kb_begin; kb < p.kb_end; ++kb) {
        // activation box of k-block kb: channel chunk and the tap's spatial offset (conv padding = TMA zero fill)
        const int tap = kb / p.cchunks;
        const int c0 = (kb - tap * p.cchunks) * TC_BK;
        int dy = 0, dx = 0;
        if (p.up) { dy = (tap >> 1) - 1 + (tc.ph >> 1); dx = (tap & 1) - 1 + (tc.ph & 1); }
        else if (ksz == 3) { dy = tap / 3 - 1; dx = tap - (tap / 3) * 3 - 1; }
        else if (EXT == 1 && ksz == 4) { dy = (tap >> 2) - 1; dx = (tap & 3) - 1; }     // 4x4 pad 1, always stride 2
        else if (EXT == 2 && ksz == 5) { dy = tap / 5 - 2; dx = tap % 5 - 2; }          // 5x5 pad 2, stride 1
        const int x = p.stride * tc.tx * p.Wt + dx, y = p.stride * tc.ty * p.Ht + dy;
        mbar_wait(empty_bar(stage), phase ^ 1u);
        const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
        mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
        tma_load_4d(sa, &map_a_hi, full_bar(stage), c0, x, y, tc.b);
        tma_load_4d(sa + A_PLANE_BYTES, &map_a_lo, full_bar(stage), c0, x, y, tc.b);
        tma_load_2d(sa + 2 * A_PLANE_BYTES, &map_b_hi, full_bar(stage), tap * p.Cin + c0, n0);
        tma_load_2d(sa + 2 * A_PLANE_BYTES + Cfg::B_PLANE_BYTES, &map_b_lo, full_bar(stage), tap * p.Cin + c0, n0);
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ===================== consumers: two warpgroups x 64 accumulator rows =====================
  // Accumulator fragment of m64nBNk16 (per warp 16 rows): d[4j + 2h + e] = row 16 * (warp % 4) + lane / 4 + 8h,
  // column 8j + 2 (lane % 4) + e.
  const int wg = warp >> 2;
  const int rsub = lane >> 2, q = lane & 3;
  const float inv_scale = __ldg(p.inv_scale);
  const bool sliced = p.slice_kb > 0;
  const int slice_len = sliced ? p.slice_kb : (p.kb_end - p.kb_begin);
  float acc[NF], ext[NF];          // ext: the F8 cross products, or the running sum of the K slices
#pragma unroll
  for (int i = 0; i < NF; ++i) { acc[i] = 0.f; ext[i] = 0.f; }
  int stage = 0; uint32_t phase = 0;
  // VQ state: the running top-4 of this thread's two rows
  float td[2][4];
  int tj[2][4];
  float a_row[2] = {0.f, 0.f};

  for (int it = 0, work; (work = work_of(it)) >= 0; ++it) {
    const TileCoord tc = decode(work);
    // ---------------- main loop
    bool have_ext = F8;
    for (int kb0 = p.kb_begin; kb0 < p.kb_end; kb0 += slice_len) {
      const int kb1 = min(kb0 + slice_len, p.kb_end);
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
        const uint64_t a_hi = make_sw128_desc(sa + wg * (A_PLANE_BYTES / 2));
        const uint64_t a_lo = make_sw128_desc(sa + A_PLANE_BYTES + wg * (A_PLANE_BYTES / 2));
        const uint64_t b_hi = make_sw128_desc(sa + 2 * A_PLANE_BYTES);
        const uint64_t b_lo = make_sw128_desc(sa + 2 * A_PLANE_BYTES + Cfg::B_PLANE_BYTES);
        fence_regs(acc); fence_regs(ext);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
          const uint64_t ko = (uint64_t)((k * 32) >> 4);   // +32 bytes per k-step inside the 128B swizzle atom
          const uint32_t more = (kb != kb0 || k != 0) ? 1u : 0u;
          // small cross terms first, the dominant hi*hi product last
          if constexpr (F8) {
            Wgmma<BN>::e4m3(ext, a_lo + ko, b_lo + ko, more);     // sum a_lo8 w_hi8 + sum a_hi8 w_lo8
            Wgmma<BN>::f16(acc, a_hi + ko, b_hi + ko, more);
          } else {
            Wgmma<BN>::f16(acc, a_lo + ko, b_hi + ko, more);
            Wgmma<BN>::f16(acc, a_hi + ko, b_lo + ko, 1u);
            Wgmma<BN>::f16(acc, a_hi + ko, b_hi + ko, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_regs(acc); fence_regs(ext);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(stage));     // this warp's reads of the stage are complete
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      if (kb1 < p.kb_end) {           // sliced: fold the finished partial into the running sum
#pragma unroll
        for (int i = 0; i < NF; ++i) ext[i] = have_ext ? acc[i] + ext[i] : acc[i];
        have_ext = true;
      }
    }
    if (have_ext) {
#pragma unroll
      for (int i = 0; i < NF; ++i) acc[i] += ext[i];
    }

    if constexpr (VQ) {
      // ===================== VQ epilogue: running top-4 of d_j = fl(fl(A + B_j) - 2 C_j) per feature row =====================
      // The thread owns two accumulator rows (features) and BN / 4 columns (codes) of every code tile; its codes arrive
      // in increasing order, so a strict '<' insertion keeps (distance, code) lexicographic order.  C_j here carries the
      // tensor core's split-fp16 accumulation error (~1e-8 against a distance grid of ulp(A) ~ 3e-5), so the FOUR best
      // are handed to femasr_vq_finish, which recomputes the exact fp32 distance of every candidate within a few ulps
      // of the best and applies the reference's tie rule.
      long token[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = wg * 64 + (warp & 3) * 16 + rsub + 8 * h;
        token[h] = (long)tc.tx * p.Wt + row;             // ksize 1: the features are one long row of tokens
        if (tc.nt == 0) {
#pragma unroll
          for (int k = 0; k < 4; ++k) { td[h][k] = INFINITY; tj[h][k] = 0x7fffffff; }
          a_row[h] = token[h] < p.W ? __ldg(p.vq_a + token[h]) : 0.f;
        }
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = tc.nt * BN + 8 * j + 2 * q;
        const float2 es = __ldg(reinterpret_cast<const float2*>(p.vq_esq + col));
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float c = acc[4 * j + 2 * h + e] * inv_scale;                                   // exact (power of two)
            const float d = __fsub_rn(__fadd_rn(a_row[h], e ? es.y : es.x), __fmul_rn(2.0f, c));   // fl(fl(A + B_j) - 2 C_j)
            if (d < td[h][3]) top4_insert(td[h], tj[h], d, col + e);
          }
      }
      if (tc.nt == p.n_tiles - 1) {
        // the four lanes of a row hold interleaved column sets: merge their lists into lane q = 0
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int pp = 1; pp < 4; ++pp)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float d = __shfl_sync(0xffffffffu, td[h][k], (lane & ~3) | pp);
              const int j = __shfl_sync(0xffffffffu, tj[h][k], (lane & ~3) | pp);
              if (q == 0 && (d < td[h][3] || (d == td[h][3] && j < tj[h][3]))) top4_insert(td[h], tj[h], d, j);
            }
          if (q == 0 && token[h] < p.W) {
            uint4* out = reinterpret_cast<uint4*>(p.vq_cand + token[h] * 4);
            out[0] = make_uint4(__float_as_uint(td[h][0]), (uint32_t)tj[h][0], __float_as_uint(td[h][1]), (uint32_t)tj[h][1]);
            out[1] = make_uint4(__float_as_uint(td[h][2]), (uint32_t)tj[h][2], __float_as_uint(td[h][3]), (uint32_t)tj[h][3]);
          }
        }
      }
      continue;
    }

    // ===================== epilogue: acc * 2^-s + bias -> GELU | ReLU -> + res1 + res2 -> store =====================
    const int Ho = p.up ? 2 * p.H : p.H, Wo = p.up ? 2 * p.W : p.W;
    long off[2];                                         // output element offset of this thread's two rows (-1: outside)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = wg * 64 + (warp & 3) * 16 + rsub + 8 * h;
      const int y = tc.ty * p.Ht + (row >> p.wt_shift), x = tc.tx * p.Wt + (row & (p.Wt - 1));
      const int oy = p.up ? 2 * y + (tc.ph >> 1) : y, ox = p.up ? 2 * x + (tc.ph & 1) : x;
      off[h] = (y < p.H && x < p.W) ? (((long)tc.b * Ho + oy) * Wo + ox) * p.Cout : -1;
    }
    const int gpl = BN / p.cpg;                           // GroupNorm groups of this n-tile
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = tc.nt * BN + 8 * j + 2 * q;
      const float2 bb = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
      float gs = 0.f, gss = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2 o;
        o.x = fmaf(acc[4 * j + 2 * h], inv_scale, bb.x);     // acc * 2^-s is exact: == (acc * inv) + bias
        o.y = fmaf(acc[4 * j + 2 * h + 1], inv_scale, bb.y);
        if (p.act == FEMASR_ACT_GELU) { o.x = gelu_erf_fast_f(o.x); o.y = gelu_erf_fast_f(o.y); }
        else if (p.act == FEMASR_ACT_RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
        else if (EXT == 1 && p.act == FEMASR_ACT_LRELU) { o.x = lrelu02_f(o.x); o.y = lrelu02_f(o.y); }
        if (off[h] >= 0) {
          const long o_off = off[h] + col;
          if (RES) { const float2 r = *reinterpret_cast<const float2*>(p.res1 + o_off); o.x += r.x; o.y += r.y; }
          if (p.res2) { const float2 r = *reinterpret_cast<const float2*>(p.res2 + o_off); o.x += r.x; o.y += r.y; }
          if (p.out_hi) {
            uint32_t hh, ll;
            split_pack2(o.x, o.y, hh, ll);
            *reinterpret_cast<uint32_t*>(p.out_hi + o_off) = hh;
            *reinterpret_cast<uint32_t*>(p.out_lo + o_off) = ll;
          } else {
            *reinterpret_cast<float2*>(p.y + o_off) = o;
          }
          gs += o.x + o.y; gss = fmaf(o.x, o.x, fmaf(o.y, o.y, gss));
        }
      }
      if (p.gn_partial) {
        // fixed-order reduction over the warp's 16 rows (lanes sharing q), then over the lanes of one group
#pragma unroll
        for (int o = 4; o <= 16; o <<= 1) { gs += __shfl_xor_sync(0xffffffffu, gs, o); gss += __shfl_xor_sync(0xffffffffu, gss, o); }
        if (p.cpg >= 4) { gs += __shfl_xor_sync(0xffffffffu, gs, 1); gss += __shfl_xor_sync(0xffffffffu, gss, 1); }
        if (p.cpg >= 8) { gs += __shfl_xor_sync(0xffffffffu, gs, 2); gss += __shfl_xor_sync(0xffffffffu, gss, 2); }
        if (rsub == 0 && (q & (p.cpg / 2 - 1)) == 0) {
          const int g = (8 * j + 2 * q) / p.cpg;
          red[(warp * 64 + g) * 2] = gs;
          red[(warp * 64 + g) * 2 + 1] = gss;
        }
      }
    }
    if (p.gn_partial) {
      // one partial row per 32-row quarter of the tile (= the two warps of 16 rows that cover it)
      asm volatile("bar.sync 1, %0;" ::"r"(32 * TC_CONSUMER_WARPS) : "memory");
      const int tile_in_img = (tc.ph * p.tiles_y + tc.ty) * p.tiles_x + tc.tx;
      for (int i = threadIdx.x; i < 4 * gpl; i += 32 * TC_CONSUMER_WARPS) {
        const int quarter = i / gpl, g = i - quarter * gpl;
        const float* r0 = red + ((2 * quarter) * 64 + g) * 2;
        const float* r1 = red + ((2 * quarter + 1) * 64 + g) * 2;
        float* gp = p.gn_partial + (((long)tc.b * p.gn_rows + tile_in_img * 4 + quarter) * 32 + tc.nt * gpl + g) * 2;
        *reinterpret_cast<float2*>(gp) = make_float2(r0[0] + r1[0], r0[1] + r1[1]);
      }
      asm volatile("bar.sync 1, %0;" ::"r"(32 * TC_CONSUMER_WARPS) : "memory");
    }
  }
}

// ------------------------------------------------------------------------------------------------ operand preparation
__device__ __forceinline__ void split_store8(const float (&v)[8], __half* hi, __half* lo) {
  __align__(16) __half h[8], l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float c = fminf(fmaxf(v[i], -65504.f), 65504.f);
    h[i] = __float2half_rn(c);
    l[i] = __float2half_rn(c - __half2float(h[i]));
  }
  *reinterpret_cast<uint4*>(hi) = *reinterpret_cast<const uint4*>(h);
  *reinterpret_cast<uint4*>(lo) = *reinterpret_cast<const uint4*>(l);
}

// x fp32 NHWC [B,H,W,C] -> fp16 hi/lo planes [B,H*up,W*up,C] with an optional GroupNorm+SiLU transform
// (scale/shift tables [B,C]) and optional nearest x2 replication.  8 channels per thread.
template <int MODE>
__global__ void __launch_bounds__(256) tc_prepare_kernel(const float* __restrict__ x, __half* __restrict__ hi,
                                                         __half* __restrict__ lo, const float* __restrict__ sc,
                                                         const float* __restrict__ sh, int H, int W, int C, int up,
                                                         long total8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  const int c8 = C / 8;
  const int cq = (int)(i % c8);
  const long pix = i / c8;
  const int xw = (int)(pix % W);
  const long t = pix / W;
  const int yh = (int)(t % H);
  const int b = (int)(t / H);
  const float4* src = reinterpret_cast<const float4*>(x + pix * C + cq * 8);
  const float4 a = __ldg(src), bq = __ldg(src + 1);
  float v[8] = {a.x, a.y, a.z, a.w, bq.x, bq.y, bq.z, bq.w};
  if (MODE == FEMASR_PRO_GN_SILU) {
    const float4* ps = reinterpret_cast<const float4*>(sc + (long)b * C + cq * 8);
    const float4* pt = reinterpret_cast<const float4*>(sh + (long)b * C + cq * 8);
    const float4 s0 = __ldg(ps), s1 = __ldg(ps + 1), t0 = __ldg(pt), t1 = __ldg(pt + 1);
    const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float tt[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = silu_f(fmaf(v[k], s[k], tt[k]));
  }
  if (!up) {
    split_store8(v, hi + pix * C + cq * 8, lo + pix * C + cq * 8);
  } else {
    const int W2 = 2 * W;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const long op = (((long)b * 2 * H + 2 * yh + dy) * W2 + 2 * xw + dx) * C + cq * 8;
        split_store8(v, hi + op, lo + op);
      }
  }
}

// nn.MaxPool2d(K, 2) (floor; K = 2 or 3) fused into the staging of the next conv's operand: the max is taken on fp32 and
// then split, so the planes are exactly the split of the pooled tensor.  x [B,H,W,C] -> [B,(H-K)/2+1,(W-K)/2+1,C], 8
// channels per thread.
template <int K>
__global__ void __launch_bounds__(256) tc_prepare_pool_kernel(const float* __restrict__ x, __half* __restrict__ hi,
                                                              __half* __restrict__ lo, int H, int W, int C, long total8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  float v[8];
  const long o = pool_max8<K>(x, i, H, W, C, v);
  split_store8(v, hi + o, lo + o);
}

// Bilinear x2 (align_corners=False) fused into the staging the same way: interpolated on fp32, then split.
// x [B,H,W,C] -> [B,2H,2W,C], 8 channels per thread.
__global__ void __launch_bounds__(256) tc_prepare_bilinear_kernel(const float* __restrict__ x, __half* __restrict__ hi,
                                                                  __half* __restrict__ lo, int H, int W, int C, long total8) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total8) return;
  float v[8];
  const long o = bilinear2_8(x, i, H, W, C, v);
  split_store8(v, hi + o, lo + o);
}

// Same transform without replication, organised for bandwidth: the image is a flat array of float4 (4 channels), a warp
// reads 512 contiguous bytes per request and every thread keeps PREP_U independent requests in flight; blockIdx.y = b.
constexpr int PREP_U = 4;
template <int MODE>
__global__ void __launch_bounds__(256) tc_prepare_flat_kernel(const float4* __restrict__ x, uint2* __restrict__ hi,
                                                              uint2* __restrict__ lo, const float* __restrict__ sc,
                                                              const float* __restrict__ sh, int C, int per_image4) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.y;
  const long base = (long)b * per_image4;
  const int i0 = blockIdx.x * (256 * PREP_U) + threadIdx.x;
  const int c4 = C >> 2;
  float4 v[PREP_U];
#pragma unroll
  for (int u = 0; u < PREP_U; ++u) {
    const int i = i0 + u * 256;
    if (i < per_image4) v[u] = __ldg(x + base + i);
  }
#pragma unroll
  for (int u = 0; u < PREP_U; ++u) {
    const int i = i0 + u * 256;
    if (i >= per_image4) break;
    float w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
    if (MODE == FEMASR_PRO_GN_SILU || MODE == FEMASR_PRO_GN_SILU_FAST) {
      const int c = (i % c4) * 4;
      const float4 s = __ldg(reinterpret_cast<const float4*>(sc + (long)b * C + c));
      const float4 t = __ldg(reinterpret_cast<const float4*>(sh + (long)b * C + c));
      const float ss[4] = {s.x, s.y, s.z, s.w}, tt[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float n = fmaf(w[k], ss[k], tt[k]);
        // fast form: 2 MUFU + 3 FP32 ops instead of ~25 instructions (this pass is issue-bound with the exact one)
        w[k] = MODE == FEMASR_PRO_GN_SILU_FAST ? __fdividef(n, 1.0f + __expf(-n)) : silu_f(n);
      }
    }
    __align__(8) __half h[4], l[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float cl = fminf(fmaxf(w[k], -65504.f), 65504.f);
      h[k] = __float2half_rn(cl);
      l[k] = __float2half_rn(cl - __half2float(h[k]));
    }
    hi[base + i] = *reinterpret_cast<const uint2*>(h);
    lo[base + i] = *reinterpret_cast<const uint2*>(l);
  }
}

// F8 staging (layers behind the VQ): the hi plane as above; the second plane holds, per pixel and 64-channel chunk, 128
// bytes = [e4m3((v - hi) * 2^10) x 64 | e4m3(v * 2^-2) x 64] - the A operand of the single K = 128 fp8 MMA group that
// replaces the two fp16 cross products (the weights carry [e4m3(w_hi * 2^-10) | e4m3(w_lo * 2^2)] at the matching offsets,
// so both power-of-two scales cancel inside the dot product).
// Error budget: scripts/exp_fp8_cross.py, 1.2e-4 output max-abs for the whole post-VQ scope (bar 1e-3).
// The scales place the operands in e4m3's normal range (4 significant bits down to 2^-6, fewer below, nothing under 2^-10).
// The first recipe, (2^12, 2^0), was tuned on the kaiming-uniform random-init weights, whose magnitudes all lie within a
// factor 2 of the per-tensor maximum; a TRAINED conv is bell-shaped with typical |w| ~ max / 10 ... max / 50, for which
// e4m3(w_hi * 2^-12) <= 0.25 * |w| / max is already subnormal.  scripts/exp_fp8_scales.py (weights of the layers behind the
// VQ redrawn from a normal / a Student-t(3) distribution of the same standard deviation; output max-abs uniform / normal /
// t(3)): (12, 0) 1.2e-4 / 1.1e-4 / 5.8e-4, (10, 2) 1.3e-4 / 1.4e-4 / 1.8e-4 - the minimax choice over a 10-recipe sweep.
// Activations keep full e4m3 precision for |a| in [2^-4, 1792] (a_lo * 2^10 ~ a / 4 likewise).
constexpr float F8_LO_SCALE = 1024.0f;       // a_lo * 2^10 against w_hi * 2^-10
constexpr float F8_VAL_SCALE = 0.25f;        // a * 2^-2 against w_lo * 2^2
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
template <int MODE>
__global__ void __launch_bounds__(256) tc_prepare_flat_f8_kernel(const float4* __restrict__ x, uint4* __restrict__ hi,
                                                                 uint2* __restrict__ x8, const float* __restrict__ sc,
                                                                 const float* __restrict__ sh, int C, int per_image8) {
  // one thread = 8 consecutive channels of a pixel: 32 bytes in, 16 (hi) + 8 (lo8) + 8 (value8) bytes out
  constexpr int U = 2;
  const int b = blockIdx.y;
  const long base = (long)b * per_image8;
  const int i0 = blockIdx.x * (256 * U) + threadIdx.x;
  const int c8 = C >> 3;
  float4 v[U][2];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int i = i0 + u * 256;
    if (i < per_image8) { v[u][0] = __ldg(x + 2 * (base + i)); v[u][1] = __ldg(x + 2 * (base + i) + 1); }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int i = i0 + u * 256;
    if (i >= per_image8) break;
    float w[8] = {v[u][0].x, v[u][0].y, v[u][0].z, v[u][0].w, v[u][1].x, v[u][1].y, v[u][1].z, v[u][1].w};
    const int c = (i % c8) * 8;
    if (MODE == FEMASR_PRO_GN_SILU || MODE == FEMASR_PRO_GN_SILU_FAST) {
      const float4* ps = reinterpret_cast<const float4*>(sc + (long)b * C + c);
      const float4* pt = reinterpret_cast<const float4*>(sh + (long)b * C + c);
      const float4 s0 = __ldg(ps), s1 = __ldg(ps + 1), t0 = __ldg(pt), t1 = __ldg(pt + 1);
      const float ss[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      const float tt[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float n = fmaf(w[k], ss[k], tt[k]);
        w[k] = MODE == FEMASR_PRO_GN_SILU_FAST ? __fdividef(n, 1.0f + __expf(-n)) : silu_f(n);
      }
    }
    float l[8];
    uint32_t hp[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t lo_unused;
      const float a = fminf(fmaxf(w[2 * k], -65504.f), 65504.f), bq = fminf(fmaxf(w[2 * k + 1], -65504.f), 65504.f);
      asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hp[k]) : "f"(bq), "f"(a));
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hp[k]));
      l[2 * k] = (a - hf.x) * F8_LO_SCALE; l[2 * k + 1] = (bq - hf.y) * F8_LO_SCALE;
      w[2 * k] = a; w[2 * k + 1] = bq;
      (void)lo_unused;
    }
    hi[base + i] = make_uint4(hp[0], hp[1], hp[2], hp[3]);
    // byte layout of the pixel's x8 row: chunk (c / 64) * 128 + (c % 64) for the lo part, + 64 for the value part
    const long pix = (base + i) / c8;
    const long q = pix * (C >> 2) + (c >> 6) * 16 + ((c & 63) >> 3);          // index in 8-byte units
    x8[q] = make_uint2(pack_e4m3x4(l[0], l[1], l[2], l[3]), pack_e4m3x4(l[4], l[5], l[6], l[7]));
    x8[q + 8] = make_uint2(pack_e4m3x4(w[0] * F8_VAL_SCALE, w[1] * F8_VAL_SCALE, w[2] * F8_VAL_SCALE, w[3] * F8_VAL_SCALE),
                           pack_e4m3x4(w[4] * F8_VAL_SCALE, w[5] * F8_VAL_SCALE, w[6] * F8_VAL_SCALE, w[7] * F8_VAL_SCALE));
  }
}

// LayerNorm (C = 256, eps) fused with the split: one warp per token row.
__global__ void __launch_bounds__(256) tc_prepare_ln_kernel(const float* __restrict__ x, __half* __restrict__ hi,
                                                            __half* __restrict__ lo, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, long M, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  // two rows per warp, all four 512-byte requests of the warp in flight before the first reduction
  constexpr int LN_ROWS = 2;
  const long row0 = ((long)blockIdx.x * 8 + (threadIdx.x >> 5)) * LN_ROWS;
  if (row0 >= M) return;
  const int lane = threadIdx.x & 31;
  // lane owns columns [4 lane, 4 lane + 4) and [128 + 4 lane, ...): two fully coalesced 512-byte requests per row
  float4 a[LN_ROWS], b[LN_ROWS];
#pragma unroll
  for (int rr = 0; rr < LN_ROWS; ++rr) {
    if (row0 + rr < M) {
      const float4* r = reinterpret_cast<const float4*>(x + (row0 + rr) * 256) + lane;
      a[rr] = __ldg(r); b[rr] = __ldg(r + 32);
    }
  }
  const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + lane), g1 = __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32);
  const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta) + lane), b1 = __ldg(reinterpret_cast<const float4*>(beta) + lane + 32);
  const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
  const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
  for (int rr = 0; rr < LN_ROWS; ++rr) {
    const long row = row0 + rr;
    if (row >= M) break;
    float v[8] = {a[rr].x, a[rr].y, a[rr].z, a[rr].w, b[rr].x, b[rr].y, b[rr].z, b[rr].w};
    float s = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
    s = warp_sum(s);
    const float mu = s * (1.0f / 256.0f);
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { const float d = v[k] - mu; q = fmaf(d, d, q); }
    q = warp_sum(q) * (1.0f / 256.0f);
    const float rs = 1.0f / sqrtf(q + eps);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (v[k] - mu) * rs * g[k] + be[k];
    uint2 h0, l0, h1, l1;
    split_pack2(v[0], v[1], h0.x, l0.x); split_pack2(v[2], v[3], h0.y, l0.y);
    split_pack2(v[4], v[5], h1.x, l1.x); split_pack2(v[6], v[7], h1.y, l1.y);
    uint2* ph = reinterpret_cast<uint2*>(hi + row * 256) + lane;
    uint2* pl = reinterpret_cast<uint2*>(lo + row * 256) + lane;
    ph[0] = h0; ph[32] = h1;
    pl[0] = l0; pl[32] = l1;
  }
}

// weights: OIHW fp32 -> [Cout][taps*Cin] fp16 hi/lo planes of w * 2^s, s chosen so max|w|*2^s is in [512,1024)
__global__ void absmax_kernel(const float* __restrict__ w, unsigned int* __restrict__ out, long n) {
  float m = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));   // non-negative floats order like uints
}
__global__ void tc_pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ hi, __half* __restrict__ lo,
                                      const unsigned int* __restrict__ absmax, float* __restrict__ inv_scale, int Cout,
                                      int Cin, int KH, int KW) {
  const float mx = __uint_as_float(*absmax);
  int ex = 0;
  if (mx > 0.f) frexpf(mx, &ex);          // mx = f * 2^ex, f in [0.5,1)
  const int s = mx > 0.f ? 10 - ex : 0;   // mx * 2^s in [512, 1024)
  const float scale = ldexpf(1.0f, s);
  const long n = (long)Cout * Cin * KH * KW;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *inv_scale = ldexpf(1.0f, -s);
  if (i >= n) return;
  // i indexes the packed layout [co][(kh*KW+kw)*Cin + ci]
  const long K = (long)Cin * KH * KW;
  const int co = (int)(i / K);
  const long k = i - (long)co * K;
  const int tap = (int)(k / Cin), ci = (int)(k - (long)tap * Cin);
  const int kh = tap / KW, kw = tap - kh * KW;
  const float v = w[(((long)co * Cin + ci) * KH + kh) * KW + kw] * scale;   // exact (power of two)
  const __half h = __float2half_rn(v);
  hi[i] = h;
  lo[i] = __float2half_rn(v - __half2float(h));
}

// F8 variant of the packed weights: hi plane as above; the second plane holds per (row, 64-wide k chunk) 128 bytes =
// [e4m3(w_hi * 2^-10) x 64 | e4m3(w_lo * 2^2) x 64] (see tc_prepare_flat_f8_kernel)
__global__ void tc_pack_weight_f8_kernel(const float* __restrict__ w, __half* __restrict__ hi, uint8_t* __restrict__ x8,
                                         const unsigned int* __restrict__ absmax, float* __restrict__ inv_scale, int Cout,
                                         int Cin, int KH, int KW) {
  const float mx = __uint_as_float(*absmax);
  int ex = 0;
  if (mx > 0.f) frexpf(mx, &ex);
  const int s = mx > 0.f ? 10 - ex : 0;
  const float scale = ldexpf(1.0f, s);
  const long n = (long)Cout * Cin * KH * KW;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *inv_scale = ldexpf(1.0f, -s);
  if (i >= n) return;
  const long K = (long)Cin * KH * KW;
  const int co = (int)(i / K);
  const long k = i - (long)co * K;
  const int tap = (int)(k / Cin), ci = (int)(k - (long)tap * Cin);
  const int kh = tap / KW, kw = tap - kh * KW;
  const float v = w[(((long)co * Cin + ci) * KH + kh) * KW + kw] * scale;
  const __half h = __float2half_rn(v);
  hi[i] = h;
  const float hf = __half2float(h);
  uint8_t* row = x8 + (long)co * K * 2 + (k >> 6) * 128 + (k & 63);
  row[0] = (uint8_t)__nv_cvt_float_to_fp8(hf * (1.0f / F8_LO_SCALE), __NV_SATFINITE, __NV_E4M3);
  row[64] = (uint8_t)__nv_cvt_float_to_fp8((v - hf) * (1.0f / F8_VAL_SCALE), __NV_SATFINITE, __NV_E4M3);
}

// nearest-x2 upsample followed by a 3x3 conv == four 2x2 convs on the low-res grid (one per output phase
// (py,px)), whose weights are sums of the 3x3 taps that land on the same source pixel:
//   rows: py=0 -> {kh=0 | kh=1,2},  py=1 -> {kh=0,1 | kh=2};  same for columns.  2.25x fewer MACs.
// out: fp32 [4*Cout][Cin][2][2] (OIHW of the stacked phase filters), summed in a fixed order.
__global__ void subpixel_weights_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin) {
  const long n = (long)4 * Cout * Cin * 4;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int bq = (int)(i & 1), a = (int)((i >> 1) & 1);
  long r = i >> 2;
  const int ci = (int)(r % Cin); r /= Cin;
  const int co = (int)(r % Cout);
  const int ph = (int)(r / Cout);
  const int py = ph >> 1, px = ph & 1;
  const int kh0 = py == 0 ? (a == 0 ? 0 : 1) : (a == 0 ? 0 : 2), kh1 = py == 0 ? (a == 0 ? 0 : 2) : (a == 0 ? 1 : 2);
  const int kw0 = px == 0 ? (bq == 0 ? 0 : 1) : (bq == 0 ? 0 : 2), kw1 = px == 0 ? (bq == 0 ? 0 : 2) : (bq == 0 ? 1 : 2);
  const float* wp = w + ((long)co * Cin + ci) * 9;
  float sum = 0.f;
  for (int kh = kh0; kh <= kh1; ++kh)
    for (int kw = kw0; kw <= kw1; ++kw) sum += wp[kh * 3 + kw];
  out[i] = sum;
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int make_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                    const cuuint32_t* box, int spatial_stride = 1, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                    CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return fail(FEMASR_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint32_t estr[4] = {1, (cuuint32_t)spatial_stride, (cuuint32_t)spatial_stride, 1};
  if (rank == 2) estr[1] = 1;
  CUresult r = enc(m, dtype, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(FEMASR_ERR_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
  return FEMASR_OK;
}

// Launch with the programmatic-stream-serialisation attribute when FEMASR_PDL=1.  Only kernels that execute
// griddepcontrol.wait before their first dependent global access are launched this way.  Off by default: the persistent
// GEMM CTAs take a whole SM's shared memory and cannot become resident before the predecessor's CTAs retire anyway.
static bool pdl_enabled() {
  static const int env = [] { const char* e = getenv("FEMASR_PDL"); return e ? atoi(e) : 0; }();
  return env != 0;
}
template <class... KArgs, class... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int n = 0;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

template <int BN, bool RES, bool F8, bool VQ, int EXT = 0>
static int launch_tc_v(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                       const TcP& p, cudaStream_t st) {
  using Cfg = TcCfg<BN>;
  static PerDeviceFlag attr_set;      // per template instantiation AND per device
  if (!attr_set.cur()) {
    FEMASR_CUDA(cudaFuncSetAttribute(tc_igemm_kernel<BN, RES, F8, VQ, EXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set.cur() = true;
  }
  const int items = VQ ? p.num_tiles / p.n_tiles : p.num_tiles;     // VQ: one CTA walks all code tiles of an m-tile
  const int grid = items < sm_count() ? items : sm_count();
  FEMASR_CUDA(launch_pdl(tc_igemm_kernel<BN, RES, F8, VQ, EXT>, dim3(grid), dim3(TC_THREADS), Cfg::SMEM_BYTES, st, ah, al, bh, bl, p));
  return launch_status(VQ ? "tc_igemm_kernel(vq)" : "tc_igemm_kernel");
}

template <int BN>
static int launch_tc(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                     const TcP& p, cudaStream_t st) {
  if (p.f8) return p.res1 ? launch_tc_v<BN, true, true, false>(ah, al, bh, bl, p, st) : launch_tc_v<BN, false, true, false>(ah, al, bh, bl, p, st);
  if (p.taps == 25)
    return p.res1 ? launch_tc_v<BN, true, false, false, 2>(ah, al, bh, bl, p, st) : launch_tc_v<BN, false, false, false, 2>(ah, al, bh, bl, p, st);
  if (p.taps == 16 || p.act == FEMASR_ACT_LRELU)
    return p.res1 ? launch_tc_v<BN, true, false, false, 1>(ah, al, bh, bl, p, st) : launch_tc_v<BN, false, false, false, 1>(ah, al, bh, bl, p, st);
  return p.res1 ? launch_tc_v<BN, true, false, false>(ah, al, bh, bl, p, st) : launch_tc_v<BN, false, false, false>(ah, al, bh, bl, p, st);
}

}  // namespace femasr

using namespace femasr;

static void tc_tile_shape(int H, int W, int* Wt, int* Ht) {
  int best_wt = 8; long best_cost = -1;
  for (int wt = 128; wt >= 8; wt >>= 1) {
    const int ht = 128 / wt;
    const long cost = cdiv(W, wt) * wt * cdiv(H, ht) * ht;
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_wt = wt; }
  }
  *Wt = best_wt; *Ht = 128 / best_wt;
}

// Tiling decisions shared by femasr_tc_igemm and femasr_tc_gn_partial_rows.  (H, W) = the grid the tiles run over.
// 128-wide tiles where Cout allows (a 128 x 128 fp32 accumulator is 64 registers per consumer thread, which leaves room
// for the F8 cross-product / K-slice accumulator beside it), else 64-wide.  femasr_tc_args.pair / .strip select
// schedules of other GPU generations and do not change the tiling here.
struct TilePlan { int Wt, Ht, wt_shift, tiles_x, tiles_y, BN; };
static TilePlan plan_tiles(const femasr_tc_args* a, int H, int W) {
  TilePlan t;
  t.BN = a->Cout % 128 == 0 ? 128 : 64;
  tc_tile_shape(H, W, &t.Wt, &t.Ht);   // the widest power-of-two Wt <= 128 that wastes the fewest padded pixels
  t.wt_shift = 0; while ((1 << t.wt_shift) < t.Wt) ++t.wt_shift;
  t.tiles_x = (int)cdiv(W, t.Wt); t.tiles_y = (int)cdiv(H, t.Ht);
  return t;
}

// rows of GroupNorm partials femasr_tc_igemm will write per image for this conv (same decision logic as the launch)
extern "C" int femasr_tc_gn_partial_rows(const femasr_tc_args* a) {
  if (!a) return 0;
  int H = a->H, W = a->W;
  if (a->stride == 2) { H = (H + 2 - a->ksize) / 2 + 1; W = (W + 2 - a->ksize) / 2 + 1; }
  const TilePlan t = plan_tiles(a, H, W);
  return (a->upsample ? 4 : 1) * t.tiles_x * t.tiles_y * 4;
}

extern "C" size_t femasr_tc_weight_bytes(int Cout, int Cin, int kh, int kw) {
  return (size_t)2 * Cout * Cin * kh * kw * sizeof(__half) + 256;   // hi plane, lo plane, then {absmax, inv_scale}
}

// Layout of the packed tensor-core weight blob: [hi plane][lo plane | F8: interleaved e4m3 plane][uint absmax][float inv_scale].
static int tc_pack_weight_impl(const float* w_oihw, void* blob, int Cout, int Cin, int kh, int kw, bool f8, void* stream) {
  FEMASR_CHECK_ARG(w_oihw && blob && Cout > 0 && Cin > 0 && kh > 0 && kw > 0, "tc_pack_weight: bad argument");
  FEMASR_CHECK_ARG(!f8 || Cin % 64 == 0, "tc_pack_weight_f8: Cin must be a multiple of 64");
  const long n = (long)Cout * Cin * kh * kw;
  __half* hi = reinterpret_cast<__half*>(blob);
  __half* lo = hi + n;
  unsigned int* amax = reinterpret_cast<unsigned int*>(lo + n);
  float* inv = reinterpret_cast<float*>(amax + 1);
  cudaStream_t st = as_stream(stream);
  FEMASR_CUDA(cudaMemsetAsync(amax, 0, 8, st));
  absmax_kernel<<<(unsigned)std::min<long>(cdiv(n, 256), 1024), 256, 0, st>>>(w_oihw, amax, n);
  int s = launch_status("absmax_kernel");
  if (s) return s;
  if (f8) {
    tc_pack_weight_f8_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(w_oihw, hi, reinterpret_cast<uint8_t*>(lo), amax, inv, Cout, Cin, kh, kw);
    return launch_status("tc_pack_weight_f8_kernel");
  }
  tc_pack_weight_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(w_oihw, hi, lo, amax, inv, Cout, Cin, kh, kw);
  return launch_status("tc_pack_weight_kernel");
}
extern "C" int femasr_tc_pack_weight(const float* w_oihw, void* blob, int Cout, int Cin, int kh, int kw, void* stream) {
  return tc_pack_weight_impl(w_oihw, blob, Cout, Cin, kh, kw, false, stream);
}
extern "C" int femasr_tc_pack_weight_f8(const float* w_oihw, void* blob, int Cout, int Cin, int kh, int kw, void* stream) {
  return tc_pack_weight_impl(w_oihw, blob, Cout, Cin, kh, kw, true, stream);
}

// Packed phase filters for the fused upsample+conv: a blob like femasr_tc_pack_weight's for the stacked
// [4*Cout][Cin][2][2] filter bank (femasr_tc_weight_bytes(4*Cout, Cin, 2, 2) bytes).
static int tc_pack_weight_up2_impl(const float* w_oihw, void* blob, int Cout, int Cin, bool f8, void* stream) {
  FEMASR_CHECK_ARG(w_oihw && blob && Cout > 0 && Cin > 0, "tc_pack_weight_up2: bad argument");
  cudaStream_t st = as_stream(stream);
  float* tmp = nullptr;
  const long n = (long)16 * Cout * Cin;
  FEMASR_CUDA(cudaMallocAsync(&tmp, n * sizeof(float), st));
  subpixel_weights_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(w_oihw, tmp, Cout, Cin);
  int s = launch_status("subpixel_weights_kernel");
  if (!s) s = tc_pack_weight_impl(tmp, blob, 4 * Cout, Cin, 2, 2, f8, stream);
  cudaFreeAsync(tmp, st);
  return s;
}
extern "C" int femasr_tc_pack_weight_up2(const float* w_oihw, void* blob, int Cout, int Cin, void* stream) {
  return tc_pack_weight_up2_impl(w_oihw, blob, Cout, Cin, false, stream);
}
extern "C" int femasr_tc_pack_weight_up2_f8(const float* w_oihw, void* blob, int Cout, int Cin, void* stream) {
  return tc_pack_weight_up2_impl(w_oihw, blob, Cout, Cin, true, stream);
}

// F8 operand staging (see tc_prepare_flat_f8_kernel): modes NONE / GN_SILU / GN_SILU_FAST, no replication
extern "C" int femasr_tc_prepare_f8(const float* x, void* a_hi, void* a_x8, int mode, const float* pro_a, const float* pro_b,
                                    int B, int H, int W, int C, void* stream) {
  FEMASR_CHECK_ARG(x && a_hi && a_x8 && B > 0 && H > 0 && W > 0, "tc_prepare_f8: bad argument");
  FEMASR_CHECK_ARG(C % 64 == 0, "tc_prepare_f8: C must be a multiple of 64");
  FEMASR_CHECK_ARG((long)H * W * (C / 4) < (1l << 30) && B <= 65535, "tc_prepare_f8: tensor too large for the flat kernel");
  cudaStream_t st = as_stream(stream);
  const int per8 = H * W * (C / 8);
  const dim3 grid((unsigned)cdiv(per8, 256 * 2), (unsigned)B);
  const float4* x4 = reinterpret_cast<const float4*>(x);
  uint4* hi = reinterpret_cast<uint4*>(a_hi);
  uint2* x8 = reinterpret_cast<uint2*>(a_x8);
  if (mode == FEMASR_PRO_GN_SILU || mode == FEMASR_PRO_GN_SILU_FAST) {
    FEMASR_CHECK_ARG(pro_a && pro_b, "tc_prepare_f8: GN mode needs the scale/shift tables");
    if (mode == FEMASR_PRO_GN_SILU) tc_prepare_flat_f8_kernel<FEMASR_PRO_GN_SILU><<<grid, 256, 0, st>>>(x4, hi, x8, pro_a, pro_b, C, per8);
    else tc_prepare_flat_f8_kernel<FEMASR_PRO_GN_SILU_FAST><<<grid, 256, 0, st>>>(x4, hi, x8, pro_a, pro_b, C, per8);
  } else if (mode == FEMASR_PRO_NONE) {
    tc_prepare_flat_f8_kernel<FEMASR_PRO_NONE><<<grid, 256, 0, st>>>(x4, hi, x8, nullptr, nullptr, C, per8);
  } else {
    return fail(FEMASR_ERR_ARG, "tc_prepare_f8: bad mode");
  }
  return launch_status("tc_prepare_flat_f8_kernel");
}

extern "C" int femasr_tc_prepare(const float* x, void* a_hi, void* a_lo, int mode, const float* pro_a, const float* pro_b,
                                 const float* gamma, const float* beta, int B, int H, int W, int C, int upsample,
                                 float eps, void* stream) {
  FEMASR_CHECK_ARG(x && a_hi && a_lo && B > 0 && H > 0 && W > 0, "tc_prepare: bad argument");
  FEMASR_CHECK_ARG(C % 8 == 0, "tc_prepare: C must be a multiple of 8");
  cudaStream_t st = as_stream(stream);
  __half* hi = reinterpret_cast<__half*>(a_hi);
  __half* lo = reinterpret_cast<__half*>(a_lo);
  if (mode == FEMASR_PRO_LN) {
    FEMASR_CHECK_ARG(C == 256 && gamma && beta && !upsample, "tc_prepare: LN mode needs C=256, gamma/beta, no upsample");
    const long M = (long)B * H * W;
    FEMASR_CUDA(launch_pdl(tc_prepare_ln_kernel, dim3((unsigned)cdiv(M, 16)), dim3(256), 0, st, x, hi, lo, gamma, beta, M, eps));
    return launch_status("tc_prepare_ln_kernel");
  }
  if (mode == FEMASR_PRO_MAXPOOL2) {
    FEMASR_CHECK_ARG(!upsample && H >= 2 && W >= 2, "tc_prepare: max-pool mode needs H, W >= 2 and no upsample");
    const long total8 = (long)B * (H / 2) * (W / 2) * (C / 8);
    tc_prepare_pool_kernel<2><<<(unsigned)cdiv(total8, 256), 256, 0, st>>>(x, hi, lo, H, W, C, total8);
    return launch_status("tc_prepare_pool_kernel");
  }
  if (mode == FEMASR_PRO_MAXPOOL3S2) {
    FEMASR_CHECK_ARG(!upsample && H >= 3 && W >= 3, "tc_prepare: 3x3 max-pool mode needs H, W >= 3 and no upsample");
    const long total8 = (long)B * ((H - 3) / 2 + 1) * ((W - 3) / 2 + 1) * (C / 8);
    tc_prepare_pool_kernel<3><<<(unsigned)cdiv(total8, 256), 256, 0, st>>>(x, hi, lo, H, W, C, total8);
    return launch_status("tc_prepare_pool_kernel");
  }
  if (mode == FEMASR_PRO_BILINEAR2) {
    FEMASR_CHECK_ARG(!upsample, "tc_prepare: bilinear mode has its own x2 (upsample must be 0)");
    const long total8 = (long)B * 2 * H * 2 * W * (C / 8);
    tc_prepare_bilinear_kernel<<<(unsigned)cdiv(total8, 256), 256, 0, st>>>(x, hi, lo, H, W, C, total8);
    return launch_status("tc_prepare_bilinear_kernel");
  }
  static const int flat_env = [] { const char* e = getenv("FEMASR_PREP_FLAT"); return e ? atoi(e) : 1; }();
  if (!upsample && flat_env && (long)H * W * (C / 4) < (1l << 30) && B <= 65535 &&
      (mode == FEMASR_PRO_GN_SILU || mode == FEMASR_PRO_GN_SILU_FAST || mode == FEMASR_PRO_NONE)) {
    const int per4 = H * W * (C / 4);
    const dim3 grid((unsigned)cdiv(per4, 256 * PREP_U), (unsigned)B);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    if (mode == FEMASR_PRO_GN_SILU) {
      FEMASR_CHECK_ARG(pro_a && pro_b, "tc_prepare: GN mode needs the scale/shift tables");
      FEMASR_CUDA(launch_pdl(tc_prepare_flat_kernel<FEMASR_PRO_GN_SILU>, grid, dim3(256), 0, st, x4, reinterpret_cast<uint2*>(hi), reinterpret_cast<uint2*>(lo), pro_a, pro_b, C, per4));
    } else if (mode == FEMASR_PRO_GN_SILU_FAST) {
      FEMASR_CHECK_ARG(pro_a && pro_b, "tc_prepare: GN mode needs the scale/shift tables");
      FEMASR_CUDA(launch_pdl(tc_prepare_flat_kernel<FEMASR_PRO_GN_SILU_FAST>, grid, dim3(256), 0, st, x4, reinterpret_cast<uint2*>(hi), reinterpret_cast<uint2*>(lo), pro_a, pro_b, C, per4));
    } else {
      FEMASR_CUDA(launch_pdl(tc_prepare_flat_kernel<FEMASR_PRO_NONE>, grid, dim3(256), 0, st, x4, reinterpret_cast<uint2*>(hi), reinterpret_cast<uint2*>(lo), (const float*)nullptr, (const float*)nullptr, C, per4));
    }
    return launch_status("tc_prepare_flat_kernel");
  }
  const long total8 = (long)B * H * W * (C / 8);
  const unsigned grid = (unsigned)cdiv(total8, 256);
  if (mode == FEMASR_PRO_GN_SILU_FAST) mode = FEMASR_PRO_GN_SILU;     // replicating variant: exact SiLU only
  if (mode == FEMASR_PRO_GN_SILU) {
    FEMASR_CHECK_ARG(pro_a && pro_b, "tc_prepare: GN mode needs the scale/shift tables");
    tc_prepare_kernel<FEMASR_PRO_GN_SILU><<<grid, 256, 0, st>>>(x, hi, lo, pro_a, pro_b, H, W, C, upsample, total8);
  } else if (mode == FEMASR_PRO_NONE) {
    tc_prepare_kernel<FEMASR_PRO_NONE><<<grid, 256, 0, st>>>(x, hi, lo, nullptr, nullptr, H, W, C, upsample, total8);
  } else {
    return fail(FEMASR_ERR_ARG, "tc_prepare: bad mode");
  }
  return launch_status("tc_prepare_kernel");
}

// VectorQuantizer distance stage on the tensor cores (femasr_arch.py:35-38, 63-66): for every feature row the four
// smallest d_j = fl(fl(A + B_j) - 2 z.e_j) with their codes, ascending in (d, j); the [N, n_e] product never leaves the SM.
extern "C" int femasr_vq_match_tc(const void* z_hi, const void* z_lo, const void* cb_blob, const float* a, const float* esq,
                                  void* cand, int N, int n_e, int e_dim, void* stream) {
  FEMASR_CHECK_ARG(z_hi && z_lo && cb_blob && a && esq && cand, "vq_match_tc: null pointer");
  FEMASR_CHECK_ARG(N > 0 && n_e > 0 && e_dim > 0 && n_e % 64 == 0 && e_dim % 64 == 0, "vq_match_tc: n_e and e_dim must be positive multiples of 64");
  const long nw = (long)n_e * e_dim;
  const __half* w_hi = reinterpret_cast<const __half*>(cb_blob);
  const __half* w_lo = w_hi + nw;
  TcP p;
  memset(&p, 0, sizeof(p));
  p.inv_scale = reinterpret_cast<const float*>(reinterpret_cast<const unsigned int*>(w_lo + nw) + 1);
  p.vq_a = a; p.vq_esq = esq; p.vq_cand = reinterpret_cast<uint2*>(cand);
  p.B = 1; p.H = 1; p.W = N; p.Cin = e_dim; p.Cout = n_e; p.taps = 1; p.stride = 1;
  p.Wt = 128; p.Ht = 1; p.wt_shift = 7; p.tiles_x = (int)cdiv(N, 128); p.tiles_y = 1;
  const int BN = n_e % 128 == 0 ? 128 : 64;
  p.n_tiles = n_e / BN;
  p.num_tiles = p.tiles_x * p.n_tiles; p.cchunks = e_dim / 64;
  p.kb_begin = 0; p.kb_end = p.cchunks; p.cpg = 1;
  CUtensorMap mah, mal, mbh, mbl;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)e_dim, (cuuint64_t)N, 1, 1};
    const cuuint64_t str[3] = {(cuuint64_t)e_dim * 2, (cuuint64_t)N * e_dim * 2, (cuuint64_t)N * e_dim * 2};
    const cuuint32_t box[4] = {64, 128, 1, 1};
    int s = make_map(&mah, z_hi, 4, dims, str, box);
    if (s) return s;
    s = make_map(&mal, z_lo, 4, dims, str, box);
    if (s) return s;
  }
  {
    const cuuint64_t dims[2] = {(cuuint64_t)e_dim, (cuuint64_t)n_e};
    const cuuint64_t str[1] = {(cuuint64_t)e_dim * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)BN};
    int s = make_map(&mbh, w_hi, 2, dims, str, box);
    if (s) return s;
    s = make_map(&mbl, w_lo, 2, dims, str, box);
    if (s) return s;
  }
  cudaStream_t st = as_stream(stream);
  if (BN == 128) return launch_tc_v<128, false, false, true>(mah, mal, mbh, mbl, p, st);
  return launch_tc_v<64, false, false, true>(mah, mal, mbh, mbl, p, st);
}

// y = act(conv(a) + bias) + res1 + res2 with a given as fp16 hi/lo planes at the conv-input resolution.
extern "C" int femasr_tc_igemm(const femasr_tc_args* a, void* stream) {
  FEMASR_CHECK_ARG(a && a->a_hi && a->a_lo && a->w_blob, "tc_igemm: null pointer");
  FEMASR_CHECK_ARG(a->y || (a->out_hi && a->out_lo), "tc_igemm: need y or the out_hi/out_lo planes");
  FEMASR_CHECK_ARG(!a->out_hi == !a->out_lo, "tc_igemm: out_hi and out_lo go together");
  FEMASR_CHECK_ARG(a->B > 0 && a->H > 0 && a->W > 0, "tc_igemm: empty input");
  FEMASR_CHECK_ARG(a->ksize == 1 || a->ksize == 3 || a->ksize == 4 || a->ksize == 5, "tc_igemm: ksize must be 1, 3, 4 or 5");
  FEMASR_CHECK_ARG(!a->upsample || a->ksize == 3, "tc_igemm: upsample fusion needs ksize 3 (and an up2 weight blob)");
  FEMASR_CHECK_ARG(a->Cin % 64 == 0 && a->Cout % 64 == 0, "tc_igemm: Cin and Cout must be multiples of 64");
  int B = a->B, H = a->H, W = a->W;
  const int stride = a->stride == 2 ? 2 : 1;
  FEMASR_CHECK_ARG(a->stride >= 0 && a->stride <= 2, "tc_igemm: stride must be 1 or 2");
  FEMASR_CHECK_ARG(stride == 1 || (a->ksize != 1 && !a->upsample), "tc_igemm: stride 2 needs a plain 3x3 or 4x4 conv");
  FEMASR_CHECK_ARG(a->ksize != 4 || stride == 2, "tc_igemm: ksize 4 needs stride 2");
  FEMASR_CHECK_ARG(a->ksize != 4 || (H >= 2 && W >= 2), "tc_igemm: a 4x4 stride-2 conv needs H, W >= 2");
  FEMASR_CHECK_ARG(a->ksize != 5 || (stride == 1 && !a->upsample), "tc_igemm: ksize 5 (pad 2) needs stride 1, no upsample");
  // the 5x5 instantiations (EXT = 2) carry no LeakyReLU epilogue: refused rather than returned without the activation
  FEMASR_CHECK_ARG(a->ksize != 5 || a->act != FEMASR_ACT_LRELU, "tc_igemm: no LeakyReLU epilogue for ksize 5");
  if (a->ksize == 1) { W = B * H * W; H = 1; B = 1; }     // pointwise: one long row of tokens
  const int Hin = H, Win = W;                             // activation-plane dims
  if (stride == 2) { H = (H + 2 - a->ksize) / 2 + 1; W = (W + 2 - a->ksize) / 2 + 1; }   // tiles run over the output grid
  FEMASR_CHECK_ARG((long)W < (1l << 31), "tc_igemm: too many rows");
  const int taps = a->upsample ? 4 : a->ksize * a->ksize;
  const int phases = a->upsample ? 4 : 1;
  const long Ktot = (long)taps * a->Cin;
  const long nw = (long)phases * a->Cout * Ktot;
  const __half* w_hi = reinterpret_cast<const __half*>(a->w_blob);
  const __half* w_lo = w_hi + nw;
  const float* inv_scale = reinterpret_cast<const float*>(reinterpret_cast<const unsigned int*>(w_lo + nw) + 1);

  TcP p;
  memset(&p, 0, sizeof(p));
  p.bias = a->bias; p.res1 = a->res1; p.res2 = a->res2; p.y = a->y; p.inv_scale = inv_scale;
  p.out_hi = reinterpret_cast<__half*>(a->out_hi); p.out_lo = reinterpret_cast<__half*>(a->out_lo);
  p.gn_partial = a->gn_partial; p.cpg = a->Cout / 32; p.gn_rows = 0;
  FEMASR_CHECK_ARG(!a->gn_partial || (a->ksize == 3 && (a->Cout == 64 || a->Cout == 128 || a->Cout == 256)),
                   "tc_igemm: gn_partial needs a 3x3 conv with Cout in {64,128,256}");
  p.B = B; p.H = H; p.W = W; p.Cin = a->Cin; p.Cout = a->Cout; p.taps = taps; p.act = a->act;
  p.up = a->upsample ? 1 : 0; p.stride = stride;
  p.f8 = a->f8 ? 1 : 0;
  FEMASR_CHECK_ARG(!a->f8 || a->slice_kb == 0, "tc_igemm: the F8 cross-term mode is for the layers behind the VQ (no K slicing)");
  FEMASR_CHECK_ARG(!a->f8 || (a->ksize != 4 && a->ksize != 5 && a->act != FEMASR_ACT_LRELU),
                   "tc_igemm: no F8 cross-term mode for 4x4 / 5x5 convs or LeakyReLU");
  const TilePlan plan = plan_tiles(a, H, W);
  p.Wt = plan.Wt; p.Ht = plan.Ht; p.wt_shift = plan.wt_shift; p.tiles_x = plan.tiles_x; p.tiles_y = plan.tiles_y;
  const int BN = plan.BN;
  p.n_tiles = a->Cout / BN;
  p.gn_rows = phases * p.tiles_x * p.tiles_y * 4;           // one partial row per (128-pixel tile, 32-row quarter)
  const long ntile = (long)phases * B * p.tiles_x * p.tiles_y * p.n_tiles;
  FEMASR_CHECK_ARG(ntile < (1l << 31), "tc_igemm: too many tiles");
  p.num_tiles = (int)ntile; p.cchunks = a->Cin / 64;
  const int nkb_total = taps * p.cchunks;
  p.kb_begin = a->kb_begin; p.kb_end = a->kb_count > 0 ? a->kb_begin + a->kb_count : nkb_total;
  FEMASR_CHECK_ARG(p.kb_begin >= 0 && p.kb_begin < p.kb_end && p.kb_end <= nkb_total, "tc_igemm: bad k-block slice");
  FEMASR_CHECK_ARG(a->slice_kb >= 0, "tc_igemm: slice_kb must be >= 0");
  p.slice_kb = (a->slice_kb > 0 && a->slice_kb < p.kb_end - p.kb_begin) ? a->slice_kb : 0;

  CUtensorMap mah, mal, mbh, mbl;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)a->Cin, (cuuint64_t)Win, (cuuint64_t)Hin, (cuuint64_t)B};
    const cuuint64_t str[3] = {(cuuint64_t)a->Cin * 2, (cuuint64_t)Win * a->Cin * 2, (cuuint64_t)Hin * Win * a->Cin * 2};
    // with a traversal stride s the box spans s*Wt x s*Ht source pixels and lands Wt x Ht of them in smem
    const cuuint32_t box[4] = {64, (cuuint32_t)(p.Wt * stride), (cuuint32_t)(p.Ht * stride), 1};
    int s = make_map(&mah, a->a_hi, 4, dims, str, box, stride);
    if (s) return s;
    s = make_map(&mal, a->a_lo, 4, dims, str, box, stride);
    if (s) return s;
  }
  {
    const cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)phases * a->Cout};
    const cuuint64_t str[1] = {(cuuint64_t)Ktot * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)BN};
    int s = make_map(&mbh, w_hi, 2, dims, str, box);
    if (s) return s;
    s = make_map(&mbl, w_lo, 2, dims, str, box);
    if (s) return s;
  }
  cudaStream_t st = as_stream(stream);
  if (BN == 128) return launch_tc<128>(mah, mal, mbh, mbl, p, st);
  return launch_tc<64>(mah, mal, mbh, mbl, p, st);
}
