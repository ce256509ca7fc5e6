// Host-side engine: the FeMaSRNet inference graph (femasr_arch.py:311-385) as a fixed kernel sequence
// over a caller-provided device workspace.  No arithmetic happens here; every step is one of the
// exported operator kernels.  The graph is data-independent, so one forward = one launch list that a
// caller may capture in a CUDA graph.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include <cuda_fp16.h>

#include "common.cuh"

namespace femasr {

static thread_local std::string g_err;
thread_local long g_launches = 0;
void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) { g_err = msg; return code; }

// ---------------------------------------------------------------------------------------------
// Offset allocator over the workspace (first fit + coalescing).  Deterministic, so a dry run with
// base == nullptr yields the exact high-water mark the real run needs.
struct Arena {
  struct Blk { size_t off, size; bool free; };
  std::vector<Blk> blks;
  char* base = nullptr;
  size_t top = 0, peak = 0, cap = 0;
  bool dry = true;
  bool overflow = false;      // real run only: an allocation ran past the caller's workspace (sizing bug) - never launch on it
  static size_t align(size_t n) { return (n + 255) & ~size_t(255); }
  size_t alloc_off(size_t bytes) {
    bytes = align(std::max<size_t>(bytes, 256));
    for (size_t i = 0; i < blks.size(); ++i) {
      if (blks[i].free && blks[i].size >= bytes) {
        if (blks[i].size > bytes) {
          Blk rest{blks[i].off + bytes, blks[i].size - bytes, true};
          blks[i].size = bytes;
          blks.insert(blks.begin() + i + 1, rest);
        }
        blks[i].free = false;
        return blks[i].off;
      }
    }
    Blk b{top, bytes, false};
    blks.push_back(b);
    top += bytes;
    peak = std::max(peak, top);
    if (!dry && top > cap) overflow = true;
    return b.off;
  }
  float* alloc(size_t nfloats) {
    size_t off = alloc_off(nfloats * sizeof(float));
    return reinterpret_cast<float*>(base + off);   // only dereferenced when !dry
  }
  void release(const void* p) {
    size_t off = (size_t)(reinterpret_cast<const char*>(p) - base);
    for (size_t i = 0; i < blks.size(); ++i) {
      if (blks[i].off == off && !blks[i].free) {
        blks[i].free = true;
        if (i + 1 < blks.size() && blks[i + 1].free) { blks[i].size += blks[i + 1].size; blks.erase(blks.begin() + i + 1); }
        if (i > 0 && blks[i - 1].free) { blks[i - 1].size += blks[i].size; blks.erase(blks.begin() + i); }
        while (!blks.empty() && blks.back().free) { top = blks.back().off; blks.pop_back(); }
        return;
      }
    }
  }
};


// The device forms femasr_net_set_param packs a parameter into, besides its fp32 copy in the reference layout.  The spec
// decides them once from the layer's role and the net's configuration; the graph reads the same flags.
constexpr unsigned
  FORM_KMAJOR = 1u << 0,   // K-major fp32 GEMM operand (conv / linear weight; codebook^T): the SIMT GEMM's weight
  FORM_TC = 1u << 1,       // split-fp16 blob: the tensor-core GEMM's weight (codebook: the fused VQ's B operand)
  FORM_TC8 = 1u << 2,      // the same in the F8 cross-term packing (3x3 convs that may run behind the VQ)
  FORM_UP = 1u << 3,       // sub-pixel phase filters of a nearest-x2 -> conv3x3 site, split fp16
  FORM_UP8 = 1u << 4,      // the same in the F8 packing
  FORM_IM2COL = 1u << 5,   // [Cout][kpad] zero-padded im2col matrix (in_conv, VGG conv1_1, AlexNet conv1; kpad = im2col_k):
                           // split-fp16 blob on gemm_path 1, K-major fp32 on gemm_path 0
  FORM_RELB = 1u << 6,     // rel-pos table expanded to [8][64][64] (SIMT attention) and in the mma kernel's fragment order
  FORM_ESQ = 1u << 7;      // sum e^2 per codebook row

struct ParamInfo {
  size_t numel;
  int Cout, Cin, k;   // conv / linear weight [Cout,Cin,k,k]; codebook [n_e,e_dim] as Cout, Cin, k = 1
  unsigned forms;     // FORM_*
  std::string sn;     // spectral-norm layer this tensor belongs to (weight_orig / weight_u / weight_v), else empty
};

// every device buffer of one parameter; nullptr where its ParamInfo lists no such form
struct DevParam {
  float* raw = nullptr;        // fp32 copy in the reference layout
  float* packed = nullptr;     // FORM_KMAJOR, or the expanded rel bias of FORM_RELB
  float* relb_mma = nullptr;   // FORM_RELB, fragment order
  float* esq = nullptr;        // FORM_ESQ
  void *tc = nullptr, *tc8 = nullptr, *up = nullptr, *up8 = nullptr, *im2col = nullptr;
  float* sigma = nullptr;      // spectral-norm weight_orig: {u . (W v), |W v|} (femasr_spectral_sigma); the forms above
  float sn[2] = {0.f, 0.f};    // are packed from weight_orig / sigma.  sn: the same two values on the host
  void release() { for (void* p : {(void*)raw, (void*)packed, (void*)relb_mma, (void*)esq, tc, tc8, up, up8, im2col, (void*)sigma}) cudaFree(p); }
};

struct Tap { float* dst; size_t cap; };

struct ProfRec { const char* name; double flops; cudaEvent_t e0, e1; };

}  // namespace femasr

using namespace femasr;

struct femasr_net {
  femasr_net_config cfg;
  int depth;   // encode depth (1 for x4, 2 for x2, 3 for the HQ autoencoder)
  bool hq = false;   // scale_factor 1: LQ_stage=False graph (no Swin, no up branches, no skip adds)
  std::map<std::string, ParamInfo> spec;
  std::map<std::string, DevParam> dev;
  struct Codebook { int scale, n_e, e_dim; };
  std::vector<Codebook> cbs;              // codebook_params rows; cbs[0].scale == 32
  int level_cb[3] = {0, -1, -1};          // decoder level i (resolution 32 << i) -> codebook index or -1
  int last_q_level = 0;                   // last decoder level that quantises (everything before it is index-critical)
  std::map<std::string, Tap> taps;
  int last_launches = 0;
  bool profile = false;
  bool tc_precise = true;                 // K-sliced fp32 accumulation for the layers in front of the VQ
  bool f8_cross = true;                   // layers behind the VQ: the two cross products of the split as one fp8 product (FEMASR_F8_CROSS=0: three fp16 products)
  int tc_slice_kb = 4;                    // K-slice length in 64-wide k-blocks (FEMASR_TC_SLICE_KB; study knob)
  bool vq_fused = true;                   // VQ distances on the tensor cores with the argmin fused (FEMASR_VQ_FUSED=0: fp32 SIMT z.E^T + vq_select)
  bool fast_silu = true;                  // approximate-unit SiLU in the operand staging behind the VQ (FEMASR_FAST_SILU=0: exact)
  bool semantic = false;                  // femasr_net_enable_semantic: the VGG19 / conv_semantic tensors are part of the spec
  int sem_slice_kb = 0;                   // K-slice length of the semantic branch's GEMMs (FEMASR_SEM_SLICE_KB; study knob, 0 = one pass)
  bool disc = false;                      // femasr_disc_create: a UNetDiscriminatorSN (dcfg); cfg holds only gemm_path
  femasr_disc_config dcfg{};
  bool lpips = false;                     // femasr_lpips_create: an LPIPS metric (lcfg); cfg holds only gemm_path
  femasr_lpips_config lcfg{};
  std::vector<ProfRec> prof;
  std::string prof_json;
  ~femasr_net() {
    for (auto& r : prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    for (auto& kv : dev) kv.second.release();
  }
};

namespace femasr {

// the generator's entry points refuse the discriminator and LPIPS handles
static bool generator(const femasr_net* n) { return !n->disc && !n->lpips; }

// width of the zero-padded im2col rows of a 3-channel first conv with k x k taps (3 k^2 values): 64, or 384 for
// AlexNet's 11x11 conv1
static int im2col_k(int k) { return k == 11 ? 384 : 64; }

static int chan(int res) {
  switch (res) { case 8: case 16: case 32: case 64: return 256; case 128: return 128; case 256: return 64; case 512: return 32; }
  return -1;
}

// DISC_CONV: a discriminator conv (spectral-norm 3x3 or 4x4 stride 2), never F8
enum Role { CONV, UP_CONV, IN_CONV, VGG_CONV, VGG_CONV1, DISC_CONV };

static unsigned weight_forms(const femasr_net* n, Role r, int ci, int co, int k) {
  const bool tc = n->cfg.gemm_path == 1;
  if (r == VGG_CONV1 || (r == IN_CONV && tc)) return FORM_KMAJOR | FORM_IM2COL;   // K = 27 / 48 -> 64, 363 -> 384
  if (!tc || (k != 1 && k != 3 && k != 4 && k != 5) || ci % 64 || co % 64) return FORM_KMAJOR;
  unsigned f = FORM_KMAJOR | FORM_TC;
  if (n->f8_cross && k == 3 && r != VGG_CONV && r != DISC_CONV) f |= FORM_TC8;   // may run behind the VQ; the VGG and
                                                                                  // discriminator convs never use F8
  if (r == UP_CONV) f |= FORM_UP | (n->f8_cross ? FORM_UP8 : 0);
  return f;
}
static void add_conv(femasr_net* n, const std::string& p, int ci, int co, int k, Role r = CONV) {
  n->spec[p + ".weight"] = ParamInfo{(size_t)co * ci * k * k, co, ci, k, weight_forms(n, r, ci, co, k)};
  n->spec[p + ".bias"] = ParamInfo{(size_t)co, 0, 0, 0, 0};
}
static void add_vec(femasr_net* n, const std::string& name, size_t c) { n->spec[name] = ParamInfo{c, 0, 0, 0, 0}; }
static void add_resblock(femasr_net* n, const std::string& p, int c) {
  add_vec(n, p + ".conv.0.norm.weight", c); add_vec(n, p + ".conv.0.norm.bias", c);
  add_conv(n, p + ".conv.2", c, c, 3);
  add_vec(n, p + ".conv.3.norm.weight", c); add_vec(n, p + ".conv.3.norm.bias", c);
  add_conv(n, p + ".conv.5", c, c, 3);
}
// nearest-x2 -> conv3x3 (p.1) -> ResBlock (p.2) -> ResBlock (p.3): femasr_arch.py:168-180, 195-211
static void add_up_block(femasr_net* n, const std::string& p, int ci, int co) {
  add_conv(n, p + ".1", ci, co, 3, UP_CONV);
  add_resblock(n, p + ".2", co);
  add_resblock(n, p + ".3", co);
}

static void build_spec(femasr_net* n) {
  const int scale = n->cfg.scale_factor;
  const int d = n->depth;
  int res = 256 / scale;
  const std::string enc = "multiscale_encoder";
  add_conv(n, enc + ".in_conv", n->cfg.in_channel, chan(res), 4, IN_CONV);
  for (int i = 0; i < d; ++i) {
    const std::string b = enc + ".blocks." + std::to_string(i);
    add_conv(n, b + ".0", chan(res), chan(res / 2), 3);
    add_resblock(n, b + ".1", chan(res / 2));
    add_resblock(n, b + ".2", chan(res / 2));
    res /= 2;
  }
  const std::string sw = enc + ".blocks." + std::to_string(d) + ".swin_blks.";
  for (int r = 0; r < (n->hq ? 0 : 4); ++r) {
    for (int b = 0; b < 6; ++b) {
      const std::string p = sw + std::to_string(r) + ".residual_group.blocks." + std::to_string(b);
      add_vec(n, p + ".norm1.weight", 256); add_vec(n, p + ".norm1.bias", 256);
      n->spec[p + ".attn.relative_position_bias_table"] = ParamInfo{225 * 8, 0, 0, 0, FORM_RELB};
      add_conv(n, p + ".attn.qkv", 256, 768, 1);
      add_conv(n, p + ".attn.proj", 256, 256, 1);
      add_vec(n, p + ".norm2.weight", 256); add_vec(n, p + ".norm2.bias", 256);
      add_conv(n, p + ".mlp.fc1", 256, 1024, 1);
      add_conv(n, p + ".mlp.fc2", 1024, 256, 1);
    }
    add_conv(n, sw + std::to_string(r) + ".conv", 256, 256, 3);
  }
  for (int j = d + 1; j <= (n->hq ? d : d + 2); ++j) {
    add_up_block(n, enc + ".blocks." + std::to_string(j), chan(res), chan(res * 2));
    res *= 2;
  }
  for (int i = 0; i < 3; ++i) add_up_block(n, "decoder_group." + std::to_string(i) + ".block", chan(32 << i), chan(64 << i));
  add_conv(n, "out_conv", 64, 3, 3);
  const unsigned cb_forms = FORM_KMAJOR | FORM_ESQ | (n->cfg.gemm_path == 1 && n->vq_fused ? FORM_TC : 0);
  for (size_t k = 0; k < n->cbs.size(); ++k) {           // femasr_arch.py:280-299
    const femasr_net::Codebook& cb = n->cbs[k];
    const std::string ks = std::to_string(k);
    const int ch = chan(cb.scale);
    n->spec["quantize_group." + ks + ".embedding.weight"] = ParamInfo{(size_t)cb.n_e * cb.e_dim, cb.n_e, cb.e_dim, 1, cb_forms};
    add_conv(n, "before_quant_group." + ks, k == 0 ? ch : 2 * ch, cb.e_dim, 1);
    add_conv(n, "after_quant_group." + ks + ".conv", k == 0 ? cb.e_dim : n->cbs[k - 1].e_dim + cb.e_dim, ch, 3);
  }
}

// A VGG-style stack: every conv is 3x3 pad 1 + ReLU, some have a 2x2/2 max-pool in front; `tap`: the ReLU output is a
// feature the caller consumes (besides the last conv's).
struct VggLayer { const char* w; int cout; bool pool_before, tap; };
// VGG19 features up to relu4_4 (vgg_arch.py:55-139 with layer_name_list ['relu4_4']), under vgg_feat_extractor.vgg_net.
static const VggLayer VGG19_RELU4_4[12] = {
    {"conv1_1", 64, false, false}, {"conv1_2", 64, false, false}, {"conv2_1", 128, true, false}, {"conv2_2", 128, false, false},
    {"conv3_1", 256, true, false}, {"conv3_2", 256, false, false}, {"conv3_3", 256, false, false}, {"conv3_4", 256, false, false},
    {"conv4_1", 512, true, false}, {"conv4_2", 512, false, false}, {"conv4_3", 512, false, false}, {"conv4_4", 512, false, false}};
// LPIPS' VGG16 (torchvision vgg16().features to relu5_3 as the lpips package's net.slice{1..5}.{i}); taps relu1_2, relu2_2,
// relu3_3, relu4_3, relu5_3
static const VggLayer VGG16_LPIPS[13] = {
    {"net.slice1.0", 64, false, false},  {"net.slice1.2", 64, false, true},
    {"net.slice2.5", 128, true, false},  {"net.slice2.7", 128, false, true},
    {"net.slice3.10", 256, true, false}, {"net.slice3.12", 256, false, false}, {"net.slice3.14", 256, false, true},
    {"net.slice4.17", 512, true, false}, {"net.slice4.19", 512, false, false}, {"net.slice4.21", 512, false, true},
    {"net.slice5.24", 512, true, false}, {"net.slice5.26", 512, false, false}, {"net.slice5.28", 512, false, true}};
// LPIPS' AlexNet (torchvision alexnet().features): the five convs (Cin, Cout, k); the ReLU after each is a tap
struct AlexLayer { const char* w; int cin, cout, k; };
static const AlexLayer ALEX_LPIPS[5] = {{"net.slice1.0", 3, 64, 11}, {"net.slice2.3", 64, 192, 5}, {"net.slice3.6", 192, 384, 3},
                                        {"net.slice4.8", 384, 256, 3}, {"net.slice5.10", 256, 256, 3}};
static const int LPIPS_TAP_C[2][5] = {{64, 192, 384, 256, 256}, {64, 128, 256, 512, 512}};   // [alex, vgg][tap]

// use_semantic_loss=True (femasr_arch.py:301-309): conv_semantic = Sequential(Conv2d(512, 512, 1), ReLU) and the extractor
static void add_semantic(femasr_net* n) {
  add_conv(n, "conv_semantic.0", 512, 512, 1, VGG_CONV);
  add_vec(n, "vgg_feat_extractor.mean", 3);
  add_vec(n, "vgg_feat_extractor.std", 3);
  int cin = 3;
  for (int i = 0; i < 12; ++i) {
    const VggLayer& l = VGG19_RELU4_4[i];
    add_conv(n, std::string("vgg_feat_extractor.vgg_net.") + l.w, cin, l.cout, 3, i == 0 ? VGG_CONV1 : VGG_CONV);
    cin = l.cout;
  }
}

// LPIPS v0.1 (lpips package): the ScalingLayer buffers, the backbone convs and the five lin weights [1,C,1,1]
static void build_lpips_spec(femasr_net* n) {
  add_vec(n, "scaling_layer.shift", 3);
  add_vec(n, "scaling_layer.scale", 3);
  const bool vgg = n->lcfg.net == 1;
  if (vgg) {
    int cin = 3;
    for (int i = 0; i < 13; ++i) {
      add_conv(n, VGG16_LPIPS[i].w, cin, VGG16_LPIPS[i].cout, 3, i == 0 ? VGG_CONV1 : VGG_CONV);
      cin = VGG16_LPIPS[i].cout;
    }
  } else {
    for (int i = 0; i < 5; ++i)   // conv1: im2col GEMM, K = 363 -> 384
      add_conv(n, ALEX_LPIPS[i].w, ALEX_LPIPS[i].cin, ALEX_LPIPS[i].cout, ALEX_LPIPS[i].k, i == 0 ? VGG_CONV1 : VGG_CONV);
  }
  for (int k = 0; k < 5; ++k) add_vec(n, "lin" + std::to_string(k) + ".model.1.weight", LPIPS_TAP_C[vgg][k]);
}

// UNetDiscriminatorSN (discriminator_arch.py): conv0 and conv9 plain convs with bias; conv1 ... conv8 spectral_norm convs
// without bias, whose state_dict entries are weight_orig [Cout,Cin,k,k], weight_u [Cout] and weight_v [Cin*k*k]
static void add_sn_conv(femasr_net* n, const std::string& p, int ci, int co, int k) {
  n->spec[p + ".weight_orig"] = ParamInfo{(size_t)co * ci * k * k, co, ci, k, weight_forms(n, DISC_CONV, ci, co, k), p};
  n->spec[p + ".weight_u"] = ParamInfo{(size_t)co, 0, 0, 0, 0, p};
  n->spec[p + ".weight_v"] = ParamInfo{(size_t)ci * k * k, 0, 0, 0, 0, p};
}
static void build_disc_spec(femasr_net* n) {
  const int F = n->dcfg.num_feat;
  add_conv(n, "conv0", n->dcfg.num_in_ch, F, 3, VGG_CONV1);     // im2col GEMM, K = 27 -> 64
  add_sn_conv(n, "conv1", F, 2 * F, 4);
  add_sn_conv(n, "conv2", 2 * F, 4 * F, 4);
  add_sn_conv(n, "conv3", 4 * F, 8 * F, 4);
  add_sn_conv(n, "conv4", 8 * F, 4 * F, 3);
  add_sn_conv(n, "conv5", 4 * F, 2 * F, 3);
  add_sn_conv(n, "conv6", 2 * F, F, 3);
  add_sn_conv(n, "conv7", F, F, 3);
  add_sn_conv(n, "conv8", F, F, 3);
  add_conv(n, "conv9", F, 1, 3);                                 // femasr_out_conv3x3_n, Cout 1
}

// ---------------------------------------------------------------------------------------------
// One conv / linear layer of the graph.  H, W: the conv-input size (low-res when upsample).  The operand is fp32 x, or
// split-fp16 planes a_hi/a_lo a producer already wrote (tensor-core GEMM only); the result is fp32 y, or split planes
// o_hi/o_lo for the next tensor-core GEMM.
struct ConvDesc {
  std::string w;                                   // parameter prefix: w.weight, w.bias
  const char* name = nullptr;                      // profile name (nullptr: "igemm_simt" / "tc_igemm" with detail labels)
  const float* x = nullptr;
  const void *a_hi = nullptr, *a_lo = nullptr;
  float* y = nullptr;
  void *o_hi = nullptr, *o_lo = nullptr;
  int B = 0, H = 0, W = 0, Cin = 0, Cout = 0, k = 3;
  int stride = 1, upsample = 0;
  int pro = FEMASR_PRO_NONE;                       // prologue; pa/pb: GN scale/shift or LN mean/rstd tables
  const float *pa = nullptr, *pb = nullptr, *gamma = nullptr, *beta = nullptr;
  int act = FEMASR_ACT_NONE;
  const float *res1 = nullptr, *res2 = nullptr;
  float* gn_partial = nullptr;                     // GroupNorm partials of the output (tensor-core GEMM)
  bool bias = true;
  bool im2col = false;                             // the weight's FORM_IM2COL: a 1x1 GEMM over 64-wide im2col rows
  bool semantic = false;                           // a GEMM of the semantic branch (its own numerics)
  bool sn = false;                                 // a spectral-norm layer: the weight's forms live on w.weight_orig
  int macs = 0;                                    // algorithmic MACs per output element if not Cin*k*k (im2col GEMMs)
  std::string wname() const { return w + (sn ? ".weight_orig" : ".weight"); }
};

static ConvDesc geom(const std::string& w, int B, int H, int W, int Cin, int Cout, int k) {
  ConvDesc d;
  d.w = w; d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.k = k;
  return d;
}

static double conv_flops(const ConvDesc& d) {   // algorithmic (reference) count
  const int u = d.upsample ? 2 : 1;
  const int Ho = d.stride == 2 ? (d.H + 2 - d.k) / 2 + 1 : d.H * u, Wo = d.stride == 2 ? (d.W + 2 - d.k) / 2 + 1 : d.W * u;
  return 2.0 * d.B * Ho * (double)Wo * d.Cout * (d.macs ? d.macs : d.Cin * d.k * d.k);
}

// How a tensor-core conv computes: K-slicing, the F8 cross product and the staging prologue
struct Numerics { int slice_kb = 0; bool f8 = false; int prologue = FEMASR_PRO_NONE; };

struct Ctx {
  femasr_net* net;
  Arena ar;
  cudaStream_t st;
  long l0;                       // g_launches when the run started
  int status = FEMASR_OK;
  double flops = 0;              // sizing run: sum of the launches' algorithmic FLOPs
  float* sem_loss = nullptr;     // forward_sem: the semantic loss output (non-NULL = run the VGG branch)
  float* vgg_feat = nullptr;     // relu4_4 [B,H/8,W/8,512], alive from the VGG stage to the loss at quantising level 0
  bool precise_region = false;   // true while emitting the layers in front of the VQ (index-critical)

  // workspace == nullptr: a sizing run (allocations and FLOPs only, nothing launched); else a run over the caller's
  // workspace, aligned up to 256 bytes
  Ctx(femasr_net* n, void* workspace, size_t bytes, void* stream) : net(n), st(as_stream(stream)), l0(g_launches) {
    const uintptr_t mis = (256 - ((uintptr_t)workspace & 255)) & 255;
    ar.dry = !workspace;
    ar.base = ar.dry ? reinterpret_cast<char*>(uintptr_t(1) << 40) : reinterpret_cast<char*>(workspace) + mis;
    ar.cap = ar.dry ? 0 : bytes - mis;
  }
  bool dry() const { return ar.dry; }
  bool ok() const { return status == FEMASR_OK; }
  void check(int s) { if (status == FEMASR_OK && s != FEMASR_OK) status = s; }
  size_t bytes_needed() const { return ar.peak + 256; }
  int finish() {
    if (!dry()) net->last_launches = (int)(g_launches - l0);
    return status;
  }

  // every kernel launch of the graph goes through here; in profile mode it is bracketed by CUDA events
  template <class F>
  void run(const char* name, double fl, F&& f) {
    if (dry()) { flops += fl; return; }
    if (!ok()) return;
    if (ar.overflow) { check(fail(FEMASR_ERR_STATE, "workspace plan mismatch: the graph needs more than femasr_net_workspace_bytes reported")); return; }
    if (net->profile) {
      ProfRec r{name, fl, nullptr, nullptr};
      cudaEventCreate(&r.e0); cudaEventCreate(&r.e1);
      cudaEventRecord(r.e0, st);
      check(f());
      cudaEventRecord(r.e1, st);
      net->prof.push_back(r);
    } else {
      check(f());
    }
  }

  // FEMASR_PROFILE_DETAIL=1: per-shape kernel labels in the profile ("tc_igemm:k3:64->64@512x512"); the strings are
  // interned for the life of the process because the profile records keep only the pointer
  const char* detail_name(const char* base, int k, int Cin, int Cout, int H, int W, int up, int stride, int slice) {
    static const bool detail = [] { const char* e = getenv("FEMASR_PROFILE_DETAIL"); return e && atoi(e) != 0; }();
    if (!detail || !net->profile) return base;
    static std::set<std::string> names;
    std::string s = std::string(base) + ":k" + std::to_string(k) + ":" + std::to_string(Cin) + "->" + std::to_string(Cout) + "@" +
                    std::to_string(H) + "x" + std::to_string(W) + (up ? ":up" : "") + (stride == 2 ? ":s2" : "") + (slice ? ":sliced" : "");
    return names.insert(s).first->c_str();
  }

  // a parameter's device buffers: all nullptr in a sizing run, and for a parameter that was never set (which fails the run)
  const DevParam& D(const std::string& name) {
    static const DevParam none;
    if (dry()) return none;
    auto it = net->dev.find(name);
    if (it == net->dev.end()) { check(fail(FEMASR_ERR_STATE, "parameter not set: " + name)); return none; }
    return it->second;
  }
  const float* P(const std::string& name) {      // packed (or raw when there is no packed form)
    const DevParam& d = D(name);
    return d.packed ? d.packed : d.raw;
  }
  bool has(const std::string& name, unsigned form) const { return (net->spec.at(name).forms & form) != 0; }
  bool tapped(const char* stage) const {
    auto it = net->taps.find(stage);
    return it != net->taps.end() && it->second.dst;
  }
  void tap(const char* stage, const float* src, size_t n) {
    if (dry() || !ok() || !tapped(stage)) return;
    const Tap& t = net->taps.at(stage);
    if (t.cap < n) { check(fail(FEMASR_ERR_ARG, std::string("tap buffer too small: ") + stage)); return; }
    cudaError_t e = cudaMemcpyAsync(t.dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) check(fail(FEMASR_ERR_CUDA, cudaGetErrorString(e)));
  }

  // the wgmma implicit GEMM wherever the spec gave the weight its tensor-core form (gemm_path 1), else the SIMT one
  bool use_tc(const ConvDesc& d) const {
    return net->cfg.gemm_path == 1 && (d.im2col || has(d.wname(), d.upsample ? FORM_UP : FORM_TC));
  }

  // The numerics policy.  In front of the VQ (index-critical): every tc_slice_kb k-blocks the tensor core's truncating
  // accumulator is folded into an fp32 round-to-nearest running sum (see femasr_tc_args.slice_kb).  Behind it (bar: 1e-3
  // on the output): approximate-unit SiLU, and the two cross products of the split as one fp8 product.  The semantic
  // branch runs in one pass (or FEMASR_SEM_SLICE_KB) without F8, wherever in the graph it sits.
  Numerics numerics(const ConvDesc& d) const {
    Numerics m;
    m.prologue = d.pro;
    if (d.semantic) {
      m.slice_kb = net->sem_slice_kb;
    } else if (precise_region) {
      const int nkb = (d.upsample ? 4 : d.k * d.k) * (d.Cin / 64);
      if (net->tc_precise && nkb > net->tc_slice_kb) m.slice_kb = net->tc_slice_kb;
    } else {
      m.f8 = !d.a_hi && d.k == 3 && d.pro != FEMASR_PRO_LN && has(d.wname(), d.upsample ? FORM_UP8 : FORM_TC8);
      if (d.pro == FEMASR_PRO_GN_SILU && net->fast_silu) m.prologue = FEMASR_PRO_GN_SILU_FAST;
    }
    return m;
  }

  const void* weight(const ConvDesc& d, bool tc, bool f8) {
    const DevParam& p = D(d.wname());
    const void* w = d.im2col ? p.im2col : !tc ? p.packed : d.upsample ? (f8 ? p.up8 : p.up) : (f8 ? p.tc8 : p.tc);
    if (!dry() && !w) check(fail(FEMASR_ERR_STATE, "parameter not packed: " + d.wname()));
    return w;
  }

  // the tensor-core GEMM's arguments for d over the operand planes a_hi/a_lo
  femasr_tc_args tc_args(const ConvDesc& d, const Numerics& m, const void* a_hi, const void* a_lo) {
    femasr_tc_args t;
    memset(&t, 0, sizeof(t));
    t.a_hi = a_hi; t.a_lo = a_lo; t.w_blob = weight(d, true, m.f8); t.bias = d.bias ? P(d.w + ".bias") : nullptr;
    t.res1 = d.res1; t.res2 = d.res2; t.y = d.y; t.out_hi = d.o_hi; t.out_lo = d.o_lo; t.gn_partial = d.gn_partial;
    t.B = d.B; t.H = d.H; t.W = d.W; t.Cin = d.Cin; t.Cout = d.Cout; t.ksize = d.k; t.act = d.act; t.upsample = d.upsample;
    t.stride = d.stride; t.slice_kb = m.slice_kb; t.f8 = m.f8 ? 1 : 0; t.pair = -1; t.strip = -1;
    return t;
  }

  // y = conv(x) (+epilogue).  The tensor-core path stages the activation operand (prologue + fp16 split, or the F8
  // plane) unless the producer already wrote split planes; a fused nearest-x2 upsample runs as four sub-pixel 2x2 convs
  // on the low-res operand.  Allocation happens in sizing runs too.
  void conv(const ConvDesc& d) {
    if (!use_tc(d)) {
      femasr_igemm_args a;
      memset(&a, 0, sizeof(a));
      a.x = d.x; a.w = static_cast<const float*>(weight(d, false, false)); a.bias = d.bias ? P(d.w + ".bias") : nullptr;
      a.res1 = d.res1; a.res2 = d.res2; a.y = d.y; a.pro_a = d.pa; a.pro_b = d.pb; a.gamma = d.gamma; a.beta = d.beta;
      a.B = d.B; a.Hin = d.H; a.Win = d.W; a.Cin = d.Cin; a.Cout = d.Cout; a.ksize = d.k; a.stride = d.stride;
      a.upsample = d.upsample; a.prologue = d.pro; a.act = d.act;
      run(d.name ? d.name : "igemm_simt", conv_flops(d), [&] { return femasr_igemm_simt(&a, st); });
      return;
    }
    const Numerics m = numerics(d);
    float *ahi = nullptr, *alo = nullptr;
    if (!d.a_hi) {
      const size_t plane_halves = (size_t)d.B * d.H * d.W * d.Cin;
      ahi = ar.alloc((plane_halves + 1) / 2);
      alo = ar.alloc((plane_halves + 1) / 2);
      run(detail_name(m.f8 ? "tc_prepare_f8" : "tc_prepare", m.prologue, d.Cin, d.Cin, d.H, d.W, 0, 1, 0), 0.0, [&] {
        return m.f8 ? femasr_tc_prepare_f8(d.x, ahi, alo, m.prologue, d.pa, d.pb, d.B, d.H, d.W, d.Cin, st)
                    : femasr_tc_prepare(d.x, ahi, alo, m.prologue, d.pa, d.pb, d.gamma, d.beta, d.B, d.H, d.W, d.Cin, 0,
                                        d.pro == FEMASR_PRO_LN ? 1e-5f : 1e-6f, st);
      });
    }
    const femasr_tc_args t = tc_args(d, m, ahi ? ahi : d.a_hi, ahi ? alo : d.a_lo);
    run(d.name ? d.name : detail_name("tc_igemm", d.k, d.Cin, d.Cout, d.H, d.W, d.upsample, d.stride, t.slice_kb),
        conv_flops(d), [&] { return femasr_tc_igemm(&t, st); });
    if (alo) ar.release(alo);
    if (ahi) ar.release(ahi);
  }

  // GroupNorm partial sums produced by a tensor-core conv epilogue (see femasr_tc_args.gn_partial)
  struct Stats { float* partial = nullptr; int rows = 0; };
  // for the conv d that will produce them (none on the SIMT path)
  Stats alloc_stats(const ConvDesc& d) {
    Stats s;
    if (!use_tc(d)) return s;
    const femasr_tc_args t = tc_args(d, numerics(d), nullptr, nullptr);
    s.rows = femasr_tc_gn_partial_rows(&t);
    s.partial = ar.alloc((size_t)d.B * s.rows * 32 * 2);
    return s;
  }

  // scale/shift tables for `norm` applied to x: from epilogue partials when available, else a stats pass over x
  void gn_tables(const std::string& norm, const float* x, const Stats& sx, float* sc, float* sh, int B, int HW, int C) {
    const float *gw = P(norm + ".weight"), *gb = P(norm + ".bias");
    if (sx.partial) {
      run("gn_finalize_rows", 0.0, [&] { return femasr_gn_finalize_rows(sx.partial, gw, gb, sc, sh, B, sx.rows, HW, C, 1e-6f, st); });
    } else {
      float* scratch = ar.alloc(femasr_gn_scratch_floats(B, HW, C));
      run("gn_stats", 0.0, [&] { return femasr_gn_stats(x, gw, gb, sc, sh, scratch, B, HW, C, 1e-6f, st); });
      ar.release(scratch);
    }
  }

  // fema_utils.py:65-84, in place on x; optional extra residual added after the block (encoder skip).
  // sx: GroupNorm partials of x from its producer (consumed/released here); returns the partials of the block's
  // output when want_out (for the next ResBlock's first norm), which the caller releases after use.
  Stats resblock(const std::string& p, float* x, int B, int H, int W, int C, const float* extra, Stats sx, bool want_out) {
    const size_t n = (size_t)B * H * W * C;
    float* sc = ar.alloc((size_t)B * C);
    float* sh = ar.alloc((size_t)B * C);
    float* t = ar.alloc(n);
    gn_tables(p + ".conv.0.norm", x, sx, sc, sh, B, H * W, C);
    if (sx.partial) ar.release(sx.partial);
    ConvDesc c = geom(p + ".conv.2", B, H, W, C, C, 3);
    c.x = x; c.y = t; c.pro = FEMASR_PRO_GN_SILU; c.pa = sc; c.pb = sh;
    const Stats s1 = alloc_stats(c);
    c.gn_partial = s1.partial;
    conv(c);
    gn_tables(p + ".conv.3.norm", t, s1, sc, sh, B, H * W, C);
    if (s1.partial) ar.release(s1.partial);
    c.w = p + ".conv.5"; c.x = t; c.y = x; c.res1 = x; c.res2 = extra;
    const Stats s2 = want_out ? alloc_stats(c) : Stats{};
    c.gn_partial = s2.partial;
    conv(c);
    ar.release(t); ar.release(sh); ar.release(sc);
    return s2;
  }

  // nn.Upsample(2) -> conv3x3 -> ResBlock -> ResBlock  (femasr_arch.py:168-180, 195-211); returns new buffer
  float* up_block(const std::string& p, const float* x, int B, int H, int W, int Cin, int Cout, const float* extra) {
    float* y = ar.alloc((size_t)B * 2 * H * 2 * W * Cout);
    ConvDesc c = geom(p + ".1", B, H, W, Cin, Cout, 3);
    c.x = x; c.y = y; c.upsample = 1;
    const Stats s0 = alloc_stats(c);
    c.gn_partial = s0.partial;
    conv(c);
    Stats s1 = resblock(p + ".2", y, B, 2 * H, 2 * W, Cout, nullptr, s0, true);
    resblock(p + ".3", y, B, 2 * H, 2 * W, Cout, extra, s1, false);
    return y;
  }

  // SwinLayers (femasr_arch.py:126-132): 4 x RSTB on tokens X [B, H*W, 256], in place.
  void swin(const std::string& p, float* X, int B, int H, int W) {
    const int C = 256;
    const size_t M = (size_t)B * H * W;
    float* T = ar.alloc(M * C);
    float* qkv = ar.alloc(M * 3 * C);
    float* ao = ar.alloc(M * C);
    float* hid = ar.alloc(M * 4 * C);
    float* mu = ar.alloc(M);
    float* rs = ar.alloc(M);
    const bool tc = net->cfg.gemm_path == 1;
    for (int r = 0; r < 4; ++r) {
      const std::string rp = p + ".swin_blks." + std::to_string(r);
      for (int b = 0; b < 6; ++b) {
        const std::string bp = rp + ".residual_group.blocks." + std::to_string(b);
        const float* in = b == 0 ? X : T;
        const std::string rbname = bp + ".attn.relative_position_bias_table";
        const double attn_flops = 2.0 * 2.0 * 64 * C * (double)M;
        ConvDesc q = geom(bp + ".attn.qkv", B, H, W, C, 3 * C, 1), o = geom(bp + ".attn.proj", B, H, W, C, C, 1);
        ConvDesc f1 = geom(bp + ".mlp.fc1", B, H, W, C, 4 * C, 1), f2 = geom(bp + ".mlp.fc2", B, H, W, 4 * C, C, 1);
        q.x = in; q.y = qkv; q.pro = FEMASR_PRO_LN; q.gamma = P(bp + ".norm1.weight"); q.beta = P(bp + ".norm1.bias");
        o.y = T; o.res1 = in;
        f1.x = T; f1.pro = FEMASR_PRO_LN; f1.gamma = P(bp + ".norm2.weight"); f1.beta = P(bp + ".norm2.bias");
        f1.act = FEMASR_ACT_GELU;
        f2.y = T; f2.res1 = T;
        if (tc) {
          // operands travel between the kernels as split fp16 planes: `ao` and `hid` are reinterpreted as
          // [hi plane | lo plane] (same byte size as the fp32 tensors they replace); LayerNorm runs in the staging
          __half* ao_hi = reinterpret_cast<__half*>(ao);  __half* ao_lo = ao_hi + M * C;
          __half* hd_hi = reinterpret_cast<__half*>(hid); __half* hd_lo = hd_hi + M * 4 * C;
          o.a_hi = ao_hi; o.a_lo = ao_lo; f1.o_hi = hd_hi; f1.o_lo = hd_lo; f2.a_hi = hd_hi; f2.a_lo = hd_lo;
          conv(q);
          const float* rbm = D(rbname).relb_mma;
          run("window_attention_mma", attn_flops, [&] {
            return femasr_window_attention_mma(qkv, rbm, nullptr, ao_hi, ao_lo, B, H, W, C, 8, (b & 1) ? 4 : 0, st);
          });
          conv(o); conv(f1); conv(f2);
          continue;
        }
        q.pa = f1.pa = mu; q.pb = f1.pb = rs; o.x = ao; f1.y = hid; f2.x = hid;
        const float* rb = P(rbname);
        run("ln_stats", 0.0, [&] { return femasr_ln_stats(in, mu, rs, (int)M, C, 1e-5f, st); });
        conv(q);
        run("window_attention", attn_flops,
            [&] { return femasr_window_attention(qkv, rb, ao, B, H, W, C, 8, (b & 1) ? 4 : 0, st); });
        conv(o);
        run("ln_stats", 0.0, [&] { return femasr_ln_stats(T, mu, rs, (int)M, C, 1e-5f, st); });
        conv(f1); conv(f2);
      }
      ConvDesc c = geom(rp + ".conv", B, H, W, C, C, 3);
      c.x = T; c.y = X; c.res1 = X;
      conv(c);
    }
    ar.release(rs); ar.release(mu); ar.release(hid); ar.release(ao); ar.release(qkv); ar.release(T);
  }

  // vgg_feat = relu4_4((x - mean) / std) (femasr_arch.py:318-320).  Runs before the encoder: relu4_4 is allocated first
  // and every full-resolution VGG buffer is released before the encoder's peak.
  void semantic_vgg(const float* x_nchw, int B, int H, int W) {
    const bool tc = net->cfg.gemm_path == 1;
    vgg_feat = ar.alloc((size_t)B * (H / 8) * (W / 8) * 512);
    float *ahi = nullptr, *alo = nullptr, *af = nullptr;   // conv1_1's operand: split planes (tc) or fp32
    const size_t rows = (size_t)B * H * W;
    if (tc) { ahi = ar.alloc(rows * 32); alo = ar.alloc(rows * 32); } else { af = ar.alloc(rows * 64); }
    const float *mean = P("vgg_feat_extractor.mean"), *sd = P("vgg_feat_extractor.std");
    run("vgg_im2col", 0.0, [&] { return femasr_vgg_im2col(x_nchw, mean, sd, ahi, alo, af, B, H, W, st); });
    vgg_stack(VGG19_RELU4_4, 12, "vgg_feat_extractor.vgg_net.", "vgg_conv", "vgg_pool", B, H, W, ahi, alo, af, vgg_feat,
              [](const float*, int, int, int) {});
    tap("vgg", vgg_feat, (size_t)B * (H / 8) * (W / 8) * 512);
  }

  // The convs of a VggLayer table over B images of H x W, from conv 0's im2col operand (K = 27 -> 64: split planes ahi/alo
  // on gemm_path 1, fp32 rows af on gemm_path 0), which this releases.  gemm_path 1 hands the activations from conv to
  // conv as split fp16 planes; the pools read fp32 (pooling before the split) and write the next conv's planes.  Every
  // conv is bias + ReLU: the 3-product split-fp16 wgmma GEMM on gemm_path 1, the fp32 SIMT GEMM on gemm_path 0.
  // on_tap(f, h, w, c) sees the fp32 output of every tap layer while it is alive.  The last conv writes into `last` if
  // given, else into an arena buffer that is returned for the caller to release.
  template <class F>
  float* vgg_stack(const VggLayer* L, int nl, const std::string& pre, const char* conv_name, const char* pool_name, int B,
                   int H, int W, float* ahi, float* alo, float* af, float* last, F&& on_tap) {
    const bool tc = net->cfg.gemm_path == 1;
    int h = H, w = W, c = 64;
    float* f = nullptr;                                    // fp32 output in front of a pool
    float* y = nullptr;
    for (int i = 0; i < nl; ++i) {
      const int co = L[i].cout;
      if (L[i].pool_before) {
        const size_t n2 = (size_t)B * (h / 2) * (w / 2) * c;
        if (tc) {
          ahi = ar.alloc((n2 + 1) / 2); alo = ar.alloc((n2 + 1) / 2);
          const int hh = h, ww = w, cc = c;
          run(pool_name, 0.0, [&] {
            return femasr_tc_prepare(f, ahi, alo, FEMASR_PRO_MAXPOOL2, nullptr, nullptr, nullptr, nullptr, B, hh, ww, cc, 0, 0.f, st);
          });
        } else {
          af = ar.alloc(n2);
          const int hh = h, ww = w, cc = c;
          run(pool_name, 0.0, [&] { return femasr_maxpool2(f, af, B, hh, ww, cc, st); });
        }
        ar.release(f); f = nullptr;
        h /= 2; w /= 2;
      }
      const bool lastl = i == nl - 1, to_f32 = !tc || lastl || L[i].tap || L[i + 1].pool_before;
      const size_t n = (size_t)B * h * w * co;
      y = lastl && last ? last : (to_f32 ? ar.alloc(n) : nullptr);
      float *ohi = nullptr, *olo = nullptr;
      if (!to_f32) { ohi = ar.alloc((n + 1) / 2); olo = ar.alloc((n + 1) / 2); }
      // conv 0: 1x1 GEMM over the K = 27 -> 64 im2col rows (27 algorithmic MACs)
      ConvDesc g = geom(pre + L[i].w, B, h, w, i == 0 ? 64 : c, co, i == 0 ? 1 : 3);
      g.name = conv_name; g.semantic = true; g.im2col = i == 0; g.macs = i == 0 ? 27 : 0; g.act = FEMASR_ACT_RELU;
      g.x = af; g.a_hi = ahi; g.a_lo = alo; g.y = y; g.o_hi = ohi; g.o_lo = olo;
      conv(g);
      if (tc) { ar.release(alo); ar.release(ahi); ahi = ohi; alo = olo; }
      else { ar.release(af); af = y; }
      if (L[i].tap) on_tap(y, h, w, co);
      if (to_f32 && !lastl) f = y;
      c = co;
    }
    return y;
  }

  // LPIPS v0.1 (lpips package, LPIPS.forward): d(x0, x1) for B pairs.  The backbone runs once over the 2B images [x0; x1]
  // (the im2col writes x0's rows first, no concatenated copy); each tap's ReLU output goes through femasr_lpips_head while
  // it is alive and is released as soon as the next layer has read it.  r [5][B] is per_layer, or workspace.  Numerics
  // are those of the semantic loss's VGG convs: the 3-product split-fp16 GEMM without F8 on gemm_path 1, fp32 SIMT on 0.
  void lpips(const float* x0, const float* x1, float* dist, float* per_layer, int B, int H, int W, int normalize) {
    const bool tc = net->cfg.gemm_path == 1, vgg = net->lcfg.net == 1;
    const int N = 2 * B;
    float* r = per_layer ? per_layer : ar.alloc((size_t)5 * B);
    int tap_k = 0;
    auto head = [&](const float* f, int h, int w, int c) {
      float* scratch = ar.alloc((femasr_lpips_head_scratch_bytes(B, h * w) + 3) / 4);
      const float* lw = P("lin" + std::to_string(tap_k) + ".model.1.weight");
      const int k = tap_k;
      run("lpips_head", 0.0, [&] { return femasr_lpips_head(f, lw, B, h * w, c, r, k, k == 4 ? dist : nullptr, scratch, st); });
      ar.release(scratch);
      ++tap_k;
    };
    // first conv's operand: im2col of the scaled pair (vgg: 3x3 pad 1, K = 27 -> 64; alex: 11x11 stride 4 pad 2, K = 363 -> 384)
    const int ks = vgg ? 3 : 11, stride = vgg ? 1 : 4, pad = vgg ? 1 : 2, kpad = im2col_k(ks);
    const int h1 = (H + 2 * pad - ks) / stride + 1, w1 = (W + 2 * pad - ks) / stride + 1;
    const size_t rows = (size_t)N * h1 * w1;
    float *ahi = nullptr, *alo = nullptr, *af = nullptr;
    if (tc) { ahi = ar.alloc(rows * kpad / 2); alo = ar.alloc(rows * kpad / 2); } else { af = ar.alloc(rows * kpad); }
    const float *shift = P("scaling_layer.shift"), *scale = P("scaling_layer.scale");
    run("lpips_im2col", 0.0, [&] {
      return femasr_vgg_im2col_ex(x0, x1, B, H, W, ks, stride, pad, kpad, shift, scale, normalize, ahi, alo, af, st);
    });
    if (vgg) ar.release(vgg_stack(VGG16_LPIPS, 13, "", "lpips_conv", "lpips_pool", N, H, W, ahi, alo, af, nullptr, head));
    else alex(ahi, alo, af, N, h1, w1, head);
    if (!per_layer) ar.release(r);
  }

  // AlexNet features (torchvision): conv1 (the im2col GEMM) | pool 3/2, conv2 5x5 pad 2 | pool 3/2, conv3 | conv4 | conv5,
  // each conv + ReLU and each ReLU a tap.  h, w: conv1's output size.  Releases conv1's operand.
  template <class F>
  void alex(float* ahi, float* alo, float* af, int N, int h, int w, F&& head) {
    const bool tc = net->cfg.gemm_path == 1;
    float* f = nullptr;                                    // the previous conv's fp32 output
    for (int i = 0; i < 5; ++i) {
      const AlexLayer& l = ALEX_LPIPS[i];
      float *phi = nullptr, *plo = nullptr, *pf = nullptr;  // max-pool 3/2 output in front of conv2 and conv3
      if (i == 1 || i == 2) {
        const int hp = (h - 3) / 2 + 1, wp = (w - 3) / 2 + 1, hh = h, ww = w, cc = l.cin;
        const size_t n2 = (size_t)N * hp * wp * l.cin;
        const float* src = f;
        if (tc) {
          phi = ar.alloc((n2 + 1) / 2); plo = ar.alloc((n2 + 1) / 2);
          run("lpips_pool", 0.0, [&] {
            return femasr_tc_prepare(src, phi, plo, FEMASR_PRO_MAXPOOL3S2, nullptr, nullptr, nullptr, nullptr, N, hh, ww, cc, 0, 0.f, st);
          });
        } else {
          pf = ar.alloc(n2);
          run("lpips_pool", 0.0, [&] { return femasr_maxpool3s2(src, pf, N, hh, ww, cc, st); });
        }
        ar.release(f); f = nullptr;
        h = hp; w = wp;
      }
      float* y = ar.alloc((size_t)N * h * w * l.cout);
      // conv1: 1x1 GEMM over the K = 363 -> 384 im2col rows (363 algorithmic MACs)
      ConvDesc g = geom(l.w, N, h, w, i == 0 ? im2col_k(l.k) : l.cin, l.cout, i == 0 ? 1 : l.k);
      g.name = "lpips_conv"; g.semantic = true; g.act = FEMASR_ACT_RELU; g.y = y;
      if (i == 0) { g.im2col = true; g.macs = 3 * l.k * l.k; g.x = af; g.a_hi = ahi; g.a_lo = alo; }
      else if (phi) { g.a_hi = phi; g.a_lo = plo; }
      else { g.x = pf ? pf : f; }
      conv(g);
      if (i == 0) { if (tc) { ar.release(alo); ar.release(ahi); } else { ar.release(af); } }
      if (phi) { ar.release(plo); ar.release(phi); }
      if (pf) ar.release(pf);
      if (f) ar.release(f);
      f = y;
      head(f, h, w, l.cout);
    }
    ar.release(f);
  }

  // semantic_loss = mse(ReLU(conv_semantic(z_quant)), vgg_feat) (femasr_arch.py:344-347) on the quantiser's output
  // (before the use_quantize override, :349-350); the only quantising level where the shapes agree is level 0 of the HQ
  // stage, so the sum over levels (:372) is this one term.
  void semantic_loss(const float* zq, int B, int hh, int ww) {
    const size_t N = (size_t)B * hh * ww;
    const bool tc = net->cfg.gemm_path == 1;
    float* s = ar.alloc(N * 512);
    float* rows = ar.alloc(N);
    float *zhi = nullptr, *zlo = nullptr;
    if (tc) {
      zhi = ar.alloc(N * 256); zlo = ar.alloc(N * 256);
      run("tc_prepare", 0.0, [&] { return femasr_tc_prepare(zq, zhi, zlo, FEMASR_PRO_NONE, nullptr, nullptr, nullptr, nullptr, B, hh, ww, 512, 0, 0.f, st); });
    }
    ConvDesc g = geom("conv_semantic.0", B, hh, ww, 512, 512, 1);
    g.name = "semantic_conv"; g.semantic = true; g.act = FEMASR_ACT_RELU; g.x = zq; g.a_hi = zhi; g.a_lo = zlo; g.y = s;
    conv(g);
    tap("semantic", s, N * 512);
    const float* v = vgg_feat;
    run("semantic_mse", 0.0, [&] { return femasr_sq_diff_rows(s, v, rows, (int)N, 512, st); });
    run("semantic_mse", 0.0, [&] { return femasr_sum_scaled(rows, sem_loss, N, 1.0 / ((double)N * 512), st); });
    if (tc) { ar.release(zlo); ar.release(zhi); }
    ar.release(rows); ar.release(s);
    ar.release(vgg_feat); vgg_feat = nullptr;
  }

  // One quantiser (femasr_arch.py:337-342 + VectorQuantizer.forward :50-100): z = before_quant(src) [N,e], argmin over
  // codebook k, zq = z + (E[idx] - z); loss terms accumulate into cb_loss.  Returns z and zq (caller releases both).
  void quantise(int k, const float* src, int Cin, int B, int hh, int ww, int64_t* indices, float* cb_loss,
                const int64_t* gt, float** z_out, float** zq_out) {
    const femasr_net::Codebook& cb = net->cbs[k];
    const std::string ks = std::to_string(k);
    const size_t N = (size_t)B * hh * ww;
    const int e = cb.e_dim;
    float* z = ar.alloc(N * e);
    ConvDesc bq = geom("before_quant_group." + ks, B, hh, ww, Cin, e, 1);
    bq.x = src; bq.y = z;
    conv(bq);
    tap(k == 0 ? "z" : (k == 1 ? "z1" : "z2"), z, N * e);
    const std::string cname = "quantize_group." + ks + ".embedding.weight";
    const bool fused = has(cname, FORM_TC);
    // fused: tensor-core distances + in-kernel top-4 (no [N, n_e] tensor); else the fp32 SIMT product + vq_select
    float *zc = nullptr, *arow = nullptr, *zhi = nullptr, *zlo = nullptr, *cand = nullptr;
    if (fused) {
      arow = ar.alloc(N);
      zhi = ar.alloc((N * e + 1) / 2);
      zlo = ar.alloc((N * e + 1) / 2);
      cand = ar.alloc(N * 8);
    } else {
      zc = ar.alloc(N * cb.n_e);
      ConvDesc d = geom("quantize_group." + ks + ".embedding", B, hh, ww, e, cb.n_e, 1);
      d.x = z; d.y = zc; d.bias = false;
      conv(d);
    }
    float* zq = ar.alloc(N * e);
    float* lrows = ar.alloc(N);
    const bool gt_loss = gt && !net->hq;                 // :84: only the LQ stage uses gt_indices for the loss
    float *zq_gt = nullptr, *gpart = nullptr;
    const int gtiles = femasr_gram_diff_tiles(e);
    if (gt_loss) { zq_gt = ar.alloc(N * e); gpart = ar.alloc((size_t)B * gtiles); }
    const DevParam& cbd = D(cname);
    const float *cbw = cbd.raw, *esq = cbd.esq;
    if (fused) {
      const void* cbt = cbd.tc;
      run("vq_row_sumsq", 0.0, [&] { return femasr_row_sumsq(z, arow, (int)N, e, st); });
      run("tc_prepare", 0.0, [&] { return femasr_tc_prepare(z, zhi, zlo, FEMASR_PRO_NONE, nullptr, nullptr, nullptr, nullptr, B, hh, ww, e, 0, 0.f, st); });
      run("vq_match_tc", 2.0 * (double)N * cb.n_e * e, [&] { return femasr_vq_match_tc(zhi, zlo, cbt, arow, esq, cand, (int)N, cb.n_e, e, st); });
      run("vq_finish", 0.0, [&] { return femasr_vq_finish(z, arow, cand, cbw, esq, indices, zq, lrows, nullptr, (int)N, cb.n_e, e, st); });
    } else {
      run("vq_select", 0.0, [&] { return femasr_vq_select(z, zc, cbw, esq, indices, zq, lrows, (int)N, cb.n_e, e, 0, st); });
    }
    if (cb_loss && !gt_loss) {
      const double s = 1.25 / ((double)N * e);         // q_latent + 0.25 * e_latent, :92
      run("sum_scaled", 0.0, [&] { return k == 0 ? femasr_sum_scaled(lrows, cb_loss, N, s, st) : femasr_sum_scaled_add(lrows, cb_loss, N, s, st); });
    } else if (cb_loss) {
      run("vq_gt_rows", 0.0, [&] { return femasr_vq_gt_rows(z, cbw, gt, zq_gt, lrows, (int)N, cb.n_e, e, st); });
      const double s = 0.25 / ((double)N * e);         // beta * mean((z_q_gt - z)^2), :87
      run("sum_scaled", 0.0, [&] { return k == 0 ? femasr_sum_scaled(lrows, cb_loss, N, s, st) : femasr_sum_scaled_add(lrows, cb_loss, N, s, st); });
      run("gram_diff", 4.0 * B * (double)hh * ww * e * e, [&] { return femasr_gram_diff(z, zq_gt, gpart, B, hh * ww, e, st); });
      run("sum_scaled", 0.0, [&] { return femasr_sum_scaled_add(gpart, cb_loss, (size_t)B * gtiles, 1.0 / ((double)B * e * e), st); });
    }
    if (gt_loss) { ar.release(gpart); ar.release(zq_gt); }
    ar.release(lrows);
    if (fused) { ar.release(cand); ar.release(zlo); ar.release(zhi); ar.release(arow); }
    else ar.release(zc);
    if (k == 0) tap("zq", zq, N * e);
    *z_out = z; *zq_out = zq;
  }

  // The decoder loop of encode_and_decode (femasr_arch.py:327-369) from decoder level 0 on.
  //   feats[i]   enc_feats[i] (NHWC, level i = resolution 32 << i) or nullptr when that level needs none
  //   zq0_given  decode_indices: the gathered codebook-0 entries; no quantiser runs at any level (:376-385)
  void decode_loop(const float* const* feats, const float* zq0_given, float* y_nchw, int64_t* indices, float* cb_loss,
                   const int64_t* gt, int B, int h, int w) {
    const femasr_net_config& cfg = net->cfg;
    const bool lq = !net->hq;
    float* t = nullptr;                       // decoder stream
    float* prev_q = nullptr; int pq_h = 0, pq_w = 0, pq_e = 0;   // previous z_quant (:358)
    float* prev_z = nullptr;
    size_t idx_off = 0;
    for (int i = 0; i < 3; ++i) {
      const int hh = h << i, ww = w << i, ch = chan(32 << i), co = chan(64 << i);
      const int k = zq0_given ? (i == 0 ? 0 : -1) : net->level_cb[i];
      if (k >= 0) {
        const femasr_net::Codebook& cb = net->cbs[k];
        const size_t N = (size_t)B * hh * ww;
        const float* aq = zq0_given;
        float *z = nullptr, *zq = nullptr;
        if (!zq0_given) {
          precise_region = true;
          const float* src = feats[i];
          float* cat = nullptr;
          int Cin = ch;
          if (t) {                            // cat(enc_feats[i], prev_dec_feat), :332-333
            cat = ar.alloc(N * 2 * ch);
            run("concat_channels", 0.0, [&] { return femasr_concat_channels(feats[i], ch, t, hh, ww, ch, cat, B, hh, ww, st); });
            ar.release(t); t = nullptr;
            src = cat; Cin = 2 * ch;
          }
          quantise(k, src, Cin, B, hh, ww, indices ? indices + idx_off : nullptr, cb_loss,
                   gt ? gt + idx_off : nullptr, &z, &zq);
          if (k == 0 && sem_loss) semantic_loss(zq, B, hh, ww);
          idx_off += N;
          if (cat) ar.release(cat);
          aq = cfg.use_quantize ? zq : z;     // :349-350
          if (i >= net->last_q_level) precise_region = false;
        }
        int e_in = cb.e_dim;
        float* cat2 = nullptr;
        if (prev_q) {                         // CombineQuantBlock: cat(z_quant, interpolate(prev_quant)), fema_utils.py:92-99
          cat2 = ar.alloc(N * (cb.e_dim + pq_e));
          const float* a0 = aq; const int pe = pq_e, ph = pq_h, pw = pq_w; const float* pq = prev_q;
          run("concat_channels", 0.0, [&] { return femasr_concat_channels(a0, cb.e_dim, pq, ph, pw, pe, cat2, B, hh, ww, st); });
          aq = cat2; e_in += pq_e;
        }
        t = ar.alloc(N * ch);
        ConvDesc c = geom("after_quant_group." + std::to_string(k) + ".conv", B, hh, ww, e_in, ch, 3);
        c.x = aq; c.y = t;
        conv(c);
        if (k == 0) tap("after_quant", t, N * ch);
        if (cat2) ar.release(cat2);
        if (prev_q) { ar.release(prev_q); ar.release(prev_z); }
        if (!zq0_given) {                     // prev_quant_feat = z_quant (after the use_quantize override), :358
          prev_q = cfg.use_quantize ? zq : z; prev_z = cfg.use_quantize ? z : zq;
          pq_h = hh; pq_w = ww; pq_e = cb.e_dim;
        }
      }
      // the skip add of the NEXT level (x = x + enc_feats[i+1], :361-362) rides on this block's last epilogue
      const bool next_quant = i + 1 < 3 && !zq0_given && net->level_cb[i + 1] >= 0;
      const float* extra = (i + 1 < 3 && !zq0_given && lq && cfg.use_residual && !next_quant) ? feats[i + 1] : nullptr;
      float* nt = up_block("decoder_group." + std::to_string(i) + ".block", t, B, hh, ww, ch, co, extra);
      ar.release(t);
      t = nt;
      tap(i == 0 ? "dec0" : (i == 1 ? "dec1" : "dec2"), t, (size_t)B * 2 * hh * 2 * ww * co);
    }
    if (prev_q) { ar.release(prev_q); ar.release(prev_z); }
    const float *ow = P("out_conv.weight"), *ob = P("out_conv.bias");
    const float* d2 = t;
    run("out_conv", 2.0 * 9 * 64 * 3 * (double)B * 64 * h * w,
        [&] { return net->cfg.gemm_path == 1 ? femasr_out_conv3x3_mma(d2, ow, ob, y_nchw, B, 8 * h, 8 * w, 64, st)
                                             : femasr_out_conv3x3(d2, ow, ob, y_nchw, B, 8 * h, 8 * w, 64, st); });
    ar.release(t);
  }

  void forward(const float* x_nchw, float* y_nchw, int64_t* indices, float* cb_loss, const int64_t* gt, int B, int H, int W) {
    const femasr_net_config& cfg = net->cfg;
    const int d = net->depth;
    const std::string enc = "multiscale_encoder";
    int c = chan(256 / cfg.scale_factor);
    int h = H - 1, w = W - 1;
    const bool tc = cfg.gemm_path == 1;
    if (sem_loss) semantic_vgg(x_nchw, B, H, W);
    precise_region = true;
    const float *iw = P(enc + ".in_conv.weight"), *ib = P(enc + ".in_conv.bias");
    float* cur = nullptr;                 // fp32 in_conv output (SIMT path, or when its tap is requested)
    float* in_hi = nullptr; float* in_lo = nullptr;   // tensor-core path: in_conv writes the split operand planes directly
    const size_t in_elems = (size_t)B * h * w * c;
    if (!tc || tapped("in_conv")) {       // identical in the sizing run and the real run: taps are registered first
      cur = ar.alloc(in_elems);
      const int c0 = c;
      run("in_conv", 2.0 * 16 * cfg.in_channel * c * (double)B * h * w,
          [&] { return femasr_in_conv4x4(x_nchw, iw, ib, cur, B, cfg.in_channel, H, W, c0, st); });
      tap("in_conv", cur, in_elems);
    }
    if (tc) {
      // K = 48 (-> 64) GEMM over im2col rows on the tensor cores, writing the down conv's split planes
      in_hi = ar.alloc((in_elems + 1) / 2);
      in_lo = ar.alloc((in_elems + 1) / 2);
      const size_t rows = (size_t)B * h * w;
      float* ic_hi = ar.alloc(rows * 64 / 2);
      float* ic_lo = ar.alloc(rows * 64 / 2);
      run("in_conv_im2col", 0.0, [&] { return femasr_in_conv_im2col(x_nchw, ic_hi, ic_lo, B, cfg.in_channel, H, W, st); });
      ConvDesc g = geom(enc + ".in_conv", B, h, w, 64, c, 1);
      g.name = "in_conv"; g.im2col = true; g.macs = 16 * cfg.in_channel;
      g.a_hi = ic_hi; g.a_lo = ic_lo; g.o_hi = in_hi; g.o_lo = in_lo;
      conv(g);
      ar.release(ic_lo); ar.release(ic_hi);
    }
    // which enc_feats the decoder loop reads: at quantising levels (before_quant input) and, in the LQ stage with
    // use_residual, at the other levels > 0 (skip adds)
    bool need[3];
    for (int i = 0; i < 3; ++i)
      need[i] = net->level_cb[i] >= 0 || (i > 0 && !net->hq && cfg.use_residual);
    float* feats[3] = {nullptr, nullptr, nullptr};
    for (int i = 0; i < d; ++i) {
      const std::string b = enc + ".blocks." + std::to_string(i);
      const int ho = (h + 2 - 3) / 2 + 1, wo = (w + 2 - 3) / 2 + 1, co = chan((256 / cfg.scale_factor) >> (i + 1));
      float* nxt = ar.alloc((size_t)B * ho * wo * co);
      ConvDesc g = geom(b + ".0", B, h, w, c, co, 3);
      g.stride = 2; g.x = cur; g.y = nxt;
      if (i == 0) { g.a_hi = in_hi; g.a_lo = in_lo; }
      const Stats sd0 = alloc_stats(g);
      g.gn_partial = sd0.partial;
      conv(g);
      if (i == 0 && in_lo) { ar.release(in_lo); ar.release(in_hi); in_lo = in_hi = nullptr; }
      // HQ stage: enc_feats = the down blocks' outputs reversed (:316); block i-1's output is level d-i
      if (cur) { if (net->hq && i > 0 && need[d - i]) feats[d - i] = cur; else ar.release(cur); }
      cur = nxt; h = ho; w = wo; c = co;
      Stats sd = resblock(b + ".1", cur, B, h, w, c, nullptr, sd0, true);
      resblock(b + ".2", cur, B, h, w, c, nullptr, sd, false);
    }
    tap("down", cur, (size_t)B * h * w * c);
    if (!net->hq) swin(enc + ".blocks." + std::to_string(d), cur, B, h, w);
    tap("swin", cur, (size_t)B * h * w * c);
    feats[0] = cur;
    // the up branches reach the decoder's skip adds (femasr_arch.py:361-362) and, in multi-scale nets, the later quantisers
    precise_region = net->last_q_level >= 1;
    if (!net->hq && (need[1] || need[2])) {
      feats[1] = up_block(enc + ".blocks." + std::to_string(d + 1), cur, B, h, w, 256, 256, nullptr);
      tap("up1", feats[1], (size_t)B * 2 * h * 2 * w * 256);
      if (need[2]) {
        precise_region = net->last_q_level >= 2;
        feats[2] = up_block(enc + ".blocks." + std::to_string(d + 2), feats[1], B, 2 * h, 2 * w, 256, 128, nullptr);
        tap("up2", feats[2], (size_t)B * 4 * h * 4 * w * 128);
      }
    }
    precise_region = false;
    decode_loop(feats, nullptr, y_nchw, indices, cb_loss, gt, B, h, w);
    for (int i = 2; i >= 0; --i) if (feats[i]) ar.release(feats[i]);
  }

  void decode_indices(const int64_t* idx, float* y_nchw, int B, int h, int w) {
    const femasr_net::Codebook& cb = net->cbs[0];
    const size_t N = (size_t)B * h * w;
    float* zq = ar.alloc(N * cb.e_dim);
    const float* cbw = D("quantize_group.0.embedding.weight").raw;
    run("codebook_gather", 0.0, [&] { return femasr_codebook_gather(idx, cbw, zq, (int)N, cb.n_e, cb.e_dim, st); });
    const float* none[3] = {nullptr, nullptr, nullptr};
    decode_loop(none, zq, y_nchw, nullptr, nullptr, nullptr, B, h, w);
    ar.release(zq);
  }

  // UNetDiscriminatorSN.forward (discriminator_arch.py), x [B,3,H,W] -> y [B,1,H,W], H and W multiples of 8.  Every conv
  // is lrelu(conv + bias) [+ skip] in its epilogue (the skip add comes after the activation, like the reference); on
  // gemm_path 1 they are the K-sliced 3-product split-fp16 GEMM of the precise region (no F8), the bilinear x2 is fused
  // into the next conv's operand staging, and conv6 -> conv7 -> conv8 hand their outputs on as split planes.
  void disc(const float* x_nchw, float* y_nchw, int B, int H, int W) {
    const bool tc = net->cfg.gemm_path == 1, skip = net->dcfg.skip_connection != 0;
    const int F = net->dcfg.num_feat;
    precise_region = true;
    const int hs[4] = {H, H / 2, H / 4, H / 8}, ws[4] = {W, W / 2, W / 4, W / 8};
    float* xs[4] = {nullptr, nullptr, nullptr, nullptr};   // x0 .. x3, fp32 NHWC; x0 .. x2 live until their skip add
    auto sn_conv = [&](int i, int h, int w, int ci, int co, int k) {
      ConvDesc g = geom("conv" + std::to_string(i), B, h, w, ci, co, k);
      g.name = "disc_conv"; g.sn = true; g.bias = false; g.act = FEMASR_ACT_LRELU;
      return g;
    };
    {  // conv0: 3x3 pad 1, 3 -> F, as a 1x1 GEMM over femasr_vgg_im2col's unnormalised K = 27 (-> 64) rows
      const size_t rows = (size_t)B * H * W;
      xs[0] = ar.alloc(rows * F);
      float *ahi = nullptr, *alo = nullptr, *af = nullptr;
      if (tc) { ahi = ar.alloc(rows * 32); alo = ar.alloc(rows * 32); } else { af = ar.alloc(rows * 64); }
      run("disc_im2col", 0.0, [&] { return femasr_vgg_im2col(x_nchw, nullptr, nullptr, ahi, alo, af, B, H, W, st); });
      ConvDesc g = geom("conv0", B, H, W, 64, F, 1);
      g.name = "disc_conv"; g.im2col = true; g.macs = 27; g.act = FEMASR_ACT_LRELU;
      g.x = af; g.a_hi = ahi; g.a_lo = alo; g.y = xs[0];
      conv(g);
      if (tc) { ar.release(alo); ar.release(ahi); } else { ar.release(af); }
    }
    for (int i = 1; i <= 3; ++i) {   // conv1 .. conv3: 4x4 stride 2 pad 1
      xs[i] = ar.alloc((size_t)B * hs[i] * ws[i] * (F << i));
      ConvDesc g = sn_conv(i, hs[i - 1], ws[i - 1], F << (i - 1), F << i, 4);
      g.stride = 2; g.x = xs[i - 1]; g.y = xs[i];
      conv(g);
    }
    // conv4 .. conv6: 3x3 on bilinear_x2 of the previous output, then + x2 / x1 / x0
    float* cur = xs[3];
    void *p_hi = nullptr, *p_lo = nullptr;                 // conv6's output as split planes (tensor-core path)
    for (int lv = 2; lv >= 0; --lv) {
      const int ci = F << (lv + 1), co = F << lv, h = hs[lv], w = ws[lv], hl = hs[lv + 1], wl = ws[lv + 1];
      const size_t n_in = (size_t)B * h * w * ci, n_out = (size_t)B * h * w * co;
      ConvDesc g = sn_conv(6 - lv, h, w, ci, co, 3);
      g.res1 = skip ? xs[lv] : nullptr;
      float *uhi = nullptr, *ulo = nullptr, *uf = nullptr;
      const float* src = cur;
      if (tc) {
        uhi = ar.alloc((n_in + 1) / 2); ulo = ar.alloc((n_in + 1) / 2);
        run("disc_up", 0.0, [&] {
          return femasr_tc_prepare(src, uhi, ulo, FEMASR_PRO_BILINEAR2, nullptr, nullptr, nullptr, nullptr, B, hl, wl, ci, 0, 0.f, st);
        });
        g.a_hi = uhi; g.a_lo = ulo;
      } else {
        uf = ar.alloc(n_in);
        run("disc_up", 0.0, [&] { return femasr_bilinear_up2(src, uf, B, hl, wl, ci, st); });
        g.x = uf;
      }
      ar.release(cur);
      cur = nullptr;
      if (lv == 0 && tc) {
        p_hi = ar.alloc((n_out + 1) / 2); p_lo = ar.alloc((n_out + 1) / 2);
        g.o_hi = p_hi; g.o_lo = p_lo;
      } else {
        cur = ar.alloc(n_out);
        g.y = cur;
      }
      conv(g);
      if (tc) { ar.release(ulo); ar.release(uhi); } else { ar.release(uf); }
      ar.release(xs[lv]);
    }
    // conv7, conv8 (3x3 F -> F), then conv9 (3x3 F -> 1, bias) on the out_conv kernels
    const size_t nf = (size_t)B * H * W * F;
    ConvDesc g7 = sn_conv(7, H, W, F, F, 3), g8 = sn_conv(8, H, W, F, F, 3);
    float* x8 = ar.alloc(nf);
    if (tc) {
      void* q_hi = ar.alloc((nf + 1) / 2);
      void* q_lo = ar.alloc((nf + 1) / 2);
      g7.a_hi = p_hi; g7.a_lo = p_lo; g7.o_hi = q_hi; g7.o_lo = q_lo;
      conv(g7);
      ar.release(p_lo); ar.release(p_hi);
      g8.a_hi = q_hi; g8.a_lo = q_lo; g8.y = x8;
      conv(g8);
      ar.release(q_lo); ar.release(q_hi);
    } else {
      float* x7 = ar.alloc(nf);
      g7.x = cur; g7.y = x7;
      conv(g7);
      ar.release(cur);
      g8.x = x7; g8.y = x8;
      conv(g8);
      ar.release(x7);
    }
    const float *w9 = P("conv9.weight"), *b9 = P("conv9.bias");
    run("disc_head", 2.0 * 9 * F * (double)B * H * W,
        [&] { return femasr_out_conv3x3_n(x8, w9, b9, y_nchw, B, H, W, F, 1, tc ? 1 : 0, st); });
    ar.release(x8);
    precise_region = false;
  }
};

static int check_geometry(femasr_net* net, int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return fail(FEMASR_ERR_ARG, "forward: empty input");
  if (net->hq) {
    if (H % 8 || W % 8) return fail(FEMASR_ERR_ARG, "forward (HQ stage): H and W must be multiples of 8");
    return FEMASR_OK;
  }
  const int div = net->cfg.scale_factor == 4 ? 2 : 4;
  if (H % 2 || W % 2) return fail(FEMASR_ERR_ARG, "forward: H and W must be even");
  const int hs = H / div, ws = W / div;
  if (H % div || W % div || hs % 8 || ws % 8 || hs == 0 || ws == 0)
    return fail(FEMASR_ERR_ARG, "forward: Swin stage (H/" + std::to_string(div) + " x W/" + std::to_string(div) +
                                    ") must be a non-empty multiple of the 8x8 window");
  return FEMASR_OK;
}

// the semantic loss exists where ReLU(conv_semantic(z_quant)) [B,512,h,w] meets relu4_4 [B,512,H/8,W/8] at every
// quantising level; elsewhere the reference raises from conv_semantic (channels) or mse_loss (sizes)
static int check_semantic(femasr_net* net, int H, int W) {
  if (!net->semantic) return fail(FEMASR_ERR_STATE, "forward_sem: the net was created without femasr_net_enable_semantic");
  const int div = net->hq ? 8 : (net->cfg.scale_factor == 4 ? 2 : 4);
  const std::string vgg = "relu4_4 is [B,512," + std::to_string(H / 8) + "," + std::to_string(W / 8) + "]";
  for (size_t k = 0; k < net->cbs.size(); ++k) {
    const femasr_net::Codebook& cb = net->cbs[k];
    const int m = cb.scale / 32, zh = H / div * m, zw = W / div * m;
    const std::string z = "[B," + std::to_string(cb.e_dim) + "," + std::to_string(zh) + "," + std::to_string(zw) + "]";
    if (cb.e_dim != 512)
      return fail(FEMASR_ERR_ARG, "semantic loss: conv_semantic takes 512 channels but z_quant of codebook " +
                                      std::to_string(k) + " is " + z + "; " + vgg);
    if (zh != H / 8 || zw != W / 8)
      return fail(FEMASR_ERR_ARG, "semantic loss: ReLU(conv_semantic(z_quant)) of codebook " + std::to_string(k) + " is " + z +
                                      " but " + vgg);
  }
  return FEMASR_OK;
}

static int workspace_impl(femasr_net* net, int B, int H, int W, bool with_sem, size_t* bytes) {
  int s = check_geometry(net, B, H, W);
  if (s) return s;
  if (with_sem && (s = check_semantic(net, H, W))) return s;
  Ctx c(net, nullptr, 0, nullptr);
  if (with_sem) c.sem_loss = reinterpret_cast<float*>(uintptr_t(8));
  // sized for the gt_indices loss branch too (its scratch is small): one workspace serves forward and forward_gt
  c.forward(nullptr, nullptr, nullptr, nullptr, reinterpret_cast<const int64_t*>(uintptr_t(8)), B, H, W);
  *bytes = c.bytes_needed();
  return c.status;
}

// cudaMalloc on the first set_param of a parameter; later calls repack into the same buffer
template <class T>
static int ensure(T** p, size_t bytes) {
  if (!*p) FEMASR_CUDA(cudaMalloc(reinterpret_cast<void**>(p), bytes));
  return FEMASR_OK;
}

// Packs every device form pi lists into d, from the fp32 tensor src in the reference layout (d.raw, or for a
// spectral-norm layer weight_orig / sigma).
static int pack_forms(femasr_net* net, DevParam& d, const ParamInfo& pi, const float* src, cudaStream_t st) {
  int s = FEMASR_OK;
  const unsigned f = pi.forms;
  const int co = pi.Cout, ci = pi.Cin, k = pi.k;
  const size_t tcb = femasr_tc_weight_bytes(co, ci, k, k), upb = femasr_tc_weight_bytes(4 * co, ci, 2, 2);
  if ((f & FORM_KMAJOR) && ((s = ensure(&d.packed, pi.numel * sizeof(float))) || (s = femasr_pack_weight(src, d.packed, co, ci, k, k, st))))
    return s;
  if (f & FORM_IM2COL) {
    // the im2col GEMM's weight: the [Cout][kp] zero-padded matrix (K = 48 for in_conv, 27 for VGG conv1_1 and the
    // discriminator's conv0, 363 for AlexNet's conv1), packed for this net's GEMM path
    const bool tc = net->cfg.gemm_path == 1;
    const int kp = im2col_k(k);
    float* tmp = nullptr;
    FEMASR_CUDA(cudaMallocAsync(&tmp, (size_t)co * kp * sizeof(float), st));
    s = k == 4 ? femasr_in_conv_pad_weight(src, tmp, co, st) : femasr_vgg_pad_weight_ex(src, tmp, co, k, kp, st);
    if (!s) s = ensure(&d.im2col, tc ? femasr_tc_weight_bytes(co, kp, 1, 1) : (size_t)co * kp * sizeof(float));
    if (!s) s = tc ? femasr_tc_pack_weight(tmp, d.im2col, co, kp, 1, 1, st)
                   : femasr_pack_weight(tmp, static_cast<float*>(d.im2col), co, kp, 1, 1, st);
    cudaFreeAsync(tmp, st);
    if (s) return s;
  }
  if ((f & FORM_TC) && ((s = ensure(&d.tc, tcb)) || (s = femasr_tc_pack_weight(src, d.tc, co, ci, k, k, st)))) return s;
  if ((f & FORM_TC8) && ((s = ensure(&d.tc8, tcb)) || (s = femasr_tc_pack_weight_f8(src, d.tc8, co, ci, k, k, st)))) return s;
  if ((f & FORM_UP) && ((s = ensure(&d.up, upb)) || (s = femasr_tc_pack_weight_up2(src, d.up, co, ci, st)))) return s;
  if ((f & FORM_UP8) && ((s = ensure(&d.up8, upb)) || (s = femasr_tc_pack_weight_up2_f8(src, d.up8, co, ci, st)))) return s;
  if ((f & FORM_RELB) &&
      ((s = ensure(&d.packed, 8 * 64 * 64 * sizeof(float))) || (s = ensure(&d.relb_mma, 8 * 64 * 64 * sizeof(float))) ||
       (s = femasr_expand_rel_bias_mma(src, d.relb_mma, 8, st)) || (s = femasr_expand_rel_bias(src, d.packed, 8, st))))
    return s;
  if ((f & FORM_ESQ) && ((s = ensure(&d.esq, co * sizeof(float))) || (s = femasr_row_sumsq(src, d.esq, co, ci, st)))) return s;
  return FEMASR_OK;
}

// Spectral-norm layer l (eval mode, torch.nn.utils.spectral_norm): once weight_orig, weight_u and weight_v are all set,
// sigma = u . (W v) and the layer's forms are packed from weight_orig / sigma.  The host copy of {sigma, |W v|} feeds
// the gemm_path 1 range check of femasr_disc_forward.
static int sn_pack(femasr_net* net, const std::string& l, cudaStream_t st) {
  auto w = net->dev.find(l + ".weight_orig"), u = net->dev.find(l + ".weight_u"), v = net->dev.find(l + ".weight_v");
  if (w == net->dev.end() || u == net->dev.end() || v == net->dev.end()) return FEMASR_OK;
  const ParamInfo& pi = net->spec.at(l + ".weight_orig");
  DevParam& d = w->second;
  int s = ensure(&d.sigma, 2 * sizeof(float));
  if (s) return s;
  float* wn = nullptr;
  FEMASR_CUDA(cudaMallocAsync(&wn, pi.numel * sizeof(float), st));
  s = femasr_spectral_sigma(d.raw, u->second.raw, v->second.raw, pi.Cout, (int)(pi.numel / pi.Cout), d.sigma, st);
  if (!s) s = femasr_spectral_normalize(d.raw, d.sigma, wn, pi.numel, st);
  if (!s) s = pack_forms(net, d, pi, wn, st);
  cudaFreeAsync(wn, st);
  if (s) return s;
  FEMASR_CUDA(cudaMemcpyAsync(d.sn, d.sigma, 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
  FEMASR_CUDA(cudaStreamSynchronize(st));
  return FEMASR_OK;
}

static int check_disc_geometry(int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return fail(FEMASR_ERR_ARG, "disc: empty input");
  if (H % 8 || W % 8)
    return fail(FEMASR_ERR_ARG, "disc: H and W must be multiples of 8 (three stride-2 convs, then x2 upsamples that must "
                                "meet the skip tensors; the reference raises at the skip add)");
  return FEMASR_OK;
}

// Study knobs read from the environment at create time (every kind of handle)
static void read_knobs(femasr_net* n) {
  if (const char* ev = getenv("FEMASR_TC_PRECISE")) n->tc_precise = atoi(ev) != 0;
  if (const char* ev = getenv("FEMASR_FAST_SILU")) n->fast_silu = atoi(ev) != 0;
  if (const char* ev = getenv("FEMASR_VQ_FUSED")) n->vq_fused = atoi(ev) != 0;
  if (const char* ev = getenv("FEMASR_F8_CROSS")) n->f8_cross = atoi(ev) != 0;
  if (const char* ev = getenv("FEMASR_TC_SLICE_KB")) n->tc_slice_kb = std::max(1, atoi(ev));
  if (const char* ev = getenv("FEMASR_SEM_SLICE_KB")) n->sem_slice_kb = std::max(0, atoi(ev));
}

}  // namespace femasr

extern "C" const char* femasr_last_error(void) { return g_err.c_str(); }
extern "C" int femasr_abi_version(void) { return 4; }   // 3: fused VQ + im2col in_conv entries; 4: femasr_tc_args.f8 + the F8 staging / packing entries

extern "C" int femasr_device_cc(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(FEMASR_ERR_NO_DEVICE, "no CUDA device");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return fail(FEMASR_ERR_NO_DEVICE, "no CUDA device");
  return prop.major * 10 + prop.minor;
}

extern "C" int femasr_net_create(const femasr_net_config* cfg, femasr_net** out) {
  FEMASR_CHECK_ARG(cfg && out, "net_create: null pointer");
  FEMASR_CHECK_ARG(cfg->scale_factor == 1 || cfg->scale_factor == 2 || cfg->scale_factor == 4,
                   "net_create: scale_factor must be 4, 2 (LQ stage) or 1 (HQ autoencoder stage)");
  FEMASR_CHECK_ARG(cfg->in_channel == 3, "net_create: in_channel must be 3");
  FEMASR_CHECK_ARG(cfg->gemm_path == 0 || cfg->gemm_path == 1, "net_create: gemm_path must be 0 or 1");
  FEMASR_CHECK_ARG(cfg->n_codebooks >= 0 && cfg->n_codebooks <= FEMASR_MAX_CODEBOOKS, "net_create: at most 3 codebooks");
  std::vector<femasr_net::Codebook> cbs;
  if (cfg->n_codebooks <= 1 && !(cfg->n_codebooks == 1 && cfg->cb_scale[0]))
    cbs.push_back({32, cfg->n_e, cfg->e_dim});
  else
    for (int k = 0; k < cfg->n_codebooks; ++k) cbs.push_back({cfg->cb_scale[k], cfg->cb_n_e[k], cfg->cb_e_dim[k]});
  FEMASR_CHECK_ARG(cbs[0].scale == 32, "net_create: the first codebook must be at scale 32 (femasr_arch.py:255-256)");
  for (size_t k = 0; k < cbs.size(); ++k) {
    FEMASR_CHECK_ARG(cbs[k].e_dim > 0 && cbs[k].e_dim % 64 == 0 && cbs[k].e_dim <= 1024, "net_create: e_dim must be a multiple of 64");
    FEMASR_CHECK_ARG(cbs[k].n_e > 0 && cbs[k].n_e % 64 == 0, "net_create: n_e must be a multiple of 64");
    FEMASR_CHECK_ARG(k == 0 || ((cbs[k].scale == 64 || cbs[k].scale == 128) && cbs[k].scale > cbs[k - 1].scale),
                     "net_create: further codebooks must sit at increasing scales out of 64, 128");
  }
  femasr_net* n = new femasr_net();
  n->cfg = *cfg;
  n->cfg.n_e = cbs[0].n_e; n->cfg.e_dim = cbs[0].e_dim;
  n->cbs = cbs;
  for (size_t k = 0; k < cbs.size(); ++k) {
    const int lvl = cbs[k].scale == 32 ? 0 : (cbs[k].scale == 64 ? 1 : 2);
    n->level_cb[lvl] = (int)k;
    n->last_q_level = lvl;
  }
  n->depth = cfg->scale_factor == 4 ? 1 : (cfg->scale_factor == 2 ? 2 : 3);
  n->hq = cfg->scale_factor == 1;
  read_knobs(n);
  build_spec(n);
  *out = n;
  return FEMASR_OK;
}

extern "C" void femasr_net_destroy(femasr_net* net) { delete net; }

extern "C" int femasr_net_enable_semantic(femasr_net* net) {
  FEMASR_CHECK_ARG(net, "enable_semantic: null");
  FEMASR_CHECK_ARG(generator(net), "enable_semantic: a discriminator or LPIPS handle");
  if (net->semantic) return FEMASR_OK;
  if (!net->dev.empty()) return fail(FEMASR_ERR_STATE, "enable_semantic: call it before the first set_param");
  add_semantic(net);
  net->semantic = true;
  return FEMASR_OK;
}

// Copies the parameter and packs every device form its ParamInfo lists.
extern "C" int femasr_net_set_param(femasr_net* net, const char* name, const float* data, size_t numel, int on_device,
                                    void* stream) {
  FEMASR_CHECK_ARG(net && name && data, "set_param: null pointer");
  auto it = net->spec.find(name);
  if (it == net->spec.end()) return fail(FEMASR_ERR_ARG, std::string("set_param: unknown parameter ") + name);
  const ParamInfo& pi = it->second;
  if (pi.numel != numel) return fail(FEMASR_ERR_ARG, std::string("set_param: wrong size for ") + name);
  cudaStream_t st = as_stream(stream);
  DevParam& d = net->dev[name];
  int s = ensure(&d.raw, numel * sizeof(float));
  if (s) return s;
  FEMASR_CUDA(cudaMemcpyAsync(d.raw, data, numel * sizeof(float), on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  if (!on_device) FEMASR_CUDA(cudaStreamSynchronize(st));   // the host buffer may be pageable / freed by the caller
  if (!pi.sn.empty()) return sn_pack(net, pi.sn, st);
  return pack_forms(net, d, pi, d.raw, st);
}

extern "C" int femasr_net_params_complete(femasr_net* net) {
  FEMASR_CHECK_ARG(net, "params_complete: null");
  for (auto& kv : net->spec)
    if (net->dev.find(kv.first) == net->dev.end()) return fail(FEMASR_ERR_STATE, "parameter not set: " + kv.first);
  return FEMASR_OK;
}

extern "C" int femasr_net_workspace_bytes(femasr_net* net, int B, int H, int W, size_t* bytes) {
  FEMASR_CHECK_ARG(net && bytes, "workspace_bytes: null pointer");
  FEMASR_CHECK_ARG(generator(net), "workspace_bytes: a discriminator or LPIPS handle");
  return workspace_impl(net, B, H, W, false, bytes);
}

extern "C" int femasr_net_workspace_bytes_sem(femasr_net* net, int B, int H, int W, int with_sem, size_t* bytes) {
  FEMASR_CHECK_ARG(net && bytes, "workspace_bytes_sem: null pointer");
  FEMASR_CHECK_ARG(generator(net), "workspace_bytes_sem: a discriminator or LPIPS handle");
  return workspace_impl(net, B, H, W, with_sem != 0, bytes);
}

extern "C" int femasr_net_forward(femasr_net* net, const float* x, float* y, int64_t* indices, float* cb_loss, int B,
                                  int H, int W, void* workspace, size_t workspace_bytes, void* stream) {
  return femasr_net_forward_gt(net, x, y, indices, cb_loss, nullptr, B, H, W, workspace, workspace_bytes, stream);
}

extern "C" int femasr_net_forward_gt(femasr_net* net, const float* x, float* y, int64_t* indices, float* cb_loss,
                                     const int64_t* gt_indices, int B, int H, int W, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  return femasr_net_forward_sem(net, x, y, indices, cb_loss, gt_indices, nullptr, B, H, W, workspace, workspace_bytes, stream);
}

extern "C" int femasr_net_forward_sem(femasr_net* net, const float* x, float* y, int64_t* indices, float* cb_loss,
                                      const int64_t* gt_indices, float* sem_loss, int B, int H, int W, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  FEMASR_CHECK_ARG(net && x && y && workspace, "forward: null pointer");
  FEMASR_CHECK_ARG(generator(net), "forward: a discriminator or LPIPS handle (use femasr_disc_forward / femasr_lpips_forward)");
  int s = check_geometry(net, B, H, W);
  if (s) return s;
  s = femasr_net_params_complete(net);
  if (s) return s;
  size_t need = 0;
  s = workspace_impl(net, B, H, W, sem_loss != nullptr, &need);
  if (s) return s;
  if (workspace_bytes < need) return fail(FEMASR_ERR_STATE, "forward: workspace too small (need " + std::to_string(need) + " bytes)");
  Ctx c(net, workspace, workspace_bytes, stream);
  c.sem_loss = sem_loss;
  c.forward(x, y, indices, cb_loss, gt_indices, B, H, W);
  return c.finish();
}

extern "C" int femasr_net_decode_workspace_bytes(femasr_net* net, int B, int h, int w, size_t* bytes) {
  FEMASR_CHECK_ARG(net && bytes && B > 0 && h > 0 && w > 0, "decode_workspace_bytes: bad argument");
  FEMASR_CHECK_ARG(generator(net), "decode_workspace_bytes: a discriminator or LPIPS handle");
  Ctx c(net, nullptr, 0, nullptr);
  c.decode_indices(nullptr, nullptr, B, h, w);
  *bytes = c.bytes_needed();
  return c.status;
}

extern "C" int femasr_net_decode_indices(femasr_net* net, const int64_t* indices, float* y, int B, int h, int w,
                                         void* workspace, size_t workspace_bytes, void* stream) {
  FEMASR_CHECK_ARG(net && indices && y && workspace && B > 0 && h > 0 && w > 0, "decode_indices: bad argument");
  FEMASR_CHECK_ARG(generator(net), "decode_indices: a discriminator or LPIPS handle");
  int s = femasr_net_params_complete(net);
  if (s) return s;
  size_t need = 0;
  s = femasr_net_decode_workspace_bytes(net, B, h, w, &need);
  if (s) return s;
  if (workspace_bytes < need) return fail(FEMASR_ERR_STATE, "decode_indices: workspace too small");
  Ctx c(net, workspace, workspace_bytes, stream);
  c.decode_indices(indices, y, B, h, w);
  return c.finish();
}

extern "C" int femasr_net_set_tap(femasr_net* net, const char* stage, float* dst, size_t capacity) {
  FEMASR_CHECK_ARG(net && stage, "set_tap: null pointer");
  FEMASR_CHECK_ARG(generator(net), "set_tap: a discriminator or LPIPS handle");
  static const char* names[] = {"in_conv", "down", "swin", "up1", "up2", "z", "zq", "after_quant", "dec0", "dec1", "dec2", "z1", "z2",
                                "vgg", "semantic"};
  bool known = false;
  for (const char* n : names) known = known || strcmp(n, stage) == 0;
  if (!known) return fail(FEMASR_ERR_ARG, std::string("set_tap: unknown stage ") + stage);
  if (dst) net->taps[stage] = Tap{dst, capacity};
  else net->taps.erase(stage);
  return FEMASR_OK;
}

extern "C" int femasr_net_last_launch_count(femasr_net* net) { return net ? net->last_launches : 0; }

extern "C" int femasr_net_set_profile(femasr_net* net, int enable) {
  FEMASR_CHECK_ARG(net, "set_profile: null");
  for (auto& r : net->prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
  net->prof.clear();
  net->profile = enable != 0;
  return FEMASR_OK;
}

// JSON {"kernel": {"launches": n, "ms": total, "flops": total}, ...} of the launches recorded since
// femasr_net_set_profile(net, 1).  Synchronises on the recorded events.
extern "C" const char* femasr_net_profile_json(femasr_net* net) {
  if (!net) return "{}";
  struct Agg { long n = 0; double ms = 0, flops = 0; };
  std::map<std::string, Agg> agg;
  for (auto& r : net->prof) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.e1) != cudaSuccess || cudaEventElapsedTime(&ms, r.e0, r.e1) != cudaSuccess) continue;
    Agg& a = agg[r.name];
    a.n += 1; a.ms += ms; a.flops += r.flops;
  }
  std::string js = "{";
  bool first = true;
  for (auto& kv : agg) {
    char buf[256];
    snprintf(buf, sizeof(buf), "%s\"%s\": {\"launches\": %ld, \"ms\": %.6f, \"flops\": %.6e}", first ? "" : ", ",
             kv.first.c_str(), kv.second.n, kv.second.ms, kv.second.flops);
    js += buf;
    first = false;
  }
  js += "}";
  net->prof_json = js;
  return net->prof_json.c_str();
}

// The sum of the algorithmic FLOPs the launches of one plain forward report (no taps, no gt_indices, no semantic loss),
// counted by a sizing run; 0 for a geometry forward rejects.
extern "C" double femasr_net_flops(femasr_net* net, int B, int H, int W) {
  if (!net || !generator(net) || check_geometry(net, B, H, W)) return 0.0;
  std::map<std::string, Tap> taps;
  taps.swap(net->taps);          // a registered in_conv tap adds the fp32 in_conv to the tensor-core plan
  Ctx c(net, nullptr, 0, nullptr);
  c.forward(nullptr, nullptr, nullptr, nullptr, nullptr, B, H, W);
  taps.swap(net->taps);
  return c.flops;
}

// ------------------------------------------------------------------------------------------------ UNetDiscriminatorSN
extern "C" int femasr_disc_create(const femasr_disc_config* cfg, femasr_net** out) {
  FEMASR_CHECK_ARG(cfg && out, "disc_create: null pointer");
  FEMASR_CHECK_ARG(cfg->num_in_ch == 3, "disc_create: num_in_ch must be 3");
  FEMASR_CHECK_ARG(cfg->num_feat == 64, "disc_create: num_feat must be 64 (conv9 runs on the Cin = 64 head kernels)");
  FEMASR_CHECK_ARG(cfg->skip_connection == 0 || cfg->skip_connection == 1, "disc_create: skip_connection must be 0 or 1");
  FEMASR_CHECK_ARG(cfg->gemm_path == 0 || cfg->gemm_path == 1, "disc_create: gemm_path must be 0 or 1");
  femasr_net* n = new femasr_net();
  n->cfg = femasr_net_config{};
  n->cfg.gemm_path = cfg->gemm_path;
  n->disc = true;
  n->dcfg = *cfg;
  read_knobs(n);
  build_disc_spec(n);
  *out = n;
  return FEMASR_OK;
}

extern "C" int femasr_disc_workspace_bytes(femasr_net* net, int B, int H, int W, size_t* bytes) {
  FEMASR_CHECK_ARG(net && bytes, "disc_workspace_bytes: null pointer");
  FEMASR_CHECK_ARG(net->disc, "disc_workspace_bytes: not a discriminator handle");
  int s = check_disc_geometry(B, H, W);
  if (s) return s;
  Ctx c(net, nullptr, 0, nullptr);
  c.disc(nullptr, nullptr, B, H, W);
  *bytes = c.bytes_needed();
  return c.status;
}

extern "C" int femasr_disc_forward(femasr_net* net, const float* x, float* y, int B, int H, int W, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  FEMASR_CHECK_ARG(net && x && y && workspace, "disc_forward: null pointer");
  FEMASR_CHECK_ARG(net->disc, "disc_forward: not a discriminator handle");
  int s = check_disc_geometry(B, H, W);
  if (s) return s;
  s = femasr_net_params_complete(net);
  if (s) return s;
  if (net->cfg.gemm_path == 1) {
    // u never power-iterated: sigma = u.(W v) is a small fraction of the spectral norm, the normalised weights are large
    // and the activations leave the fp16 operand range (a finite reference result would come back as inf)
    for (auto& kv : net->spec) {
      if (kv.second.sn.empty() || kv.first != kv.second.sn + ".weight_orig") continue;
      const float* sn = net->dev.at(kv.first).sn;
      if (!(sn[0] >= 0.5f * sn[1]))
        return fail(FEMASR_ERR_STATE, kv.second.sn + ": u.(W v) = " + std::to_string(sn[0]) + " is below half of |W v| = " +
                                          std::to_string(sn[1]) + ": weight_u / weight_v were never power-iterated, and " +
                                          "gemm_path 1's fp16 operands cannot hold the activations; use gemm_path 0 or "
                                          "iterated u, v (as a trained checkpoint carries)");
    }
  }
  size_t need = 0;
  s = femasr_disc_workspace_bytes(net, B, H, W, &need);
  if (s) return s;
  if (workspace_bytes < need) return fail(FEMASR_ERR_STATE, "disc_forward: workspace too small (need " + std::to_string(need) + " bytes)");
  Ctx c(net, workspace, workspace_bytes, stream);
  c.disc(x, y, B, H, W);
  return c.finish();
}

// The sum of the algorithmic FLOPs of one femasr_disc_forward's launches, counted by a sizing run; 0 for a rejected
// geometry or a generator handle.
extern "C" double femasr_disc_flops(femasr_net* net, int B, int H, int W) {
  if (!net || !net->disc || check_disc_geometry(B, H, W)) return 0.0;
  Ctx c(net, nullptr, 0, nullptr);
  c.disc(nullptr, nullptr, B, H, W);
  return c.flops;
}

// ------------------------------------------------------------------------------------------------ LPIPS
static int check_lpips_geometry(femasr_net* net, int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return fail(FEMASR_ERR_ARG, "lpips: empty input");
  const std::string got = " (got " + std::to_string(H) + "x" + std::to_string(W) + ")";
  if (net->lcfg.net == 1 && (H % 16 || W % 16))
    return fail(FEMASR_ERR_ARG, "lpips (vgg): H and W must be multiples of 16, so that each of the four 2x2 max-pools is exact" + got);
  if (net->lcfg.net == 0 && (H < 31 || W < 31))
    return fail(FEMASR_ERR_ARG, "lpips (alex): H and W must be at least 31, the smallest input AlexNet's features accept" + got);
  return FEMASR_OK;
}

extern "C" int femasr_lpips_create(const femasr_lpips_config* cfg, femasr_net** out) {
  FEMASR_CHECK_ARG(cfg && out, "lpips_create: null pointer");
  FEMASR_CHECK_ARG(cfg->net == 0 || cfg->net == 1, "lpips_create: net must be 0 (alex) or 1 (vgg)");
  FEMASR_CHECK_ARG(cfg->gemm_path == 0 || cfg->gemm_path == 1, "lpips_create: gemm_path must be 0 or 1");
  femasr_net* n = new femasr_net();
  n->cfg = femasr_net_config{};
  n->cfg.gemm_path = cfg->gemm_path;
  n->lpips = true;
  n->lcfg = *cfg;
  read_knobs(n);
  build_lpips_spec(n);
  *out = n;
  return FEMASR_OK;
}

extern "C" int femasr_lpips_workspace_bytes(femasr_net* net, int B, int H, int W, size_t* bytes) {
  FEMASR_CHECK_ARG(net && bytes, "lpips_workspace_bytes: null pointer");
  FEMASR_CHECK_ARG(net->lpips, "lpips_workspace_bytes: not an LPIPS handle");
  int s = check_lpips_geometry(net, B, H, W);
  if (s) return s;
  Ctx c(net, nullptr, 0, nullptr);
  c.lpips(nullptr, nullptr, nullptr, nullptr, B, H, W, 0);
  *bytes = c.bytes_needed();
  return c.status;
}

extern "C" int femasr_lpips_forward(femasr_net* net, const float* x0, const float* x1, float* dist, float* per_layer, int B,
                                    int H, int W, int normalize, void* workspace, size_t workspace_bytes, void* stream) {
  FEMASR_CHECK_ARG(net && x0 && x1 && dist && workspace, "lpips_forward: null pointer");
  FEMASR_CHECK_ARG(net->lpips, "lpips_forward: not an LPIPS handle");
  int s = check_lpips_geometry(net, B, H, W);
  if (s) return s;
  s = femasr_net_params_complete(net);
  if (s) return s;
  size_t need = 0;
  s = femasr_lpips_workspace_bytes(net, B, H, W, &need);
  if (s) return s;
  if (workspace_bytes < need) return fail(FEMASR_ERR_STATE, "lpips_forward: workspace too small (need " + std::to_string(need) + " bytes)");
  Ctx c(net, workspace, workspace_bytes, stream);
  c.lpips(x0, x1, dist, per_layer, B, H, W, normalize);
  return c.finish();
}

// The sum of the algorithmic FLOPs of one femasr_lpips_forward's launches (both images of every pair), counted by a sizing
// run; 0 for a rejected geometry or another kind of handle.
extern "C" double femasr_lpips_flops(femasr_net* net, int B, int H, int W) {
  if (!net || !net->lpips || check_lpips_geometry(net, B, H, W)) return 0.0;
  Ctx c(net, nullptr, 0, nullptr);
  c.lpips(nullptr, nullptr, nullptr, nullptr, B, H, W, 0);
  return c.flops;
}
