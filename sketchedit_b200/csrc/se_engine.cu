// Host side of the library: weight packing, the generator forward graph, the C ABI
// (include/sketchedit_b200.h). Graph structure follows
//   MDGenerator.forward            reference models/networks/editline2_g.py:59-94
//   DeepFillC2Generator.forward    reference models/networks/editline_g.py:119-221
//   EditLine2Model inference       reference models/editline2_model.py:128-133,338-370
#include <stdlib.h>

#include <cuda_fp16.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_conv_direct.h"
#include "se_conv_c8.h"
#include "se_cam.h"
#include "se_gemm_split.h"
#include "se_conv_tc.h"
#include "se_misc.h"
#include "se_detail.h"

namespace se {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const char* last_error() { return g_err.c_str(); }

static thread_local int g_launches = 0;

// bytes the contextual attention's quadratic temporaries (probabilities, logits) may take; se_set_attention_workspace_limit
constexpr long long kDefaultAttnLimit = 16LL << 30;
static std::atomic<long long> g_attn_limit{kDefaultAttnLimit};

// ------------------------------------------------------------------------------------------ launch timing
// se_timing_enable(1): every launch of a forward is bracketed by CUDA events on its stream and accounted to a kernel
// class (kernel + layer shape) together with its ALGORITHMIC work: 2*MAC of the reference op (SURVEY.md 8d), the MACs
// this implementation really issues (sub-pixel deconvs: 4/9 of the reference's), and the bytes the op must move (input
// once, output once, weights once). bench.py runs ONE instrumented pass for the roofline table; the throughput passes
// run with timing off. Process-wide, guarded by a mutex.
struct TimedLaunch { cudaEvent_t a, b; int cls; };
struct ClassAgg { std::string name; int tensor; double flops_alg, flops_exec, bytes_alg; int launches; double ms; };
static std::mutex g_time_mu;
static bool g_timing = false;
static std::vector<TimedLaunch> g_tl;
static size_t g_tl_used = 0;
static std::vector<ClassAgg> g_classes;
static std::map<std::string, int> g_class_idx;

struct LaunchTag {
  std::string name;
  int tensor = 0;
  double flops_alg = 0, flops_exec = 0, bytes_alg = 0;
  bool set = false;
};

static int timing_begin(const LaunchTag& t, cudaStream_t st, size_t* slot) {
  std::lock_guard<std::mutex> lk(g_time_mu);
  const std::string key = t.set ? t.name : std::string("other");
  auto it = g_class_idx.find(key);
  int ci;
  if (it == g_class_idx.end()) {
    ci = (int)g_classes.size();
    g_class_idx[key] = ci;
    g_classes.push_back(ClassAgg{key, t.tensor, 0, 0, 0, 0, 0});
  } else ci = it->second;
  ClassAgg& a = g_classes[ci];
  a.flops_alg += t.flops_alg; a.flops_exec += t.flops_exec; a.bytes_alg += t.bytes_alg; a.launches += 1;
  if (g_tl_used == g_tl.size()) {
    TimedLaunch tl;
    SE_CUDA_OK(cudaEventCreate(&tl.a));
    SE_CUDA_OK(cudaEventCreate(&tl.b));
    g_tl.push_back(tl);
  }
  *slot = g_tl_used++;
  g_tl[*slot].cls = ci;
  SE_CUDA_OK(cudaEventRecord(g_tl[*slot].a, st));
  return 0;
}
static int timing_end(size_t slot, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_time_mu);
  SE_CUDA_OK(cudaEventRecord(g_tl[slot].b, st));
  return 0;
}

// ------------------------------------------------------------------------------------------ architecture
struct Spec {
  int cin, cout, k, stride, rate;
  bool deconv;
  int act;   // 0 elu, 1 relu, -1 none
};

struct ArchTable {
  std::vector<std::string> names;
  std::vector<Spec> specs;
  void add(const std::string& n, int ci, int co, int k = 3, int s = 1, int r = 1, bool deconv = false, int act = 0) {
    if (co == 3) act = -1;   // reference utils.py:27
    names.push_back(n);
    specs.push_back(Spec{ci, co, k, s, r, deconv, act});
  }
  void add_encoder(const std::string& pfx, int cin0) {
    const int c = 48;
    add(pfx + "conv1", cin0, c, 5);
    add(pfx + "conv2_downsample", c / 2, 2 * c, 3, 2);
    add(pfx + "conv3", c, 2 * c);
    add(pfx + "conv4_downsample", c, 4 * c, 3, 2);
    add(pfx + "conv5", 2 * c, 4 * c);
    add(pfx + "conv6", 2 * c, 4 * c);
    add(pfx + "conv7_atrous", 2 * c, 4 * c, 3, 1, 2);
    add(pfx + "conv8_atrous", 2 * c, 4 * c, 3, 1, 4);
    add(pfx + "conv9_atrous", 2 * c, 4 * c, 3, 1, 8);
    add(pfx + "conv10_atrous", 2 * c, 4 * c, 3, 1, 16);
  }
  void add_decoder(const std::string& pfx, int cin11, int cout17) {
    const int c = 48;
    add(pfx + "11", cin11, 4 * c);
    add(pfx + "12", 2 * c, 4 * c);
    add(pfx + "13_upsample_conv", 2 * c, 2 * c, 3, 1, 1, true);
    add(pfx + "14", c, 2 * c);
    add(pfx + "15_upsample_conv", c, c, 3, 1, 1, true);
    add(pfx + "16", c / 2, c / 2);
    add(pfx + "17", c / 4, cout17, 3, 1, 1, false, -1);
  }
};

static ArchTable make_arch(char net) {
  ArchTable t;
  const int c = 48;
  if (net == 'M') {
    t.add_encoder("", 4);
    t.add_decoder("conv", 2 * c, 3);
    t.add_decoder("conv_mask_", 2 * c, 1);
  } else {
    t.add_encoder("", 5);
    t.add_decoder("conv", 4 * c, 3);
    t.add_encoder("w", 5);
    t.add("xconv1", 3, c, 5);
    t.add("xconv2_downsample", c / 2, c, 3, 2);
    t.add("xconv3", c / 2, 2 * c);
    t.add("xconv4_downsample", c, 2 * c, 3, 2);
    t.add("xconv5", c, 4 * c);
    t.add("xconv6", 2 * c, 4 * c);
    t.add("xconv7_atrous", 2 * c, 4 * c, 3, 1, 2);
    t.add("xconv8_atrous", 2 * c, 4 * c, 3, 1, 4);
    t.add("xconv9_atrous", 2 * c, 4 * c, 3, 1, 8);
    t.add("xconv10_atrous", 2 * c, 4 * c, 3, 1, 16);
    t.add("pmconv1", 3, c, 5);
    t.add("pmconv2_downsample", c / 2, c, 3, 2);
    t.add("pmconv3", c / 2, 2 * c);
    t.add("pmconv4_downsample", c, 4 * c, 3, 2);
    t.add("pmconv5", 2 * c, 4 * c);
    t.add("pmconv6", 2 * c, 4 * c, 3, 1, 1, false, 1);   // ReLU gate, editline_g.py:89-90
    t.add("pmconv9", 2 * c, 4 * c);
    t.add("pmconv10", 2 * c, 4 * c);
    t.add_decoder("allconv", 4 * c, 3);
  }
  return t;
}

// ------------------------------------------------------------------------------------------ packed layers
// the taps of one launch form: tap t reads the input at offset (dy, dx) from its position, starting at channel block cb
struct Taps {
  int n = 0;
  int8_t dy[MAX_TAPS] = {}, dx[MAX_TAPS] = {}, cb[MAX_TAPS] = {};
};

struct ClassW {
  Taps direct;                 // CUDA-core form (se_conv_direct.cu) over NHWC input
  float* w_direct = nullptr;   // device fp32 [tap][Ci][CoutP]
  int CoutP = 0;
  int osy = 1, ooy = 0, osx = 1, oox = 0;
  // channel-blocked wgmma forms (se_conv_c8.cu): every gated layer has them, the heads (CUDA-core only) do not
  bool tc = false;
  // stride-2 3x3 layers on the tensor-core path read a SPACE-TO-DEPTH channel-blocked input (written that way by
  // the producing layer's epilogue): tap (ky,kx) of output (y,x) reads input row 2y+ky-1 = row y+dy of parity
  // (ky-1)&1, i.e. a stride-1 read at offset (dy, dx) starting at channel block cb = parity * Ci/8
  bool s2d = false;
  Taps bf16;                   // bf16 form: the direct taps, in space-to-depth form on s2d layers
  C8Layer c8;
  // split-half twin (SE_PREC_FP32_TC, DT_F16X2): every tap becomes three virtual taps (x_hi, w_hi), (x_hi, w_lo), (x_lo, w_hi); a
  // virtual tap reads the hi or lo channel blocks of the input (cb) and its weight image holds fp16(w) or fp16(w - fp16(w))
  Taps split;
  C8Layer c8s;
  float s_wscale = 1.0f;   // power of two the split-half weight images are multiplied by
};

struct Layer {
  Spec spec;
  char net = 0;                // 'M' or 'G'
  std::string name;
  int Ci = 0;                  // stored input channels (stems are packed to 8)
  bool is_head = false;
  bool is_stem = false;
  bool set = false;
  std::vector<float> w_host, b_host;
  std::vector<ClassW> cls;
  std::vector<C8Group> groups; // deconv layers on the tensor-core path: sub-pixel classes fused per launch (se_conv_c8.h)
  int pair_cin_sum = 0;        // fused_pair: real input channels of the two source layers together (algorithmic FLOPs)
  bool fused_pair = false;     // two 5x5 stems over the same packed input fused along N (tensor-core path; see make_stem_pair)
  float* bias = nullptr;       // device [cout]
  std::vector<float> w_head_host;   // heads: host [9][12][cout], the head kernel's by-value weights are built from it
};

}  // namespace se

using namespace se;

struct se_model {
  std::map<std::string, Layer> layers;   // key = net + "." + name
  int opt[8] = {1, 0, 0, 0, 1, 0, 0, 0};
  bool finalized = false;
  void* arena = nullptr;
  size_t arena_bytes = 0;
  std::vector<void*> owned;              // device allocations of packed weights
  // one forward at a time per model (the workspace arena is shared by every call); the model lives on ONE device; a call
  // on another stream than the previous one waits for that stream's work on the arena first
  std::mutex mu;
  // whole-forward CUDA graphs, one per call signature (entry point, shape, precision, options, every pointer argument): the
  // ~85 launches of a forward (each with its tensor-map encodes) become one cudaGraphLaunch. A signature is captured the
  // second time it is seen (one-off calls stay eager); entries die with the arena they were captured on.
  struct GraphEntry { std::vector<uintptr_t> key; cudaGraphExec_t exec = nullptr; void* arena = nullptr; int launches = 0; unsigned long long tick = 0; };
  std::vector<GraphEntry> graphs;
  std::map<std::vector<uintptr_t>, int> seen;
  unsigned long long tick = 0;
  cudaStream_t gstream = nullptr;          // graphs cannot be captured on / launched into the legacy default stream: callers that pass it
  cudaEvent_t bridge_in = nullptr, bridge_out = nullptr;   // (torch's default) are bridged through this stream with two events
  int device = -1;
  cudaStream_t last_stream = nullptr;
  bool used = false;
  cudaEvent_t order_ev = nullptr;
  // activation taps (se_taps_enable): device copies of the stage inputs of the last forward, recorded by se::tap
  struct Tap { std::string name; int desc[SE_TAP_DESC_LEN] = {}; void* p = nullptr; size_t bytes = 0; };
  bool taps_on = false;
  std::vector<Tap> taps;
};

namespace se {

// 5x5 stems read an 8-channel packed input through overlapping 8-pixel windows: 64 virtual channels
// (pixel pitch 8 elements), see pack_layer / run_layer.
constexpr int STEM_PADL = 2;                       // zero pixels left of the image in the packed buffer
static inline int stem_wp(int W) { return W + 8; } // packed row length (2 left + 6 right zero pixels)
static int stored_ci(const Spec& s) { return s.k == 5 ? 64 : s.cin; }

static int upload(se_model* m, const void* host, size_t bytes, void** dev) {
  SE_CUDA_OK(cudaMalloc(dev, bytes));
  m->owned.push_back(*dev);
  SE_CUDA_OK(cudaMemcpy(*dev, host, bytes, cudaMemcpyHostToDevice));
  return 0;
}

static inline uint16_t f32_to_bf16_rn(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

// effective tap = sum of source taps (ky,kx) of the OIHW kernel (deconv parity classes merge taps)
// each source adds W[:, :, ky, kx] into the virtual input channels [ci_off, ci_off + cin)
struct SrcTap { int ky, kx, ci_off; };
struct EffTap { int dy, dx; std::vector<SrcTap> src; };

static int pack_class(se_model* m, Layer& L, const std::vector<EffTap>& taps, ClassW& cw) {
  const Spec& s = L.spec;
  const int Ci = L.Ci, Cout = s.cout, k = s.k;
  const int ntaps = (int)taps.size();
  SE_REQUIRE(ntaps <= MAX_TAPS, "too many taps");
  cw.direct.n = ntaps;
  cw.CoutP = (Cout + 3) / 4 * 4;
  std::vector<float> weff((size_t)ntaps * Ci * Cout, 0.0f);
  for (int t = 0; t < ntaps; ++t) {
    cw.direct.dy[t] = (int8_t)taps[t].dy;
    cw.direct.dx[t] = (int8_t)taps[t].dx;
    for (auto& sk : taps[t].src)
      for (int ci = 0; ci < s.cin; ++ci)
        for (int co = 0; co < Cout; ++co)
          weff[((size_t)t * Ci + sk.ci_off + ci) * Cout + co] += L.w_host[(((size_t)co * s.cin + ci) * k + sk.ky) * k + sk.kx];
  }
  {
    std::vector<float> wd((size_t)ntaps * Ci * cw.CoutP, 0.0f);
    for (int t = 0; t < ntaps; ++t)
      for (int ci = 0; ci < Ci; ++ci)
        for (int co = 0; co < Cout; ++co) wd[((size_t)t * Ci + ci) * cw.CoutP + co] = weff[((size_t)t * Ci + ci) * Cout + co];
    int rc = upload(m, wd.data(), wd.size() * 4, (void**)&cw.w_direct);
    if (rc) return rc;
  }
  cw.tc = !L.is_head;
  if (cw.tc) {
    cw.s2d = (s.stride == 2 && s.k == 3 && s.rate == 1 && !s.deconv && !L.is_stem);
    SE_REQUIRE(Ci % 8 == 0 && (s.stride == 1 || cw.s2d), "layer " + L.name + " has no tensor-core form");   // every gated layer of the two generators has one
    cw.bf16 = cw.direct;
    if (cw.s2d) {
      for (int t = 0; t < ntaps; ++t) {
        const int oy = cw.direct.dy[t], ox = cw.direct.dx[t];   // -1, 0, +1 (input row 2y + oy)
        const int py = oy & 1, px = ox & 1;                     // parity of that row / column
        cw.bf16.dy[t] = (int8_t)((oy - py) / 2);                // -1 for oy = -1, else 0
        cw.bf16.dx[t] = (int8_t)((ox - px) / 2);
        cw.bf16.cb[t] = (int8_t)((py * 2 + px) * (Ci / 8));
      }
    }
    {
      int rc = c8_configure(&cw.c8, ntaps, cw.bf16.dy, cw.bf16.dx, Ci, Cout, L.is_stem, cw.bf16.cb);
      if (rc) return rc;
      rc = c8_instantiated(cw.c8, false, L.name);
      if (rc) return rc;
    }
    TcWeights* tcp = &cw.c8.w;
    // the exact (swizzled) shared-memory image of every pipeline stage, see se_conv_tc.h. Gate channels (n >= Cout/2) are stored
    // pre-multiplied by 0.5 (exact): the accumulator then holds 0.5*g and the epilogue's sigmoid(g + b) = 0.5*tanh(0.5*g + 0.5*b) + 0.5
    // needs one add (with a constant operand) before the MUFU
    auto build_images = [&](TcWeights& tc, const std::function<uint16_t(int, int, int)>& wv) -> int {
      const int ksteps = tc_ksteps(tc), sb = tc_stage_b_bytes(tc);
      std::vector<uint16_t> img((size_t)ksteps * sb / 2, 0);
      for (int ks = 0; ks < ksteps; ++ks) {
        uint16_t* base = img.data() + (size_t)ks * sb / 2;
        for (int j = 0; j < tc.r64 && tc.n64; ++j) {
          const int u = ks * tc.r64 + j, t = u / tc.n64, chunk = u % tc.n64;
          for (int n = 0; n < Cout; ++n)
            for (int k = 0; k < 64; ++k) base[tc_b_image_offset(tc.NT, tc.r64, true, j, gated_column(Cout, n), k) / 2] = wv(t, chunk * 64 + k, n);
        }
        for (int j = 0; j < tc.r32 && tc.n32; ++j) {
          const int t = ks * tc.r32 + j;
          for (int n = 0; n < Cout; ++n)
            for (int k = 0; k < 32; ++k)
              base[tc_b_image_offset(tc.NT, tc.n64 ? tc.r64 : 0, false, j, gated_column(Cout, n), k) / 2] = wv(t, tc.n64 * 64 + k, n);
        }
      }
      return upload(m, img.data(), img.size() * 2, (void**)&tc.data);
    };
    auto wval = [&](int t, int ci, int n) -> float { return ci < Ci ? weff[((size_t)t * Ci + ci) * Cout + n] * (n >= Cout / 2 ? 0.5f : 1.0f) : 0.0f; };
    int rc = build_images(*tcp, [&](int t, int ci, int n) -> uint16_t { return f32_to_bf16_rn(wval(t, ci, n)); });
    if (rc) return rc;
    // ---- split-half twin: virtual tap 3t + p, p = 0: (x_hi, w_hi), 1: (x_hi, w_lo), 2: (x_lo, w_hi)
    const int CB = L.is_stem ? 1 : Ci / 8;   // channel blocks of one half of the input (the packed stem input is one block)
    cw.split.n = 3 * ntaps;
    SE_REQUIRE(cw.split.n <= MAX_TAPS, "too many virtual taps");
    for (int t = 0; t < ntaps; ++t)
      for (int pp = 0; pp < 3; ++pp) {
        cw.split.dy[3 * t + pp] = cw.bf16.dy[t];
        cw.split.dx[3 * t + pp] = cw.bf16.dx[t];
        cw.split.cb[3 * t + pp] = (int8_t)(2 * cw.bf16.cb[t] + (pp == 2 ? CB : 0));   // a parity group holds 2 * CB blocks
      }
    rc = c8_configure(&cw.c8s, cw.split.n, cw.split.dy, cw.split.dx, Ci, Cout, L.is_stem, cw.split.cb);
    if (rc) return rc;
    rc = c8_instantiated(cw.c8s, true, L.name);
    if (rc) return rc;
    // weights times a power of two (exact) that brings the largest one to [8192, 16384): the lo halves of all but negligible
    // weights are then normal fp16 numbers (22 bits for the pair); the epilogue undoes it (se_common.cuh: kSplitActScale)
    float wmax = 0.0f;
    for (int t = 0; t < ntaps; ++t)
      for (int ci = 0; ci < Ci; ++ci)
        for (int n = 0; n < Cout; ++n) wmax = std::max(wmax, std::fabs(wval(t, ci, n)));
    int kw = 0;
    if (wmax > 0.0f && std::isfinite(wmax)) kw = std::min(24, std::max(0, 13 - (int)std::floor(std::log2(wmax))));
    cw.s_wscale = std::ldexp(1.0f, kw);
    auto half_bits = [](float v) -> uint16_t { return __half_as_ushort(__float2half_rn(v)); };
    rc = build_images(cw.c8s.w, [&](int vt, int ci, int n) -> uint16_t {
      const float w = wval(vt / 3, ci, n) * cw.s_wscale;
      const float hi = __half2float(__float2half_rn(w));
      return (vt % 3) == 1 ? half_bits(w - hi) : half_bits(w);
    });
    if (rc) return rc;
  }
  return 0;
}

static int pack_layer(se_model* m, Layer& L) {
  const Spec& s = L.spec;
  L.Ci = stored_ci(s);
  L.is_head = (s.cin == 12);
  L.is_stem = (s.k == 5);
  int rc = upload(m, L.b_host.data(), L.b_host.size() * 4, (void**)&L.bias);
  if (rc) return rc;
  if (L.is_head) {
    std::vector<float> wh((size_t)9 * 12 * s.cout);
    for (int t = 0; t < 9; ++t)
      for (int c = 0; c < 12; ++c)
        for (int o = 0; o < s.cout; ++o) wh[((size_t)t * 12 + c) * s.cout + o] = L.w_host[(((size_t)o * 12 + c) * 3 + t / 3) * 3 + t % 3];
    L.w_head_host = wh;
  }
  if (L.is_stem) {
    // 5x5 / pad 2 over <= 5 real channels: K per tap would be 3-5. Instead one 64-wide GEMM-K chunk covers a
    // window of 8 horizontally adjacent pixels x 8 packed channels (kernel columns 0..4 + three zero columns):
    // 5 K-units (one per kernel row) instead of 25 taps. Window start in packed-buffer pixels:
    // (x + STEM_PADL) - 2 = x, so dx = 0.
    std::vector<EffTap> taps;
    for (int ky = 0; ky < 5; ++ky) {
      EffTap e;
      e.dy = ky - 2;
      e.dx = 0;
      for (int pxl = 0; pxl < 5; ++pxl) e.src.push_back(SrcTap{ky, pxl, pxl * 8});
      taps.push_back(e);
    }
    L.cls.resize(1);
    return pack_class(m, L, taps, L.cls[0]);
  }
  if (!s.deconv) {
    std::vector<EffTap> taps;
    const int p = s.rate * (s.k - 1) / 2;   // reference utils.py:21
    for (int ky = 0; ky < s.k; ++ky)
      for (int kx = 0; kx < s.k; ++kx) taps.push_back(EffTap{ky * s.rate - p, kx * s.rate - p, {SrcTap{ky, kx, 0}}});
    L.cls.resize(1);
    return pack_class(m, L, taps, L.cls[0]);
  }
  // nearest x2 upsample + 3x3 conv == four sub-pixel 2x2 convs over the low-res map with merged taps:
  // output row 2i   reads rows {i-1: W[0], i: W[1]+W[2]};  row 2i+1 reads {i: W[0]+W[1], i+1: W[2]}
  L.cls.resize(4);
  for (int pc = 0; pc < 4; ++pc) {
    const int py = pc / 2, px = pc % 2;
    std::vector<EffTap> taps;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        EffTap e;
        e.dy = (py == 0) ? (a - 1) : a;
        e.dx = (px == 0) ? (b - 1) : b;
        std::vector<int> rows = (py == 0) ? (a == 0 ? std::vector<int>{0} : std::vector<int>{1, 2})
                                          : (a == 0 ? std::vector<int>{0, 1} : std::vector<int>{2});
        std::vector<int> cols = (px == 0) ? (b == 0 ? std::vector<int>{0} : std::vector<int>{1, 2})
                                          : (b == 0 ? std::vector<int>{0, 1} : std::vector<int>{2});
        for (int r : rows)
          for (int c : cols) e.src.push_back(SrcTap{r, c, 0});
        taps.push_back(e);
      }
    ClassW& cw = L.cls[pc];
    cw.osy = 2; cw.ooy = py; cw.osx = 2; cw.oox = px;
    rc = pack_class(m, L, taps, cw);
    if (rc) return rc;
  }
  // fuse the classes into as few launches as shared memory allows: all four (48->48), else one launch per output-row
  // parity (96->96: classes {0,1} and {2,3}); the per-class launches stay available as the fallback
  if (L.cls[0].tc && L.cls[0].c8.resident && L.cls[0].c8.mode == C8_HALO) {
    for (int per : {4, 2}) {
      std::vector<C8Group> gs;
      bool ok = true;
      for (int g0 = 0; g0 < 4 && ok; g0 += per) {
        int8_t dy[C8_MAX_CLS][8], dx[C8_MAX_CLS][8];
        int ooy[C8_MAX_CLS], oox[C8_MAX_CLS];
        for (int k = 0; k < per; ++k) {
          const ClassW& cw = L.cls[g0 + k];
          for (int t = 0; t < cw.bf16.n; ++t) { dy[k][t] = cw.bf16.dy[t]; dx[k][t] = cw.bf16.dx[t]; }
          ooy[k] = cw.ooy; oox[k] = cw.oox;
        }
        C8Group G;
        if (c8_configure_group(&G, per, L.cls[0].bf16.n, dy, dx, ooy, oox, L.Ci, s.cout)) { ok = false; break; }
        const C8Layer& c0 = L.cls[g0].c8;
        ok = (G.geo.w.r64 == c0.w.r64 && G.geo.w.r32 == c0.w.r32 && G.geo.w.NT == c0.w.NT && G.cls_bytes == (int)tc_weight_bytes_per_image(c0.w));
        if (!ok) break;
        rc = c8_instantiated(G.geo, false, L.name + " (fused classes)");
        if (rc) return rc;
        void* d = nullptr;
        SE_CUDA_OK(cudaMalloc(&d, (size_t)per * G.cls_bytes));
        m->owned.push_back(d);
        for (int k = 0; k < per; ++k)
          SE_CUDA_OK(cudaMemcpy((char*)d + (size_t)k * G.cls_bytes, L.cls[g0 + k].c8.w.data, G.cls_bytes, cudaMemcpyDeviceToDevice));
        G.w_all = d;
        gs.push_back(G);
      }
      if (ok) { L.groups = gs; break; }
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------ arena
// Offsets inside one device slab, first-fit with coalescing. The forward graph is replayed twice per
// call: a dry pass (no launches) finds the peak, then the slab is grown if needed and the real pass runs.
struct Arena {
  struct Blk { size_t off, size; };
  std::vector<Blk> free_list;
  size_t top = 0, peak = 0;
  char* base = nullptr;
  void reset(char* b) { free_list.clear(); top = 0; peak = 0; base = b; }
  void* alloc(size_t bytes) {
    bytes = (bytes + 1023) & ~size_t(1023);
    for (size_t i = 0; i < free_list.size(); ++i)
      if (free_list[i].size >= bytes) {
        size_t off = free_list[i].off;
        if (free_list[i].size == bytes) free_list.erase(free_list.begin() + i);
        else { free_list[i].off += bytes; free_list[i].size -= bytes; }
        return base + off;
      }
    size_t off = top;
    top += bytes;
    if (top > peak) peak = top;
    return base + off;
  }
  void release(void* p, size_t bytes) {
    bytes = (bytes + 1023) & ~size_t(1023);
    size_t off = (char*)p - base;
    if (off + bytes == top) {
      top = off;
      // merge trailing free blocks
      bool again = true;
      while (again) {
        again = false;
        for (size_t i = 0; i < free_list.size(); ++i)
          if (free_list[i].off + free_list[i].size == top) { top = free_list[i].off; free_list.erase(free_list.begin() + i); again = true; break; }
      }
      return;
    }
    free_list.push_back({off, bytes});
    // coalesce neighbours
    bool again = true;
    while (again) {
      again = false;
      for (size_t i = 0; i < free_list.size() && !again; ++i)
        for (size_t j = 0; j < free_list.size(); ++j)
          if (i != j && free_list[i].off + free_list[i].size == free_list[j].off) {
            free_list[i].size += free_list[j].size;
            free_list.erase(free_list.begin() + j);
            again = true;
            break;
          }
    }
  }
};

struct Buf { void* p = nullptr; size_t bytes = 0; };

// activation view. c8 == 0: NHWC, channels [0,C) at pixel pitch ld. c8 == 1: [B][ld blocks][H][W][8], the view's
// channels start at block cb_off. c8 == 2: channel-blocked space-to-depth, [B][ld blocks][H/2][W/2][8] with the four
// (row, column) parity groups of ld / 4 blocks one after the other (H, W: the full-resolution size)
struct View { void* p; int H, W, C, ld; int c8 = 0; int cb_off = 0; };
static inline View nhwc(void* p, int H, int W, int C, int ld) { return View{p, H, W, C, ld, 0, 0}; }
static inline View c8view(void* p, int H, int W, int C, int cbtot, int cb_off = 0) { return View{p, H, W, C, cbtot, 1, cb_off}; }
static inline View s2dview(void* p, int H, int W, int C, int cbtot, int cb_off = 0) { return View{p, H, W, C, cbtot, 2, cb_off}; }

// an activation: its view plus the workspace buffer it owns (own.p == nullptr: a view into a buffer owned elsewhere)
struct Act {
  View v;
  Buf own;
  Act borrow() const { return Act{v, Buf()}; }
};

struct Ctx {
  se_model* m;
  cudaStream_t stream;
  int prec;
  bool dry;
  Arena arena;
  int B;
  long long attn_limit;   // se_set_attention_workspace_limit, read once per call (the dry and the real pass plan alike)
  LaunchTag tag_;
  // label + algorithmic work of the NEXT launch (consumed by CK); see "launch timing" above
  void tag(const std::string& name, int tensor, double flops_alg, double flops_exec, double bytes_alg) {
    if (!g_timing || dry) return;
    tag_.name = name; tag_.tensor = tensor; tag_.flops_alg = flops_alg; tag_.flops_exec = flops_exec; tag_.bytes_alg = bytes_alg; tag_.set = true;
  }
  // the mode's activation storage: bf16 and split-half channel-blocked for the wgmma kernels, fp32 NHWC for the CUDA-core kernels
  bool tc() const { return prec != SE_PREC_FP32_EXACT; }
  bool split() const { return prec == SE_PREC_FP32_TC; }
  int sp() const { return split() ? 2 : 1; }                                        // channel-block multiplier of the storage
  int act_dt() const { return split() ? DT_F16X2 : tc() ? DT_BF16 : DT_F32; }
  size_t esz() const { return prec == SE_PREC_BF16_TC ? 2 : 4; }
  Buf get(size_t bytes) { Buf b; b.bytes = bytes; b.p = arena.alloc(bytes); return b; }
  void put(Buf& b) { if (b.p) arena.release(b.p, b.bytes); b.p = nullptr; }
  void put(Act& a) { put(a.own); }
  size_t act_bytes(int H, int W, int C, int c8) const { return c8 ? (size_t)B * ((C + 7) / 8) * H * W * 16 * sp() : (size_t)B * H * W * C * esz(); }
  // a dense activation of layout c8 at p
  View dense(void* p, int H, int W, int C, int c8) const {
    if (c8 == 2) return s2dview(p, H, W, C, 4 * (C / 8) * sp());   // split-half: twice the blocks per parity group
    if (c8 == 1) return c8view(p, H, W, C, (C + 7) / 8 * sp());
    return nhwc(p, H, W, C, C);
  }
};

#define CK(expr)                                                    \
  do {                                                              \
    if (!c.dry) {                                                   \
      size_t _slot = 0;                                             \
      const bool _timed = g_timing;                                 \
      if (_timed) { int _rt = timing_begin(c.tag_, c.stream, &_slot); if (_rt) return _rt; } \
      c.tag_.set = false;                                           \
      int _rc = (expr);                                             \
      if (_rc) return _rc;                                          \
      if (_timed) { int _rt = timing_end(_slot, c.stream); if (_rt) return _rt; } \
      ++g_launches;                                                 \
    }                                                               \
  } while (0)

static Layer* find_layer(se_model* m, char net, const std::string& name) {
  auto it = m->layers.find(std::string(1, net) + "." + name);
  return it == m->layers.end() ? nullptr : &it->second;
}
// layer that has weights (forward paths); nullptr + error text otherwise
static Layer* find_ready(se_model* m, char net, const std::string& name) {
  Layer* L = find_layer(m, net, name);
  if (L && !L->set) {
    set_error(std::string("weights of net") + net + " were never loaded (layer " + name + ")");
    return nullptr;
  }
  return L;
}

// layout a layer wants for its input: 0 NHWC (CUDA-core path, heads), 1 channel-blocked (C8), 2 channel-blocked
// space-to-depth (stride-2 layers on the tensor-core path)
static int wants_c8(const Ctx& c, const Layer& L) {
  if (!c.tc() || L.is_head) return 0;
  if (L.spec.stride == 1) return 1;
  return (!L.cls.empty() && L.cls[0].s2d) ? 2 : 0;
}
// the packed 8-channel network input (zero-padded rows of stem_wp(W) pixels): NHWC with C = ld = 8 for the CUDA-core
// kernels, the same bytes seen as one channel block of width stem_wp(W) for the tensor-core path
static View stem_view(const Ctx& c, void* p, int H, int W) {
  if (c.tc()) return c8view(p, H, W, 8, c.sp(), 0);
  return nhwc(p, H, W, 8, 8);
}

// ------------------------------------------------------------------------------------------ activation taps
static void drop_taps(se_model* m) {
  if (m->taps.empty()) return;
  cudaDeviceSynchronize();   // a se_tap_copy may still read them
  for (auto& t : m->taps) cudaFree(t.p);
  m->taps.clear();
}

// records the bytes of view v as tap `name` (se_taps_enable): layout 0..2 = v.c8, 3 = packed stem rows; dtype -1 = the
// mode's activation storage. Enqueued on the forward's stream before the consumer's launch, so the buffer is still live.
static int tap(Ctx& c, const std::string& name, const View& v, int layout, int dtype = -1) {
  if (c.dry || !c.m->taps_on) return 0;
  se_model::Tap t;
  t.name = name;
  if (dtype < 0) dtype = c.act_dt() == DT_F32 ? 0 : (c.split() ? 2 : 1);
  int* d = t.desc;
  d[SE_TAP_LAYOUT] = layout; d[SE_TAP_DTYPE] = dtype; d[SE_TAP_B] = c.B; d[SE_TAP_C] = v.C; d[SE_TAP_H] = v.H; d[SE_TAP_W] = v.W;
  d[SE_TAP_LD] = v.ld; d[SE_TAP_CB_OFF] = v.cb_off;
  size_t elems;
  if (layout == 3) {
    d[SE_TAP_WP] = stem_wp(v.W); d[SE_TAP_PADL] = STEM_PADL;
    elems = (size_t)c.B * v.H * stem_wp(v.W) * 8 * (dtype == 2 ? 2 : 1);
  } else if (layout == 0) {
    elems = (size_t)c.B * v.H * v.W * v.ld;
  } else {
    elems = (size_t)c.B * v.ld * (layout == 2 ? (size_t)(v.H / 2) * (v.W / 2) : (size_t)v.H * v.W) * 8;
  }
  t.bytes = elems * (dtype == 0 ? 4 : 2);
  SE_CUDA_OK(cudaMalloc(&t.p, t.bytes));
  c.m->taps.push_back(t);
  SE_CUDA_OK(cudaMemcpyAsync(t.p, v.p, t.bytes, cudaMemcpyDeviceToDevice, c.stream));
  return 0;
}
#define TAP(...)                  \
  do {                            \
    int _rt = tap(c, __VA_ARGS__); \
    if (_rt) return _rt;          \
  } while (0)

// one gated conv / deconv layer: in (Hi x Wi x Ci) -> out (channels written at [choff, choff+cout_g), layout out_c8)
static int run_layer(Ctx& c, Layer& L, const View& in, void* out, int ldo, int choff, int out_c8 = 0) {
  SE_REQUIRE(in.c8 == wants_c8(c, L), "activation layout mismatch at layer " + L.name);
  TAP("in:" + std::string(1, L.net) + "." + L.name, in, L.is_stem ? 3 : in.c8);
  const Spec& s = L.spec;
  const int Ho = s.deconv ? in.H : (in.H + s.stride - 1) / s.stride;   // position grid
  const int Wo = s.deconv ? in.W : (in.W + s.stride - 1) / s.stride;
  const bool fused = c.prec == SE_PREC_BF16_TC && !L.groups.empty() && in.c8 == 1;
  const bool split = c.split();
  const int n_launch = fused ? (int)L.groups.size() : (int)L.cls.size();
  if (c8_log_on() && !c.dry) c8_log_label(std::string(1, L.net) + "." + L.name);
  for (int li = 0; li < n_launch; ++li) {
    const C8Group* grp = fused ? &L.groups[li] : nullptr;
    ClassW& cw = L.cls[fused ? li * grp->ncls : li];
    ConvParams cp;
    memset(&cp, 0, sizeof(cp));
    cp.x = in.p; cp.in_dt = c.act_dt();
    cp.N = c.B; cp.Hi = in.H; cp.Wi = in.W; cp.Ci = L.Ci; cp.ldx = in.ld;
    if (L.is_stem && !in.c8) {   // `in` is the packed 8-channel buffer with zero-padded rows of stem_wp(W) pixels
      cp.ldx = 8;
      cp.Wi = stem_wp(in.W) - 7;
      cp.x_row_pitch = (long long)stem_wp(in.W) * 8;
      cp.x_img_pitch = (long long)in.H * cp.x_row_pitch;
    }
    if (in.c8) {
      cp.in_c8 = 1; cp.x_cb_off = in.cb_off; cp.ldx = in.ld;
      if (L.is_stem) cp.Wi = stem_wp(in.W);   // the window starts at buffer pixel x (image sits at x + STEM_PADL)
    }
    cp.out_c8 = out_c8;
    cp.Ho = Ho; cp.Wo = Wo; cp.stride = s.deconv ? 1 : s.stride;
    // the taps of the form this mode launches (the tensor-core forms are already in space-to-depth form where that applies)
    const Taps& tp = split ? cw.split : c.tc() ? cw.bf16 : cw.direct;
    cp.ntaps = tp.n;
    memcpy(cp.dy, tp.dy, sizeof(cp.dy));
    memcpy(cp.dx, tp.dx, sizeof(cp.dx));
    memcpy(cp.tap_cb, tp.cb, sizeof(cp.tap_cb));
    if (split) {
      SE_REQUIRE(in.c8 && out_c8, "split-half mode runs on channel-blocked activations (layer " + L.name + ")");
      cp.f16x2 = 1;
      // hi blocks first, lo blocks after them: per image (channel-blocked) or per parity group (space-to-depth)
      cp.out_split_stride = out_c8 == 2 ? (long long)(ldo / 8) * (Ho * cw.osy / 2) * (Wo * cw.osx / 2) : (long long)(ldo / 2) * (Ho * cw.osy) * (Wo * cw.osx);
    }
    if (in.c8 == 2) {   // space-to-depth input: a stride-1 problem on the half-resolution grid with per-tap parity blocks
      SE_REQUIRE(cw.s2d && in.H % 2 == 0 && in.W % 2 == 0, "space-to-depth input at layer " + L.name);
      cp.Hi = in.H / 2; cp.Wi = in.W / 2; cp.stride = 1;
    }
    cp.w = nullptr; cp.w_img_stride = 0;
    cp.bias = L.bias; cp.bias_host = L.b_host.data(); cp.Cout = s.cout;
    cp.y = out; cp.out_dt = c.act_dt();
    cp.Hout = Ho * cw.osy; cp.Wout = Wo * cw.osx; cp.ldo = ldo; cp.choff = choff;
    cp.osy = cw.osy; cp.ooy = cw.ooy; cp.osx = cw.osx; cp.oox = cw.oox;
    cp.epi = s.act == 1 ? EPI_GATE_RELU : EPI_GATE_ELU;
    cp.scale = split ? 1.0f / (kSplitActScale * cw.s_wscale) : 1.0f;   // split-half: accumulator -> true pre-activation (exact: powers of two)
    cp.colscale = nullptr;
    if (L.fused_pair) {
      // two space-to-depth tensors of 4 x 3 blocks each, back to back per image (ldo = 24 blocks): blocks 3..5 of the fused
      // output are blocks 0..2 of the second one, 12 - 3 = 9 block planes further on
      SE_REQUIRE(out_c8 == 2 && ldo == 24, "a fused stem pair writes two space-to-depth tensors");
      cp.out_blk_split = 3; cp.out_par_stride = 3; cp.out_blk_jump = 9 * (cp.Hout / 2) * (cp.Wout / 2);
    }
    if (g_timing && !c.dry) {
      // algorithmic work of this launch. A deconv layer is 4 sub-pixel class launches: each gets a quarter of the
      // reference op's 2*MAC (nearest x2 + 3x3 over the (2Ho x 2Wo) output) and issues 4 taps instead of 9.
      // (a fused launch carries `gc` classes)
      const double gc = grp ? grp->ncls : 1.0;
      const double pos = (double)c.B * Ho * Wo * gc, ncls = (double)L.cls.size() / gc;
      const double cin_alg = L.fused_pair ? L.pair_cin_sum / 2.0 : (double)s.cin;   // a stem pair: two 48-output layers over their own channels
      const double f_alg = 2.0 * pos * s.cout * cin_alg * (s.deconv ? 9.0 : (double)s.k * s.k);
      const double f_exec = 2.0 * pos * s.cout * cin_alg * (s.deconv ? 4.0 : (double)s.k * s.k) * (split ? 3.0 : 1.0);   // split-half: 3 products per tap
      const double bytes = ((double)c.B * in.H * in.W * (L.fused_pair ? 8.0 : (double)s.cin) / ncls + pos * (s.cout / 2) + (double)s.cout * s.cin * s.k * s.k / ncls) * c.esz();
      char buf[160];
      snprintf(buf, sizeof(buf), "%s|%s %d->%d k%d s%d d%d @%dx%d", c.tc() ? (split ? "conv_c8_kernel (split-half fp16 x3)" : "conv_c8_kernel") : "conv_direct_kernel",
               s.deconv ? (grp ? (grp->ncls == 4 ? "deconv (4 classes fused)" : "deconv (2 classes fused)") : "deconv-class") : (L.fused_pair ? "stem pair" : "conv"), s.cin, s.cout, s.k, s.stride, s.rate, Ho * cw.osy, Wo * cw.osx);
      c.tag(buf, c.tc() ? 1 : 0, f_alg, f_exec, bytes);
    }
    if (split) CK(c8_launch(cp, cw.c8s, c.stream));
    else if (c.tc()) CK(c8_launch(cp, cw.c8, c.stream, grp));
    else {
      cp.w = cw.w_direct;
      CK(direct_launch(cp, cw.CoutP, c.stream));
    }
  }
  return 0;
}

static void out_dims(const Spec& s, int H, int W, int* Ho, int* Wo) {
  if (s.deconv) { *Ho = 2 * H; *Wo = 2 * W; }
  else { *Ho = (H + s.stride - 1) / s.stride; *Wo = (W + s.stride - 1) / s.stride; }
}

// where the last layer of a chain writes: into p (ld pixel pitch / channel blocks, channel offset choff) when given, else
// into a fresh workspace buffer. c8: layout of the result, -1 = the mode's own (channel-blocked on the tensor-core path)
struct Dst { void* p = nullptr; int ld = 0, choff = 0, c8 = -1; };

// run a chain of gated layers; intermediate buffers come from the arena. Each intermediate is written in the layout
// its consumer wants. The chain releases `in` when it owns its buffer; *out (may be null when dst.p is given) receives
// the result.
static int run_chain(Ctx& c, char net, const std::vector<std::string>& names, Act in, Act* out, Dst dst = Dst()) {
  Act cur = in;
  if (dst.c8 < 0) dst.c8 = c.tc() ? 1 : 0;
  for (size_t i = 0; i < names.size(); ++i) {
    Layer* L = find_ready(c.m, net, names[i]);
    SE_REQUIRE(L != nullptr, "unknown or unloaded layer " + names[i] + ": " + last_error());
    int Ho, Wo;
    out_dims(L->spec, cur.v.H, cur.v.W, &Ho, &Wo);
    const int cg = L->spec.cout / 2;
    const bool last = (i + 1 == names.size());
    Act nxt;
    if (last && dst.p) {
      nxt.v = dst.c8 ? c8view(dst.p, Ho, Wo, cg, dst.ld, dst.choff / 8) : nhwc(dst.p, Ho, Wo, cg, dst.ld);
      int rc = run_layer(c, *L, cur.v, dst.p, dst.ld, dst.choff, dst.c8);
      if (rc) return rc;
    } else {
      int oc8 = dst.c8;
      if (!last) {
        Layer* nx = find_ready(c.m, net, names[i + 1]);
        SE_REQUIRE(nx != nullptr, "unknown or unloaded layer " + names[i + 1]);
        oc8 = wants_c8(c, *nx);
      }
      nxt.own = c.get(c.act_bytes(Ho, Wo, cg, oc8));
      nxt.v = c.dense(nxt.own.p, Ho, Wo, cg, oc8);
      int rc = run_layer(c, *L, cur.v, nxt.own.p, nxt.v.ld, 0, oc8);
      if (rc) return rc;
    }
    c.put(cur);
    cur = nxt;
  }
  if (out) *out = cur;
  return 0;
}

// pfx + each name of l from the skip-th on
static std::vector<std::string> with_prefix(const std::string& pfx, std::initializer_list<const char*> l, int skip = 0) {
  std::vector<std::string> v;
  for (auto s = l.begin() + skip; s != l.end(); ++s) v.push_back(pfx + *s);
  return v;
}

// io: the tensors of the head (HeadIO); its input map, sizes and mode are filled in here
static int run_head(Ctx& c, char net, const std::string& name, const View& in, int mode, HeadIO io) {
  Layer* L = find_ready(c.m, net, name);
  SE_REQUIRE(L != nullptr && L->is_head, "head layer " + name + ": " + last_error());
  TAP("in:" + std::string(1, net) + "." + name, in, in.c8);
  {
    // 12-channel map in (two channel blocks on the C8 path), image / mask planes in, cout (+ blend / pack) planes out
    const double px = (double)c.B * in.H * in.W;
    const int outs = !!io.mask + !!io.mask_bin + !!io.stage + !!io.composed;
    const double bytes = px * ((in.c8 ? 16 : 12) * c.esz() + (io.img ? 12 : 0) + (io.blend ? 4 : 0) + outs * 4 * L->spec.cout + (io.packed ? 8 * c.esz() : 0));
    const double fl = 2.0 * px * 9 * 12 * L->spec.cout;
    c.tag(std::string("head_kernel|12->") + std::to_string(L->spec.cout) + " k3 + " +
              (mode == HEAD_MASK ? "sigmoid+threshold" : mode == HEAD_TANH ? "tanh" : mode == HEAD_COARSE ? "tanh+blend+pack8" : "tanh+soft blend"),
          0, fl, fl, bytes);
  }
  SE_REQUIRE(in.c8 == (c.tc() ? 1 : 0) && in.ld == (c.tc() ? 2 * c.sp() : 12), "head input: dense 12 channels in the mode's storage");
  io.x = in.p; io.B = c.B; io.H = in.H; io.W = in.W; io.mode = mode;
  io.Wp = stem_wp(in.W); io.padl = STEM_PADL; io.no_mask_coarse = c.m->opt[SE_OPT_NO_MASK_COARSE];
  CK(head(io, c.act_dt(), L->w_head_host.data(), L->b_host.data(), L->spec.cout, c.stream));
  return 0;
}

// ------------------------------------------------------------------------------------------ contextual attention
// cam_1 + cam_2 (reference splitcam.py:57-108,147-174) on an NHWC feature map f [B,h,w,C]:
//   S = Q K^T  as a stride-2, 4x4-tap "convolution" of f with per-image kernels K   (utils.py:72-99)
//   A = softmax_l(10 * S * m_l),  out = fold_sum(A V) as four sub-pixel 2x2 convolutions over A
// bf16 tensor-core path (se_cam.cu): f is the space-to-depth channel-blocked map, out is channel-blocked [B][12][h][w][8]
static int run_cam_tc(Ctx& c, const View& f, const float* mask_s, void* out, float* attn_out) {
  SE_REQUIRE(f.c8 == 2 && f.C == 96, "tensor-core attention reads a 96-channel space-to-depth channel-blocked map");
  CamPlan pl;
  int rc = cam_plan(c.B, f.H, f.W, c.attn_limit, attn_out != nullptr, &pl);
  if (rc) return rc;
  Buf fn = c.get(pl.fn_bytes), cs = c.get(pl.cs_bytes), P = c.get(pl.p_bytes);
  if (g_timing && !c.dry) {
    const double L = (double)pl.hs * pl.ws;
    const double fl = 4.0 * c.B * L * L * 96 * 16;   // QK^T + PV (SURVEY.md 8d); the statistics sweep repeats QK^T: executed = 1.5x
    c.tag("cam_s_kernel + cam_pv_kernel (+ norm, colscale)|contextual attention", 1, fl, 1.5 * fl,
          (double)c.B * f.H * f.W * 96 * 2 * 2 + 2.0 * (double)c.B * pl.KB * pl.hs * pl.ws * 16);   // P of all bands
  }
  CK(cam_forward_tc(f.p, mask_s, out, pl, fn.p, (float*)cs.p, P.p, attn_out, c.stream));
  if (!c.dry) g_launches += 1 + 2 * pl.n_bands + (attn_out ? 1 : 0);   // norm, colscale and an S + PV pair per band behind one call
  c.put(P); c.put(cs); c.put(fn);
  return 0;
}

static int run_cam(Ctx& c, const View& f, const float* mask_s, void* out, int out_ld, float* attn_out /*fp32 [B,L,N] or null*/, int out_c8 = 0) {
  SE_REQUIRE(f.c8 == 0 && c.act_dt() == DT_F32, "the CUDA-core attention reads an fp32 NHWC feature map");
  const int B = c.B, h = f.H, w = f.W, C = f.C;
  SE_REQUIRE(h % 2 == 0 && w % 2 == 0 && h >= 4 && w >= 4, "attention map must be even-sized and >= 4");
  const int hs = (h - 4) / 2 + 1, ws = (w - 4) / 2 + 1, L = hs * ws;
  const int Lpad = (L + 127) / 128 * 128;
  // CUDA-core path (fp32 modes; bf16 with channel counts other than netG's 96): the tensor-core attention is run_cam_tc / se_cam.cu
  const float* fp = (const float*)f.p;
  Buf rnorm = c.get((size_t)B * C * 4);
  Buf colm = c.get((size_t)B * L * 4);
  c.tag("plane_reduce|attention key norm", 0, 0, 0, (double)B * h * w * C * 4);
  CK(plane_reduce(fp, DT_F32, B, h * w, C, f.ld, RED_RNORM, (float*)rnorm.p, c.stream));
  c.tag("cam_colmask_kernel", 0, 0, 0, (double)B * h * w * 4);
  CK(cam_colmask(mask_s, (float*)colm.p, B, h, w, hs, ws, 0.1f, c.stream));

  // ---- keys
  const size_t kbytes = (size_t)B * 16 * C * Lpad * 4;   // keys as per-image conv kernels: fp32 [b][tap][c][Lpad]
  Buf kbuf = c.get(kbytes);
  SE_REQUIRE(f.ld == C, "attention input must be dense NHWC");
  c.tag("cam_pack_k|attention key operand", 0, 0, 0, (double)B * h * w * C * 4 + (double)kbytes);
  CK(cam_pack_k(fp, (const float*)rnorm.p, (float*)kbuf.p, B, h, w, C, ws, L, Lpad, c.stream));

  // ---- bands of output class rows [y0, y1): S and P hold the query rows [qa, q1) those rows read (y0 - 1 .. y1 - 1, clipped
  // to the patch grid; the boundary query row is computed by both bands that read it). R = class rows per band: the tallest
  // whose S + P fit the attention workspace limit, every row when the attention map is wanted.
  const int Hs = h / 2;
  const size_t qrow_bytes = (size_t)B * ws * Lpad * 8;   // one query row of S and P (fp32)
  int R = Hs;
  if (!attn_out && qrow_bytes * hs > (size_t)c.attn_limit) {
    R = (int)((size_t)c.attn_limit / qrow_bytes) - 1;
    SE_REQUIRE(R >= 1, "attention workspace limit of " + std::to_string(c.attn_limit) + " bytes is below the " +
                           std::to_string(qrow_bytes * (hs < 2 ? hs : 2)) + " bytes one band of 1 output row needs at this size and batch");
  }
  const size_t per_pc_bytes = (size_t)B * 4 * Lpad * C * 4;   // values per sub-pixel class: fp32 [b][tap][key][c]
  Buf vbuf;
  for (int y0 = 0; y0 < Hs; y0 += R) {
    const int y1 = y0 + R < Hs ? y0 + R : Hs;
    const int qa = y0 ? y0 - 1 : 0, q1 = y1 < hs ? y1 : hs, nq = q1 - qa;
    const bool last = y1 == Hs;
    // ---- logits S[b, n, l] of query rows [qa, q1) (fp32, row pitch Lpad), scaled by 10 * m_l in the GEMM epilogue
    Buf sbuf = c.get((size_t)B * nq * ws * Lpad * 4);
    {
      ConvParams cp;
      memset(&cp, 0, sizeof(cp));
      cp.x = fp + (size_t)2 * qa * w * f.ld; cp.in_dt = DT_F32; cp.N = B; cp.Hi = h - 2 * qa; cp.Wi = w; cp.Ci = C; cp.ldx = f.ld;
      cp.x_img_pitch = (long long)h * w * f.ld;
      cp.Ho = nq; cp.Wo = ws; cp.stride = 2; cp.ntaps = 16;
      for (int t = 0; t < 16; ++t) { cp.dy[t] = (int8_t)(t / 4); cp.dx[t] = (int8_t)(t % 4); }
      cp.bias = nullptr; cp.Cout = L;
      cp.y = sbuf.p; cp.out_dt = DT_F32; cp.Hout = nq; cp.Wout = ws; cp.ldo = Lpad; cp.choff = 0;
      cp.osy = 1; cp.ooy = 0; cp.osx = 1; cp.oox = 0;
      cp.epi = EPI_LINEAR; cp.scale = 10.0f; cp.colscale = (const float*)colm.p;
      cp.w = kbuf.p; cp.w_img_stride = (long long)16 * C * Lpad;
      const double nL = (double)nq * ws;
      c.tag("conv_direct_kernel|attention S=QK^T", 0, 2.0 * B * nL * (double)L * C * 16,
            2.0 * B * nL * (double)L * C * 16, (double)B * h * w * C * 4 + (double)kbytes + (double)B * nL * Lpad * 4);
      CK(direct_launch(cp, Lpad, c.stream));
    }
    if (last) {
      c.put(kbuf);
      c.put(rnorm);
    }

    // ---- softmax over keys -> P[b, n, 0..Lpad)
    Buf pbuf = c.get((size_t)B * nq * ws * Lpad * 4);
    c.tag("softmax_rows|attention", 0, 0, 0, (double)B * nq * ws * Lpad * 8);
    CK(softmax_rows((const float*)sbuf.p, Lpad, (float*)pbuf.p, Lpad, (long long)B * nq * ws, L, c.stream));
    if (attn_out) {
      // cam_1 returns [B, L(keys), hs, ws]: transpose of P (one band)
      // (small, test-only path: done with the layout conversion, P viewed as an NHWC map of L x 1 pixels with C = L keys)
      CK(act_to_f32(pbuf.p, DT_F32, Layout{LAYOUT_NHWC, L, 1, Lpad}, attn_out, 0, B, L, c.stream));
    }
    c.put(sbuf);
    if (last) c.put(colm);

    // ---- values + fold-sum of class rows [y0, y1): query row y - a is P row y - a - qa
    if (!vbuf.p) {
      vbuf = c.get(4 * per_pc_bytes);
      c.tag("cam_pack_v|attention value operand", 0, 0, 0, (double)B * h * w * C * 4 + 4.0 * per_pc_bytes);
      CK(cam_pack_v(fp, (float*)vbuf.p, B, h, w, C, ws, L, Lpad, c.stream));
    }
    for (int pc = 0; pc < 4; ++pc) {
      ConvParams cp;
      memset(&cp, 0, sizeof(cp));
      cp.x = pbuf.p; cp.in_dt = DT_F32; cp.N = B; cp.Hi = nq; cp.Wi = ws; cp.Ci = Lpad; cp.ldx = Lpad;
      cp.Ho = y1 - y0; cp.Wo = w / 2; cp.stride = 1; cp.ntaps = 4;
      for (int t = 0; t < 4; ++t) { cp.dy[t] = (int8_t)(y0 - qa - t / 2); cp.dx[t] = (int8_t)(-(t % 2)); }
      cp.bias = nullptr; cp.Cout = C;
      cp.y = out; cp.out_dt = DT_F32; cp.Hout = h; cp.Wout = w; cp.ldo = out_c8 ? (C + 7) / 8 : out_ld; cp.choff = 0;
      cp.out_c8 = out_c8;
      cp.osy = 2; cp.ooy = 2 * y0 + pc / 2; cp.osx = 2; cp.oox = pc % 2;
      cp.epi = EPI_LINEAR; cp.scale = 1.0f; cp.colscale = nullptr;
      cp.w = (char*)vbuf.p + pc * per_pc_bytes; cp.w_img_stride = (long long)4 * Lpad * C;
      const double ny = y1 - y0;
      c.tag("conv_direct_kernel|attention out=fold(PV) class", 0,
            2.0 * B * ny * (w / 2) * (double)C * L * 4, 2.0 * B * ny * (w / 2) * (double)C * L * 4,
            ((double)B * nq * ws * Lpad + (double)B * 4 * Lpad * C + (double)B * ny * (w / 2) * C) * 4);
      CK(direct_launch(cp, C, c.stream));
    }
    if (last) c.put(vbuf);
    c.put(pbuf);
  }
  return 0;
}

// Attention of the fp32-on-tensor-cores mode: f fp32 NHWC [B][h][w][96] -> out fp32 NHWC, split-half fp16 wgmma GEMMs (se_gemm_split.cu)
static int run_cam_split(Ctx& c, const float* f, int h, int w, int C, const float* mask_s, float* out, float* attn_out = nullptr) {
  CamSplitPlan pl;
  {
    int rc = cam_split_plan(c.B, h, w, C, c.attn_limit, &pl);
    if (rc) return rc;
  }
  Buf rnorm = c.get((size_t)c.B * C * 4), colm = c.get((size_t)c.B * pl.L * 4);
  Buf q = c.get(pl.q_bytes), kn = c.get(pl.q_bytes), sb = c.get(pl.s_bytes), pb = c.get(pl.p_bytes), ob = c.get(pl.o_bytes);
  c.tag("plane_reduce|attention key norm", 0, 0, 0, (double)c.B * h * w * C * 4);
  CK(plane_reduce(f, DT_F32, c.B, h * w, C, C, RED_RNORM, (float*)rnorm.p, c.stream));
  c.tag("cam_colmask_kernel", 0, 0, 0, (double)c.B * h * w * 4);
  CK(cam_colmask(mask_s, (float*)colm.p, c.B, h, w, pl.hs, pl.ws, 0.1f, c.stream));
  const double fl = 2.0 * c.B * (double)pl.L * pl.L * pl.KQ * 2.0;   // S and PV, algorithmic (one product each)
  c.tag("gemm_split_kernel x2 (split-half fp16 x3) + pack / softmax / fold|contextual attention", 1, fl, 3.0 * 2.0 * c.B * (double)pl.Mp * pl.Mp * pl.KQ * 2.0,
        (double)c.B * h * w * C * 4 * 2 + 2.0 * pl.q_bytes * 2 + 2.0 * c.B * (double)pl.Mp * pl.Mp * 8 /* S + P of all bands */ + 2.0 * pl.o_bytes);
  CK(cam_forward_split(f, (const float*)rnorm.p, (const float*)colm.p, out, pl, q.p, kn.p, (float*)sb.p, pb.p, (float*)ob.p, attn_out, c.stream));
  if (!c.dry) g_launches += 1 + 3 * pl.n_bands;   // pack, S GEMM + softmax + PV GEMM per band, fold behind one call
  c.put(ob); c.put(pb); c.put(sb); c.put(kn); c.put(q); c.put(colm); c.put(rnorm);
  return 0;
}

// ------------------------------------------------------------------------------------------ networks
static const std::initializer_list<const char*> kEncoder = {"conv1", "conv2_downsample", "conv3", "conv4_downsample", "conv5", "conv6",
                                                            "conv7_atrous", "conv8_atrous", "conv9_atrous", "conv10_atrous"};
static const std::initializer_list<const char*> kDecoder = {"11", "12", "13_upsample_conv", "14", "15_upsample_conv", "16"};

// input packing / pooling glue in the activation storage of the current mode
// the packed 8-channel network input (stem_view) in a fresh workspace buffer
static int do_pack8(Ctx& c, Act* out, const float* img, const float* sk, const float* mask, int H, int W, int img_mode, float sscale, int write_mask,
                    int img2_mode = -1) {
  Buf in8 = c.get((size_t)c.B * H * stem_wp(W) * 8 * c.esz());
  c.tag("pack8_kernel|mask-mul + concat + cast", 0, 0, 0, (double)c.B * H * W * 20 + (double)c.B * H * stem_wp(W) * 8 * c.esz());
  CK(pack8(img, sk, mask, in8.p, c.act_dt(), c.B, H, W, stem_wp(W), STEM_PADL, img_mode, sscale, write_mask, c.stream, img2_mode));
  *out = Act{stem_view(c, in8.p, H, W), in8};
  return 0;
}
// global pooling of the 96-channel map v, broadcast into channels 96..191 of the concat buffer cat
static int do_pool_broadcast(Ctx& c, const View& v, int mode, void* cat, int cat_ld) {
  const int HW = v.H * v.W;
  TAP("in:G.pool", v, v.c8);
  Buf pooled = c.get((size_t)c.B * 96 * 4);
  c.tag("plane_reduce + broadcast_channels|global style pooling -> concat blocks", 0, 0, 0, 2.0 * c.B * v.H * v.W * 96 * (c.esz() > 2 ? 4 : 2));
  auto launch = [&](float* pl) -> int {   // one timed launch pair
    int rc = plane_reduce(v.p, c.act_dt(), c.B, HW, 96, v.ld, mode, pl, c.stream);
    return rc ? rc : broadcast_channels(pl, cat, c.act_dt(), c.B, HW, 96, cat_ld, 96, c.stream);
  };
  CK(launch((float*)pooled.p));
  c.put(pooled);
  return 0;
}

// MDGenerator.forward: x [B,3,H,W], guide [B,1,H,W] -> the soft mask (mask_bs elements between images, 0 = dense) with its
// binarised plane (> 0.5) and bytes where set, and x_stage1. Without a mask only the trunk (conv1-conv9) and the image decoder
// run. All fields are 8 bytes wide: they form the graph key.
struct NetMIO {
  const float *x, *guide;
  float* mask = nullptr;
  long long mask_bs = 0;
  float* mask_bin = nullptr;
  unsigned char* mask_u8 = nullptr;
  float* x_stage1 = nullptr;
};

static int run_netM(Ctx& c, int H, int W, const NetMIO& io) {
  SE_REQUIRE(io.mask || io.x_stage1, "netM with neither output");
  Act in8, x9;
  int rc = do_pack8(c, &in8, io.x, io.guide, nullptr, H, W, PACK_IMG_ONE, 1.0f, 0);
  if (rc) return rc;
  std::vector<std::string> trunk = with_prefix("", kEncoder);
  trunk.pop_back();   // conv10_atrous opens the mask branch
  rc = run_chain(c, 'M', trunk, in8, &x9);
  if (rc) return rc;
  if (io.x_stage1) {
    // image decoder reads the conv9 output too (editline2_g.py:76-77)
    Act v16;
    rc = run_chain(c, 'M', with_prefix("conv", kDecoder), x9.borrow(), &v16);
    if (rc) return rc;
    HeadIO h{};
    h.stage = io.x_stage1;
    rc = run_head(c, 'M', "conv17", v16.v, HEAD_TANH, h);
    if (rc) return rc;
    c.put(v16);
  }
  if (!io.mask) {
    c.put(x9);
    return 0;
  }
  Act v;
  rc = run_chain(c, 'M', with_prefix("", {"conv10_atrous", "conv_mask_11", "conv_mask_12", "conv_mask_13_upsample_conv", "conv_mask_14",
                                          "conv_mask_15_upsample_conv", "conv_mask_16"}),
                 x9, &v);
  if (rc) return rc;
  Buf scratch;
  HeadIO h{};
  h.mask = io.mask; h.mask_bs = io.mask_bs; h.mask_bin = io.mask_bin; h.mask_u8 = io.mask_u8;
  if (!h.mask_bin) { scratch = c.get((size_t)c.B * H * W * 4); h.mask_bin = (float*)scratch.p; }
  rc = run_head(c, 'M', "conv_mask_17", v.v, HEAD_MASK, h);
  if (rc) return rc;
  c.put(scratch);
  c.put(v);
  return 0;
}

// the fused stem pair `pair` (make_stem_pair) over the packed input `in`, which it releases: *st = the two stems' space-to-depth
// outputs side by side (24 blocks per image, 12 per stem)
static int run_stem_pair(Ctx& c, Layer& pair, Act in, Buf* st) {
  *st = c.get((size_t)c.B * 24 * (in.v.H / 2) * (in.v.W / 2) * 16);
  int rc = run_layer(c, pair, in.v, st->p, 24, 0, 2);
  if (rc) return rc;
  c.put(in);
  return 0;
}

// DeepFillC2Generator.forward. x, x2 [B,3,H,W]; mask, mask2 planes [B,H,W]; guide [B,H,W] or null (ones, editline_g.py:127-130).
// Outputs where set: x_stage1, x_stage2, composed = x_stage2 * mask_soft + x * (1 - mask_soft) (editline2_model.py:132) and its
// BGR bytes. *_bs: elements between images, 0 = dense. All fields are 8 bytes wide: they form the graph key.
struct NetGIO {
  const float *x, *x2, *mask, *mask2, *guide;
  float *x_stage1 = nullptr, *x_stage2 = nullptr, *composed = nullptr;
  long long composed_bs = 0;
  unsigned char* composed_u8 = nullptr;
  const float* mask_soft = nullptr;
  long long msoft_bs = 0;
  float* attn = nullptr;   // the attention's softmax weights [B][L][L] (cam_1's layout), one band
};

static int run_netG(Ctx& c, int H, int W, const NetGIO& io) {
  const int* opt = c.m->opt;
  const int h = H / 4, w = W / 4;
  const size_t e = c.esz();
  const int tc = c.tc() ? 1 : 0;
  const int cat_ld = tc ? 24 * c.sp() : 192;           // 192-channel concat buffers: 24 channel blocks (x2 split-half) or pixel pitch 192
  const int style_img = opt[SE_OPT_NO_MASK_CC] ? PACK_IMG_ONE : PACK_IMG_M;   // image channels of the style encoder's input
  // stem pairs (tensor-core path, make_stem_pair): conv1 + wconv1 share one packed input when both encoders see the same image
  // and mask (always true on the inference path: netG(inputs, inputs, mask_bin, mask_bin, line)); xconv1 + pmconv1 always do.
  // Each encoder then reads its half of the pair's output and its chain starts at its second layer.
  Layer* pair1 = (c.prec == SE_PREC_BF16_TC && io.x == io.x2 && io.mask == io.mask2) ? find_layer(c.m, 'G', "conv1+wconv1") : nullptr;
  Layer* pair2 = c.prec == SE_PREC_BF16_TC ? find_layer(c.m, 'G', "xconv1+pmconv1") : nullptr;
  auto pair_half = [&](const Buf& st, int which) { return s2dview(st.p, H, W, 24, 24, 12 * which); };

  // ---- stage 1: coarse encoder + style ("warp-in") encoder -> 192-channel concat -> coarse decoder
  Buf cat1 = c.get((size_t)c.B * h * w * 192 * e);
  Buf st1;
  int rc = 0;
  if (pair1) {
    Act in8;
    rc = do_pack8(c, &in8, io.x, io.guide, io.mask, H, W, PACK_IMG_ONE_MINUS_M, 1.0f, 1, style_img);
    if (rc) return rc;
    rc = run_stem_pair(c, *pair1, in8, &st1);
    if (rc) return rc;
  }
  Act in;
  if (!pair1) rc = do_pack8(c, &in, io.x, io.guide, io.mask, H, W, PACK_IMG_ONE_MINUS_M, 1.0f, 1);
  if (rc) return rc;
  rc = run_chain(c, 'G', with_prefix("", kEncoder, pair1 ? 1 : 0), pair1 ? Act{pair_half(st1, 0)} : in, nullptr, Dst{cat1.p, cat_ld, 0});
  if (rc) return rc;
  if (!pair1) rc = do_pack8(c, &in, io.x2, io.guide, io.mask2, H, W, style_img, opt[SE_OPT_JOINT_TRAIN_INP] ? 0.0f : 1.0f, 1);
  if (rc) return rc;
  Act style;
  rc = run_chain(c, 'G', with_prefix("w", kEncoder, pair1 ? 1 : 0), pair1 ? Act{pair_half(st1, 1)} : in, &style);
  if (rc) return rc;
  c.put(st1);
  rc = do_pool_broadcast(c, style.v, opt[SE_OPT_POOL_AVG] ? RED_AVG : RED_MAX, cat1.p, cat_ld);
  if (rc) return rc;
  c.put(style);
  Buf xnow = c.get((size_t)c.B * H * stem_wp(W) * 8 * e);   // stage-2 input: the blended coarse result, packed like the network input
  Act dec;
  rc = run_chain(c, 'G', with_prefix("conv", kDecoder), Act{c.dense(cat1.p, h, w, 192, tc), cat1}, &dec);
  if (rc) return rc;
  c.tag("memset|pad pixels of the packed stage-2 input", 0, 0, 0, (double)xnow.bytes);
  CK(fill_zero(xnow.p, xnow.bytes, c.stream));   // zero pad pixels of the packed stage-2 input
  HeadIO coarse{};
  coarse.img = io.x; coarse.blend = io.mask; coarse.stage = io.x_stage1; coarse.packed = xnow.p;
  rc = run_head(c, 'G', "conv17", dec.v, HEAD_COARSE, coarse);
  if (rc) return rc;
  c.put(dec);

  // ---- stage 2: hallucination branch + patch-match branch -> concat -> joint decoder
  Buf cat2 = c.get((size_t)c.B * h * w * 192 * e);
  Act in2{stem_view(c, xnow.p, H, W), xnow};
  Buf st2;
  if (pair2) {
    rc = run_stem_pair(c, *pair2, in2, &st2);
    if (rc) return rc;
  }
  rc = run_chain(c, 'G', with_prefix("x", kEncoder, pair2 ? 1 : 0), pair2 ? Act{pair_half(st2, 0)} : in2.borrow(), nullptr, Dst{cat2.p, cat_ld, 0});
  if (rc) return rc;
  // pmconv6 writes the layout the attention reads: space-to-depth channel-blocked on the tensor-core path, NHWC otherwise
  const int pm_c8 = opt[SE_OPT_USE_CAM] ? (c.split() ? 1 : (tc ? 2 : 0)) : -1;
  Act pm;
  rc = run_chain(c, 'G', with_prefix("pm", {"conv1", "conv2_downsample", "conv3", "conv4_downsample", "conv5", "conv6"}, pair2 ? 1 : 0),
                 pair2 ? Act{pair_half(st2, 1), st2} : in2, &pm, Dst{nullptr, 0, 0, pm_c8});
  if (rc) return rc;
  if (opt[SE_OPT_USE_CAM]) {
    Buf ms = c.get((size_t)c.B * h * w * 4);
    c.tag("avgpool4_kernel", 0, 0, 0, (double)c.B * H * W * 4);
    CK(avgpool4(io.mask, (float*)ms.p, c.B, H, W, c.stream));
    TAP("in:G.cam", pm.v, pm.v.c8);
    TAP("in:G.cam.mask_s", nhwc(ms.p, h, w, 1, 1), 0, 0);
    Buf camo = c.get((size_t)c.B * h * w * 96 * e);
    if (c.split()) {
      // split-half mode: fp32 NHWC in / out of the attention (split-half fp16 GEMMs over explicit patch matrices, se_gemm_split.cu)
      Buf f32 = c.get((size_t)c.B * h * w * 96 * 4), o32 = c.get((size_t)c.B * h * w * 96 * 4);
      const Layout pml{LAYOUT_C8, h, w, pm.v.ld};
      CK(act_to_f32(pm.v.p, DT_F16X2, pml, (float*)f32.p, 1, c.B, 96, c.stream));
      TAP("in:G.cam.f32", nhwc(f32.p, h, w, 96, 96), 0, 0);
      rc = run_cam_split(c, (const float*)f32.p, h, w, 96, (const float*)ms.p, (float*)o32.p, io.attn);
      if (rc) return rc;
      TAP("out:G.cam.f32", nhwc(o32.p, h, w, 96, 96), 0, 0);
      CK(f32_to_act((const float*)o32.p, 1, camo.p, DT_F16X2, pml, c.B, 96, c.stream));
      c.put(o32); c.put(f32);
    } else {
      rc = tc ? run_cam_tc(c, pm.v, (const float*)ms.p, camo.p, io.attn) : run_cam(c, pm.v, (const float*)ms.p, camo.p, 96, io.attn, 0);
      if (rc) return rc;
    }
    c.put(ms);
    c.put(pm);
    pm = Act{c.dense(camo.p, h, w, 96, tc), camo};
  }
  rc = run_chain(c, 'G', with_prefix("pm", {"conv9", "conv10"}), pm, nullptr, Dst{cat2.p, cat_ld, 96});
  if (rc) return rc;
  rc = run_chain(c, 'G', with_prefix("allconv", kDecoder), Act{c.dense(cat2.p, h, w, 192, tc), cat2}, &dec);
  if (rc) return rc;
  HeadIO fine{};
  fine.stage = io.x_stage2;
  const bool blend = io.composed || io.composed_u8;
  if (blend) {
    fine.img = io.x; fine.blend = io.mask_soft; fine.blend_bs = io.msoft_bs;
    fine.composed = io.composed; fine.composed_bs = io.composed_bs; fine.bgr_u8 = io.composed_u8;
  }
  rc = run_head(c, 'G', "allconv17", dec.v, blend ? HEAD_FINE : HEAD_TANH, fine);
  if (rc) return rc;
  c.put(dec);
  return 0;
}

// One generate_fake call (editline2_model.py:338-370): image and sketch or their bytes; netM or the caller's edit mask (fp32, or
// bytes v meaning v/255); outputs where set, *_bs elements between images (0 = dense); mask_bin_in replaces netM's binarised
// mask, mask_bin_out receives the one netG inpaints. All fields are 8 bytes wide: they form the graph key.
struct Request {
  const float *image = nullptr, *sketch = nullptr;
  const unsigned char *image_u8 = nullptr, *sketch_u8 = nullptr;
  const float* edit_mask = nullptr;
  const unsigned char* edit_mask_u8 = nullptr;
  float *composed = nullptr, *mask = nullptr;
  long long composed_bs = 0, mask_bs = 0;
  unsigned char *bgr_u8 = nullptr, *mask_u8 = nullptr;
  float *coarse = nullptr, *fine = nullptr, *mask_image = nullptr;
  const float* mask_bin_in = nullptr;
  float* mask_bin_out = nullptr;
  float* attn = nullptr;                 // netG's attention weights (NetGIO::attn)
  unsigned char* hole_u8 = nullptr;      // the mask netG inpaints as 0 / 1 bytes [B,H,W]
};

// input codec, mask source, netM (only its trunk and image decoder, for mask_image, on a caller's mask), then
// netG(inputs, inputs, mask_bin, mask_bin, line) (editline2_model.py:368) blended with the soft mask
static int run_generate(Ctx& c, int H, int W, const Request& r) {
  const size_t plane = (size_t)c.B * H * W * 4;
  const bool from_netM = !r.edit_mask && !r.edit_mask_u8;
  const float *image = r.image, *sketch = r.sketch;
  Buf img, sk, soft, mb;
  if (r.image_u8) {
    // input codec (reference data/testimage_dataset.py:89-103); the output codec is fused into the two heads (test.py:25-35):
    // the float image and masks live only in the workspace
    img = c.get(3 * plane); sk = c.get(plane); mb = c.get(plane);
    if (!r.edit_mask) soft = c.get(plane);   // a caller's fp32 edit mask is blended as given: no soft plane to decode
    image = (const float*)img.p, sketch = (const float*)sk.p;
    c.tag(r.edit_mask_u8 ? "u8_to_inputs_kernel|input codec + edit mask" : "u8_to_inputs_kernel|input codec", 0, 0, 0,
          (double)c.B * H * W * (r.edit_mask_u8 ? 5 + 24 : 4 + 16));
    CK(u8_to_inputs(r.image_u8, r.sketch_u8, r.edit_mask_u8, (float*)img.p, (float*)sk.p, (float*)soft.p, (float*)mb.p, c.B, H, W, c.stream));
  } else if (from_netM || !r.mask_bin_out) {
    mb = c.get(plane);
  }
  float* msoft = r.image_u8 ? (float*)soft.p : r.mask;   // netM's soft mask, or the decoded edit mask
  const float* mbin = r.edit_mask && r.mask_bin_out ? r.mask_bin_out : (const float*)mb.p;   // the mask netG inpaints
  if (r.edit_mask) {
    c.tag("binarise_kernel|edit mask > 0.5", 0, 0, 0, (double)c.B * H * W * 8);
    CK(binarise(r.edit_mask, (float*)mbin, (long long)c.B * H * W, c.stream));
  }
  if (from_netM || r.mask_image) {
    NetMIO nm{image, sketch};
    nm.x_stage1 = r.mask_image;
    if (from_netM) { nm.mask = msoft; nm.mask_bs = r.mask_bs; nm.mask_bin = (float*)mb.p; nm.mask_u8 = r.mask_u8; }
    int rc = run_netM(c, H, W, nm);
    if (rc) return rc;
  }
  if (from_netM && r.mask_bin_in) mbin = r.mask_bin_in;
  if (from_netM && r.mask_bin_out && !c.dry) SE_CUDA_OK(cudaMemcpyAsync(r.mask_bin_out, mbin, plane, cudaMemcpyDeviceToDevice, c.stream));
  if (r.hole_u8) {
    c.tag("detail_hole_kernel|mask_inpaint bytes", 0, 0, 0, (double)c.B * H * W * 5);
    CK(detail_hole_u8(mbin, r.hole_u8, (long long)c.B * H * W, c.stream));
  }
  NetGIO g{image, image, mbin, mbin, sketch};
  g.x_stage1 = r.coarse; g.x_stage2 = r.fine; g.attn = r.attn;
  g.composed = r.composed; g.composed_bs = r.composed_bs; g.composed_u8 = r.bgr_u8;
  g.mask_soft = r.edit_mask ? r.edit_mask : msoft;
  g.msoft_bs = r.edit_mask ? 0 : r.mask_bs;
  int rc = run_netG(c, H, W, g);
  if (rc) return rc;
  c.put(mb); c.put(soft); c.put(sk); c.put(img);
  return 0;
}

// netM's mask alone on the input codec's bytes: the soft mask (caller's, or a workspace plane) and its bytes where set, from the
// trunk and the mask branch; netM's image decoder and netG do not run. The same launches as netM's inside run_generate on a u8
// request, so the mask is that forward's bit for bit. All fields are 8 bytes wide: they form the graph key.
struct MaskRequest {
  const unsigned char *image_u8 = nullptr, *sketch_u8 = nullptr;
  float* mask = nullptr;
  unsigned char* mask_u8 = nullptr;
};

static int run_predict_mask(Ctx& c, int H, int W, const MaskRequest& r) {
  const size_t plane = (size_t)c.B * H * W * 4;
  Buf img = c.get(3 * plane), sk = c.get(plane), soft;
  if (!r.mask) soft = c.get(plane);
  c.tag("u8_to_inputs_kernel|input codec", 0, 0, 0, (double)c.B * H * W * (4 + 16));
  CK(u8_to_inputs(r.image_u8, r.sketch_u8, nullptr, (float*)img.p, (float*)sk.p, nullptr, nullptr, c.B, H, W, c.stream));
  NetMIO nm{(const float*)img.p, (const float*)sk.p};
  nm.mask = r.mask ? r.mask : (float*)soft.p;
  nm.mask_u8 = r.mask_u8;
  int rc = run_netM(c, H, W, nm);
  if (rc) return rc;
  c.put(soft); c.put(sk); c.put(img);
  return 0;
}

// run `fn` twice: dry (arena peak) then for real
static const bool g_graphs_on = getenv("SE_NO_GRAPHS") == nullptr;
static const bool g_graph_log = getenv("SE_GRAPH_LOG") != nullptr;   // one stderr line per capture / failed capture
constexpr size_t kMaxGraphs = 16;

template <typename F>
static int with_arena(se_model* m, int prec, int B, cudaStream_t stream, F fn, std::vector<uintptr_t> key = {}) {
  SE_REQUIRE(m && m->finalized, "model not finalized");
  SE_REQUIRE(prec == SE_PREC_BF16_TC || prec == SE_PREC_FP32_TC || prec == SE_PREC_FP32_EXACT,
             "precision " + std::to_string(prec) + ": the modes are SE_PREC_BF16_TC (0), SE_PREC_FP32_TC (3) and SE_PREC_FP32_EXACT (1)");
  std::lock_guard<std::mutex> model_lock(m->mu);
  {
    int dev = -1;
    SE_CUDA_OK(cudaGetDevice(&dev));
    if (m->device < 0) m->device = dev;   // model-less operator holder: bound at first use
    SE_REQUIRE(dev == m->device, "model lives on device " + std::to_string(m->device) + " but the current device is " + std::to_string(dev));
    if (m->used && m->last_stream != stream) {
      // the previous forward may still be using the workspace on its own stream: order this one after it
      if (!m->order_ev) SE_CUDA_OK(cudaEventCreateWithFlags(&m->order_ev, cudaEventDisableTiming));
      SE_CUDA_OK(cudaEventRecord(m->order_ev, m->last_stream));
      SE_CUDA_OK(cudaStreamWaitEvent(stream, m->order_ev, 0));
    }
    m->last_stream = stream;
    m->used = true;
  }
  drop_taps(m);
  // ---- replay a captured forward (a forward with taps or the launch record on runs eagerly)
  const bool graphable = g_graphs_on && !g_timing && !m->taps_on && !c8_log_on() && !key.empty();
  const bool legacy = (stream == nullptr || stream == cudaStreamLegacy);
  cudaStream_t gs = stream;   // stream the graph is captured on / launched into
  if (graphable && legacy) {
    if (!m->gstream) {
      SE_CUDA_OK(cudaStreamCreateWithFlags(&m->gstream, cudaStreamNonBlocking));
      SE_CUDA_OK(cudaEventCreateWithFlags(&m->bridge_in, cudaEventDisableTiming));
      SE_CUDA_OK(cudaEventCreateWithFlags(&m->bridge_out, cudaEventDisableTiming));
    }
    gs = m->gstream;
  }
  auto bridge_in = [&]() -> int {
    if (gs != stream) { SE_CUDA_OK(cudaEventRecord(m->bridge_in, stream)); SE_CUDA_OK(cudaStreamWaitEvent(gs, m->bridge_in, 0)); }
    return 0;
  };
  auto bridge_out = [&]() -> int {
    if (gs != stream) { SE_CUDA_OK(cudaEventRecord(m->bridge_out, gs)); SE_CUDA_OK(cudaStreamWaitEvent(stream, m->bridge_out, 0)); }
    return 0;
  };
  const long long attn_limit = g_attn_limit.load();
  if (graphable) {
    for (int k = 0; k < 8; ++k) key.push_back((uintptr_t)m->opt[k]);
    key.push_back((uintptr_t)prec);
    key.push_back((uintptr_t)B);
    key.push_back((uintptr_t)attn_limit);   // decides the attention's band plan
    for (auto& g : m->graphs)
      if (g.exec && g.arena == m->arena && g.key == key) {
        int rb = bridge_in();
        if (rb) return rb;
        SE_CUDA_OK(cudaGraphLaunch(g.exec, gs));
        rb = bridge_out();
        if (rb) return rb;
        g.tick = ++m->tick;
        g_launches = g.launches;
        return 0;
      }
  }
  Ctx c;
  c.m = m; c.stream = stream; c.prec = prec; c.B = B; c.attn_limit = attn_limit;
  c.dry = true;
  c.arena.reset(nullptr);
  int rc = fn(c);
  if (rc) return rc;
  const size_t need = c.arena.peak + 4096;
  if (need > m->arena_bytes) {
    SE_CUDA_OK(cudaDeviceSynchronize());   // every stream that ever used the old slab
    for (auto& g : m->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);   // captured on the old slab
    m->graphs.clear();
    if (m->arena) SE_CUDA_OK(cudaFree(m->arena));
    m->arena = nullptr;
    m->arena_bytes = 0;
    SE_CUDA_OK(cudaMalloc(&m->arena, need));
    m->arena_bytes = need;
  }
  c.dry = false;
  c.arena.reset((char*)m->arena);
  g_launches = 0;
  // ---- second sighting of this signature: capture the launches into a graph (first sighting runs eagerly: it also performs the
  // one-time initialisations - function attributes, driver entry points - that must not happen inside a capture)
  if (graphable && m->seen[key]++ >= 1) {
    cudaGraph_t graph = nullptr;
    int rb = bridge_in();
    if (rb) return rb;
    if (cudaStreamBeginCapture(gs, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      c.stream = gs;
      rc = fn(c);
      c.stream = stream;
      const cudaError_t ce = cudaStreamEndCapture(gs, &graph);
      cudaGraphExec_t exec = nullptr;
      if (rc == 0 && ce == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
        cudaGraphDestroy(graph);
        if (m->graphs.size() >= kMaxGraphs) {   // evict the least recently used
          size_t lru = 0;
          for (size_t i = 1; i < m->graphs.size(); ++i) if (m->graphs[i].tick < m->graphs[lru].tick) lru = i;
          cudaGraphExecDestroy(m->graphs[lru].exec);
          m->graphs.erase(m->graphs.begin() + lru);
        }
        se_model::GraphEntry e;
        e.key = key; e.exec = exec; e.arena = m->arena; e.launches = g_launches; e.tick = ++m->tick;
        m->graphs.push_back(e);
        if (g_graph_log) fprintf(stderr, "[graph] captured B=%d prec=%d launches=%d (%zu cached)\n", B, prec, e.launches, m->graphs.size());
        SE_CUDA_OK(cudaGraphLaunch(exec, gs));
        return bridge_out();
      }
      if (g_graph_log) fprintf(stderr, "[graph] capture failed: rc=%d end=%s exec=%p\n", rc, cudaGetErrorString(ce), (void*)exec);
      if (graph) cudaGraphDestroy(graph);
      (void)cudaGetLastError();
      m->seen[key] = -1000000;   // not capturable: stay eager for this signature
      if (rc) return rc;
      c.arena.reset((char*)m->arena);
      g_launches = 0;
    } else {
      if (g_graph_log) fprintf(stderr, "[graph] cudaStreamBeginCapture failed: %s\n", cudaGetErrorString(cudaPeekAtLastError()));
      (void)cudaGetLastError();  // a failed cudaStreamBeginCapture leaves a sticky error behind
      m->seen[key] = -1000000;
    }
    rb = bridge_out();           // (orders nothing new, but keeps the two streams' event pairs balanced)
    if (rb) return rb;
  }
  if (g_graph_log && graphable) fprintf(stderr, "[graph] eager run B=%d prec=%d (sighting %d of this signature, %zu signatures seen)\n", B, prec, m->seen[key], m->seen.size());
  return fn(c);
}

// Two 5x5 stems that read the SAME packed 8-channel input become ONE launch with N = 96 (a stem tile is bound by its per-tile
// protocol and the small-N MMA rate, not by math: one N = 96 launch costs about what one N = 48 launch does).
//   "G.conv1+wconv1": packed input [x(1-m) (3), sketch, m, x2*m2 (3)]: conv1 reads channels 0..4, wconv1 its own image copy in
//                     5..7, the sketch channel (weight zeroed under --joint_train_inp, where the reference feeds zeros) and m
//   "G.xconv1+pmconv1": both read the 3 channels of the blended coarse result
// Fused output channel order [fA(24) fB(24) | gA(24) gB(24)] so that it is an ordinary gated layer with 96 outputs; the epilogue
// sends output blocks 0-2 to layer A's space-to-depth tensor and blocks 3-5 to layer B's (EpiParams::blk_split).
static int make_stem_pair(se_model* m, const char* key, const char* a, const char* b, const int* chan_a, const int* chan_b, float scale_b3) {
  Layer* A = find_layer(m, 'G', a);
  Layer* B = find_layer(m, 'G', b);
  if (!A || !B || !A->set || !B->set) return 0;
  Layer F;
  F.net = 'G';
  F.name = key;
  F.spec = Spec{8, 96, 5, 1, 1, false, 0};
  F.set = true;
  F.fused_pair = true;
  F.pair_cin_sum = A->spec.cin + B->spec.cin;
  F.w_host.assign((size_t)96 * 8 * 25, 0.0f);
  F.b_host.assign(96, 0.0f);
  for (int n = 0; n < 96; ++n) {
    const bool gate = n >= 48;
    const int r = n % 48;
    const Layer* S = r < 24 ? A : B;
    const int* chan = r < 24 ? chan_a : chan_b;
    const int co = (r % 24) + (gate ? 24 : 0);           // channel of the source layer: features 0..23, gates 24..47
    F.b_host[n] = S->b_host[co];
    for (int ci = 0; ci < S->spec.cin; ++ci) {
      const float sc = (S == B && ci == 3) ? scale_b3 : 1.0f;
      for (int t = 0; t < 25; ++t) F.w_host[((size_t)n * 8 + chan[ci]) * 25 + t] = S->w_host[((size_t)co * S->spec.cin + ci) * 25 + t] * sc;
    }
  }
  int rc = pack_layer(m, F);
  if (rc) return rc;
  F.w_host.clear();
  m->layers[std::string("G.") + key] = F;
  return 0;
}

static int check_hw(int H, int W) {
  SE_REQUIRE(H % 8 == 0 && W % 8 == 0 && H >= 16 && W >= 16, "H and W must be multiples of 8 and >= 16 (two stride-2 convs, 4x4 mask pool, stride-2 patch grid)");
  return 0;
}

// run(c, H, W, a) under a graph keyed on the kind, size and every byte of the argument struct a, so that a replay never writes
// through a pointer the call did not pass (with_arena appends the options, precision, B and the attention limit)
template <class Args>
static int keyed_forward(se_model* m, int prec, int B, int H, int W, void* stream, uintptr_t kind, const Args& a,
                         int (*run)(Ctx&, int, int, const Args&)) {
  static_assert(std::has_unique_object_representations_v<Args> && sizeof(Args) % sizeof(uintptr_t) == 0,
                "argument structs hold 8-byte fields only, so that every field is part of the key");
  int rc = check_hw(H, W);
  if (rc) return rc;
  std::vector<uintptr_t> key(3 + sizeof(Args) / sizeof(uintptr_t));
  key[0] = kind; key[1] = (uintptr_t)H; key[2] = (uintptr_t)W;
  memcpy(&key[3], &a, sizeof(Args));
  return with_arena(m, prec, B, (cudaStream_t)stream, [&](Ctx& c) { return run(c, H, W, a); }, key);
}

}  // namespace se

// ============================================================================================ C ABI
extern "C" {

const char* se_last_error(void) { return se::last_error(); }
int se_abi_version(void) { return 3; }

int se_model_create(se_model** out) {
  SE_REQUIRE(out != nullptr, "out");
  se_model* m = new se_model();
  for (char net : {'M', 'G'}) {
    ArchTable t = make_arch(net);
    for (size_t i = 0; i < t.specs.size(); ++i) {
      Layer L;
      L.spec = t.specs[i];
      L.net = net;
      L.name = t.names[i];
      m->layers[std::string(1, net) + "." + t.names[i]] = L;
    }
  }
  *out = m;
  return 0;
}

void se_model_destroy(se_model* m) {
  if (!m) return;
  drop_taps(m);
  for (void* p : m->owned) cudaFree(p);
  if (m->arena) cudaFree(m->arena);
  if (m->order_ev) cudaEventDestroy(m->order_ev);
  for (auto& g : m->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (m->gstream) cudaStreamDestroy(m->gstream);
  if (m->bridge_in) cudaEventDestroy(m->bridge_in);
  if (m->bridge_out) cudaEventDestroy(m->bridge_out);
  delete m;
}

int se_model_set_layer(se_model* m, char net, const char* layer, const float* weight, const float* bias, int cout, int cin, int ksize) {
  SE_REQUIRE(m && layer && weight && bias, "null argument");
  SE_REQUIRE(!m->finalized, "model already finalized");
  Layer* L = find_layer(m, net, layer);
  SE_REQUIRE(L != nullptr, std::string("no such layer: net") + net + "." + layer);
  SE_REQUIRE(L->spec.cout == cout && L->spec.cin == cin && L->spec.k == ksize,
             std::string("shape mismatch for ") + layer + ": expected [" + std::to_string(L->spec.cout) + "," + std::to_string(L->spec.cin) + "," +
                 std::to_string(L->spec.k) + "," + std::to_string(L->spec.k) + "]");
  L->w_host.assign(weight, weight + (size_t)cout * cin * ksize * ksize);
  L->b_host.assign(bias, bias + cout);
  L->set = true;
  return 0;
}

int se_model_set_option(se_model* m, int option, int value) {
  SE_REQUIRE(m && option >= 0 && option < 8, "option");
  SE_REQUIRE(!m->finalized, "options are fixed at se_model_finalize (they shape the packed weights)");
  m->opt[option] = value;
  return 0;
}

int se_model_finalize(se_model* m) {
  SE_REQUIRE(m, "model");
  SE_REQUIRE(!m->finalized, "model already finalized");
  int ndev = 0;
  SE_CUDA_OK(cudaGetDeviceCount(&ndev));
  SE_REQUIRE(ndev > 0, "no CUDA device: sketchedit_b200 has no CPU fallback");
  SE_CUDA_OK(cudaGetDevice(&m->device));   // packed weights and the workspace live on the device current now
  // a net may be left out entirely (stand-alone netM / netG modules); a partially set net is an error
  for (char net : {'M', 'G'}) {
    int nset = 0, ntot = 0;
    std::string first_missing;
    for (auto& kv : m->layers)
      if (kv.first[0] == net) {
        ++ntot;
        if (kv.second.set) ++nset;
        else if (first_missing.empty()) first_missing = kv.first;
      }
    SE_REQUIRE(nset == 0 || nset == ntot, "layer not set: net" + first_missing);
  }
  {
    const int id5[5] = {0, 1, 2, 3, 4}, w5[5] = {5, 6, 7, 3, 4}, id3[3] = {0, 1, 2};
    int rc = make_stem_pair(m, "conv1+wconv1", "conv1", "wconv1", id5, w5, m->opt[SE_OPT_JOINT_TRAIN_INP] ? 0.0f : 1.0f);
    if (rc) return rc;
    rc = make_stem_pair(m, "xconv1+pmconv1", "xconv1", "pmconv1", id3, id3, 1.0f);
    if (rc) return rc;
  }
  for (auto& kv : m->layers) {
    if (!kv.second.set || kv.second.fused_pair) continue;
    int rc = pack_layer(m, kv.second);
    if (rc) return rc;
    kv.second.w_host.clear();
    kv.second.w_host.shrink_to_fit();
  }
  m->finalized = true;
  return 0;
}

int se_forward_inference(se_model* m, const float* image, const float* sketch, int B, int H, int W, int precision, float* composed,
                         float* mask, float* coarse, float* fine, float* mask_image, const float* mask_bin_in, float* mask_bin_out,
                         void* stream) {
  SE_REQUIRE(image && sketch && composed && mask, "null tensor");
  Request r;
  r.image = image; r.sketch = sketch; r.composed = composed; r.mask = mask;
  r.coarse = coarse; r.fine = fine; r.mask_image = mask_image; r.mask_bin_in = mask_bin_in; r.mask_bin_out = mask_bin_out;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_forward_inference_packed(se_model* m, const float* image, const float* sketch, int B, int H, int W, int precision, float* packed,
                                void* stream) {
  SE_REQUIRE(image && sketch && packed, "null tensor");
  Request r;
  r.image = image; r.sketch = sketch;
  r.composed = packed; r.mask = packed + 3LL * H * W;   // [B,4,H,W]: composed in channels 0-2, the soft mask in channel 3
  r.composed_bs = r.mask_bs = 4LL * H * W;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_forward_inference_u8(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, int B, int H, int W, int precision,
                            unsigned char* bgr_u8, unsigned char* mask_u8, void* stream) {
  SE_REQUIRE(image_u8 && sketch_u8 && bgr_u8 && mask_u8, "null tensor");
  Request r;
  r.image_u8 = image_u8; r.sketch_u8 = sketch_u8; r.bgr_u8 = bgr_u8; r.mask_u8 = mask_u8;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_forward_with_mask(se_model* m, const float* image, const float* sketch, const float* edit_mask, int B, int H, int W, int precision,
                         float* composed, float* coarse, float* fine, float* mask_image, float* mask_bin_out, void* stream) {
  SE_REQUIRE(image && sketch && edit_mask && composed, "null tensor");
  Request r;
  r.image = image; r.sketch = sketch; r.edit_mask = edit_mask; r.composed = composed;
  r.coarse = coarse; r.fine = fine; r.mask_image = mask_image; r.mask_bin_out = mask_bin_out;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_forward_with_mask_u8(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, const unsigned char* edit_mask_u8, int B,
                            int H, int W, int precision, unsigned char* bgr_u8, void* stream) {
  SE_REQUIRE(image_u8 && sketch_u8 && edit_mask_u8 && bgr_u8, "null tensor");
  Request r;
  r.image_u8 = image_u8; r.sketch_u8 = sketch_u8; r.edit_mask_u8 = edit_mask_u8; r.bgr_u8 = bgr_u8;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_predict_mask_u8(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, int B, int H, int W, int precision,
                       float* mask, unsigned char* mask_u8, void* stream) {
  SE_REQUIRE(image_u8 && sketch_u8, "null tensor");
  SE_REQUIRE(mask || mask_u8, "se_predict_mask_u8 needs mask or mask_u8");
  MaskRequest r;
  r.image_u8 = image_u8; r.sketch_u8 = sketch_u8; r.mask = mask; r.mask_u8 = mask_u8;
  return keyed_forward(m, precision, B, H, W, stream, 4, r, run_predict_mask);
}

int se_forward_u8_with_soft_mask(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, const float* edit_mask, int B,
                                 int H, int W, int precision, unsigned char* bgr_u8, void* stream) {
  SE_REQUIRE(image_u8 && sketch_u8 && edit_mask && bgr_u8, "null tensor");
  Request r;
  r.image_u8 = image_u8; r.sketch_u8 = sketch_u8; r.edit_mask = edit_mask; r.bgr_u8 = bgr_u8;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_forward_u8_export(se_model* m, const unsigned char* image_u8, const unsigned char* sketch_u8, const unsigned char* edit_mask_u8,
                         const float* edit_mask, int B, int H, int W, int precision, unsigned char* bgr_u8, unsigned char* mask_u8, float* attn,
                         unsigned char* hole_u8, void* stream) {
  SE_REQUIRE(image_u8 && sketch_u8 && bgr_u8 && attn && hole_u8, "null tensor");
  SE_REQUIRE(!(edit_mask_u8 && edit_mask), "se_forward_u8_export takes at most one of edit_mask_u8 and edit_mask");
  SE_REQUIRE(edit_mask_u8 || edit_mask || mask_u8, "se_forward_u8_export without an edit mask writes mask_u8: it must not be NULL");
  SE_REQUIRE(m && m->opt[SE_OPT_USE_CAM], "se_forward_u8_export returns the contextual attention's weights: the model runs without it "
                                          "(use_cam = 0)");
  Request r;
  r.image_u8 = image_u8; r.sketch_u8 = sketch_u8; r.edit_mask_u8 = edit_mask_u8; r.edit_mask = edit_mask; r.bgr_u8 = bgr_u8;
  r.mask_u8 = edit_mask_u8 || edit_mask ? nullptr : mask_u8;
  r.attn = attn; r.hole_u8 = hole_u8;
  return keyed_forward(m, precision, B, H, W, stream, 1, r, run_generate);
}

int se_netM_forward(se_model* m, const float* x, const float* guide, int B, int H, int W, int precision, float* mask1, float* x_stage1,
                    void* stream) {
  SE_REQUIRE(x && guide && mask1, "null tensor");
  NetMIO io{x, guide, mask1};
  io.x_stage1 = x_stage1;
  return keyed_forward(m, precision, B, H, W, stream, 2, io, run_netM);
}

int se_netG_forward(se_model* m, const float* x, const float* x2, const float* mask, const float* mask2, const float* guide, int B, int H,
                    int W, int precision, float* x_stage1, float* x_stage2, void* stream) {
  SE_REQUIRE(x && x2 && mask && mask2 && x_stage2, "null tensor");   // guide may be NULL: guide=None of the reference
  const NetGIO io{x, x2, mask, mask2, guide, x_stage1, x_stage2};
  return keyed_forward(m, precision, B, H, W, stream, 3, io, run_netG);
}

int se_gated_conv_forward(se_model* m, char net, const char* layer, const float* x, int B, int H, int W, int precision, float* y,
                          void* stream) {
  SE_REQUIRE(m && layer && x && y, "null argument");
  Layer* L = find_ready(m, net, layer);
  SE_REQUIRE(L != nullptr, std::string("no such (loaded) layer: ") + layer);
  cudaStream_t st = (cudaStream_t)stream;
  return with_arena(m, precision, B, st, [&](Ctx& c) -> int {
    const Spec& s = L->spec;
    int Ho, Wo;
    out_dims(s, H, W, &Ho, &Wo);
    if (L->is_head) {
      // raw conv (activation=None / cout==3, utils.py:27) on the fp32 direct kernel in every mode, fp32 NHWC in and out; bf16
      // rounds its input to bf16 first (through a bf16 copy), like the heads of its forward read it
      const Layout lin{LAYOUT_NHWC, H, W, 12}, lout{LAYOUT_NHWC, Ho, Wo, s.cout};
      Buf in = c.get((size_t)B * H * W * 12 * 4), o = c.get((size_t)B * Ho * Wo * s.cout * 4);
      if (c.prec == SE_PREC_BF16_TC) {
        Buf r = c.get((size_t)B * H * W * 12 * 2);
        CK(f32_to_act(x, 0, r.p, DT_BF16, lin, B, 12, c.stream));
        CK(act_to_f32(r.p, DT_BF16, lin, (float*)in.p, 1, B, 12, c.stream));
        c.put(r);
      } else {
        CK(f32_to_act(x, 0, in.p, DT_F32, lin, B, 12, c.stream));
      }
      ConvParams cp;
      memset(&cp, 0, sizeof(cp));
      ClassW& cw = L->cls[0];
      cp.x = in.p; cp.in_dt = DT_F32; cp.N = B; cp.Hi = H; cp.Wi = W; cp.Ci = 12; cp.ldx = 12;
      cp.Ho = Ho; cp.Wo = Wo; cp.stride = 1; cp.ntaps = cw.direct.n;
      memcpy(cp.dy, cw.direct.dy, sizeof(cp.dy));
      memcpy(cp.dx, cw.direct.dx, sizeof(cp.dx));
      cp.w = cw.w_direct; cp.bias = L->bias; cp.Cout = s.cout;
      cp.y = o.p; cp.out_dt = DT_F32; cp.Hout = Ho; cp.Wout = Wo; cp.ldo = s.cout; cp.choff = 0;
      cp.osy = cp.osx = 1; cp.epi = EPI_LINEAR; cp.scale = 1.0f;
      CK(direct_launch(cp, cw.CoutP, c.stream));
      CK(act_to_f32(o.p, DT_F32, lout, y, 0, B, s.cout, c.stream));
      c.put(o);
      c.put(in);
      return 0;
    }
    // input in the layout the layer reads, in the mode's storage (channel-blocked padding channels and the pad pixels of the
    // packed stem rows zeroed first); output channel-blocked in split-half, NHWC otherwise
    const int in_c8 = wants_c8(c, *L);
    Buf in = c.get(L->is_stem ? (size_t)B * H * stem_wp(W) * 8 * c.esz() : c.act_bytes(H, W, L->Ci, in_c8));
    const View vin = L->is_stem ? stem_view(c, in.p, H, W) : c.dense(in.p, H, W, L->Ci, in_c8);
    if (L->is_stem || (in_c8 && s.cin % 8)) CK(fill_zero(in.p, in.bytes, c.stream));
    const Layout lin{L->is_stem ? LAYOUT_ROWS : in_c8, H, W, vin.ld, stem_wp(W), STEM_PADL};
    CK(f32_to_act(x, 0, in.p, c.act_dt(), lin, B, s.cin, c.stream));
    const int cg = s.cout / 2, out_c8 = c.split() ? 1 : 0;
    Buf o = c.get(c.act_bytes(Ho, Wo, cg, out_c8));
    const View vo = c.dense(o.p, Ho, Wo, cg, out_c8);
    if (out_c8 && cg % 8) CK(fill_zero(o.p, o.bytes, c.stream));
    int r = run_layer(c, *L, vin, o.p, vo.ld, 0, out_c8);
    if (r) return r;
    CK(act_to_f32(o.p, c.act_dt(), Layout{out_c8, Ho, Wo, vo.ld}, y, 0, B, cg, c.stream));
    c.put(o);
    c.put(in);
    return 0;
  });
}

int se_contextual_attention_forward(const float* feat, const float* mask_s, int B, int C, int h, int w, int precision, float* out,
                                    float* attn, void* stream) {
  SE_REQUIRE(feat && mask_s && out, "null tensor");
  static se_model* holder = nullptr;   // arena owner for the model-less operator call
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  if (!holder) { holder = new se_model(); holder->finalized = true; }
  // fp32-on-tensor-cores mode: split-half GEMM attention (needs 16 * C to be a multiple of 256 and no attention-map output);
  // bf16: the tensor-core attention over netG's 96 channels. Everything else runs on the fp32 CUDA-core kernels.
  const bool even = h % 2 == 0 && w % 2 == 0;
  const bool split_cam = precision == SE_PREC_FP32_TC && C % 16 == 0 && attn == nullptr && even;
  const bool tc_cam = precision == SE_PREC_BF16_TC && C == 96 && even;
  if (precision == SE_PREC_FP32_TC || (precision == SE_PREC_BF16_TC && !tc_cam)) precision = SE_PREC_FP32_EXACT;
  cudaStream_t st = (cudaStream_t)stream;
  return with_arena(holder, precision, B, st, [&](Ctx& c) -> int {
    const Layout nhwc_l{LAYOUT_NHWC, h, w, C};
    Buf in = c.get((size_t)B * h * w * C * c.esz()), o = c.get((size_t)B * h * w * C * c.esz());
    if (tc_cam) {
      // the layouts netG uses on the tensor-core path: space-to-depth channel-blocked in, channel-blocked out
      CK(f32_to_act(feat, 0, in.p, DT_BF16, Layout{LAYOUT_S2D, h, w, 4 * (C / 8)}, B, C, c.stream));
      int r = run_cam_tc(c, c.dense(in.p, h, w, C, 2), mask_s, o.p, attn);
      if (r) return r;
      CK(act_to_f32(o.p, DT_BF16, Layout{LAYOUT_C8, h, w, C / 8}, out, 0, B, C, c.stream));
    } else {
      CK(f32_to_act(feat, 0, in.p, DT_F32, nhwc_l, B, C, c.stream));
      int r = split_cam ? run_cam_split(c, (const float*)in.p, h, w, C, mask_s, (float*)o.p)
                        : run_cam(c, nhwc(in.p, h, w, C, C), mask_s, o.p, C, attn);
      if (r) return r;
      CK(act_to_f32(o.p, DT_F32, nhwc_l, out, 0, B, C, c.stream));
    }
    c.put(o);
    c.put(in);
    return 0;
  });
}

int se_outputs_to_uint8(const float* composed, const float* mask, int B, int H, int W, unsigned char* bgr_hwc, unsigned char* mask_u8,
                        void* stream) {
  SE_REQUIRE(composed && bgr_hwc && (mask || !mask_u8), "null tensor");
  return to_uint8(composed, mask, bgr_hwc, mask_u8, B, H, W, (cudaStream_t)stream);
}

int se_set_attention_workspace_limit(long long bytes) {
  SE_REQUIRE(bytes >= 0, "attention workspace limit must be >= 0 bytes (0 = the default)");
  g_attn_limit = bytes ? bytes : kDefaultAttnLimit;
  return 0;
}

int se_taps_enable(se_model* m, int on) {
  SE_REQUIRE(m, "model");
  std::lock_guard<std::mutex> lk(m->mu);
  m->taps_on = on != 0;
  drop_taps(m);
  return 0;
}

int se_taps_count(se_model* m) {
  if (!m) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  return (int)m->taps.size();
}

int se_tap_info(se_model* m, int i, char* name, int name_cap, int* desc, long long* bytes) {
  SE_REQUIRE(m, "model");
  std::lock_guard<std::mutex> lk(m->mu);
  SE_REQUIRE(i >= 0 && i < (int)m->taps.size(), "tap index " + std::to_string(i) + " of " + std::to_string(m->taps.size()));
  const se_model::Tap& t = m->taps[i];
  if (name && name_cap > 0) {
    const size_t n = std::min(t.name.size(), (size_t)name_cap - 1);
    memcpy(name, t.name.data(), n);
    name[n] = 0;
  }
  if (desc) memcpy(desc, t.desc, sizeof(t.desc));
  if (bytes) *bytes = (long long)t.bytes;
  return 0;
}

int se_tap_copy(se_model* m, int i, void* dst, void* stream) {
  SE_REQUIRE(m && dst, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  SE_REQUIRE(i >= 0 && i < (int)m->taps.size(), "tap index " + std::to_string(i) + " of " + std::to_string(m->taps.size()));
  SE_CUDA_OK(cudaMemcpyAsync(dst, m->taps[i].p, m->taps[i].bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

int se_last_launch_count(void) { return se::g_launches; }
long long se_workspace_bytes(se_model* m) { return m ? (long long)m->arena_bytes : 0; }

int se_timing_enable(int on) {
  std::lock_guard<std::mutex> lk(g_time_mu);
  g_timing = on != 0;
  g_tl_used = 0;
  g_classes.clear();
  g_class_idx.clear();
  return 0;
}

// JSON text: {"classes":[{"name","tensor","launches","ms","flops_alg","flops_exec","bytes_alg"},...]} of everything
// launched since se_timing_enable(1). Synchronises on the recorded events. Returns the length needed (>= cap: truncated).
int se_timing_report(char* buf, int cap) {
  std::lock_guard<std::mutex> lk(g_time_mu);
  for (auto& a : g_classes) a.ms = 0.0;
  for (size_t i = 0; i < g_tl_used; ++i) {
    float t = 0.0f;
    if (cudaEventSynchronize(g_tl[i].b) != cudaSuccess || cudaEventElapsedTime(&t, g_tl[i].a, g_tl[i].b) != cudaSuccess) {
      set_error("se_timing_report: event query failed");
      return -1;
    }
    g_classes[g_tl[i].cls].ms += t;
  }
  std::string out = "{\"classes\":[";
  for (size_t i = 0; i < g_classes.size(); ++i) {
    const ClassAgg& a = g_classes[i];
    char num[256];
    snprintf(num, sizeof(num), "\",\"tensor\":%d,\"launches\":%d,\"ms\":%.6f,\"flops_alg\":%.6e,\"flops_exec\":%.6e,\"bytes_alg\":%.6e}", a.tensor, a.launches,
             a.ms, a.flops_alg, a.flops_exec, a.bytes_alg);
    out += std::string(i ? "," : "") + "{\"name\":\"" + a.name + num;
  }
  out += "]}";
  if (buf && cap > 0) {
    const size_t n = out.size() < (size_t)cap - 1 ? out.size() : (size_t)cap - 1;
    memcpy(buf, out.data(), n);
    buf[n] = 0;
  }
  return (int)out.size() + 1;
}

}  // extern "C"
