// LW-DETR forward engine (host side).  Packs a reference-format checkpoint into kernel-native
// layouts once, then runs a fixed schedule of hand-written sm_90a kernels per batch:
//   patch gather -> [LN, qkv GEMM, fused attention, proj GEMM(+layer-scale+residual), LN, fc1 GEMM(GELU),
//   fc2 GEMM(+layer-scale+residual)] x depth -> projector (1x1 / implicit 3x3 / pixel-shuffle GEMMs,
//   channel LN writing the decoder memory directly) -> two-stage selection (GEMMs, row max, top-k,
//   gathers) -> 3 decoder layers (GEMMs, fused attention, fused deformable gather, LNs) -> heads.
// Reference call stack being replaced: SURVEY.md section 3.2 (lwdetr.py:111-174 and callees).
#include "engine.h"
#include "launch.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "attn.h"
#include "gemm_tc.h"
#include "msda.h"
#include "resize.h"
#include "rowops.h"

namespace lwb {

namespace {
struct Mat {
  void* p;
  int ld;
};
inline char* cptr(void* p) { return static_cast<char*>(p); }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// One pass of Engine::plan.  Pass 0 sizes the workspace: allocations only advance the bump offset (and return null),
// weight lookups return null and nothing is recorded.  Pass 1 lays the same allocations out from the arena base, resolves
// the packed weights and records the ops.  The first error is kept.
class OpBuilder {
 public:
  OpBuilder(int pass, int dtype, void* arena, const std::map<std::string, void*>& w16s, const std::map<std::string, float*>& w32s,
            std::string too_big, std::string* err, std::vector<Op>* ops)
      : pass_(pass), dtype_(dtype), arena_(pass ? arena : nullptr), w16s_(w16s), w32s_(w32s), too_big_(std::move(too_big)),
        err_(err), ops_(ops) {}

  bool failed() const { return failed_; }
  size_t bytes() const { return off_; }
  void fail(const std::string& m) { if (!failed_) *err_ = m; failed_ = true; }
  // every kernel indexes a buffer's elements / a GEMM's rows with 32-bit integers somewhere: no buffer may exceed that range
  bool fits(long long n) { if (n > 2147483647LL) fail(too_big_); return n <= 2147483647LL; }
  void* alloc(size_t bytes) {
    off_ = align_up(off_, 1024);
    void* p = arena_ ? cptr(arena_) + off_ : nullptr;
    off_ += bytes;
    return p;
  }
  Mat buf16(long long rows, int cols) { fits(rows * cols); return Mat{alloc(static_cast<size_t>(rows) * cols * 2), cols}; }
  float* buf32(long long n) { fits(n); return static_cast<float*>(alloc(static_cast<size_t>(n) * 4)); }
  void* w16(const std::string& k) { return lookup(w16s_, k, "internal: weight "); }
  float* w32(const std::string& k) { return lookup(w32s_, k, "internal: vector "); }

  void record(const std::string& label, std::function<int(cudaStream_t)> run, const OutView& out, double flops, double bytes,
              bool reads_input) {
    if (pass_ == 0 || failed_) return;
    Op op;
    op.label = label; op.run = std::move(run);
    op.out = out;
    op.flops = flops; op.bytes = bytes; op.reads_input = reads_input;
    ops_->push_back(std::move(op));
  }
  // a further output of the op recorded last, captured as "<label>.<name>"
  void also(const std::string& name, const OutView& v) {
    if (pass_ == 0 || failed_) return;
    ops_->back().extra.emplace_back(name, v);
  }
  void op(const std::string& label, std::function<int(cudaStream_t)> run, const OutView& out, double bytes, bool reads_input = false) {
    record(label, std::move(run), out, 0.0, bytes, reads_input);
  }
  // out = epilogue(A W^T) with W = `wkey`.w, bias `wkey`.b if packed (and colsum `wkey`.cs for a LayerNorm consumer); `g` carries
  // the A mode and the epilogue, the rest is filled in here
  void gemm(const std::string& label, GemmDesc g, Mat A, long long M, int K, const std::string& wkey, int N, Mat out) {
    if (!fits(M) || pass_ == 0) return;
    g.dtype = dtype_; g.A = A.p; g.lda = A.ld; g.M = static_cast<int>(M); g.N = N; g.K = K;
    g.W = w16(wkey + ".w"); g.bias = w32s_.count(wkey + ".b") ? w32s_.at(wkey + ".b") : nullptr;
    g.out = out.p; g.ld_out = out.ld; g.stats_parts_in = stats_parts_;
    if (g.stats_in) g.colsum = w32(wkey + ".cs");
    GemmOp op;
    std::string e;
    if (failed_ || gemm_build(g, &op, &e)) return fail(label + ": " + e);
    if (g.stats_out) {   // partial (sum, sumsq) pairs per row written by the N = C producer GEMMs: the same for all of them
      if (stats_parts_ == 0) stats_parts_ = op.args.stats_parts_out;
      if (stats_parts_ != op.args.stats_parts_out || stats_parts_ > 48) return fail(label + ": inconsistent LayerNorm partial count");
    }
    const long long rows = g.hm_S ? M * g.hm_slices * g.hm_heads : (g.shuffle_cout ? M * 4 : M);
    const int cols = g.shuffle_cout ? g.shuffle_cout : (g.hm_S ? 16 : N);
    record(label, [op](cudaStream_t st) { return gemm_launch(op, st); }, {out.p, rows, cols, out.ld, g.out_fp32}, op.flops,
           2.0 * (static_cast<double>(M) * K + static_cast<double>(N) * K) + (g.out_fp32 ? 4.0 : 2.0) * M * N + (g.resid ? 2.0 * M * N : 0.0),
           false);
  }
  // the e4m3 GEMM: A e4m3 codes [M, K] with per-row scales; W, per-channel scales and bias `wkey`.w / .s / .b
  void gemm_e4m3(const std::string& label, const void* A, const float* a_scale, long long M, int K, const std::string& wkey, int N, int act,
                 Mat out) {
    if (pass_ == 0) return;
    GemmE4m3Desc g;
    g.A = A; g.lda = K; g.a_scale = a_scale; g.M = static_cast<int>(M); g.K = K; g.N = N;
    g.W = w16(wkey + ".w"); g.w_scale = w32(wkey + ".s"); g.bias = w32(wkey + ".b"); g.act = act; g.out = out.p; g.ld_out = out.ld;
    GemmOp op;
    std::string e;
    if (failed_ || gemm_e4m3_build(g, &op, &e)) return fail(label + ": " + e);
    record(label, [op](cudaStream_t st) { return gemm_launch(op, st); }, {out.p, M, N, out.ld, 0}, op.flops,
           1.0 * (static_cast<double>(M) * K + static_cast<double>(N) * K) + 4.0 * M + 8.0 * N + 2.0 * M * N, false);   // 1-byte operands
  }
  // fused ViT MLP (vit_mlp_kernel) of block `k`: LN2 statistics from stats_in, folded fc1, GELU, fc2, layer-scale and
  // residual; writes the next block's LayerNorm partials in the layout the fc2 GEMM would have used
  void mlp(const std::string& label, Mat x, long long M, const float2* stats_in, const std::string& k, float2* stats_out, Mat out) {
    if (pass_ == 0) return;
    MlpDesc g;
    g.dtype = dtype_; g.x = x.p; g.ldx = x.ld; g.M = static_cast<int>(M);
    g.stats_in = stats_in; g.stats_parts_in = stats_parts_; g.ln_eps = 1e-6f;
    g.w1 = w16(k + "fc1_ln.w"); g.colsum1 = w32(k + "fc1_ln.cs"); g.b1 = w32(k + "fc1_ln.b");
    g.w2 = w16(k + "fc2.w"); g.b2 = w32(k + "fc2.b"); g.gamma = w32(k + "g2");
    g.out = out.p; g.ld_out = out.ld; g.stats_out = stats_out; g.stats_parts_out = stats_parts_;
    MlpOp op;
    std::string e;
    if (failed_ || vit_mlp_build(g, &op, &e)) return fail(label + ": " + e);
    record(label, [op](cudaStream_t st) { return vit_mlp_launch(op, st); }, {out.p, M, MLP_C, out.ld, 0}, op.flops,
           2.0 * 3.0 * M * MLP_C + 2.0 * 2.0 * (4.0 * MLP_C) * MLP_C, false);   // x (operand and residual), out, both weights
  }
  // y = LN(x; `nkey`.w / .b, eps) over rows x C; `a` carries the optional fields (row flag / override, y2 = y + add_src, grouped
  // y rows, and the chained y3 = LN(y; `nkey3`.w / .b, eps3)), the rest is filled in here
  void layernorm(const std::string& label, Mat x, Mat y, const std::string& nkey, float eps, long long rows, int C, LayerNormArgs a = {},
                 const std::string& nkey3 = std::string()) {
    if (pass_ == 0) return;
    if (a.y3) { a.w3 = w32(nkey3 + ".w"); a.b3 = w32(nkey3 + ".b"); }
    a.x = x.p; a.ldx = x.ld; a.y = y.p; a.ldy = y.ld; a.w = w32(nkey + ".w"); a.b = w32(nkey + ".b"); a.eps = eps;
    a.rows = rows; a.C = C;
    if (a.flag_mod < 1) a.flag_mod = 1;
    const int dt = dtype_;
    const long long out_rows = a.y_group ? rows / a.y_group * a.y_group_stride : rows;
    record(label, [a, dt](cudaStream_t st) { return layernorm_launch(dt, a, st); }, {y.p, out_rows, C, y.ld, 0}, 0.0,
           4.0 * rows * C + (a.y2 ? 4.0 * rows * C : 0.0) + (a.y3 ? 2.0 * rows * C : 0.0), false);
  }
  void attention(const std::string& label, Mat q, Mat k, Mat v, Mat o, int nseq, int seqlen, int heads, int dh) {
    if (pass_ == 0) return;
    AttnArgs a;
    a.q = q.p; a.k = k.p; a.v = v.p; a.ldq = q.ld; a.ldk = k.ld; a.ldv = v.ld; a.o = o.p; a.ldo = o.ld;
    a.seqlen = seqlen; a.nseq = nseq; a.heads = heads;
    a.scale_log2 = 1.4426950408889634f / std::sqrt(static_cast<float>(dh));
    const int dt = dtype_;
    record(label, [a, dt, dh](cudaStream_t st) { return attention_launch(dt, a, dh, st); }, {o.p, 1LL * nseq * seqlen, heads * dh, o.ld, 0},
           4.0 * nseq * static_cast<double>(seqlen) * seqlen * heads * dh, 2.0 * 4.0 * nseq * seqlen * heads * dh, false);
  }

 private:
  template <typename T>
  T* lookup(const std::map<std::string, T*>& m, const std::string& k, const char* what) {   // packed weights: pass 1 only
    if (pass_ == 0) return nullptr;
    auto it = m.find(k);
    if (it == m.end()) { fail(what + k); return nullptr; }
    return it->second;
  }

  const int pass_, dtype_;
  void* const arena_;
  const std::map<std::string, void*>& w16s_;
  const std::map<std::string, float*>& w32s_;
  const std::string too_big_;
  std::string* const err_;
  std::vector<Op>* const ops_;
  size_t off_ = 0;          // workspace bump offset
  bool failed_ = false;
  int stats_parts_ = 0;     // LayerNorm partials per row of the ViT's statistics producers (0 until the first one is built)
};
}  // namespace

// ------------------------------------------------------------------------------- host math helpers
// Bicubic resize, align_corners=False, cubic-convolution kernel with A = -0.75 and border clamping:
// the semantics of F.interpolate(mode="bicubic") used by get_abs_pos (vit.py:44-52).
static void cubic_coeffs(float t, float w[4]) {
  const float A = -0.75f;
  auto c1 = [&](float x) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; };            // |x| <= 1
  auto c2 = [&](float x) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; };      // 1 < |x| < 2
  w[0] = c2(t + 1.f);
  w[1] = c1(t);
  w[2] = c1(1.f - t);
  w[3] = c2(2.f - t);
}
// source taps and weights of one output axis (F.interpolate's scale = n_in / n_out, border clamped)
static void cubic_axis(int n_in, int n_out, std::vector<int>* idx, std::vector<float>* wts) {
  const float scale = static_cast<float>(n_in) / static_cast<float>(n_out);
  idx->assign(static_cast<size_t>(n_out) * 4, 0);
  wts->assign(static_cast<size_t>(n_out) * 4, 0.f);
  for (int o = 0; o < n_out; ++o) {
    const float s = (o + 0.5f) * scale - 0.5f;
    const float f = std::floor(s);
    cubic_coeffs(s - f, &(*wts)[o * 4]);
    for (int k = 0; k < 4; ++k) (*idx)[o * 4 + k] = std::min(std::max(static_cast<int>(f) - 1 + k, 0), n_in - 1);
  }
}
void bicubic_resize_chlast_hw(const float* src, int n_in, int C, int out_h, int out_w, float* dst) {
  std::vector<int> iy, ix;
  std::vector<float> wy, wx;
  cubic_axis(n_in, out_h, &iy, &wy);
  cubic_axis(n_in, out_w, &ix, &wx);
  for (int oy = 0; oy < out_h; ++oy)
    for (int ox = 0; ox < out_w; ++ox) {
      float* d = dst + (static_cast<size_t>(oy) * out_w + ox) * C;
      for (int c = 0; c < C; ++c) d[c] = 0.f;
      for (int ky = 0; ky < 4; ++ky)
        for (int kx = 0; kx < 4; ++kx) {
          const float w = wy[oy * 4 + ky] * wx[ox * 4 + kx];
          const float* s = src + (static_cast<size_t>(iy[oy * 4 + ky]) * n_in + ix[ox * 4 + kx]) * C;
          for (int c = 0; c < C; ++c) d[c] += w * s[c];
        }
    }
}
void bicubic_resize_chlast(const float* src, int n_in, int C, int n_out, float* dst) { bicubic_resize_chlast_hw(src, n_in, C, n_out, n_out, dst); }

// fp32 -> e4m3 (OCP E4M3, "fn": no infinities, 0x7F is NaN) code, round to nearest even, saturating to +-448: what
// cvt.rn.satfinite.e4m3x2.f32 computes on the device and torch's float8_e4m3fn conversion after a clamp to +-448.
static uint8_t e4m3_code(float v) {
  const uint8_t sign = std::signbit(v) ? 0x80 : 0x00;
  const float a = std::fabs(v);
  if (!(a < 448.f)) return sign | 0x7E;                        // saturate (and +-448 itself)
  if (a < 0.015625f) return sign | static_cast<uint8_t>(std::nearbyint(a * 512.f));   // subnormal steps of 2^-9 (8 -> 2^-6)
  int e;
  const float f = std::frexp(a, &e);                            // a = f * 2^e, f in [0.5, 1)
  int m = static_cast<int>(std::nearbyint((f * 2.f - 1.f) * 8.f));
  int be = e - 1 + 7;
  if (m == 8) { m = 0; ++be; }
  const int code = (be << 3) | m;
  return sign | static_cast<uint8_t>(code > 0x7E ? 0x7E : code);
}

void host_quant_e4m3_rows(const float* src, long long rows, int K, uint8_t* q, float* scale) {
  for (long long r = 0; r < rows; ++r) {
    const float* x = src + r * K;
    float m = 0.f;
    for (int k = 0; k < K; ++k) m = std::max(m, std::fabs(x[k]));
    const float inv = m > 0.f ? 448.f / m : 1.f;
    scale[r] = m > 0.f ? m / 448.f : 1.f;
    for (int k = 0; k < K; ++k) q[r * K + k] = e4m3_code(x[k] * inv);
  }
}

// The ViT's position table at a GH x GW token grid: the 14x14 pretraining grid of pos_embed [197, C] (cls slot first)
// resized bicubically (vit.py:26-54) and laid out in window-major token order (vit.py:353-358), fp32.
static std::vector<float> window_major_pos(const float* pos_embed, int C, int GH, int GW) {
  const int T = GH * GW, wh = GH / 4, ww = GW / 4, wsz = wh * ww;
  std::vector<float> grid(static_cast<size_t>(T) * C), wm(static_cast<size_t>(T) * C);
  bicubic_resize_chlast_hw(pos_embed + C, 14, C, GH, GW, grid.data());   // drop the cls slot (vit.py:39-40)
  for (int r = 0; r < T; ++r) {   // window-major row r -> spatial (y, x)
    const int win = r / wsz, t = r % wsz;
    const int y = (win >> 2) * wh + t / ww, x = (win & 3) * ww + t % ww;
    std::memcpy(&wm[static_cast<size_t>(r) * C], &grid[(static_cast<size_t>(y) * GW + x) * C], C * sizeof(float));
  }
  return wm;
}

// ------------------------------------------------------------------------------- Engine basics
// LWDETR_F16_E4M3 is the fp16 engine with the encoder's qkv / fc1 (and their LayerNorms) in e4m3
Engine::Engine(const lwdetr_config& cfg, int dtype) : cfg_(cfg), dtype_(dtype == LWDETR_F16_E4M3 ? DT_F16 : dtype), e4m3_(dtype == LWDETR_F16_E4M3) {
  cudaGetDevice(&device_);
}

Engine::~Engine() {
  DeviceGuard guard(device_);
  plan_.reset();
  if (gstream_) cudaStreamDestroy(gstream_);
  if (ev_in_) cudaEventDestroy(ev_in_);
  if (ev_out_) cudaEventDestroy(ev_out_);
  if (warena_.p) cudaFree(warena_.p);
  if (sarena_.p) cudaFree(sarena_.p);
}

void* Engine::walloc(size_t bytes) {
  woff_ = align_up(woff_, 256);
  if (woff_ + bytes > warena_.bytes) return nullptr;
  void* p = cptr(warena_.p) + woff_;
  woff_ += bytes;
  return p;
}

std::vector<uint16_t> Engine::to16(const std::vector<float>& v) const {
  std::vector<uint16_t> h(v.size());
  if (dtype_ == DT_BF16) {
    for (size_t i = 0; i < v.size(); ++i) {
      __nv_bfloat16 b = __float2bfloat16_rn(v[i]);
      std::memcpy(&h[i], &b, 2);
    }
  } else {
    for (size_t i = 0; i < v.size(); ++i) {
      __half b = __float2half_rn(v[i]);
      std::memcpy(&h[i], &b, 2);
    }
  }
  return h;
}
void* Engine::upload16(const std::vector<float>& v) {
  void* d = walloc(v.size() * 2);
  if (!d) return nullptr;
  const std::vector<uint16_t> h = to16(v);
  cudaMemcpy(d, h.data(), h.size() * 2, cudaMemcpyHostToDevice);
  return d;
}
void* Engine::upload8(const std::vector<uint8_t>& v) {
  void* d = walloc(v.size());
  if (!d) return nullptr;
  cudaMemcpy(d, v.data(), v.size(), cudaMemcpyHostToDevice);
  return d;
}
float* Engine::upload32(const std::vector<float>& v) {
  void* d = walloc(v.size() * 4);
  if (!d) return nullptr;
  cudaMemcpy(d, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
  return static_cast<float*>(d);
}

int Engine::set_option(const char* name, int value) {
  if (std::strcmp(name, "fuse_layernorm") == 0) {
    fuse_ln_ = value;
    plan_.reset();
    return 0;
  }
  if (std::strcmp(name, "cuda_graph") == 0) {
    use_graph_ = value;
    if (plan_) plan_->clear_graphs();
    return 0;
  }
  if (std::strcmp(name, "pdl") == 0) {                 // programmatic dependent launch of every kernel (launch.h); process-wide
    pdl_enabled() = value ? 1 : 0;
    if (plan_) plan_->clear_graphs();
    return 0;
  }
  return -1;
}

// ------------------------------------------------------------------------------- weight packing
int Engine::load_weights(const std::map<std::string, HostTensor>& w, std::string* err) {
  DeviceGuard guard(device_);
  // Whatever happens below, the old packing is gone: a failed load must not leave a schedule pointing into a freed arena.
  weights_loaded_ = false;
  plan_.reset();
  const int C = cfg_.vit_dim, d = cfg_.hidden_dim, nq = cfg_.num_queries, ncls = cfg_.num_classes;
  const int G = cfg_.img_size / 16, ntap = cfg_.n_taps, c2 = d / 2;
  const int M = cfg_.ca_heads, L = cfg_.n_levels, P = cfg_.dec_points, ff = cfg_.dim_feedforward;
  bool missing = false;
  auto get = [&](const std::string& name, long long numel) -> const float* {
    auto it = w.find(name);
    if (it == w.end()) { if (!missing) *err = "missing tensor " + name; missing = true; return nullptr; }
    if (it->second.numel != numel) {
      if (!missing) *err = "tensor " + name + " has " + std::to_string(it->second.numel) + " elements, expected " + std::to_string(numel);
      missing = true; return nullptr;
    }
    return it->second.data;
  };
  auto vec = [&](const std::string& name, long long numel) {
    const float* p = get(name, numel);
    return p ? std::vector<float>(p, p + numel) : std::vector<float>(static_cast<size_t>(numel), 0.f);
  };
  // total parameter bytes bound: every tensor at most once in 16-bit + fp32 vectors + slack
  long long total = 0;
  for (auto& kv : w) total += kv.second.numel;
  if (warena_.p) { cudaFree(warena_.p); warena_.p = nullptr; }
  warena_.bytes = static_cast<size_t>(total) * 4 + (96u << 20);
  if (cudaMalloc(&warena_.p, warena_.bytes) != cudaSuccess) { *err = "cudaMalloc(weight arena) failed"; return -1; }
  woff_ = 0;
  W_.clear(); F_.clear();
  bool oom = false;
  auto put16 = [&](const std::string& key, const std::vector<float>& v) { void* p = upload16(v); if (!p) oom = true; W_[key] = p; };
  auto put32 = [&](const std::string& key, const std::vector<float>& v) { float* p = upload32(v); if (!p) oom = true; F_[key] = p; };

  const int dtl = dtype_;
  auto round16 = [dtl](float f) -> float {
    return dtl == DT_BF16 ? __bfloat162float(__float2bfloat16_rn(f)) : __half2float(__float2half_rn(f));
  };
  // fold BatchNorm (eval, eps 1e-5) into a bias-free conv: returns (W', b') with W' laid out [Co][k-order]
  auto fold_convx = [&](const std::string& p, int co, int ci, int k, std::vector<float>* Wp, std::vector<float>* bp) {
    auto cw = vec(p + ".conv.weight", 1LL * co * ci * k * k);
    auto g = vec(p + ".bn.weight", co), b = vec(p + ".bn.bias", co), mu = vec(p + ".bn.running_mean", co), var = vec(p + ".bn.running_var", co);
    Wp->assign(static_cast<size_t>(co) * ci * k * k, 0.f);
    bp->assign(co, 0.f);
    for (int o = 0; o < co; ++o) {
      const float s = g[o] / std::sqrt(var[o] + 1e-5f);
      (*bp)[o] = b[o] - mu[o] * s;
      for (int i = 0; i < ci; ++i)
        for (int t = 0; t < k * k; ++t)      // [Co, Ci, kh, kw] -> [Co, (kh*k+kw)*Ci + ci]
          (*Wp)[(static_cast<size_t>(o) * k * k + t) * ci + i] = cw[(static_cast<size_t>(o) * ci + i) * k * k + t] * s;
    }
  };
  auto put_convx = [&](const std::string& key, const std::string& p, int co, int ci, int k) {
    std::vector<float> Wp, bp;
    fold_convx(p, co, ci, k, &Wp, &bp);
    put16(key + ".w", Wp);
    put32(key + ".b", bp);
  };
  auto put_linear = [&](const std::string& key, const std::string& p, int n_out, int n_in) {
    put16(key + ".w", vec(p + ".weight", 1LL * n_out * n_in));
    put32(key + ".b", vec(p + ".bias", n_out));
  };
  auto put_norm = [&](const std::string& key, const std::string& p, int n) {
    put32(key + ".w", vec(p + ".weight", n));
    put32(key + ".b", vec(p + ".bias", n));
  };
  // ConvTranspose2d(k=2,s=2) weight [Ci, Co, 2, 2] -> GEMM weight [(dy*2+dx)*Co + co, Ci], bias x4
  auto put_convT = [&](const std::string& key, const std::string& p, int ci, int co) {
    auto cw = vec(p + ".weight", 1LL * ci * co * 4);
    auto cb = vec(p + ".bias", co);
    std::vector<float> Wp(static_cast<size_t>(4) * co * ci), bp(static_cast<size_t>(4) * co);
    for (int i = 0; i < ci; ++i)
      for (int o = 0; o < co; ++o)
        for (int q = 0; q < 4; ++q) Wp[(static_cast<size_t>(q) * co + o) * ci + i] = cw[(static_cast<size_t>(i) * co + o) * 4 + q];
    for (int q = 0; q < 4; ++q)
      for (int o = 0; o < co; ++o) bp[q * co + o] = cb[o];
    put16(key + ".w", Wp);
    put32(key + ".b", bp);
  };

  // ---- ViT
  const std::string E = "backbone.0.encoder.";
  put16("patch.w", vec(E + "patch_embed.proj.weight", 1LL * C * 768));
  put32("patch.b", vec(E + "patch_embed.proj.bias", C));
  const std::vector<float> pos_embed = vec(E + "pos_embed", 197LL * C);
  put16("pos", window_major_pos(pos_embed.data(), C, G, G));   // the table at the configured resolution
  // The encoder's LayerNorms folded into the consuming GEMM (which then runs on the raw residual stream, see gemm_tc.h):
  //   W'[n,k] = W[n,k]*ln_w[k] ; bias'[n] = bias[n] + sum_k ln_b[k]*W[n,k] (double).  16-bit: W', bias' and colsum[n] =
  //   sum_k round16(W'[n,k]).  e4m3 (lwdetr_b200.h LWDETR_F16_E4M3): per output channel n, w_scale[n] = max_k |W'[n,k]| / 448
  //   and codes e4m3(W'[n,k] * 448 / max), then bias'
  auto put_folded = [&](const std::string& key, const std::vector<float>& Wm, const std::vector<float>& bias, const std::string& ln, int n_out) {
    auto lw = vec(ln + ".weight", C), lb = vec(ln + ".bias", C);
    std::vector<float> Wf(Wm.size()), bf(n_out), per_n(n_out);   // per output channel: w_scale (e4m3) or colsum (16-bit)
    for (int n = 0; n < n_out; ++n) {
      double acc_b = bias[n];
      for (int kk = 0; kk < C; ++kk) {
        const float wv = Wm[static_cast<size_t>(n) * C + kk];
        Wf[static_cast<size_t>(n) * C + kk] = wv * lw[kk];
        acc_b += static_cast<double>(lb[kk]) * wv;
      }
      bf[n] = static_cast<float>(acc_b);
    }
    if (e4m3_) {
      std::vector<uint8_t> q(Wf.size());
      host_quant_e4m3_rows(Wf.data(), n_out, C, q.data(), per_n.data());
      void* p = upload8(q);
      if (!p) oom = true;
      W_[key + ".w"] = p;
    } else {
      for (int n = 0; n < n_out; ++n) {
        double acc_c = 0.0;
        for (int kk = 0; kk < C; ++kk) acc_c += round16(Wf[static_cast<size_t>(n) * C + kk]);
        per_n[n] = static_cast<float>(acc_c);
      }
      put16(key + ".w", Wf);
    }
    put32(key + ".b", bf);
    put32(key + (e4m3_ ? ".s" : ".cs"), per_n);
  };
  for (int i = 0; i < cfg_.vit_depth; ++i) {
    const std::string b = E + "blocks." + std::to_string(i) + ".", k = "blk" + std::to_string(i) + ".";
    // the e4m3 mode packs qkv and fc1 only as e4m3 weights with the LayerNorm affine folded in
    if (!e4m3_) {
      put_norm(k + "ln1", b + "norm1", C);
      put16(k + "qkv.w", vec(b + "attn.qkv.weight", 3LL * C * C));
    }
    auto qb = vec(b + "attn.q_bias", C), vb = vec(b + "attn.v_bias", C);
    std::vector<float> qkv_b(static_cast<size_t>(3) * C, 0.f);     // [q_bias, 0, v_bias]  (vit.py:123-125)
    std::copy(qb.begin(), qb.end(), qkv_b.begin());
    std::copy(vb.begin(), vb.end(), qkv_b.begin() + 2 * C);
    if (!e4m3_) put32(k + "qkv.b", qkv_b);
    put_folded(k + (e4m3_ ? "qkv_q" : "qkv_ln"), vec(b + "attn.qkv.weight", 3LL * C * C), qkv_b, b + "norm1", 3 * C);
    put_folded(k + (e4m3_ ? "fc1_q" : "fc1_ln"), vec(b + "mlp.fc1.weight", 4LL * C * C), vec(b + "mlp.fc1.bias", 4LL * C), b + "norm2", 4 * C);
    put_linear(k + "proj", b + "attn.proj", C, C);
    put32(k + "g1", vec(b + "gamma_1", C));
    if (!e4m3_) {
      put_norm(k + "ln2", b + "norm2", C);
      put_linear(k + "fc1", b + "mlp.fc1", 4 * C, C);
    }
    put_linear(k + "fc2", b + "mlp.fc2", C, 4 * C);
    put32(k + "g2", vec(b + "gamma_2", C));
  }
  // ---- projector
  const std::string PR = "backbone.0.projector.";
  for (int l = 0; l < L; ++l) {
    const int sc = cfg_.level_scale_log2[l];
    const std::string k = "lvl" + std::to_string(l) + ".";
    int cs = C;   // channels each tap contributes
    for (int t = 0; t < ntap; ++t) {
      const std::string s = PR + "stages_sampling." + std::to_string(l) + "." + std::to_string(t) + ".";
      const std::string ks = k + "samp" + std::to_string(t);
      if (sc == 1) {
        if (C > 512) {
          put_convx(ks + ".pre", s + "0", C / 2, C, 1);
          put_convT(ks + ".up", s + "1", C / 2, C / 4);
          cs = C / 4;
        } else {
          put_convT(ks + ".up", s + "0", C, C / 2);
          cs = C / 2;
        }
      } else if (sc == -1) {
        put_convx(ks + ".down", s + "0", C, C, 3);
      }
    }
    const std::string st = PR + "stages." + std::to_string(l) + ".";
    put_convx(k + "cv1", st + "0.cv1", 2 * c2, cs * ntap, 1);
    put_convx(k + "cv2", st + "0.cv2", d, 5 * c2, 1);
    for (int j = 0; j < 3; ++j) {
      put_convx(k + "m" + std::to_string(j) + "a", st + "0.m." + std::to_string(j) + ".cv1", c2, c2, 3);
      put_convx(k + "m" + std::to_string(j) + "b", st + "0.m." + std::to_string(j) + ".cv2", c2, c2, 3);
    }
    put_norm(k + "ln", st + "1", d);
  }
  // ---- two-stage + decoder (group 0 only in eval: lwdetr.py:141-144, transformer.py:229)
  const std::string TR = "transformer.";
  put_linear("enc_out", TR + "enc_output.0", d, d);
  put_norm("enc_ln", TR + "enc_output_norm.0", d);
  put_linear("enc_cls", TR + "enc_out_class_embed.0", ncls, d);
  for (int i = 0; i < 3; ++i) put_linear("enc_box" + std::to_string(i), TR + "enc_out_bbox_embed.0.layers." + std::to_string(i), i == 2 ? 4 : d, d);
  {
    auto re = vec("refpoint_embed.weight", 1LL * nq * cfg_.group_detr * 4);
    put32("refpoint_embed", std::vector<float>(re.begin(), re.begin() + static_cast<size_t>(nq) * 4));
    auto qf = vec("query_feat.weight", 1LL * nq * cfg_.group_detr * d);
    put16("query_feat", std::vector<float>(qf.begin(), qf.begin() + static_cast<size_t>(nq) * d));
  }
  put_linear("rph0", TR + "decoder.ref_point_head.layers.0", d, 2 * d);
  put_linear("rph1", TR + "decoder.ref_point_head.layers.1", d, d);
  std::vector<float> wval, bval;
  const int MLP = M * L * P;
  for (int i = 0; i < cfg_.dec_layers; ++i) {
    const std::string p = TR + "decoder.layers." + std::to_string(i) + ".", k = "dec" + std::to_string(i) + ".";
    auto ipw = vec(p + "self_attn.in_proj_weight", 3LL * d * d), ipb = vec(p + "self_attn.in_proj_bias", 3LL * d);
    put16(k + "qk.w", std::vector<float>(ipw.begin(), ipw.begin() + static_cast<size_t>(2) * d * d));
    put32(k + "qk.b", std::vector<float>(ipb.begin(), ipb.begin() + 2 * d));
    put16(k + "v.w", std::vector<float>(ipw.begin() + static_cast<size_t>(2) * d * d, ipw.end()));
    put32(k + "v.b", std::vector<float>(ipb.begin() + 2 * d, ipb.end()));
    put_linear(k + "so", p + "self_attn.out_proj", d, d);
    put_norm(k + "n1", p + "norm1", d);
    {
      auto ow = vec(p + "cross_attn.sampling_offsets.weight", 2LL * MLP * d), ob = vec(p + "cross_attn.sampling_offsets.bias", 2LL * MLP);
      auto aw = vec(p + "cross_attn.attention_weights.weight", 1LL * MLP * d), ab = vec(p + "cross_attn.attention_weights.bias", MLP);
      ow.insert(ow.end(), aw.begin(), aw.end());
      ob.insert(ob.end(), ab.begin(), ab.end());
      put16(k + "oa.w", ow);
      put32(k + "oa.b", ob);
    }
    {
      auto vw = vec(p + "cross_attn.value_proj.weight", 1LL * d * d), vb = vec(p + "cross_attn.value_proj.bias", d);
      wval.insert(wval.end(), vw.begin(), vw.end());
      bval.insert(bval.end(), vb.begin(), vb.end());
    }
    put_linear(k + "co", p + "cross_attn.output_proj", d, d);
    put_norm(k + "n2", p + "norm2", d);
    put_linear(k + "l1", p + "linear1", ff, d);
    put_linear(k + "l2", p + "linear2", d, ff);
    put_norm(k + "n3", p + "norm3", d);
  }
  put16("value.w", wval);
  put32("value.b", bval);
  put_norm("dec_norm", TR + "decoder.norm", d);
  put_linear("cls", "class_embed", ncls, d);
  for (int i = 0; i < 3; ++i) put_linear("box" + std::to_string(i), "bbox_embed.layers." + std::to_string(i), i == 2 ? 4 : d, d);
  // the raw pos_embed (fp32, after every other entry): plan() derives the table of any other input size from the ARENA copy,
  // which lwdetr_broadcast_weights fills on every rank
  put32("pos_raw", pos_embed);
  if (missing) return -1;
  if (oom) { *err = "weight arena exhausted"; return -1; }
  if (cudaDeviceSynchronize() != cudaSuccess) { *err = "CUDA error while uploading weights"; return -1; }
  weights_loaded_ = true;
  return 0;
}

// ------------------------------------------------------------------------------- schedule
int Engine::plan(int B, int IH, int IW, std::string* err) {
  plan_.reset();   // its graphs point into the workspace arena, which pass 0 may reallocate; a failed plan leaves none
  const int C = cfg_.vit_dim, d = cfg_.hidden_dim, nq = cfg_.num_queries, ncls = cfg_.num_classes;
  const int GH = IH / 16, GW = IW / 16, T = GH * GW, ntap = cfg_.n_taps, c2 = d / 2, heads = cfg_.vit_heads;
  const int M = cfg_.ca_heads, L = cfg_.n_levels, P = cfg_.dec_points, ff = cfg_.dim_feedforward, NL = cfg_.dec_layers;
  const long long BT = 1LL * B * T;
  int lvl_h[2] = {0, 0}, lvl_w[2] = {0, 0}, lvl_start[2] = {0, 0}, S = 0;
  for (int l = 0; l < L; ++l) {   // P3 = 2x the token grid, P4 = the grid, P5 = half of it (projector.py:165-193)
    const int sc = cfg_.level_scale_log2[l];
    lvl_h[l] = sc == 1 ? 2 * GH : (sc == -1 ? GH / 2 : GH);
    lvl_w[l] = sc == 1 ? 2 * GW : (sc == -1 ? GW / 2 : GW);
    lvl_start[l] = S;
    S += lvl_h[l] * lvl_w[l];
  }
  const long long BS = 1LL * B * S, BQ = 1LL * B * nq;
  const int ldc = static_cast<int>(align_up(static_cast<size_t>(ncls), 32));   // row pitch of the fp32 class-logit buffers
  if (d / M != 16) { *err = "deformable attention head dim must be 16"; return -1; }
  if (C / heads != 16 && C / heads != 32 && C / heads != 64) { *err = "unsupported ViT head dim"; return -1; }
  if (S < nq) {
    *err = "lwdetr_forward: a " + std::to_string(IH) + "x" + std::to_string(IW) + " input has " + std::to_string(S) +
           " memory tokens, fewer than num_queries = " + std::to_string(nq);
    return -1;
  }
  // position table of this token grid: the packed table at the configured size, else resized from the arena's raw pos_embed
  const bool own_pos = !(GH == cfg_.img_size / 16 && GW == cfg_.img_size / 16);
  std::vector<uint16_t> pos_host;
  if (own_pos) {
    std::vector<float> pe(static_cast<size_t>(197) * C);
    const float* raw = F_.count("pos_raw") ? F_["pos_raw"] : nullptr;
    // the arena may just have been filled by a stream-ordered broadcast: the whole device is synchronised first
    if (!raw || cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(pe.data(), raw, pe.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess) {
      *err = "lwdetr_forward: reading pos_embed from the weight arena failed";
      return -1;
    }
    pos_host = to16(window_major_pos(pe.data(), C, GH, GW));
  }
  const std::string too_big = "lwdetr_forward: batch " + std::to_string(B) + " at " + std::to_string(IH) + "x" + std::to_string(IW) +
                              " needs a workspace buffer of more than 2^31-1 elements";
  auto p = std::make_unique<Plan>();
  // GEMM epilogues of the call sites below
  auto act = [](int a) { GemmDesc g; g.act = a; return g; };
  auto resid = [](Mat r) { GemmDesc g; g.resid = r.p; g.ld_resid = r.ld; return g; };
  GemmDesc f32; f32.out_fp32 = 1;
  auto col = [](Mat m, int c) { return Mat{cptr(m.p) + static_cast<size_t>(c) * 2, m.ld}; };
  const int dt = dtype_;

  for (int pass = 0; pass < 2; ++pass) {   // pass 0 sizes the workspace, pass 1 builds the ops
    OpBuilder b(pass, dtype_, sarena_.p, W_, F_, too_big, err, &p->ops);

    // ================================================================ padding-mask tables (constants when the batch is unpadded)
    float* prop_b = b.buf32(BS * 4);
    float* vr_b = b.buf32(static_cast<long long>(B) * L * 2 + 4);
    uint8_t* invalid_b = static_cast<uint8_t*>(b.alloc(static_cast<size_t>(BS)));
    uint8_t* pad_b = static_cast<uint8_t*>(b.alloc(static_cast<size_t>(BS)));
    uint8_t* fmask_b = static_cast<uint8_t*>(b.alloc(static_cast<size_t>(B) * IH * IW));   // padding mask of a batch of raw frames
    {
      const int lh0 = lvl_h[0], lh1 = lvl_h[1], lw0 = lvl_w[0], lw1 = lvl_w[1], ls0 = lvl_start[0], ls1 = lvl_start[1];
      b.op("mask_setup", [this, B, IH, IW, L, S, lh0, lh1, lw0, lw1, ls0, ls1, prop_b, invalid_b, pad_b, vr_b, fmask_b](cudaStream_t st) {
        const int lh[2] = {lh0, lh1}, lw[2] = {lw0, lw1}, ls[2] = {ls0, ls1};
        const uint8_t* mask = in_.mask;
        if (in_.kind == IN_FRAMES || in_.kind == IN_FRAMES_NV12) {   // raw frames: the mask follows from their dst sizes, made on the device
          mask = frames_padded_ ? fmask_b : nullptr;
          if (frames_padded_) {
            const int rc = in_.kind == IN_FRAMES ? frame_mask_launch(in_.frames, B, IH, IW, fmask_b, st)
                                                 : frame_mask_launch(in_.frames_nv12, B, IH, IW, fmask_b, st);
            if (rc) return rc;
          }
        }
        return mask_setup_launch(mask, B, IH, IW, L, S, lh, lw, ls, prop_b, invalid_b, pad_b, vr_b, st);
      }, {prop_b, BS, 4, 4, EL_F32}, 24.0 * BS, /*reads_input=*/true);
      b.also("invalid", {invalid_b, BS, 1, 1, EL_U8});
      b.also("pad", {pad_b, BS, 1, 1, EL_U8});
      b.also("valid_ratio", {vr_b, 1LL * B * L, 2, 2, EL_F32});
    }
    // ================================================================ ViT encoder
    Mat a0 = b.buf16(BT, 768);
    Mat xa = b.buf16(BT, C), xb = b.buf16(BT, C), xm = b.buf16(BT, C), lnb = b.buf16(BT, C);
    Mat tapbuf = b.buf16(BT, ntap * C);
    // the 192-wide encoder (tiny, small) runs each block's LN2 -> fc1 -> GELU -> fc2 as one kernel (mlp.cu): no hidden buffer.
    // Only when its 128-row tiles cover every SM: below that (batch 1 - 10 at 640x640) the two GEMMs, whose narrower n-tiles
    // spread the work over more SMs, are faster.  Both paths give the same bits.
    const bool fused_mlp = fuse_ln_ != 0 && !e4m3_ && C == MLP_C && (BT + 127) / 128 >= current_device_sms();
    Mat qkv = b.buf16(BT, 3 * C), att = b.buf16(BT, C), hid = fused_mlp ? Mat{nullptr, 4 * C} : b.buf16(BT, 4 * C);
    {
      void* a0p = a0.p;
      b.op("patch_gather", [this, a0p, B, IH, IW, dt](cudaStream_t st) {
             if (in_.kind == IN_FRAMES) return resize_patches_launch(dt, in_.frames, B, IH, IW, in_.mean, in_.stdv, a0p, st);
             if (in_.kind == IN_FRAMES_NV12) return resize_patches_launch(dt, in_.frames_nv12, B, IH, IW, in_.mean, in_.stdv, a0p, st);
             if (in_.kind == IN_U8_NHWC) return patch_gather_u8_launch(dt, in_.images, in_.mean, in_.stdv, a0p, B, IH, IW, st);
             return patch_gather_launch(dt, in_.images, in_.kind == IN_F32_NCHW ? 1 : 0, a0p, B, IH, IW, st);
           },
           {a0.p, BT, 768, 768, 0}, 1.0 * B * 3 * IH * IW * 4 + 2.0 * BT * 768, /*reads_input=*/true);
    }
    float2* stats_x = static_cast<float2*>(b.alloc(static_cast<size_t>(BT) * 48 * sizeof(float2)));   // row stats of x (block input)
    float2* stats_m = static_cast<float2*>(b.alloc(static_cast<size_t>(BT) * 48 * sizeof(float2)));   // row stats of x + attn
    const bool fuse = fuse_ln_ != 0 && !e4m3_;   // the e4m3 mode has its own LayerNorm -> e4m3 pass in front of qkv / fc1
    // e4m3 mode: the LayerNorm output as e4m3 codes + per-row scales, shared by qkv and fc1
    uint8_t* lnq = e4m3_ ? static_cast<uint8_t*>(b.alloc(static_cast<size_t>(BT) * C)) : nullptr;
    float* lns = e4m3_ ? b.buf32(BT) : nullptr;
    auto ln_e4m3 = [&](const std::string& label, Mat x) {   // a capture returns the row scales
      const void* xp = x.p; const int ldx = x.ld;
      b.op(label, [xp, ldx, BT, C, lnq, lns](cudaStream_t st) { return layernorm_e4m3_launch(xp, ldx, BT, C, 1e-6f, lnq, C, lns, st); },
           {lns, BT, 1, 1, 1}, 2.0 * BT * C + 1.0 * BT * C + 4.0 * BT);
    };
    // LayerNorm consumers: the GEMM normalises its raw input rows with the statistics the producers wrote
    auto ln_fold = [&](const float2* stats, int a) { GemmDesc g = act(a); g.stats_in = stats; g.ln_C = C; g.ln_eps = 1e-6f; return g; };
    Mat xcur = xa;
    void* pos_tab = own_pos ? b.alloc(pos_host.size() * 2) : nullptr;
    if (own_pos && pass == 1 && cudaMemcpy(pos_tab, pos_host.data(), pos_host.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess) {
      *err = "lwdetr_forward: position table upload failed";
      return -1;
    }
    {
      GemmDesc g = resid(Mat{own_pos ? pos_tab : b.w16("pos"), C}); g.resid_mod = T; if (fuse) g.stats_out = stats_x;
      b.gemm("patch_embed", g, a0, BT, 768, "patch", C, xcur);
    }
    int tap_slot = 0;
    for (int i = 0; i < cfg_.vit_depth; ++i) {
      const std::string k = "blk" + std::to_string(i) + ".", lb = "block" + std::to_string(i);
      const bool window = (cfg_.window_block_mask >> i) & 1;
      if (e4m3_) {
        ln_e4m3(lb + ".ln1", xcur);
        b.gemm_e4m3(lb + ".qkv", lnq, lns, BT, C, k + "qkv_q", 3 * C, ACT_NONE, qkv);
      } else if (fuse) {
        b.gemm(lb + ".qkv", ln_fold(stats_x, ACT_NONE), xcur, BT, C, k + "qkv_ln", 3 * C, qkv);
      } else {
        b.layernorm(lb + ".ln1", xcur, lnb, k + "ln1", 1e-6f, BT, C);
        b.gemm(lb + ".qkv", GemmDesc{}, lnb, BT, C, k + "qkv", 3 * C, qkv);
      }
      b.attention(lb + (window ? ".win_attn" : ".glb_attn"), col(qkv, 0), col(qkv, C), col(qkv, 2 * C), att,
                  window ? 16 * B : B, window ? T / 16 : T, heads, C / heads);
      { GemmDesc g = resid(xcur); g.gamma = b.w32(k + "g1"); if (fuse) g.stats_out = stats_m;
        b.gemm(lb + ".proj", g, att, BT, C, k + "proj", C, xm); }
      if (fused_mlp) {
        // fc1 + fc2 in one op under the fc2 label (block taps and captures stay where they were)
      } else if (e4m3_) {
        ln_e4m3(lb + ".ln2", xm);
        b.gemm_e4m3(lb + ".fc1", lnq, lns, BT, C, k + "fc1_q", 4 * C, ACT_GELU, hid);
      } else if (fuse) {
        b.gemm(lb + ".fc1", ln_fold(stats_m, ACT_GELU), xm, BT, C, k + "fc1_ln", 4 * C, hid);
      } else {
        b.layernorm(lb + ".ln2", xm, lnb, k + "ln2", 1e-6f, BT, C);
        b.gemm(lb + ".fc1", act(ACT_GELU), lnb, BT, C, k + "fc1", 4 * C, hid);
      }
      Mat xnext;
      bool is_tap = false;
      for (int t = 0; t < ntap; ++t) is_tap = is_tap || cfg_.taps[t] == i;
      if (is_tap) xnext = col(tapbuf, (tap_slot++) * C);
      else xnext = (xcur.p == xa.p) ? xb : xa;
      if (fused_mlp) {
        b.mlp(lb, xm, BT, stats_m, k, i + 1 < cfg_.vit_depth ? stats_x : nullptr, xnext);
      } else {
        GemmDesc g = resid(xm); g.gamma = b.w32(k + "g2"); if (fuse && i + 1 < cfg_.vit_depth) g.stats_out = stats_x;
        b.gemm(lb, g, hid, BT, 4 * C, k + "fc2", C, xnext);
      }
      xcur = xnext;
    }

    // ================================================================ projector -> decoder memory [B, S, d]
    Mat memory = b.buf16(BS, d);
    for (int l = 0; l < L; ++l) {
      const int sc = cfg_.level_scale_log2[l], H = lvl_h[l], W = lvl_w[l];
      const long long rows = 1LL * B * H * W;
      const std::string k = "lvl" + std::to_string(l) + ".", lb = "level" + std::to_string(l);
      auto conv3 = [&](int a_mode, int a) { GemmDesc g = act(a); g.a_mode = a_mode; g.B = B; g.OH = H; g.OW = W; return g; };
      Mat c2f = b.buf16(rows, 5 * c2), tmp = b.buf16(rows, c2), pout = b.buf16(rows, d);
      if (sc == 0) {
        GemmDesc g = act(ACT_SILU); g.rows_in = ROWS_WINDOW_MAJOR; g.remap_rows = 1; g.IH = GH; g.IW = GW;
        b.gemm(lb + ".cv1", g, tapbuf, BT, ntap * C, k + "cv1", 2 * c2, c2f);
      } else if (sc == 1) {
        const int cs = C > 512 ? C / 4 : C / 2;
        Mat samp = b.buf16(rows, ntap * cs);
        Mat pre = C > 512 ? b.buf16(BT, C / 2) : Mat{nullptr, 0};
        for (int t = 0; t < ntap; ++t) {
          const std::string ks = k + "samp" + std::to_string(t);
          Mat src = col(tapbuf, t * C);
          int kin = C;
          if (C > 512) {
            b.gemm(lb + ".pre" + std::to_string(t), act(ACT_RELU), src, BT, C, ks + ".pre", C / 2, pre);
            src = pre; kin = C / 2;
          }
          GemmDesc g; g.rows_in = ROWS_WINDOW_MAJOR; g.shuffle_cout = cs; g.IH = GH; g.IW = GW;
          b.gemm(lb + ".up" + std::to_string(t), g, src, BT, kin, ks + ".up", 4 * cs, col(samp, t * cs));
        }
        b.gemm(lb + ".cv1", act(ACT_SILU), samp, rows, ntap * cs, k + "cv1", 2 * c2, c2f);
      } else {
        Mat spat = b.buf16(BT, ntap * C), samp = b.buf16(rows, ntap * C);
        {
          void* sp = tapbuf.p; void* dp = spat.p; const int ldx = ntap * C;
          b.op(lb + ".unwindow", [sp, dp, ldx, BT, GH, GW, dt](cudaStream_t st) { return unwindow_launch(dt, sp, ldx, dp, ldx, BT, ldx, GH, GW, st); },
               {spat.p, BT, ldx, ldx, 0}, 4.0 * BT * ldx);
        }
        for (int t = 0; t < ntap; ++t)
          b.gemm(lb + ".down" + std::to_string(t), conv3(AMODE_CONV3_S2, ACT_RELU), col(spat, t * C), rows, 9 * C,
                 k + "samp" + std::to_string(t) + ".down", C, col(samp, t * C));
        b.gemm(lb + ".cv1", act(ACT_SILU), samp, rows, ntap * C, k + "cv1", 2 * c2, c2f);
      }
      for (int j = 0; j < 3; ++j) {
        const std::string m = "m" + std::to_string(j);
        b.gemm(lb + "." + m + "a", conv3(AMODE_CONV3_S1, ACT_SILU), col(c2f, (1 + j) * c2), rows, 9 * c2, k + m + "a", c2, tmp);
        b.gemm(lb + "." + m + "b", conv3(AMODE_CONV3_S1, ACT_SILU), tmp, rows, 9 * c2, k + m + "b", c2, col(c2f, (2 + j) * c2));
      }
      b.gemm(lb + ".cv2", act(ACT_SILU), c2f, rows, 5 * c2, k + "cv2", d, pout);
      LayerNormArgs a{}; a.y_group = 1LL * H * W; a.y_group_stride = S; a.y_row_off = lvl_start[l];   // rows of the memory of each image
      b.layernorm(lb, pout, memory, k + "ln", 1e-6f, rows, d, a);
    }

    // ================================================================ two-stage query selection
    // value_proj of all decoder layers, HEAD-MAJOR [B][layer][head][S][16] (msda.cu stages whole (image, head) slabs)
    Mat value = b.buf16(BS, NL * d), om = b.buf16(BS, d), omn = b.buf16(BS, d);
    float* cls_all = b.buf32(BS * ldc);
    float* score = b.buf32(BS);
    int* topk_idx = static_cast<int*>(b.alloc(static_cast<size_t>(BQ) * 4));
    Mat sel = b.buf16(BQ, d), h1 = b.buf16(BQ, d), h2 = b.buf16(BQ, d);
    float* delta_ts = b.buf32(BQ * 4);
    float* enc_logits = b.buf32(BQ * ncls);
    float* enc_boxes = b.buf32(BQ * 4);
    float* refpoint = b.buf32(BQ * 4);
    Mat sine = b.buf16(BQ, 2 * d), qpos = b.buf16(BQ, d);
    { GemmDesc g; g.hm_S = S; g.hm_heads = M; g.hm_slices = NL; g.row_zero = pad_b; b.gemm("value_proj", g, memory, BS, d, "value", NL * d, Mat{value.p, 16}); }
    b.gemm("enc_output", GemmDesc{}, memory, BS, d, "enc_out", d, om);
    { LayerNormArgs a{}; a.row_flag = invalid_b; a.flag_mod = static_cast<int>(BS); a.override_vec = b.w32("enc_out.b");
      b.layernorm("enc_output_norm", om, omn, "enc_ln", 1e-5f, BS, d, a); }
    b.gemm("enc_class", f32, omn, BS, d, "enc_cls", ncls, Mat{cls_all, ldc});
    b.op("enc_score", [cls_all, ncls, ldc, score, BS](cudaStream_t st) { return rowmax_launch(cls_all, ldc, ncls, score, BS, st); },
         {score, BS, 1, 1, 1}, 4.0 * BS * ncls);
    b.op("topk", [this, score, B, S, nq, topk_idx](cudaStream_t st) {
      if (in_topk_override_ != nullptr)
        return static_cast<int>(cudaMemcpyAsync(topk_idx, in_topk_override_, static_cast<size_t>(B) * nq * 4, cudaMemcpyDeviceToDevice, st));
      return topk_launch(score, B, S, nq, topk_idx, st);
    }, {topk_idx, BQ, 1, 1, EL_I32}, 4.0 * BS);
    {
      void* omp = omn.p; void* selp = sel.p;
      b.op("gather_topk", [omp, d, cls_all, ncls, ldc, topk_idx, B, S, nq, selp, enc_logits, dt](cudaStream_t st) {
        return gather_topk_launch(dt, omp, d, cls_all, ldc, ncls, topk_idx, B, S, nq, d, selp, enc_logits, st);
      }, {sel.p, BQ, d, d, EL_16}, 4.0 * BQ * d);
      b.also("enc_logits", {enc_logits, BQ, ncls, ncls, EL_F32});
    }
    b.gemm("enc_box0", act(ACT_RELU), sel, BQ, d, "enc_box0", d, h1);
    b.gemm("enc_box1", act(ACT_RELU), h1, BQ, d, "enc_box1", d, h2);
    b.gemm("enc_box2", f32, h2, BQ, d, "enc_box2", 4, Mat{delta_ts, 4});
    {
      const float* rpe = b.w32("refpoint_embed");
      void* sp = sine.p;
      b.op("query_init", [delta_ts, prop_b, topk_idx, rpe, B, nq, d, enc_boxes, refpoint, sp, dt, S, L, vr_b](cudaStream_t st) {
        return query_init_launch(dt, delta_ts, prop_b, topk_idx, rpe, B, nq, d, enc_boxes, refpoint, sp, S, L, vr_b, st);
      }, {refpoint, BQ, 4, 4, EL_F32}, 4.0 * BQ * d);
      b.also("box_ts", {enc_boxes, BQ, 4, 4, EL_F32});
      b.also("sine", {sine.p, BQ, 2 * d, 2 * d, EL_16});
    }
    b.gemm("ref_point_head0", act(ACT_RELU), sine, BQ, 2 * d, "rph0", d, h1);
    b.gemm("query_pos", GemmDesc{}, h1, BQ, d, "rph1", d, qpos);

    // ================================================================ decoder
    Mat tgt = b.buf16(BQ, d), tq = b.buf16(BQ, d), t1 = b.buf16(BQ, d), ta = b.buf16(BQ, d), tb = b.buf16(BQ, d);
    Mat qk = b.buf16(BQ, 2 * d), vb = b.buf16(BQ, d), sa = b.buf16(BQ, d), oa = b.buf16(BQ, 3 * M * L * P), ms = b.buf16(BQ, d), ffh = b.buf16(BQ, ff);
    Mat hs = b.buf16(NL * BQ, d);
    {
      void* qf = b.w16("query_feat"); void* tp = tgt.p; void* tqp = tq.p; void* qp = qpos.p;
      b.op("tgt_init", [qf, d, nq, tp, BQ, dt](cudaStream_t st) { return add_rows_launch(dt, qf, d, nq, nullptr, 0, tp, d, BQ, d, st); },
           {tgt.p, BQ, d, d, 0}, 4.0 * BQ * d);
      b.op("tgt_plus_pos", [qf, d, nq, qp, tqp, BQ, dt](cudaStream_t st) { return add_rows_launch(dt, qf, d, nq, qp, d, tqp, d, BQ, d, st); },
           {tq.p, BQ, d, d, 0}, 6.0 * BQ * d);
    }
    MsdaArgs mbase;
    std::memset(&mbase, 0, sizeof mbase);
    mbase.v_b_stride = 1LL * NL * M * S * MSDA_D; mbase.valid_ratio = vr_b; mbase.offs_logits = oa.p; mbase.ld_ol = oa.ld; mbase.ref = refpoint; mbase.out = ms.p; mbase.ld_out = ms.ld;
    mbase.batch = B; mbase.nq = nq; mbase.heads = M; mbase.levels = L; mbase.points = P; mbase.S = S;
    for (int l = 0; l < L; ++l) { mbase.lvl_h[l] = lvl_h[l]; mbase.lvl_w[l] = lvl_w[l]; mbase.lvl_start[l] = lvl_start[l]; }
    if (msda_plan(&mbase)) { *err = "deformable attention: invalid level table"; return -1; }   // nbands = 0: direct-gather kernel
    LayerNormArgs plus_pos{}; plus_pos.add_src = qpos.p; plus_pos.ld_add = qpos.ld; plus_pos.y2 = tq.p; plus_pos.ldy2 = tq.ld;   // tq = y + qpos
    Mat cur = tgt;
    for (int i = 0; i < NL; ++i) {
      const std::string k = "dec" + std::to_string(i) + ".", lb = "dec" + std::to_string(i);
      b.gemm(lb + ".qk", GemmDesc{}, tq, BQ, d, k + "qk", 2 * d, qk);
      b.gemm(lb + ".v", GemmDesc{}, cur, BQ, d, k + "v", d, vb);
      b.attention(lb + ".self_attn", col(qk, 0), col(qk, d), vb, sa, B, nq, cfg_.sa_heads, d / cfg_.sa_heads);
      b.gemm(lb + ".sa_out", resid(cur), sa, BQ, d, k + "so", d, t1);
      b.layernorm(lb + ".norm1", t1, ta, k + "n1", 1e-5f, BQ, d, plus_pos);
      b.gemm(lb + ".offs_attn", GemmDesc{}, tq, BQ, d, k + "oa", 3 * M * L * P, oa);
      {
        MsdaArgs ma = mbase;
        ma.value = cptr(value.p) + static_cast<size_t>(i) * M * S * MSDA_D * 2;
        b.op(lb + ".msda", [ma, dt](cudaStream_t st) { return msda_launch(dt, ma, st); }, {ms.p, BQ, d, d, 0},
             2.0 * std::min<double>(1.0 * BS * d, 1.0 * BQ * M * L * P * 4 * 16) + 2.0 * BQ * M * L * P * 3 + 2.0 * BQ * d);
      }
      b.gemm(lb + ".ca_out", resid(ta), ms, BQ, d, k + "co", d, t1);
      b.layernorm(lb + ".norm2", t1, tb, k + "n2", 1e-5f, BQ, d);
      b.gemm(lb + ".linear1", act(ACT_RELU), tb, BQ, d, k + "l1", ff, ffh);
      b.gemm(lb + ".linear2", resid(tb), ffh, BQ, ff, k + "l2", d, t1);
      // norm3 and the decoder's output norm of this layer's hidden state (transformer.py:279-285) in one launch
      LayerNormArgs a = plus_pos; a.y3 = cptr(hs.p) + static_cast<size_t>(i) * BQ * d * 2; a.ldy3 = d; a.eps3 = 1e-5f;
      b.layernorm(lb, t1, tgt, k + "n3", 1e-5f, BQ, d, a, "dec_norm");
      cur = tgt;
    }
    // ================================================================ heads
    float* logits = b.buf32(NL * BQ * ldc);
    float* delta = b.buf32(NL * BQ * 4);
    float* boxes = b.buf32(NL * BQ * 4);
    Mat bh1 = b.buf16(NL * BQ, d), bh2 = b.buf16(NL * BQ, d);
    b.gemm("class_embed", f32, hs, NL * BQ, d, "cls", ncls, Mat{logits, ldc});
    b.gemm("bbox0", act(ACT_RELU), hs, NL * BQ, d, "box0", d, bh1);
    b.gemm("bbox1", act(ACT_RELU), bh1, NL * BQ, d, "box1", d, bh2);
    b.gemm("bbox2", f32, bh2, NL * BQ, d, "box2", 4, Mat{delta, 4});
    b.op("final_boxes", [delta, refpoint, BQ, NL, boxes](cudaStream_t st) { return final_boxes_launch(delta, refpoint, BQ, NL, boxes, st); },
         {boxes, NL * BQ, 4, 4, 1}, 32.0 * NL * BQ);
    p->logits = logits; p->boxes = boxes; p->enc_logits = enc_logits; p->enc_boxes = enc_boxes; p->topk_idx = topk_idx;
    p->hidden = hs.p;

    if (b.failed()) return -1;
    if (pass == 0) {
      const size_t need = b.bytes() + 4096;
      if (need > sarena_.bytes) {
        if (sarena_.p) cudaFree(sarena_.p);
        sarena_.p = nullptr;
        if (cudaMalloc(&sarena_.p, need) != cudaSuccess) { *err = "cudaMalloc(workspace, " + std::to_string(need >> 20) + " MiB) failed"; sarena_.bytes = 0; return -1; }
        sarena_.bytes = need;
      }
    }
  }
  p->B = B; p->H = IH; p->W = IW; p->ldc = ldc;
  plan_ = std::move(p);
  return 0;
}

int Engine::copy_view(const OutView& v, Capture* c) {
  const long long n = v.rows * v.cols;
  if (n > c->capacity) { c->written = -2; return 0; }
  const size_t esz = v.kind == EL_U8 ? 1 : (v.kind == EL_16 ? 2 : 4);
  std::vector<uint8_t> raw(static_cast<size_t>(n) * esz);
  if (cudaMemcpy2D(raw.data(), v.cols * esz, v.p, static_cast<size_t>(v.ld) * esz, v.cols * esz, static_cast<size_t>(v.rows), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  float* dst = c->dst;
  if (v.kind == EL_F32) std::memcpy(dst, raw.data(), raw.size());
  else if (v.kind == EL_I32) for (long long i = 0; i < n; ++i) { int32_t x; std::memcpy(&x, &raw[i * 4], 4); dst[i] = static_cast<float>(x); }
  else if (v.kind == EL_U8) for (long long i = 0; i < n; ++i) dst[i] = static_cast<float>(raw[i]);
  else if (dtype_ == DT_BF16) for (long long i = 0; i < n; ++i) { __nv_bfloat16 x; std::memcpy(&x, &raw[i * 2], 2); dst[i] = __bfloat162float(x); }
  else for (long long i = 0; i < n; ++i) { __half x; std::memcpy(&x, &raw[i * 2], 2); dst[i] = __half2float(x); }
  c->written = n;
  return 0;
}

int Engine::do_capture(const Op& op, cudaStream_t st) {
  bool synced = false;
  for (auto& c : captures_) {
    const OutView* v = c.label == op.label ? &op.out : nullptr;
    for (const auto& e : op.extra)
      if (!v && c.label == op.label + "." + e.first) v = &e.second;
    if (!v || v->p == nullptr) continue;
    if (!synced && cudaStreamSynchronize(st) != cudaSuccess) return -1;
    synced = true;
    if (copy_view(*v, &c)) return -1;
  }
  return 0;
}

int Engine::forward(const ForwardIn& in, int B, int H, int W, float* pred_logits, float* pred_boxes, const lwdetr_aux_out* aux,
                    const int32_t* topk_override, cudaStream_t st, std::string* err) {
  DeviceGuard guard(device_);
  if (!weights_loaded_) { *err = "lwdetr_forward: weights not loaded"; return -1; }
  if (B <= 0) { *err = "lwdetr_forward: batch must be positive"; return -1; }
  if (H % 64 || W % 64 || H < kMinSide || W < kMinSide || H > kMaxSide || W > kMaxSide) {
    *err = "lwdetr_forward: input " + std::to_string(H) + "x" + std::to_string(W) + " is not supported: height and width must be multiples of 64 in [" +
           std::to_string(kMinSide) + ", " + std::to_string(kMaxSide) + "] (4x4 windows of 16-pixel patches)";
    return -1;
  }
  if ((!plan_ || B != plan_->B || H != plan_->H || W != plan_->W) && plan(B, H, W, err)) return -1;
  Plan& p = *plan_;
  if (in.kind == IN_FRAMES ? !in.frames : in.kind == IN_FRAMES_NV12 ? !in.frames_nv12 : !in.images) { *err = "lwdetr_forward: null images"; return -1; }
  in_ = in; in_topk_override_ = topk_override;
  // the schedule (and profile_ops, later) reads the engine's copy: the caller's array is free on return.  Neither the source
  // format nor the descriptors are part of the plan or the graphs: the input ops run eagerly in front of them
  if (in.kind == IN_FRAMES) {
    frames_.assign(in.frames, in.frames + B);
    in_.frames = frames_.data();
    frames_padded_ = frames_padded(in.frames, B, H, W);
  } else if (in.kind == IN_FRAMES_NV12) {
    frames_nv12_.assign(in.frames_nv12, in.frames_nv12 + B);
    in_.frames_nv12 = frames_nv12_.data();
    frames_padded_ = frames_padded(in.frames_nv12, B, H, W);
  }
  // The first forward of a plan always runs eagerly (it also performs the one-time cudaFuncSetAttribute calls).
  const bool graph_ok = use_graph_ && captures_.empty() && p.eager_runs > 0;
  if (graph_ok) {
    if (!gstream_) {
      if (cudaStreamCreateWithFlags(&gstream_, cudaStreamNonBlocking) != cudaSuccess ||
          cudaEventCreateWithFlags(&ev_in_, cudaEventDisableTiming) != cudaSuccess ||
          cudaEventCreateWithFlags(&ev_out_, cudaEventDisableTiming) != cudaSuccess) { *err = "graph stream setup failed"; return -1; }
    }
    auto it = p.graphs.find(topk_override);
    if (it == p.graphs.end()) {
      if (p.graphs.size() >= 8) p.clear_graphs();
      cudaGraph_t g = nullptr;
      if (cudaStreamBeginCapture(gstream_, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { *err = std::string("graph capture begin failed: ") + cudaGetErrorString(cudaGetLastError()); return -1; }
      int rc = 0;
      for (auto& op : p.ops) { if (op.reads_input) continue; rc = op.run(gstream_); if (rc) break; }
      cudaError_t ce = cudaStreamEndCapture(gstream_, &g);
      if (rc || ce != cudaSuccess) { if (g) cudaGraphDestroy(g); *err = "graph capture failed"; return -1; }
      cudaGraphExec_t ex = nullptr;
      if (cudaGraphInstantiate(&ex, g, 0) != cudaSuccess) { cudaGraphDestroy(g); *err = "graph instantiate failed"; return -1; }
      cudaGraphDestroy(g);
      it = p.graphs.emplace(topk_override, ex).first;
    }
    // the input-reading ops on the caller's stream, then the graph ordered after them, then the caller's stream after the graph
    for (auto& op : p.ops) {
      if (!op.reads_input) continue;
      const int rc = op.run(st);
      if (rc) { *err = "op " + op.label + " failed to launch"; return -1; }
    }
    if (cudaEventRecord(ev_in_, st) != cudaSuccess || cudaStreamWaitEvent(gstream_, ev_in_, 0) != cudaSuccess ||
        cudaGraphLaunch(it->second, gstream_) != cudaSuccess || cudaEventRecord(ev_out_, gstream_) != cudaSuccess ||
        cudaStreamWaitEvent(st, ev_out_, 0) != cudaSuccess) { *err = std::string("graph launch failed: ") + cudaGetErrorString(cudaGetLastError()); return -1; }
  } else {
    for (auto& op : p.ops) {
      const int rc = op.run(st);
      if (rc) { *err = "op " + op.label + " failed to launch: " + (rc > 0 ? cudaGetErrorString(static_cast<cudaError_t>(rc)) : "bad arguments"); return -1; }
      if (!captures_.empty() && do_capture(op, st)) { *err = "capture after " + op.label + " failed: " + cudaGetErrorString(cudaGetLastError()); return -1; }
    }
    ++p.eager_runs;
  }
  // results -> caller buffers (dense)
  const int nq = cfg_.num_queries, ncls = cfg_.num_classes, NL = cfg_.dec_layers;
  const long long BQ = 1LL * B * nq;
  auto copy_logits = [&](float* dst, int layer) {
    return cudaMemcpy2DAsync(dst, ncls * 4, p.logits + static_cast<size_t>(layer) * BQ * p.ldc, static_cast<size_t>(p.ldc) * 4, ncls * 4, static_cast<size_t>(BQ), cudaMemcpyDeviceToDevice, st);
  };
  cudaError_t e = cudaSuccess;
  if (pred_logits) e = copy_logits(pred_logits, NL - 1);
  if (e == cudaSuccess && pred_boxes) e = cudaMemcpyAsync(pred_boxes, p.boxes + static_cast<size_t>(NL - 1) * BQ * 4, BQ * 16, cudaMemcpyDeviceToDevice, st);
  if (aux) {
    for (int l = 0; l + 1 < NL && e == cudaSuccess; ++l) {
      if (aux->aux_logits) e = copy_logits(aux->aux_logits + static_cast<size_t>(l) * BQ * ncls, l);
      if (e == cudaSuccess && aux->aux_boxes) e = cudaMemcpyAsync(aux->aux_boxes + static_cast<size_t>(l) * BQ * 4, p.boxes + static_cast<size_t>(l) * BQ * 4, BQ * 16, cudaMemcpyDeviceToDevice, st);
    }
    if (e == cudaSuccess && aux->enc_logits) e = cudaMemcpyAsync(aux->enc_logits, p.enc_logits, BQ * ncls * 4, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && aux->enc_boxes) e = cudaMemcpyAsync(aux->enc_boxes, p.enc_boxes, BQ * 16, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && aux->topk_index) e = cudaMemcpyAsync(aux->topk_index, p.topk_idx, BQ * 4, cudaMemcpyDeviceToDevice, st);
  }
  if (e != cudaSuccess) { *err = std::string("result copy failed: ") + cudaGetErrorString(e); return -1; }
  return 0;
}

int Engine::last_hidden(void* dst, int ld, cudaStream_t st, std::string* err) {
  DeviceGuard guard(device_);
  if (!plan_ || plan_->eager_runs == 0) { *err = "lwdetr_last_hidden: run a forward first"; return -1; }
  const int d = cfg_.hidden_dim;
  if (ld < d) { *err = "lwdetr_last_hidden: ld_dst is smaller than hidden_dim"; return -1; }
  const size_t BQ = static_cast<size_t>(plan_->B) * cfg_.num_queries;
  const char* src = static_cast<const char*>(plan_->hidden) + (cfg_.dec_layers - 1) * BQ * d * 2;
  const cudaError_t e = cudaMemcpy2DAsync(dst, static_cast<size_t>(ld) * 2, src, static_cast<size_t>(d) * 2, static_cast<size_t>(d) * 2, BQ,
                                          cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) { *err = std::string("lwdetr_last_hidden: ") + cudaGetErrorString(e); return -1; }
  return 0;
}

int Engine::profile_ops(int iters, std::vector<float>* ms, cudaStream_t st, std::string* err) {
  DeviceGuard guard(device_);
  if (!plan_) { *err = "profile_ops: run a forward first"; return -1; }
  const std::vector<Op>& ops = plan_->ops;
  ms->assign(ops.size(), 0.f);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (size_t i = 0; i < ops.size(); ++i) {
    ops[i].run(st);   // warm
    cudaEventRecord(e0, st);
    for (int k = 0; k < iters; ++k) ops[i].run(st);
    cudaEventRecord(e1, st);
    if (cudaEventSynchronize(e1) != cudaSuccess) { *err = "profile_ops: op " + ops[i].label + " failed"; return -1; }
    float t = 0.f;
    cudaEventElapsedTime(&t, e0, e1);
    (*ms)[i] = t / iters;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return 0;
}

}  // namespace lwb
