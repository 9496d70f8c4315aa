// C-ABI surface (include/lwdetr_b200.h): argument checking, error strings, dispatch to the kernels.
#include "lwdetr_b200.h"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdint.h>

#include <string>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <new>
#include <type_traits>
#include <vector>

#include "annotate.h"
#include "attn.h"
#include "crops.h"
#include "engine.h"
#include "flow.h"
#include "gemm_tc.h"
#include "gmc.h"
#include "msda.h"
#include "resize.h"
#include "rowops.h"
#include "speed.h"
#include "tiles.h"
#include "track.h"
#include "zones.h"


namespace {
thread_local std::string g_err;
int fail(const std::string& m) {
  g_err = m;
  return -1;
}
int cuda_fail(int e, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorString(static_cast<cudaError_t>(e));
  return -1;
}
// the GEMM both lwdetr_gemm and lwdetr_gemm_ex describe
lwb::GemmDesc gemm_desc(const lwdetr_gemm_args& a) {
  lwb::GemmDesc d;
  d.dtype = a.dtype; d.A = a.A; d.lda = a.lda; d.M = a.M; d.N = a.N; d.K = a.K; d.W = a.W; d.bias = a.bias; d.gamma = a.gamma;
  d.resid = a.resid; d.ld_resid = a.ld_resid; d.resid_mod = a.resid_mod; d.act = a.act; d.out = a.out; d.ld_out = a.ld_out;
  d.out_fp32 = a.out_fp32; d.rows_in = a.rows_in; d.remap_rows = a.remap_rows; d.shuffle_cout = a.shuffle_cout;
  d.IH = a.IH; d.IW = a.IW;
  d.stats_in = reinterpret_cast<const float2*>(a.stats_in); d.stats_parts_in = a.stats_parts_in; d.colsum = a.colsum;
  d.ln_C = a.ln_C; d.ln_eps = a.ln_eps; d.stats_out = reinterpret_cast<float2*>(a.stats_out);
  d.hm_S = a.hm_S; d.hm_heads = a.hm_heads; d.hm_slices = a.hm_slices; d.row_zero = a.row_zero;
  return d;
}
// lwdetr_attention and lwdetr_attention_ex: check and plan (no CUDA call), report the plan, launch unless a dry run
int attention_call(lwdetr_attention_args* p, void* stream, const char* fn) {
  const std::string name(fn);
  if (!p->q || !p->k || !p->v || !p->out) return fail(name + ": null pointer");
  lwb::AttnArgs a{};
  a.q = p->q; a.k = p->k; a.v = p->v; a.ldq = p->ldq; a.ldk = p->ldk; a.ldv = p->ldv; a.o = p->out; a.ldo = p->ldo;
  a.seqlen = p->seqlen; a.nseq = p->nseq; a.heads = p->heads; a.scale_log2 = p->scale * 1.4426950408889634f;
  lwb::AttnPlan plan;
  std::string err;
  if (lwb::attention_plan(p->dtype, a, p->dh, &plan, &err)) return fail(name + ": " + err);
  p->kernel = plan.kernel;
  p->warps = plan.warps;
  p->poly_mask = static_cast<int32_t>(plan.poly_mask);
  if (p->dry_run) return 0;
  int e = lwb::attention_run(p->dtype, a, p->dh, plan, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, (name + " launch").c_str());
  return 0;
}

// HOST stream ids of one call of a tracker, an estimator or a zones object: distinct and in [0, num_streams); "" when they are
std::string check_ids(int num_streams, const int32_t* ids, int n) {
  std::vector<char> seen(static_cast<size_t>(num_streams), 0);
  for (int i = 0; i < n; ++i) {
    if (ids[i] < 0 || ids[i] >= num_streams)
      return "stream id " + std::to_string(ids[i]) + " outside [0, " + std::to_string(num_streams) + ")";
    if (seen[ids[i]]++) return "stream id " + std::to_string(ids[i]) + " appears twice in one call";
  }
  return "";
}

// Buffers one after another at 256-byte aligned offsets, cudaMalloc's alignment, on which the kernels' float4, double and
// 16-byte pyramid accesses rely.  With a null base it only counts the bytes, so one layout function both sizes and assigns.
struct Carver {
  char* base = nullptr;
  size_t bytes = 0;
  template <class T> void take(T*& p, size_t n) {
    bytes = (bytes + 255) / 256 * 256;
    p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += n * sizeof(T);
  }
};

// The device side of a tracker, an estimator or a zones object: its buffers in one allocation, an event marking its last launch, and a
// non-blocking stream for its set-up and its reads, so that a read waits for the object's own work and nothing else.
struct DeviceState {
  int device = 0;
  void* arena = nullptr;
  cudaEvent_t done = nullptr;   // recorded after every launch on the state (an external event node inside a CUDA graph capture)
  cudaStream_t copy = nullptr;

  DeviceState() = default;
  DeviceState(const DeviceState&) = delete;
  DeviceState& operator=(const DeviceState&) = delete;

  // On the current device: lays the buffers out with layout(Carver&), allocates them in one piece, assigns them, then runs
  // init() (the set-up copies, enqueued on `copy`) and waits for it.  0, or -1 with the error set.
  template <class Layout, class Init> int create(const char* fn, Layout layout, Init init) {
    if (cudaGetDevice(&device) != cudaSuccess) return fail(std::string(fn) + ": no CUDA device (there is no CPU fallback)");
    Carver size;
    layout(size);
    cudaError_t e = cudaEventCreateWithFlags(&done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc(&arena, size.bytes);
    if (e == cudaSuccess) {
      Carver at{static_cast<char*>(arena)};
      layout(at);
      e = init();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(copy);
    return e == cudaSuccess ? 0 : cuda_fail(e, fn);
  }

  // marks the object's last launch on `stream`, so that read() waits for exactly that work.  Inside a stream capture the
  // record becomes an external event node, so every replay of the graph records it (the flag is accepted only while capturing)
  int mark(void* stream) const {
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaError_t e = cudaStreamIsCapturing(st, &cs)) return static_cast<int>(e);
    return static_cast<int>(cs == cudaStreamCaptureStatusActive ? cudaEventRecordWithFlags(done, st, cudaEventRecordExternal)
                                                                : cudaEventRecord(done, st));
  }

  // the call sequence of every launch on the object: run(stream) (0 or a CUDA error) on the object's device, then mark() on
  // this state and on `also` (a second object the launch wrote), in that order.  0, or -1 with "<fn> launch: <error>" set
  template <class Run> int launch(const std::string& fn, void* stream, Run run, const DeviceState* also = nullptr) const {
    lwb::DeviceGuard g(device);
    int e = run(static_cast<cudaStream_t>(stream));
    if (!e) e = mark(stream);
    if (!e && also) e = also->mark(stream);
    return e ? cuda_fail(e, (fn + " launch").c_str()) : 0;
  }

  struct Copy { void* dst; const void* src; size_t bytes; };
  // device-to-host copies once the last marked launch is done, all on `copy`, waited for once
  cudaError_t read(const std::vector<Copy>& parts) const {
    lwb::DeviceGuard g(device);
    cudaError_t e = cudaStreamWaitEvent(copy, done, 0);
    for (size_t i = 0; i < parts.size() && e == cudaSuccess; ++i)
      if (parts[i].bytes) e = cudaMemcpyAsync(parts[i].dst, parts[i].src, parts[i].bytes, cudaMemcpyDeviceToHost, copy);
    if (e == cudaSuccess) e = cudaStreamSynchronize(copy);
    return e;
  }

  // host-to-device copies once the last marked launch is done, all on `copy`, waited for once
  cudaError_t write(const std::vector<Copy>& parts) const {
    lwb::DeviceGuard g(device);
    cudaError_t e = cudaStreamWaitEvent(copy, done, 0);
    for (size_t i = 0; i < parts.size() && e == cudaSuccess; ++i)
      if (parts[i].bytes) e = cudaMemcpyAsync(parts[i].dst, parts[i].src, parts[i].bytes, cudaMemcpyHostToDevice, copy);
    if (e == cudaSuccess) e = cudaStreamSynchronize(copy);
    return e;
  }

  // the first step of an export: heads[stream_id] of a table of num_streams, once the last marked launch is done
  template <class Head> int read_head(const char* fn, const Head* heads, int num_streams, int stream_id, Head* h) const {
    if (stream_id < 0 || stream_id >= num_streams) return fail(std::string(fn) + ": stream id outside [0, num_streams)");
    if (cudaError_t e = read({{h, heads + stream_id, sizeof(Head)}})) return cuda_fail(e, fn);
    return 0;
  }

  ~DeviceState() {
    if (!done) return;          // create() failed before it made anything
    lwb::DeviceGuard g(device);
    if (copy) {
      cudaStreamSynchronize(copy);
      cudaStreamDestroy(copy);
    }
    cudaFree(arena);
    cudaEventDestroy(done);
  }
};

// lwdetr_tracker_reset, lwdetr_gmc_reset and lwdetr_zones_reset: the listed streams of obj start again through
// reset_launch(obj->table, streams, n, stream)
template <class T, class Launch> int reset_call(const char* name, T* obj, const int32_t* streams, int n, void* stream, Launch reset_launch) {
  const std::string fn(name);
  if (!obj || (n > 0 && !streams)) return fail(fn + ": null pointer");
  if (n < 0) return fail(fn + ": n must be >= 0");
  const std::string err = check_ids(obj->table.num_streams, streams, n);
  if (!err.empty()) return fail(fn + ": " + err);
  if (n == 0) return 0;
  return obj->state.launch(fn, stream, [&](cudaStream_t st) { return reset_launch(obj->table, streams, n, st); });
}

// lwdetr_layernorm and lwdetr_layernorm_ex, once each has checked its arguments: fill, launch, report the kernel instance
int layernorm_call(const char* name, int dtype, lwdetr_layernorm_args* p, void* stream) {
  const std::string fn(name);
  lwb::LayerNormArgs a{};
  a.x = p->x; a.ldx = p->ldx; a.y = p->y; a.ldy = p->ldy; a.w = p->w; a.b = p->b; a.eps = p->eps; a.rows = p->rows; a.C = p->C;
  a.row_flag = p->row_flag; a.flag_mod = p->row_flag ? p->flag_mod : 1; a.override_vec = p->override_vec;
  a.add_src = p->add_src; a.ld_add = p->ld_add; a.y2 = p->y2; a.ldy2 = p->ldy2;
  a.y_group = p->y_group; a.y_group_stride = p->y_group_stride; a.y_row_off = p->y_row_off;
  a.w3 = p->w3; a.b3 = p->b3; a.eps3 = p->eps3; a.y3 = p->y3; a.ldy3 = p->ldy3;
  int e = lwb::layernorm_launch(dtype, a, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail(fn + ": C must be a multiple of 8 and <= 1024");
  if (e) return cuda_fail(e, (fn + " launch").c_str());
  p->rows_per_warp = lwb::layernorm_rows_per_warp(p->rows, p->C);
  return 0;
}
}  // namespace

static_assert(LWDETR_ATTN_WG == lwb::ATTN_WG && LWDETR_ATTN_MMA == lwb::ATTN_MMA && LWDETR_ATTN_MMA_SHORT == lwb::ATTN_MMA_SHORT, "attention kernel codes");

extern "C" {

const char* lwdetr_last_error(void) { return g_err.c_str(); }
int lwdetr_abi_version(void) { return 1; }

int lwdetr_gemm(int dtype, const void* A, int lda, int M, int K, const void* W, int N, const float* bias,
                const float* gamma, const void* resid, int ld_resid, int resid_mod, int act, void* out, int ld_out,
                int out_fp32, int rows_in, int remap_rows, int shuffle_cout, int IH, int IW, void* stream) {
  if (!A || !W || !out) return fail("lwdetr_gemm: null pointer");
  const lwdetr_gemm_args a = {dtype, A, lda, M, K, W, N, bias, gamma, resid, ld_resid, resid_mod, act, out, ld_out, out_fp32,
                              rows_in, remap_rows, shuffle_cout, IH, IW};
  lwb::GemmOp op;
  std::string err;
  if (lwb::gemm_build(gemm_desc(a), &op, &err)) return fail("lwdetr_gemm: " + err);
  int e = lwb::gemm_launch(op, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_gemm launch");
  return 0;
}

static_assert(LWDETR_EP_GENERIC == lwb::EP_GENERIC && LWDETR_EP_BIAS == lwb::EP_BIAS && LWDETR_EP_BIAS_ACT == lwb::EP_BIAS_ACT &&
              LWDETR_EP_LN == lwb::EP_LN && LWDETR_EP_LN_GELU == lwb::EP_LN_GELU && LWDETR_EP_RESID == lwb::EP_RESID, "EP codes");

int lwdetr_gemm_ex(lwdetr_gemm_args* a, void* stream) {
  if (!a || !a->A || !a->W || !a->out) return fail("lwdetr_gemm_ex: null pointer");
  // 16-bit GEMMs only (the e4m3 GEMM has its own entry point and no epilogue variants), so `epilogue` is always an LWDETR_EP_*
  if (a->dtype != LWDETR_F16 && a->dtype != LWDETR_BF16) return fail("lwdetr_gemm_ex: dtype must be LWDETR_F16 or LWDETR_BF16");
  lwb::GemmOp op;
  std::string err;
  if (lwb::gemm_build(gemm_desc(*a), &op, &err)) return fail("lwdetr_gemm_ex: " + err);
  a->bn = op.bn;
  a->epilogue = lwb::gemm_epilogue(op);
  a->stats_parts_out = op.args.stats_parts_out;
  if (a->dry_run) return 0;
  int e = lwb::gemm_launch(op, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_gemm_ex launch");
  return 0;
}

int lwdetr_conv3x3(int dtype, const void* X, int ldx, int B, int OH, int OW, int stride, int Cin, const void* W,
                   int N, const float* bias, int act, void* out, int ld_out, void* stream) {
  if (!X || !W || !out) return fail("lwdetr_conv3x3: null pointer");
  if (stride != 1 && stride != 2) return fail("lwdetr_conv3x3: stride must be 1 or 2");
  lwb::GemmDesc d;
  d.dtype = dtype; d.a_mode = stride == 1 ? lwb::AMODE_CONV3_S1 : lwb::AMODE_CONV3_S2;
  d.A = X; d.lda = ldx; d.B = B; d.OH = OH; d.OW = OW; d.M = B * OH * OW; d.N = N; d.K = 9 * Cin; d.W = W;
  d.bias = bias; d.act = act; d.out = out; d.ld_out = ld_out;
  lwb::GemmOp op;
  std::string err;
  if (lwb::gemm_build(d, &op, &err)) return fail("lwdetr_conv3x3: " + err);
  int e = lwb::gemm_launch(op, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_conv3x3 launch");
  return 0;
}

int lwdetr_conv3x3_plan(int OH, int OW, int32_t* tw, int32_t* th) {
  if (!tw || !th) return fail("lwdetr_conv3x3_plan: null pointer");
  if (OH < 1 || OW < 1) return fail("lwdetr_conv3x3_plan: OH and OW must be positive");
  int w = 0, h = 0;
  lwb::conv_tile_plan(OH, OW, &w, &h);
  *tw = w; *th = h;
  return 0;
}


int lwdetr_layernorm(int dtype, const void* x, int ldx, void* y, int ldy, const float* w, const float* b, float eps,
                     int64_t rows, int C, void* stream) {
  if (!x || !y || !w || !b) return fail("lwdetr_layernorm: null pointer");
  lwdetr_layernorm_args a = {x, ldx, y, ldy, w, b, eps, rows, C};
  return layernorm_call("lwdetr_layernorm", dtype, &a, stream);
}

int lwdetr_layernorm_ex(int dtype, lwdetr_layernorm_args* p, void* stream) {
  if (!p || !p->x || !p->y || !p->w || !p->b) return fail("lwdetr_layernorm_ex: null pointer");
  if (p->row_flag && (!p->override_vec || p->flag_mod < 1)) return fail("lwdetr_layernorm_ex: row_flag needs override_vec and flag_mod >= 1");
  if (p->y2 && !p->add_src) return fail("lwdetr_layernorm_ex: y2 needs add_src");
  if (p->y3 && (!p->w3 || !p->b3)) return fail("lwdetr_layernorm_ex: y3 needs w3 and b3");
  if ((p->ldx | p->ldy | (p->y2 ? p->ld_add | p->ldy2 : 0) | (p->y3 ? p->ldy3 : 0)) % 8) return fail("lwdetr_layernorm_ex: leading dimensions must be multiples of 8");
  if (p->rows < 1) return fail("lwdetr_layernorm_ex: rows must be positive");
  return layernorm_call("lwdetr_layernorm_ex", dtype, p, stream);
}

int lwdetr_attention(int dtype, const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo,
                     int nseq, int seqlen, int heads, int dh, float scale, void* stream) {
  lwdetr_attention_args a = {dtype, q, ldq, k, ldk, v, ldv, out, ldo, nseq, seqlen, heads, dh, scale};
  return attention_call(&a, stream, "lwdetr_attention");
}

int lwdetr_attention_ex(lwdetr_attention_args* a, void* stream) {
  if (!a) return fail("lwdetr_attention_ex: null pointer");
  return attention_call(a, stream, "lwdetr_attention_ex");
}

int lwdetr_ms_deform_attn_forward(int etype, const void* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                  const void* sampling_loc, const void* attn_weight, void* out, int B, int S, int M, int D, int Lq, int L,
                                  int P, int im2col_step, void* stream) {
  if (!value || !spatial_shapes || !level_start_index || !sampling_loc || !attn_weight || !out) return fail("lwdetr_ms_deform_attn_forward: null pointer");
  if (etype != LWDETR_ET_F32 && etype != LWDETR_ET_F16 && etype != LWDETR_ET_BF16) return fail("lwdetr_ms_deform_attn_forward: etype must be LWDETR_ET_F32, _F16 or _BF16");
  if (B < 1 || S < 1 || M < 1 || D < 1 || Lq < 1 || L < 1 || P < 1) return fail("lwdetr_ms_deform_attn_forward: sizes must be positive");
  if (im2col_step < 1 || B % (B < im2col_step ? B : im2col_step) != 0)
    return fail("lwdetr_ms_deform_attn_forward: batch(" + std::to_string(B) + ") must divide im2col_step(" + std::to_string(im2col_step) + ")");   // ms_deform_attn_cuda.cu:50-52
  lwb::MsdaOpArgs a{};
  a.value = value; a.spatial_shapes = spatial_shapes; a.level_start_index = level_start_index; a.sampling_loc = sampling_loc;
  a.attn_weight = attn_weight; a.out = out; a.B = B; a.S = S; a.M = M; a.D = D; a.Lq = Lq; a.L = L; a.P = P;
  int e = lwb::msda_op_launch(etype, a, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail("lwdetr_ms_deform_attn_forward: unsupported element type / head dim");
  if (e) return cuda_fail(e, "lwdetr_ms_deform_attn_forward launch");
  return 0;
}

int lwdetr_ms_deform_attn_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index, const float* sampling_loc,
                                   const float* attn_weight, const float* grad_output, float* grad_value, float* grad_sampling_loc,
                                   float* grad_attn_weight, int B, int S, int M, int D, int Lq, int L, int P, int im2col_step, void* stream) {
  if (!value || !spatial_shapes || !level_start_index || !sampling_loc || !attn_weight || !grad_output || !grad_value || !grad_sampling_loc || !grad_attn_weight)
    return fail("lwdetr_ms_deform_attn_backward: null pointer");
  if (B < 1 || S < 1 || M < 1 || D < 1 || Lq < 1 || L < 1 || P < 1) return fail("lwdetr_ms_deform_attn_backward: sizes must be positive");
  if (im2col_step < 1 || B % (B < im2col_step ? B : im2col_step) != 0)
    return fail("lwdetr_ms_deform_attn_backward: batch(" + std::to_string(B) + ") must divide im2col_step(" + std::to_string(im2col_step) + ")");   // ms_deform_attn_cuda.cu:116-118
  lwb::MsdaOpArgs a{};
  a.value = value; a.spatial_shapes = spatial_shapes; a.level_start_index = level_start_index; a.sampling_loc = sampling_loc;
  a.attn_weight = attn_weight; a.out = nullptr; a.B = B; a.S = S; a.M = M; a.D = D; a.Lq = Lq; a.L = L; a.P = P;
  int e = lwb::msda_op_backward_launch(a, grad_output, grad_value, grad_sampling_loc, grad_attn_weight, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_ms_deform_attn_backward launch");
  return 0;
}


static const char kMsdaBadTable[] = ": invalid level table (a level is empty or extends past S)";
static_assert(LWDETR_MSDA_MAX_BANDS == lwb::MSDA_MAX_BANDS, "band table size");

int lwdetr_msda_plan(int L, const int32_t* spatial_shapes_host, const int32_t* level_start_host, int S, int32_t* nbands, int32_t* bands) {
  if (!spatial_shapes_host || !level_start_host || !nbands || !bands) return fail("lwdetr_msda_plan: null pointer");
  if (L < 1 || L > lwb::MSDA_MAX_LEVELS) return fail("lwdetr_msda_plan: 1..4 levels supported");
  lwb::MsdaArgs a{};
  a.levels = L; a.S = S;
  for (int l = 0; l < L; ++l) { a.lvl_h[l] = spatial_shapes_host[2 * l]; a.lvl_w[l] = spatial_shapes_host[2 * l + 1]; a.lvl_start[l] = level_start_host[l]; }
  if (lwb::msda_plan(&a)) return fail(std::string("lwdetr_msda_plan") + kMsdaBadTable);
  *nbands = a.nbands;
  for (int k = 0; k < a.nbands; ++k) {
    const lwb::MsdaBand& b = a.bands[k];
    const int32_t row[6] = {b.level, b.row0, b.own0, b.own1, b.tok0, b.bytes};
    for (int j = 0; j < 6; ++j) bands[6 * k + j] = row[j];
  }
  return 0;
}

int lwdetr_msda_forward(int dtype, const void* value_hm, int64_t v_image_stride, const void* offs_logits, int ld_ol, const float* ref,
                        const float* valid_ratio, void* out, int ld_out, int B, int S, int Lq, int M, int L, int P,
                        const int32_t* spatial_shapes_host, const int32_t* level_start_host, void* stream) {
  if (!value_hm || !offs_logits || !ref || !out || !spatial_shapes_host || !level_start_host) return fail("lwdetr_msda_forward: null pointer");
  if (L < 1 || L > lwb::MSDA_MAX_LEVELS) return fail("lwdetr_msda_forward: 1..4 levels supported");
  if ((ld_out % 8) || (ld_ol % 2) || (v_image_stride % 8) || (reinterpret_cast<uintptr_t>(value_hm) & 15)) return fail("lwdetr_msda_forward: misaligned leading dimension / base");
  if (v_image_stride < static_cast<int64_t>(M) * S * lwb::MSDA_D) return fail("lwdetr_msda_forward: v_image_stride smaller than one image's M*S*16 values");
  lwb::MsdaArgs a{};
  a.value = value_hm; a.v_b_stride = v_image_stride; a.offs_logits = offs_logits; a.ld_ol = ld_ol; a.ref = ref; a.valid_ratio = valid_ratio;
  a.out = out; a.ld_out = ld_out; a.batch = B; a.nq = Lq; a.heads = M; a.levels = L; a.points = P; a.S = S;
  for (int l = 0; l < L; ++l) { a.lvl_h[l] = spatial_shapes_host[2 * l]; a.lvl_w[l] = spatial_shapes_host[2 * l + 1]; a.lvl_start[l] = level_start_host[l]; }
  if (lwb::msda_plan(&a)) return fail(std::string("lwdetr_msda_forward") + kMsdaBadTable);
  int e = lwb::msda_launch(dtype, a, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail("lwdetr_msda_forward: unsupported (levels, points) combination");
  if (e) return cuda_fail(e, "lwdetr_msda_forward launch");
  return 0;
}

int lwdetr_topk(const float* score, int B, int S, int k, int32_t* idx, void* stream) {
  if (!score || !idx) return fail("lwdetr_topk: null pointer");
  int e = lwb::topk_launch(score, B, S, k, idx, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail("lwdetr_topk: need k <= S, and k <= 4096 when S > 16384");
  if (e) return cuda_fail(e, "lwdetr_topk launch");
  return 0;
}

int lwdetr_postprocess(const float* pred_logits, const float* pred_boxes, const float* target_sizes, int B, int nq, int num_classes,
                       int num_select, int32_t* work, float* scores, int32_t* labels, float* boxes, void* stream) {
  if (!pred_logits || !pred_boxes || !target_sizes || !work || !scores || !labels || !boxes) return fail("lwdetr_postprocess: null pointer");
  if (B < 1 || nq < 1 || num_classes < 1 || num_select < 1) return fail("lwdetr_postprocess: bad sizes");
  int e = lwb::postprocess_launch(pred_logits, pred_boxes, target_sizes, B, nq, num_classes, num_select, work, scores, labels, boxes,
                                  static_cast<cudaStream_t>(stream));
  if (e == -2) return fail("lwdetr_postprocess: need num_select <= slice length and slices * num_select <= 16384");
  if (e) return cuda_fail(e, "lwdetr_postprocess launch");
  return 0;
}

static_assert(sizeof(lwdetr_tile_view) == sizeof(lwb::TileViewHost) && LWDETR_TILE_IOU == lwb::TILE_IOU &&
              LWDETR_TILE_IOS == lwb::TILE_IOS, "tile view layout");

int lwdetr_tile_merge(const float* scores, const int32_t* labels, const float* boxes, int V, int k, const lwdetr_tile_view* views,
                      int num_frames, float score_threshold, float iou_threshold, int metric, int max_det, float* out_scores,
                      int32_t* out_labels, float* out_boxes, int32_t* counts, void* stream) {
  if (V < 1 || k < 1 || num_frames < 1) return fail("lwdetr_tile_merge: need V >= 1, k >= 1 and num_frames >= 1");
  if (max_det < 1 || max_det > lwb::TILE_MAX_DET) return fail("lwdetr_tile_merge: max_det must be in [1, 1024]");
  if (!scores || !labels || !boxes || !views || !out_scores || !out_labels || !out_boxes || !counts)
    return fail("lwdetr_tile_merge: null pointer");
  if (reinterpret_cast<uintptr_t>(boxes) % 16 || reinterpret_cast<uintptr_t>(out_boxes) % 16)
    return fail("lwdetr_tile_merge: boxes and out_boxes must be 16-byte aligned");
  if (metric != LWDETR_TILE_IOU && metric != LWDETR_TILE_IOS) return fail("lwdetr_tile_merge: metric must be LWDETR_TILE_IOU or LWDETR_TILE_IOS");
  if (!(iou_threshold >= 0.f && iou_threshold <= 1.f)) return fail("lwdetr_tile_merge: iou_threshold must be in [0, 1]");
  if (score_threshold != score_threshold) return fail("lwdetr_tile_merge: score_threshold is NaN");
  for (int v = 0; v < V; ++v) {
    if (views[v].frame < 0 || views[v].frame >= num_frames)
      return fail("lwdetr_tile_merge: view " + std::to_string(v) + " names frame " + std::to_string(views[v].frame) + " outside [0, " +
                  std::to_string(num_frames) + ")");
    if (v > 0 && views[v].frame < views[v - 1].frame)
      return fail("lwdetr_tile_merge: view frames must be non-decreasing (each frame's views contiguous); view " + std::to_string(v) +
                  " goes back to frame " + std::to_string(views[v].frame));
  }
  int e = lwb::tile_merge_launch(scores, labels, boxes, V, k, reinterpret_cast<const lwb::TileViewHost*>(views), num_frames, score_threshold,
                                 iou_threshold, metric, max_det, out_scores, out_labels, out_boxes, counts, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail("lwdetr_tile_merge: a frame has more than 16384 candidates (views * k) or more than 2048 views");
  if (e) return cuda_fail(e, "lwdetr_tile_merge launch");
  return 0;
}

static_assert(sizeof(lwdetr_track_record) == 192, "track record layout");

struct lwdetr_tracker {
  lwb::TrackTable table;
  lwb::ReidTable reid;   // embedding_dim 0 and null pointers without appearance
  lwdetr_track_params params;
  DeviceState state;
};

void lwdetr_track_params_default(lwdetr_track_params* p) {
  if (!p) return;
  p->track_thresh = 0.5f;
  p->low_thresh = 0.1f;
  p->new_track_thresh = static_cast<float>(0.5 + 0.1);
  p->match_thresh = 0.8f;
  p->second_thresh = 0.5f;
  p->unconfirmed_thresh = 0.7f;
  p->duplicate_thresh = 0.15f;
  p->track_buffer = 30;
  p->frame_rate = 30;
  p->fuse_score = 1;
  p->class_aware = 0;
  p->capacity = 512;
}

// lwdetr_tracker_create and, with reid (already checked), lwdetr_tracker_create_reid: the tracker's checks (their messages
// name lwdetr_tracker_create for both calls), then the table and any appearance state in one arena
static int tracker_create(const char* fn, int num_streams, const lwdetr_track_params& p, const lwdetr_reid_params* reid,
                          lwdetr_tracker** out) {
  if (num_streams < 1) return fail("lwdetr_tracker_create: num_streams must be >= 1");
  const float th[] = {p.track_thresh, p.low_thresh, p.new_track_thresh, p.duplicate_thresh};
  for (float v : th)
    if (!(v >= 0.f && v <= 1.f)) return fail("lwdetr_tracker_create: track_thresh, low_thresh, new_track_thresh and duplicate_thresh must be in [0, 1]");
  const float lim[] = {p.match_thresh, p.second_thresh, p.unconfirmed_thresh};
  for (float v : lim)
    if (!(v > 0.f && v <= 1.f)) return fail("lwdetr_tracker_create: match_thresh, second_thresh and unconfirmed_thresh must be in (0, 1]");
  if (p.capacity < 1 || p.capacity > lwb::TRACK_MAX) return fail("lwdetr_tracker_create: capacity must be in [1, 1024]");
  if (p.track_buffer < 0 || p.frame_rate < 1) return fail("lwdetr_tracker_create: need track_buffer >= 0 and frame_rate >= 1");
  if ((p.fuse_score != 0 && p.fuse_score != 1) || (p.class_aware != 0 && p.class_aware != 1))
    return fail("lwdetr_tracker_create: fuse_score and class_aware must be 0 or 1");
  std::unique_ptr<lwdetr_tracker> t(new (std::nothrow) lwdetr_tracker{});
  if (!t) return fail(std::string(fn) + ": out of memory");
  t->params = p;
  t->table.num_streams = num_streams;
  t->table.capacity = p.capacity;
  if (reid) t->reid.params = *reid;
  const size_t ns = static_cast<size_t>(num_streams), cap = static_cast<size_t>(p.capacity), pairs = ns * lwb::TRACK_PAIRS;
  const std::vector<lwb::TrackHead> h(ns, lwb::TrackHead{1, 1});     // every stream at frame 1, next id 1
  const auto layout = [&](Carver& c) {
    c.take(t->table.head, ns);
    c.take(t->table.rec, ns * 2 * cap);
    if (!reid) return;
    c.take(t->reid.slot, ns * 2 * cap);
    c.take(t->reid.has, ns * cap);
    c.take(t->reid.emb, ns * cap * reid->embedding_dim);
    c.take(t->reid.pkey, pairs);
    c.take(t->reid.pval, pairs);
  };
  const auto init = [&] {
    return cudaMemcpyAsync(t->table.head, h.data(), ns * sizeof(lwb::TrackHead), cudaMemcpyHostToDevice, t->state.copy);
  };
  if (int rc = t->state.create(fn, layout, init)) return rc;
  *out = t.release();
  return 0;
}

int lwdetr_tracker_create(int num_streams, const lwdetr_track_params* params, lwdetr_tracker** out) {
  if (!params || !out) return fail("lwdetr_tracker_create: null pointer");
  return tracker_create("lwdetr_tracker_create", num_streams, *params, nullptr, out);
}

void lwdetr_tracker_destroy(lwdetr_tracker* t) { delete t; }

int lwdetr_tracker_reset(lwdetr_tracker* t, const int32_t* streams, int n, void* stream) {
  return reset_call("lwdetr_tracker_reset", t, streams, n, stream, lwb::track_reset_launch);
}

static int track_common(const char* name, lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes,
                        const double* motion, int B, int k, const int32_t* stream_ids, int max_out, int32_t* out_ids, float* out_scores,
                        int32_t* out_labels, float* out_boxes, int32_t* out_index, int32_t* counts, void* stream,
                        const lwb::ReidInput* reid = nullptr) {
  const std::string fn(name);
  if (!t || !scores || !labels || !boxes || !stream_ids || !out_ids || !out_scores || !out_labels || !out_boxes || !out_index || !counts)
    return fail(fn + ": null pointer");
  if (B < 1 || k < 1 || k > lwb::TRACK_MAX || max_out < 1) return fail(fn + ": need B >= 1, k in [1, 1024] and max_out >= 1");
  if (reinterpret_cast<uintptr_t>(boxes) % 16 || reinterpret_cast<uintptr_t>(out_boxes) % 16)
    return fail(fn + ": boxes and out_boxes must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(motion) % 8) return fail(fn + ": motion must be 8-byte aligned");
  const std::string err = check_ids(t->table.num_streams, stream_ids, B);
  if (!err.empty()) return fail(fn + ": " + err);
  // a tracker with appearance always runs the appearance instantiation (without embeddings when none are given: ByteTrack's
  // bits), which keeps each record's embedding slot; the ByteTrack one would leave the slot array stale
  const lwb::ReidInput none{&t->reid, nullptr, LWDETR_ET_F32, 0};
  if (!reid && t->reid.emb) reid = &none;
  return t->state.launch(fn, stream, [&](cudaStream_t st) {
    return lwb::track_launch(t->table, t->params, scores, labels, boxes, motion, B, k, stream_ids, max_out, out_ids, out_scores, out_labels,
                             out_boxes, out_index, counts, st, reid);
  });
}

int lwdetr_track(lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes, int B, int k, const int32_t* stream_ids,
                 int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes, int32_t* out_index,
                 int32_t* counts, void* stream) {
  return track_common("lwdetr_track", t, scores, labels, boxes, nullptr, B, k, stream_ids, max_out, out_ids, out_scores, out_labels,
                      out_boxes, out_index, counts, stream);
}

int lwdetr_track_ex(lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes, const double* motion, int B, int k,
                    const int32_t* stream_ids, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes,
                    int32_t* out_index, int32_t* counts, void* stream) {
  return track_common("lwdetr_track_ex", t, scores, labels, boxes, motion, B, k, stream_ids, max_out, out_ids, out_scores, out_labels,
                      out_boxes, out_index, counts, stream);
}

void lwdetr_reid_params_default(lwdetr_reid_params* p) {
  if (!p) return;
  p->embedding_dim = 256;
  p->proximity_thresh = 0.5f;
  p->appearance_thresh = 0.25f;
  p->ema_alpha = 0.9f;
}

int lwdetr_tracker_create_reid(int num_streams, const lwdetr_track_params* params, const lwdetr_reid_params* reid, lwdetr_tracker** out) {
  if (!params || !reid || !out) return fail("lwdetr_tracker_create_reid: null pointer");
  const lwdetr_reid_params& r = *reid;
  if (r.embedding_dim < 1 || r.embedding_dim > 2048) return fail("lwdetr_tracker_create_reid: embedding_dim must be in [1, 2048]");
  if (!(r.proximity_thresh >= 0.f && r.proximity_thresh < 1.f)) return fail("lwdetr_tracker_create_reid: proximity_thresh must be in [0, 1)");
  if (!(r.appearance_thresh >= 0.f && r.appearance_thresh <= 1.f) || !(r.ema_alpha >= 0.f && r.ema_alpha <= 1.f))
    return fail("lwdetr_tracker_create_reid: appearance_thresh and ema_alpha must be in [0, 1]");
  return tracker_create("lwdetr_tracker_create_reid", num_streams, *params, reid, out);
}

int lwdetr_track_reid(lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes, const double* motion,
                      const void* embeddings, int emb_dtype, int ld_emb, int B, int k, const int32_t* stream_ids, int max_out,
                      int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes, int32_t* out_index, int32_t* counts,
                      void* stream) {
  if (t && t->reid.emb && embeddings) {
    if (emb_dtype != LWDETR_ET_F32 && emb_dtype != LWDETR_ET_F16 && emb_dtype != LWDETR_ET_BF16)
      return fail("lwdetr_track_reid: emb_dtype must be LWDETR_ET_F32, _F16 or _BF16");
    if (ld_emb < t->reid.params.embedding_dim) return fail("lwdetr_track_reid: ld_emb is smaller than embedding_dim");
    if (reinterpret_cast<uintptr_t>(embeddings) % (emb_dtype == LWDETR_ET_F32 ? 4 : 2))
      return fail("lwdetr_track_reid: embeddings must be aligned to their element size");
  }
  const lwb::ReidInput in{t ? &t->reid : nullptr, embeddings, emb_dtype, ld_emb};
  return track_common("lwdetr_track_reid", t, scores, labels, boxes, motion, B, k, stream_ids, max_out, out_ids, out_scores, out_labels,
                      out_boxes, out_index, counts, stream, t && t->reid.emb && embeddings ? &in : nullptr);
}

int lwdetr_tracker_export_embeddings(lwdetr_tracker* t, int stream_id, float* host, int cap, int32_t* count, int8_t* has) {
  if (!t || !count || (cap > 0 && (!host || !has))) return fail("lwdetr_tracker_export_embeddings: null pointer");
  if (!t->reid.emb) return fail("lwdetr_tracker_export_embeddings: the tracker was made without appearance (lwdetr_tracker_create_reid)");
  lwb::TrackHead h;
  if (int rc = t->state.read_head("lwdetr_tracker_export_embeddings", t->table.head, t->table.num_streams, stream_id, &h)) return rc;
  const int n = h.n_tracked + h.n_lost;
  const int m = n < cap ? n : (cap > 0 ? cap : 0);
  if (m > 0) {
    // the stream's whole embedding block in one copy, the rows gathered into record order here
    const size_t s0 = static_cast<size_t>(stream_id), C = static_cast<size_t>(t->table.capacity), D = t->reid.params.embedding_dim;
    std::vector<int16_t> slot(static_cast<size_t>(m));
    std::vector<uint8_t> full(C);
    std::vector<float> emb(C * D);
    const cudaError_t e = t->state.read({{slot.data(), t->reid.slot + (s0 * 2 + h.parity) * C, slot.size() * sizeof(int16_t)},
                                         {full.data(), t->reid.has + s0 * C, C},
                                         {emb.data(), t->reid.emb + s0 * C * D, emb.size() * sizeof(float)}});
    if (e != cudaSuccess) return cuda_fail(e, "lwdetr_tracker_export_embeddings");
    for (int i = 0; i < m; ++i) {
      has[i] = static_cast<int8_t>(full[slot[i]]);
      std::copy_n(emb.data() + slot[i] * D, D, host + i * D);
    }
  }
  *count = n;
  return 0;
}

int lwdetr_tracker_export(lwdetr_tracker* t, int stream_id, lwdetr_track_record* host, int cap, int32_t* count, int32_t frame_next_overflow[3]) {
  if (!t || !count || !frame_next_overflow || (cap > 0 && !host)) return fail("lwdetr_tracker_export: null pointer");
  lwb::TrackHead h;
  if (int rc = t->state.read_head("lwdetr_tracker_export", t->table.head, t->table.num_streams, stream_id, &h)) return rc;
  const int n = h.n_tracked + h.n_lost;
  const int m = n < cap ? n : (cap > 0 ? cap : 0);
  const lwdetr_track_record* src = t->table.rec + (static_cast<size_t>(stream_id) * 2 + h.parity) * t->table.capacity;
  if (cudaError_t e = t->state.read({{host, src, static_cast<size_t>(m) * sizeof(lwdetr_track_record)}}))
    return cuda_fail(e, "lwdetr_tracker_export");
  *count = n;
  frame_next_overflow[0] = h.frame;
  frame_next_overflow[1] = h.next_id;
  frame_next_overflow[2] = h.overflow;
  return 0;
}

static_assert(sizeof(lwdetr_zone_record) == 176, "zone record layout");

struct lwdetr_zones {
  lwb::ZoneTable table;
  lwdetr_zones_params params;
  std::vector<int32_t> n_lines, n_polys;   // each stream's geometry, as the last lwdetr_zones_set gave it
  DeviceState state;
};

void lwdetr_zones_params_default(lwdetr_zones_params* p) {
  if (!p) return;
  p->num_classes = 91;
  p->capacity = 1024;
  p->forget_after = 30;
  p->zone_anchor = LWDETR_ANCHOR_BOTTOM_CENTER;
  p->line_anchors = (1 << LWDETR_ANCHOR_TOP_LEFT) | (1 << LWDETR_ANCHOR_TOP_RIGHT) | (1 << LWDETR_ANCHOR_BOTTOM_LEFT) |
                    (1 << LWDETR_ANCHOR_BOTTOM_RIGHT);
}

int lwdetr_zones_create(int num_streams, const lwdetr_zones_params* params, lwdetr_zones** out) {
  if (!params || !out) return fail("lwdetr_zones_create: null pointer");
  const lwdetr_zones_params& p = *params;
  if (num_streams < 1) return fail("lwdetr_zones_create: num_streams must be >= 1");
  if (p.num_classes < 1 || p.num_classes > lwb::ZONE_CLASSES) return fail("lwdetr_zones_create: num_classes must be in [1, 1024]");
  if (p.capacity < 1 || p.capacity > lwb::ZONE_CAPACITY) return fail("lwdetr_zones_create: capacity must be in [1, 4096]");
  if (p.forget_after < 0) return fail("lwdetr_zones_create: forget_after must be >= 0");
  if (p.zone_anchor < 0 || p.zone_anchor > 8) return fail("lwdetr_zones_create: zone_anchor must be in [0, 9)");
  if (p.line_anchors <= 0 || p.line_anchors >= 1 << 9) return fail("lwdetr_zones_create: line_anchors must be a non-zero mask below 1 << 9");
  std::unique_ptr<lwdetr_zones> z(new (std::nothrow) lwdetr_zones{});
  if (!z) return fail("lwdetr_zones_create: out of memory");
  z->params = p;
  z->n_lines.assign(static_cast<size_t>(num_streams), 0);
  z->n_polys.assign(static_cast<size_t>(num_streams), 0);
  lwb::ZoneTable& t = z->table;
  t.num_streams = num_streams;
  t.capacity = p.capacity;
  t.num_classes = p.num_classes;
  t.forget_after = p.forget_after;
  t.zone_anchor = p.zone_anchor;
  t.line_anchors = p.line_anchors;
  const size_t ns = static_cast<size_t>(num_streams), cap = static_cast<size_t>(p.capacity), ncol = static_cast<size_t>(p.num_classes) + 1;
  const std::vector<lwb::ZoneHead> h(ns, lwb::ZoneHead{1, 0, 0, 0});    // every stream at frame 1, no records
  const auto layout = [&](Carver& c) {
    c.take(t.head, ns);
    c.take(t.geom, ns);
    c.take(t.verts, ns * lwb::ZONE_VERTS);
    c.take(t.index, ns * cap);
    c.take(t.rec, ns * cap);
    c.take(t.line_counts, ns * lwb::ZONE_LINES * ncol * 2);
    c.take(t.entries, ns * lwb::ZONE_POLYS * ncol);
  };
  const auto init = [&] {
    cudaError_t e = cudaMemcpyAsync(t.head, h.data(), ns * sizeof(lwb::ZoneHead), cudaMemcpyHostToDevice, z->state.copy);
    if (e == cudaSuccess) e = cudaMemsetAsync(t.geom, 0, ns * sizeof(lwb::ZoneGeom), z->state.copy);     // no lines, no polygons
    if (e == cudaSuccess) e = cudaMemsetAsync(t.line_counts, 0, ns * lwb::ZONE_LINES * ncol * 2 * sizeof(int32_t), z->state.copy);
    if (e == cudaSuccess) e = cudaMemsetAsync(t.entries, 0, ns * lwb::ZONE_POLYS * ncol * sizeof(int32_t), z->state.copy);
    return e;
  };
  if (int rc = z->state.create("lwdetr_zones_create", layout, init)) return rc;
  *out = z.release();
  return 0;
}

void lwdetr_zones_destroy(lwdetr_zones* z) { delete z; }

int lwdetr_zones_set(lwdetr_zones* z, int stream_id, const double* lines, int n_lines, const int32_t* polygon_sizes, int n_polygons,
                     const double* vertices) {
  if (!z || (n_lines > 0 && !lines) || (n_polygons > 0 && (!polygon_sizes || !vertices))) return fail("lwdetr_zones_set: null pointer");
  const lwb::ZoneTable& t = z->table;
  if (stream_id < 0 || stream_id >= t.num_streams) return fail("lwdetr_zones_set: stream id outside [0, num_streams)");
  if (n_lines < 0 || n_lines > lwb::ZONE_LINES) return fail("lwdetr_zones_set: n_lines must be in [0, 32]");
  if (n_polygons < 0 || n_polygons > lwb::ZONE_POLYS) return fail("lwdetr_zones_set: n_polygons must be in [0, 32]");
  lwb::ZoneGeom g{};
  g.n_lines = n_lines;
  g.n_polys = n_polygons;
  for (int l = 0; l < n_lines; ++l) {
    for (int c = 0; c < 4; ++c) {
      g.line[l][c] = lines[4 * l + c];
      if (!std::isfinite(g.line[l][c])) return fail("lwdetr_zones_set: line " + std::to_string(l) + " has a non-finite coordinate");
    }
    if (g.line[l][0] == g.line[l][2] && g.line[l][1] == g.line[l][3]) return fail("lwdetr_zones_set: line " + std::to_string(l) + " has zero length");
  }
  for (int q = 0; q < n_polygons; ++q) {
    if (polygon_sizes[q] < 3 || polygon_sizes[q] > lwb::ZONE_POLY_VERTS)
      return fail("lwdetr_zones_set: polygon " + std::to_string(q) + " must have 3 to 256 vertices");
    g.start[q + 1] = g.start[q] + polygon_sizes[q];
    if (g.start[q + 1] > lwb::ZONE_VERTS) return fail("lwdetr_zones_set: more than 2048 vertices");
  }
  const int nv = g.start[n_polygons];
  for (int i = 0; i < 2 * nv; ++i)
    if (!std::isfinite(vertices[i])) return fail("lwdetr_zones_set: vertex " + std::to_string(i / 2) + " has a non-finite coordinate");
  // after the object's last launch: the frame count goes on, the records and counters are cleared
  lwb::ZoneHead h;
  if (int rc = z->state.read_head("lwdetr_zones_set", t.head, t.num_streams, stream_id, &h)) return rc;
  h.n = 0;
  h.overflow = 0;
  const size_t s = static_cast<size_t>(stream_id), ncol = static_cast<size_t>(t.num_classes) + 1;
  lwb::DeviceGuard guard(z->state.device);
  const cudaStream_t cs = z->state.copy;
  cudaError_t e = cudaMemcpyAsync(t.geom + s, &g, sizeof(g), cudaMemcpyHostToDevice, cs);
  if (e == cudaSuccess && nv) e = cudaMemcpyAsync(t.verts + s * lwb::ZONE_VERTS, vertices, nv * sizeof(double2), cudaMemcpyHostToDevice, cs);
  if (e == cudaSuccess) e = cudaMemsetAsync(t.line_counts + s * lwb::ZONE_LINES * ncol * 2, 0, lwb::ZONE_LINES * ncol * 2 * sizeof(int32_t), cs);
  if (e == cudaSuccess) e = cudaMemsetAsync(t.entries + s * lwb::ZONE_POLYS * ncol, 0, lwb::ZONE_POLYS * ncol * sizeof(int32_t), cs);
  if (e == cudaSuccess) e = cudaMemcpyAsync(t.head + s, &h, sizeof(h), cudaMemcpyHostToDevice, cs);
  if (e == cudaSuccess) e = cudaStreamSynchronize(cs);
  if (e != cudaSuccess) return cuda_fail(e, "lwdetr_zones_set");
  z->n_lines[s] = n_lines;
  z->n_polys[s] = n_polygons;
  return 0;
}

int lwdetr_zones_reset(lwdetr_zones* z, const int32_t* streams, int n, void* stream) {
  return reset_call("lwdetr_zones_reset", z, streams, n, stream, lwb::zones_reset_launch);
}

int lwdetr_zones_update(lwdetr_zones* z, const int32_t* ids, const int32_t* labels, const float* boxes, const int32_t* counts, int B,
                        int max_out, const int32_t* stream_ids, uint32_t* inside, int32_t* occupancy, int32_t* events, int max_events,
                        int32_t* event_counts, void* stream) {
  if (!z || !ids || !labels || !boxes || !counts || !stream_ids || !inside || !occupancy || !event_counts || (max_events > 0 && !events))
    return fail("lwdetr_zones_update: null pointer");
  if (B < 1 || max_out < 1 || max_out > lwb::ZONE_MAX_OUT || max_events < 0)
    return fail("lwdetr_zones_update: need B >= 1, max_out in [1, 1024] and max_events >= 0");
  if (reinterpret_cast<uintptr_t>(boxes) % 16) return fail("lwdetr_zones_update: boxes must be 16-byte aligned");
  const std::string err = check_ids(z->table.num_streams, stream_ids, B);
  if (!err.empty()) return fail("lwdetr_zones_update: " + err);
  return z->state.launch("lwdetr_zones_update", stream, [&](cudaStream_t st) {
    return lwb::zones_launch(z->table, ids, labels, boxes, counts, B, max_out, stream_ids, inside, occupancy, events, max_events,
                             event_counts, st);
  });
}

int lwdetr_zones_export(lwdetr_zones* z, int stream_id, int32_t frame_overflow[2], int32_t info[3], int32_t* line_counts, int32_t* entries,
                        lwdetr_zone_record* records, int cap) {
  if (!z || !frame_overflow || !info || !line_counts || !entries || (cap > 0 && !records)) return fail("lwdetr_zones_export: null pointer");
  const lwb::ZoneTable& t = z->table;
  lwb::ZoneHead h;
  if (int rc = z->state.read_head("lwdetr_zones_export", t.head, t.num_streams, stream_id, &h)) return rc;
  const size_t s = static_cast<size_t>(stream_id), C = static_cast<size_t>(t.capacity), ncol = static_cast<size_t>(t.num_classes) + 1;
  const int L = z->n_lines[s], Z = z->n_polys[s];
  std::vector<lwb::ZoneIndex> idx(static_cast<size_t>(h.n));
  std::vector<lwb::ZoneRec> rec(C);
  const cudaError_t e = z->state.read({{line_counts, t.line_counts + s * lwb::ZONE_LINES * ncol * 2, L * ncol * 2 * sizeof(int32_t)},
                                       {entries, t.entries + s * lwb::ZONE_POLYS * ncol, Z * ncol * sizeof(int32_t)},
                                       {idx.data(), t.index + s * C, idx.size() * sizeof(lwb::ZoneIndex)},
                                       {rec.data(), t.rec + s * C, h.n ? C * sizeof(lwb::ZoneRec) : 0}});
  if (e != cudaSuccess) return cuda_fail(e, "lwdetr_zones_export");
  for (int i = 0; i < h.n && i < cap; ++i) {
    const lwb::ZoneRec& r = rec[static_cast<size_t>(idx[i].slot)];
    lwdetr_zone_record& o = records[i];
    o = lwdetr_zone_record{};
    o.id = idx[i].id;
    o.last_seen = idx[i].last_seen;
    o.label = r.label;
    o.inside = r.inside;
    for (int l = 0; l < L; ++l) o.sides[l] = static_cast<int8_t>(r.side_set >> l & 1 ? (r.side_pos >> l & 1 ? 1 : -1) : 0);
    for (int q = 0; q < Z; ++q) o.entry[q] = r.entry[q];
  }
  frame_overflow[0] = h.frame;
  frame_overflow[1] = h.overflow;
  info[0] = L;
  info[1] = Z;
  info[2] = h.n;
  return 0;
}

struct lwdetr_speed {
  lwb::SpeedTable table;
  DeviceState state;
};

int lwdetr_speed_create(int num_streams, int capacity, int window, int min_samples, int forget_after, int anchor, double frame_rate,
                        lwdetr_speed** out) {
  if (!out) return fail("lwdetr_speed_create: null pointer");
  if (num_streams < 1) return fail("lwdetr_speed_create: num_streams must be >= 1");
  if (capacity < 1 || capacity > lwb::SPEED_CAPACITY) return fail("lwdetr_speed_create: capacity must be in [1, 4096]");
  if (window < 2 || window > lwb::SPEED_WINDOW) return fail("lwdetr_speed_create: window must be in [2, 64]");
  if (min_samples < 2 || min_samples > window) return fail("lwdetr_speed_create: min_samples must be in [2, window]");
  if (forget_after < 0) return fail("lwdetr_speed_create: forget_after must be >= 0");
  if (anchor < 0 || anchor > 8) return fail("lwdetr_speed_create: anchor must be in [0, 9)");
  if (!std::isfinite(frame_rate) || frame_rate <= 0.0) return fail("lwdetr_speed_create: frame_rate must be finite and > 0");
  std::unique_ptr<lwdetr_speed> s(new (std::nothrow) lwdetr_speed{});
  if (!s) return fail("lwdetr_speed_create: out of memory");
  lwb::SpeedTable& t = s->table;
  t.num_streams = num_streams;
  t.capacity = capacity;
  t.window = window;
  t.min_samples = min_samples;
  t.forget_after = forget_after;
  t.anchor = anchor;
  t.frame_rate = frame_rate;
  const size_t ns = static_cast<size_t>(num_streams), cap = static_cast<size_t>(capacity);
  // every stream at frame 1, no records, no timestamp yet, H the identity
  const std::vector<lwb::SpeedHead> h(ns, lwb::SpeedHead{1, 0, 0, 0, -HUGE_VAL});
  std::vector<double> H(ns * 9, 0.0);
  for (size_t i = 0; i < ns; ++i) H[i * 9] = H[i * 9 + 4] = H[i * 9 + 8] = 1.0;
  const auto layout = [&](Carver& c) {
    c.take(t.head, ns);
    c.take(t.homography, ns * 9);
    c.take(t.index, ns * cap);
    c.take(t.rec, ns * cap);
    c.take(t.ring, ns * cap * static_cast<size_t>(window) * 3);
  };
  const auto init = [&] {
    cudaError_t e = cudaMemcpyAsync(t.head, h.data(), ns * sizeof(lwb::SpeedHead), cudaMemcpyHostToDevice, s->state.copy);
    if (e == cudaSuccess) e = cudaMemcpyAsync(t.homography, H.data(), H.size() * sizeof(double), cudaMemcpyHostToDevice, s->state.copy);
    return e;
  };
  if (int rc = s->state.create("lwdetr_speed_create", layout, init)) return rc;
  *out = s.release();
  return 0;
}

void lwdetr_speed_destroy(lwdetr_speed* s) { delete s; }

int lwdetr_speed_set(lwdetr_speed* s, int stream_id, const double* homography) {
  if (!s || !homography) return fail("lwdetr_speed_set: null pointer");
  const lwb::SpeedTable& t = s->table;
  if (stream_id < 0 || stream_id >= t.num_streams) return fail("lwdetr_speed_set: stream id outside [0, num_streams)");
  const double* h = homography;
  for (int i = 0; i < 9; ++i)
    if (!std::isfinite(h[i])) return fail("lwdetr_speed_set: the homography has a non-finite entry");
  const double det = h[0] * (h[4] * h[8] - h[5] * h[7]) - h[1] * (h[3] * h[8] - h[5] * h[6]) + h[2] * (h[3] * h[7] - h[4] * h[6]);
  if (det == 0.0 || !std::isfinite(det)) return fail("lwdetr_speed_set: the homography is singular");
  const cudaError_t e = s->state.write({{t.homography + static_cast<size_t>(stream_id) * 9, h, 9 * sizeof(double)}});
  return e == cudaSuccess ? 0 : cuda_fail(e, "lwdetr_speed_set");
}

int lwdetr_speed_reset(lwdetr_speed* s, const int32_t* streams, int n, void* stream) {
  return reset_call("lwdetr_speed_reset", s, streams, n, stream, lwb::speed_reset_launch);
}

int lwdetr_speed_update(lwdetr_speed* s, const int32_t* ids, const float* boxes, const int32_t* counts, int B, int max_out,
                        const int32_t* stream_ids, const double* timestamps, float* kin, int32_t* samples, void* stream) {
  if (!s || !ids || !boxes || !counts || !stream_ids || !kin || !samples) return fail("lwdetr_speed_update: null pointer");
  if (B < 1 || max_out < 1 || max_out > lwb::SPEED_MAX_OUT) return fail("lwdetr_speed_update: need B >= 1 and max_out in [1, 1024]");
  if (reinterpret_cast<uintptr_t>(boxes) % 16) return fail("lwdetr_speed_update: boxes must be 16-byte aligned");
  const std::string err = check_ids(s->table.num_streams, stream_ids, B);
  if (!err.empty()) return fail("lwdetr_speed_update: " + err);
  return s->state.launch("lwdetr_speed_update", stream, [&](cudaStream_t st) {
    return lwb::speed_launch(s->table, ids, boxes, counts, B, max_out, stream_ids, timestamps, kin, samples, st);
  });
}

int lwdetr_speed_export(lwdetr_speed* s, int stream_id, int32_t head[4], double* last_t, double* homography, int32_t* ids,
                        int32_t* last_seen, int32_t* counts, double* samples, int cap) {
  if (!s || !head || !last_t || !homography || (cap > 0 && (!ids || !last_seen || !counts || !samples)))
    return fail("lwdetr_speed_export: null pointer");
  const lwb::SpeedTable& t = s->table;
  lwb::SpeedHead h;
  if (int rc = s->state.read_head("lwdetr_speed_export", t.head, t.num_streams, stream_id, &h)) return rc;
  const size_t st = static_cast<size_t>(stream_id), C = static_cast<size_t>(t.capacity), W = static_cast<size_t>(t.window);
  std::vector<lwb::RecordIndex> idx(static_cast<size_t>(h.n));
  std::vector<lwb::SpeedRec> rec(h.n ? C : 0);
  std::vector<double> ring(h.n ? C * W * 3 : 0);
  const cudaError_t e = s->state.read({{homography, t.homography + st * 9, 9 * sizeof(double)},
                                       {idx.data(), t.index + st * C, idx.size() * sizeof(lwb::RecordIndex)},
                                       {rec.data(), t.rec + st * C, rec.size() * sizeof(lwb::SpeedRec)},
                                       {ring.data(), t.ring + st * C * W * 3, ring.size() * sizeof(double)}});
  if (e != cudaSuccess) return cuda_fail(e, "lwdetr_speed_export");
  for (int i = 0; i < h.n && i < cap; ++i) {
    const size_t slot = static_cast<size_t>(idx[i].slot);
    const lwb::SpeedRec r = rec[slot];
    ids[i] = idx[i].id;
    last_seen[i] = idx[i].last_seen;
    counts[i] = r.n;
    for (int k = 0; k < r.n; ++k)
      for (int c = 0; c < 3; ++c) samples[(i * W + k) * 3 + c] = ring[(slot * W + (r.pos + k) % W) * 3 + c];
  }
  head[0] = h.frame;
  head[1] = h.n;
  head[2] = h.overflow;
  head[3] = h.clock_errors;
  *last_t = h.last_t;
  return 0;
}

// the annotator's default palette (include/lwdetr_b200.h)
static const uint8_t kAnnPalette[16][3] = {{230, 25, 75},   {60, 180, 75},  {255, 225, 25},  {0, 130, 200},  {245, 130, 48}, {145, 30, 180},
                                           {70, 240, 240},  {240, 50, 230}, {210, 245, 60},  {250, 190, 212}, {0, 128, 128},  {220, 190, 255},
                                           {170, 110, 40},  {255, 250, 200}, {128, 0, 0},    {170, 255, 195}};

struct lwdetr_annotator {
  lwb::AnnTable table;
  lwb::AnnOptions options;
  DeviceState state;
};

int lwdetr_annotator_create(int num_classes, lwdetr_annotator** out) {
  if (!out) return fail("lwdetr_annotator_create: null pointer");
  if (num_classes < 1 || num_classes > lwb::ANN_CLASSES) return fail("lwdetr_annotator_create: num_classes must be in [1, 1024]");
  std::unique_ptr<lwdetr_annotator> a(new (std::nothrow) lwdetr_annotator{});
  if (!a) return fail("lwdetr_annotator_create: out of memory");
  a->options = lwb::AnnOptions{2, 2, 0, LWDETR_LABEL_NAME | LWDETR_LABEL_ID | LWDETR_LABEL_SCORE, 64, 2, 16};
  lwb::AnnTable& t = a->table;
  t.num_classes = num_classes;
  const size_t nc = static_cast<size_t>(num_classes);
  const int32_t n16 = 16;
  const auto layout = [&](Carver& c) {
    c.take(t.palette, lwb::ANN_PALETTE * 3);
    c.take(t.palette_n, 1);
    c.take(t.names, nc * lwb::ANN_NAME);
    c.take(t.privacy, nc);
    c.take(t.prims, static_cast<size_t>(lwb::ANN_GROUP) * lwb::ANN_PRIMS);
    c.take(t.nprims, static_cast<size_t>(lwb::ANN_GROUP) * 2);
    c.take(t.texts, static_cast<size_t>(lwb::ANN_GROUP) * lwb::ANN_TEXTS * lwb::ANN_TEXT);
  };
  const auto init = [&] {
    cudaError_t e = cudaMemcpyAsync(t.palette, kAnnPalette, sizeof(kAnnPalette), cudaMemcpyHostToDevice, a->state.copy);
    if (e == cudaSuccess) e = cudaMemcpyAsync(t.palette_n, &n16, sizeof(n16), cudaMemcpyHostToDevice, a->state.copy);
    if (e == cudaSuccess) e = cudaMemsetAsync(t.names, 0, nc * lwb::ANN_NAME, a->state.copy);     // every class named by its id
    if (e == cudaSuccess) e = cudaMemsetAsync(t.privacy, 0, nc, a->state.copy);
    return e;
  };
  if (int rc = a->state.create("lwdetr_annotator_create", layout, init)) return rc;
  *out = a.release();
  return 0;
}

void lwdetr_annotator_destroy(lwdetr_annotator* a) { delete a; }

int lwdetr_annotator_set_option(lwdetr_annotator* a, const char* name, int value) {
  if (!a || !name) return fail("lwdetr_annotator_set_option: null pointer");
  const std::string n(name), fn = "lwdetr_annotator_set_option: ";
  lwb::AnnOptions& o = a->options;
  const auto in = [&](int lo, int hi, int* dst) {
    if (value < lo || value > hi) return fail(fn + n + " must be in [" + std::to_string(lo) + ", " + std::to_string(hi) + "], got " + std::to_string(value));
    *dst = value;
    return 0;
  };
  if (n == "thickness") return in(1, 32, &o.thickness);
  if (n == "text_scale") return in(1, 8, &o.text_scale);
  if (n == "box_fill_alpha") return in(0, 256, &o.box_fill_alpha);
  if (n == "label") return in(0, 7, &o.label);
  if (n == "zone_fill_alpha") return in(0, 256, &o.zone_fill_alpha);
  if (n == "zone_thickness") return in(1, 32, &o.zone_thickness);
  if (n == "privacy_block") {
    if (value < 2 || value > 64 || (value & (value - 1))) return fail(fn + "privacy_block must be 2, 4, 8, 16, 32 or 64, got " + std::to_string(value));
    o.privacy_block = value;
    return 0;
  }
  return fail(fn + "unknown option " + n + " (thickness, text_scale, box_fill_alpha, label, zone_fill_alpha, zone_thickness, privacy_block)");
}

int lwdetr_annotator_set_names(lwdetr_annotator* a, const char* names) {
  if (!a || !names) return fail("lwdetr_annotator_set_names: null pointer");
  const lwb::AnnTable& t = a->table;
  std::vector<char> tab(static_cast<size_t>(t.num_classes) * lwb::ANN_NAME, 0);
  int cls = 0, len = 0;
  for (const char* c = names; *c; ++c) {
    if (*c == '\n') {
      ++cls;
      len = 0;
      continue;
    }
    if (cls >= t.num_classes) return fail("lwdetr_annotator_set_names: more than num_classes = " + std::to_string(t.num_classes) + " names");
    if (len == lwb::ANN_NAME - 1) return fail("lwdetr_annotator_set_names: the name of class " + std::to_string(cls) + " is longer than 31 characters");
    tab[static_cast<size_t>(cls) * lwb::ANN_NAME + len++] = *c;
  }
  if (cudaError_t e = a->state.write({{t.names, tab.data(), tab.size()}})) return cuda_fail(e, "lwdetr_annotator_set_names");
  return 0;
}

int lwdetr_annotator_set_palette(lwdetr_annotator* a, const uint8_t* rgb, int n) {
  if (!a || !rgb) return fail("lwdetr_annotator_set_palette: null pointer");
  if (n < 1 || n > lwb::ANN_PALETTE) return fail("lwdetr_annotator_set_palette: n must be in [1, 256]");
  const int32_t nn = n;
  if (cudaError_t e = a->state.write({{a->table.palette, rgb, 3 * static_cast<size_t>(n)}, {a->table.palette_n, &nn, sizeof(nn)}}))
    return cuda_fail(e, "lwdetr_annotator_set_palette");
  return 0;
}

int lwdetr_annotator_set_privacy(lwdetr_annotator* a, const int32_t* classes, int n) {
  if (!a || (n > 0 && !classes)) return fail("lwdetr_annotator_set_privacy: null pointer");
  if (n < 0) return fail("lwdetr_annotator_set_privacy: n must be >= 0");
  const lwb::AnnTable& t = a->table;
  std::vector<uint8_t> mask(static_cast<size_t>(t.num_classes), 0);
  for (int i = 0; i < n; ++i) {
    if (classes[i] < 0 || classes[i] >= t.num_classes)
      return fail("lwdetr_annotator_set_privacy: class " + std::to_string(classes[i]) + " outside [0, " + std::to_string(t.num_classes) + ")");
    mask[static_cast<size_t>(classes[i])] = 1;
  }
  if (cudaError_t e = a->state.write({{t.privacy, mask.data(), mask.size()}})) return cuda_fail(e, "lwdetr_annotator_set_privacy");
  return 0;
}

struct lwdetr_gmc {
  lwb::GmcTable table;
  DeviceState state;
};

void lwdetr_gmc_params_default(lwdetr_gmc_params* p) {
  if (!p) return;
  p->downscale = 2;
  p->max_points = 1024;
  p->quality = 0.01f;
  p->levels = 3;
  p->window = 21;
  p->iterations = 30;
  p->eps = 0.01f;
  p->min_eig = 1e-4f;
  p->ransac_thresh = 3.0f;
  p->hypotheses = 1024;
  p->min_inliers = 10;
  p->max_height = 2160;
  p->max_width = 3840;
}

int lwdetr_gmc_create(int num_streams, const lwdetr_gmc_params* params, lwdetr_gmc** out) {
  if (!params || !out) return fail("lwdetr_gmc_create: null pointer");
  const lwdetr_gmc_params& p = *params;
  if (num_streams < 1) return fail("lwdetr_gmc_create: num_streams must be >= 1");
  if (p.downscale < 1 || p.downscale > 8) return fail("lwdetr_gmc_create: downscale must be in [1, 8]");
  if (p.max_points < 16 || p.max_points > lwb::GMC_MAX_POINTS) return fail("lwdetr_gmc_create: max_points must be in [16, 4096]");
  if (!(p.quality > 0.f && p.quality <= 1.f)) return fail("lwdetr_gmc_create: quality must be in (0, 1]");
  if (p.levels < 0 || p.levels > lwb::GMC_MAX_LEVELS) return fail("lwdetr_gmc_create: levels must be in [0, 5]");
  if (p.window < 5 || p.window > lwb::GMC_MAX_WINDOW || p.window % 2 == 0) return fail("lwdetr_gmc_create: window must be odd in [5, 31]");
  if (p.iterations < 1 || p.iterations > 100) return fail("lwdetr_gmc_create: iterations must be in [1, 100]");
  if (!(p.eps > 0.f && p.eps < 1e30f) || !(p.min_eig >= 0.f && p.min_eig < 1e30f) || !(p.ransac_thresh > 0.f && p.ransac_thresh < 1e30f))
    return fail("lwdetr_gmc_create: need eps > 0, min_eig >= 0 and ransac_thresh > 0, all finite");
  if (p.hypotheses < 1 || p.hypotheses > lwb::GMC_MAX_HYPOTHESES) return fail("lwdetr_gmc_create: hypotheses must be in [1, 4096]");
  if (p.min_inliers < 2 || p.min_inliers > p.max_points) return fail("lwdetr_gmc_create: min_inliers must be in [2, max_points]");
  const int lo = lwb::GMC_MIN_SIDE * p.downscale;
  if (p.max_height < lo || p.max_width < lo || p.max_height > 8192 || p.max_width > 8192)
    return fail("lwdetr_gmc_create: max_height and max_width must be in [16 * downscale, 8192]");
  std::unique_ptr<lwdetr_gmc> g(new (std::nothrow) lwdetr_gmc{});
  if (!g) return fail("lwdetr_gmc_create: out of memory");
  lwb::GmcTable& t = g->table;
  t.num_streams = num_streams;
  t.p = p;
  lwb::GmcGeo geo;
  lwb::gmc_geometry(p.max_height, p.max_width, p, &geo);
  long long off = 0;
  for (int l = 0; l <= lwb::GMC_MAX_LEVELS; ++l) {
    t.off[l] = off;
    if (l <= p.levels) off += (static_cast<long long>(geo.lw[l]) * geo.lh[l] + 15) / 16 * 16;
  }
  t.slot_bytes = off;
  const size_t ns = static_cast<size_t>(num_streams), mp = static_cast<size_t>(p.max_points);
  const auto layout = [&](Carver& c) {
    c.take(t.head, ns);
    c.take(t.pyr, ns * 2 * static_cast<size_t>(t.slot_bytes));
    c.take(t.pts, ns * 2 * mp);
    c.take(t.cell_r, ns * mp);
    c.take(t.cell_i, ns * mp);
    c.take(t.flow, ns * mp);
    c.take(t.found, ns * mp);
  };
  const auto init = [&] { return cudaMemsetAsync(t.head, 0, ns * sizeof(lwb::GmcHead), g->state.copy); };
  if (int rc = g->state.create("lwdetr_gmc_create", layout, init)) return rc;
  *out = g.release();
  return 0;
}

void lwdetr_gmc_destroy(lwdetr_gmc* g) { delete g; }

int lwdetr_gmc_reset(lwdetr_gmc* g, const int32_t* streams, int n, void* stream) {
  return reset_call("lwdetr_gmc_reset", g, streams, n, stream, lwb::gmc_reset_launch);
}

int lwdetr_gmc_export(lwdetr_gmc* g, int stream_id, uint8_t* levels, int64_t levels_bytes, float* corners, float* flow, int8_t* found,
                      int32_t info[6]) {
  if (!g || !info || (levels_bytes > 0 && !levels) || !corners || !flow || !found) return fail("lwdetr_gmc_export: null pointer");
  const lwb::GmcTable& t = g->table;
  lwb::GmcHead h;
  if (int rc = g->state.read_head("lwdetr_gmc_export", t.head, t.num_streams, stream_id, &h)) return rc;
  lwb::GmcGeo geo;
  lwb::gmc_geometry(h.valid ? h.h : lwb::GMC_MIN_SIDE * t.p.downscale, h.valid ? h.w : lwb::GMC_MIN_SIDE * t.p.downscale, t.p, &geo);
  const int nlev = h.valid ? geo.nlev : -1;
  long long need = 0;
  for (int l = 0; l <= nlev; ++l) need += static_cast<long long>(geo.lw[l]) * geo.lh[l];
  if (need > levels_bytes) return fail("lwdetr_gmc_export: levels buffer too small");
  const size_t mp = static_cast<size_t>(t.p.max_points), sid = static_cast<size_t>(stream_id);
  const uint8_t* slot = t.pyr + (sid * 2 + h.cur) * static_cast<size_t>(t.slot_bytes);
  std::vector<DeviceState::Copy> parts;
  long long o = 0;
  for (int l = 0; l <= nlev; ++l) {
    const size_t n = static_cast<size_t>(geo.lw[l]) * geo.lh[l];
    parts.push_back({levels + o, slot + t.off[l], n});
    o += static_cast<long long>(n);
  }
  parts.push_back({corners, t.pts + (sid * 2 + h.cur) * mp, mp * sizeof(float2)});
  parts.push_back({flow, t.flow + sid * mp, mp * sizeof(float4)});
  parts.push_back({found, t.found + sid * mp, mp});
  if (cudaError_t e = g->state.read(parts)) return cuda_fail(e, "lwdetr_gmc_export");
  info[0] = h.valid;
  info[1] = h.h;
  info[2] = h.w;
  info[3] = nlev;
  info[4] = h.npts[h.cur];
  info[5] = h.npts[h.cur ^ 1];
  return 0;
}

}  // extern "C"

// a frame as the estimator reads it: RGB, or NV12 through its luma plane
static lwb::GmcFrameHost gmc_frame(const lwdetr_frame& f) { return {f.data, f.pitch_bytes, f.height, f.width, 0}; }
static lwb::GmcFrameHost gmc_frame(const lwdetr_frame_nv12& f) { return {f.luma, f.luma_pitch, f.height, f.width, 1}; }

// lwdetr_gmc_estimate / _nv12, and with observe lwdetr_gmc_observe / _nv12 (no outputs)
template <typename F>
static int gmc_call(const char* name, lwdetr_gmc* g, const F* frames, int B, const int32_t* stream_ids, double* motion, int32_t* status,
                    int32_t* inliers, void* stream, bool observe) {
  const std::string fn(name);
  if (!g || !frames || !stream_ids) return fail(fn + ": null pointer");
  if (B < 1) return fail(fn + ": B must be >= 1");
  if (!observe && (!motion || !status || !inliers)) return fail(fn + ": null pointer");
  if (reinterpret_cast<uintptr_t>(motion) % 8) return fail(fn + ": motion must be 8-byte aligned");
  const std::string err = check_ids(g->table.num_streams, stream_ids, B);
  if (!err.empty()) return fail(fn + ": " + err);
  const lwdetr_gmc_params& p = g->table.p;
  const int lo = lwb::GMC_MIN_SIDE * p.downscale;
  std::vector<lwb::GmcFrameHost> fr(static_cast<size_t>(B));
  for (int i = 0; i < B; ++i) {
    const lwb::GmcFrameHost& f = fr[i] = gmc_frame(frames[i]);
    if (!f.data) return fail(fn + ": null frame pointer");
    if (f.h < lo || f.w < lo || f.h > p.max_height || f.w > p.max_width)
      return fail(fn + ": frame " + std::to_string(i) + " is " + std::to_string(f.h) + " x " + std::to_string(f.w) + "; sides must be in [" +
                  std::to_string(lo) + ", max_height / max_width = " + std::to_string(p.max_height) + " x " + std::to_string(p.max_width) + "]");
    if (f.pitch < static_cast<long long>(f.w) * (f.nv12 ? 1 : 3)) return fail(fn + ": frame " + std::to_string(i) + ": pitch too small");
  }
  return g->state.launch(fn, stream, [&](cudaStream_t st) {
    return lwb::gmc_estimate_launch(g->table, fr.data(), B, stream_ids, motion, status, inliers, st, observe);
  });
}

extern "C" {

int lwdetr_gmc_estimate(lwdetr_gmc* g, const lwdetr_frame* frames, int B, const int32_t* stream_ids, double* motion, int32_t* status,
                        int32_t* inliers, void* stream) {
  return gmc_call("lwdetr_gmc_estimate", g, frames, B, stream_ids, motion, status, inliers, stream, false);
}

int lwdetr_gmc_estimate_nv12(lwdetr_gmc* g, const lwdetr_frame_nv12* frames, int B, const int32_t* stream_ids, double* motion,
                             int32_t* status, int32_t* inliers, void* stream) {
  return gmc_call("lwdetr_gmc_estimate_nv12", g, frames, B, stream_ids, motion, status, inliers, stream, false);
}

int lwdetr_gmc_observe(lwdetr_gmc* g, const lwdetr_frame* frames, int B, const int32_t* stream_ids, void* stream) {
  return gmc_call("lwdetr_gmc_observe", g, frames, B, stream_ids, nullptr, nullptr, nullptr, stream, true);
}

int lwdetr_gmc_observe_nv12(lwdetr_gmc* g, const lwdetr_frame_nv12* frames, int B, const int32_t* stream_ids, void* stream) {
  return gmc_call("lwdetr_gmc_observe_nv12", g, frames, B, stream_ids, nullptr, nullptr, nullptr, stream, true);
}

struct lwdetr_flow {
  lwb::FlowTable table;
  lwdetr_gmc* gmc;
  DeviceState state;
};

void lwdetr_flow_params_default(lwdetr_flow_params* p) {
  if (!p) return;
  p->grid = 10;
  p->window = 15;
  p->iterations = 30;
  p->eps = 0.01f;
  p->min_eig = 1e-4f;
  p->ncc_window = 11;
  p->min_points = 8;
  p->fb_max = 10.f;
  p->scale_min = 0.5f;
  p->scale_max = 2.f;
  p->max_tracks = 256;
}

int lwdetr_flow_create(lwdetr_gmc* gmc, const lwdetr_flow_params* params, lwdetr_flow** out) {
  if (!gmc || !params || !out) return fail("lwdetr_flow_create: null pointer");
  const lwdetr_flow_params& p = *params;
  if (p.grid < 2 || p.grid > lwb::FLOW_MAX_GRID) return fail("lwdetr_flow_create: grid must be in [2, 16]");
  if (p.window < 5 || p.window > lwb::GMC_MAX_WINDOW || p.window % 2 == 0) return fail("lwdetr_flow_create: window must be odd in [5, 31]");
  if (p.iterations < 1 || p.iterations > 100) return fail("lwdetr_flow_create: iterations must be in [1, 100]");
  if (!(p.eps > 0.f && p.eps < 1e30f) || !(p.min_eig >= 0.f && p.min_eig < 1e30f)) return fail("lwdetr_flow_create: need eps > 0 and min_eig >= 0, both finite");
  if (p.ncc_window < 3 || p.ncc_window > 31 || p.ncc_window % 2 == 0) return fail("lwdetr_flow_create: ncc_window must be odd in [3, 31]");
  if (p.min_points < 1 || p.min_points > p.grid * p.grid) return fail("lwdetr_flow_create: min_points must be in [1, grid^2]");
  if (!(p.fb_max > 0.f && p.fb_max < 1e30f)) return fail("lwdetr_flow_create: fb_max must be > 0 and finite");
  if (!(p.scale_min > 0.f && p.scale_min <= 1.f && p.scale_max >= 1.f && p.scale_max < 1e30f))
    return fail("lwdetr_flow_create: need 0 < scale_min <= 1 <= scale_max, finite");
  if (p.max_tracks < 1 || p.max_tracks > lwb::TRACK_MAX) return fail("lwdetr_flow_create: max_tracks must be in [1, 1024]");
  std::unique_ptr<lwdetr_flow> f(new (std::nothrow) lwdetr_flow{});
  if (!f) return fail("lwdetr_flow_create: out of memory");
  lwb::DeviceGuard dg(gmc->state.device);   // the flow's scratch lives beside the estimator's pyramids, which its kernels read
  lwb::FlowTable& t = f->table;
  t.p = p;
  t.num_streams = gmc->table.num_streams;
  t.g2 = p.grid * p.grid;
  f->gmc = gmc;
  const size_t ns = static_cast<size_t>(t.num_streams), nt = ns * static_cast<size_t>(p.max_tracks), np = nt * static_cast<size_t>(t.g2);
  const auto layout = [&](Carver& c) {
    c.take(t.ntracks, ns);
    c.take(t.slot, nt);
    c.take(t.status, nt);
    c.take(t.meas, nt * 8);
    c.take(t.seed, np);
    c.take(t.fwd, np);
    c.take(t.bwd, np);
    c.take(t.fb, np);
    c.take(t.ncc, np);
    c.take(t.valid, np);
  };
  const auto init = [&] { return cudaMemsetAsync(t.ntracks, 0, ns * sizeof(int32_t), f->state.copy); };
  if (int rc = f->state.create("lwdetr_flow_create", layout, init)) return rc;
  *out = f.release();
  return 0;
}

void lwdetr_flow_destroy(lwdetr_flow* f) { delete f; }

int lwdetr_track_flow(lwdetr_tracker* t, lwdetr_flow* flow, const double* motion, int B, const int32_t* stream_ids, int max_out,
                      int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes, int32_t* out_index, int32_t* counts,
                      void* stream) {
  const std::string fn("lwdetr_track_flow");
  if (!t || !flow || !stream_ids || !out_ids || !out_scores || !out_labels || !out_boxes || !out_index || !counts)
    return fail(fn + ": null pointer");
  if (B < 1 || max_out < 1) return fail(fn + ": need B >= 1 and max_out >= 1");
  if (reinterpret_cast<uintptr_t>(out_boxes) % 16) return fail(fn + ": out_boxes must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(motion) % 8) return fail(fn + ": motion must be 8-byte aligned");
  std::string err = check_ids(t->table.num_streams, stream_ids, B);
  if (err.empty()) err = check_ids(flow->table.num_streams, stream_ids, B);
  if (!err.empty()) return fail(fn + ": " + err);
  if (flow->state.device != t->state.device) return fail(fn + ": the tracker and the flow live on different devices");
  const auto run = [&](cudaStream_t st) {
    int e = lwb::flow_launch(flow->table, flow->gmc->table, t->table, B, stream_ids, st);
    if (!e) e = lwb::track_flow_launch(t->table, t->params, flow->table, motion, t->reid.slot, B, stream_ids, max_out, out_ids, out_scores,
                                       out_labels, out_boxes, out_index, counts, st);
    return e;
  };
  return flow->state.launch(fn, stream, run, &t->state);   // the devices are one: checked above
}

int lwdetr_flow_export(lwdetr_flow* f, int stream_id, int cap, float* seeds, float* fwd, float* bwd, int8_t* valid, double* fb,
                       double* ncc, int32_t* status, double* meas, int32_t info[3]) {
  if (!f || !info || (cap > 0 && (!seeds || !fwd || !bwd || !valid || !fb || !ncc || !status || !meas)))
    return fail("lwdetr_flow_export: null pointer");
  const lwb::FlowTable& t = f->table;
  int32_t n = 0;
  if (int rc = f->state.read_head("lwdetr_flow_export", t.ntracks, t.num_streams, stream_id, &n)) return rc;
  const int m = std::min(std::min(n, t.p.max_tracks), std::max(cap, 0));
  const size_t o = static_cast<size_t>(stream_id) * t.p.max_tracks, g2 = static_cast<size_t>(t.g2), k = static_cast<size_t>(m);
  if (cudaError_t e = f->state.read({{seeds, t.seed + o * g2, k * g2 * sizeof(float2)},
                                     {fwd, t.fwd + o * g2, k * g2 * sizeof(float2)},
                                     {bwd, t.bwd + o * g2, k * g2 * sizeof(float2)},
                                     {valid, t.valid + o * g2, k * g2},
                                     {fb, t.fb + o * g2, k * g2 * sizeof(double)},
                                     {ncc, t.ncc + o * g2, k * g2 * sizeof(double)},
                                     {status, t.status + o, k * sizeof(int32_t)},
                                     {meas, t.meas + o * 8, k * 8 * sizeof(double)}}))
    return cuda_fail(e, "lwdetr_flow_export");
  info[0] = n;
  info[1] = std::min(n, t.p.max_tracks);
  info[2] = t.p.grid;
  return 0;
}

int lwdetr_query_best(const float* pred_logits, const float* pred_boxes, const float* target_sizes, int B, int nq, int num_classes,
                      float* scores, int32_t* labels, float* boxes, void* stream) {
  if (!pred_logits || !pred_boxes || !target_sizes || !scores || !labels || !boxes) return fail("lwdetr_query_best: null pointer");
  if (B < 1 || nq < 1 || num_classes < 1) return fail("lwdetr_query_best: bad sizes");
  if (reinterpret_cast<uintptr_t>(pred_boxes) % 16 || reinterpret_cast<uintptr_t>(boxes) % 16)
    return fail("lwdetr_query_best: pred_boxes and boxes must be 16-byte aligned");
  int e = lwb::query_best_launch(pred_logits, pred_boxes, target_sizes, B, nq, num_classes, scores, labels, boxes,
                                 static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_query_best launch");
  return 0;
}

int lwdetr_layernorm_e4m3(const void* x, int ldx, int64_t rows, int C, float eps, uint8_t* q, int ldq, float* row_scale, void* stream) {
  if (!x || !q || !row_scale) return fail("lwdetr_layernorm_e4m3: null pointer");
  int e = lwb::layernorm_e4m3_launch(x, ldx, rows, C, eps, q, ldq, row_scale, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail("lwdetr_layernorm_e4m3: need rows >= 1, C % 8 == 0, 8 <= C <= 1024, ldx and ldq multiples of 8 and >= C");
  if (e) return cuda_fail(e, "lwdetr_layernorm_e4m3 launch");
  return 0;
}

int lwdetr_gemm_e4m3(const void* A, int lda, const float* a_scale, int M, int K, const void* W, const float* w_scale, int N,
                     const float* bias, int act, void* out, int ld_out, void* stream) {
  lwb::GemmE4m3Desc d;
  d.A = A; d.lda = lda; d.a_scale = a_scale; d.M = M; d.K = K; d.W = W; d.w_scale = w_scale; d.N = N; d.bias = bias;
  d.act = act; d.out = out; d.ld_out = ld_out;
  lwb::GemmOp op;
  std::string err;
  if (lwb::gemm_e4m3_build(d, &op, &err)) return fail("lwdetr_gemm_e4m3: " + err);
  int e = lwb::gemm_launch(op, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_gemm_e4m3 launch");
  return 0;
}

int lwdetr_vit_mlp(int dtype, const void* x, int ldx, int M, const float* stats_in, int stats_parts, float eps,
                   const void* W1, const float* colsum1, const float* b1, const void* W2, const float* b2,
                   const float* gamma, void* out, int ld_out, float* stats_out, int stats_parts_out, void* stream) {
  lwb::MlpDesc d;
  d.dtype = dtype; d.x = x; d.ldx = ldx; d.M = M;
  d.stats_in = reinterpret_cast<const float2*>(stats_in); d.stats_parts_in = stats_parts; d.ln_eps = eps;
  d.w1 = W1; d.colsum1 = colsum1; d.b1 = b1; d.w2 = W2; d.b2 = b2; d.gamma = gamma;
  d.out = out; d.ld_out = ld_out; d.stats_out = reinterpret_cast<float2*>(stats_out); d.stats_parts_out = stats_parts_out;
  lwb::MlpOp op;
  std::string err;
  if (lwb::vit_mlp_build(d, &op, &err)) return fail("lwdetr_vit_mlp: " + err);
  int e = lwb::vit_mlp_launch(op, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_vit_mlp launch");
  return 0;
}

int lwdetr_host_quant_e4m3_rows(const float* src, int64_t rows, int K, uint8_t* q, float* scale) {
  if (!src || !q || !scale || rows < 0 || K < 1) return fail("lwdetr_host_quant_e4m3_rows: bad arguments");
  lwb::host_quant_e4m3_rows(src, rows, K, q, scale);
  return 0;
}

int lwdetr_host_bicubic(const float* src, int n_in, int C, int n_out, float* dst) {
  if (!src || !dst || n_in < 1 || n_out < 1 || C < 1) return fail("lwdetr_host_bicubic: bad arguments");
  lwb::bicubic_resize_chlast(src, n_in, C, n_out, dst);
  return 0;
}

int lwdetr_host_bicubic_hw(const float* src, int n_in, int C, int out_h, int out_w, float* dst) {
  if (!src || !dst || n_in < 1 || out_h < 1 || out_w < 1 || C < 1) return fail("lwdetr_host_bicubic_hw: bad arguments");
  lwb::bicubic_resize_chlast_hw(src, n_in, C, out_h, out_w, dst);
  return 0;
}

// ------------------------------------------------------------------------------------------ model level
struct lwdetr_handle {
  lwb::Engine* eng;
};

int lwdetr_create(const lwdetr_config* cfg, int dtype, lwdetr_handle** out) {
  if (!cfg || !out) return fail("lwdetr_create: null pointer");
  if (dtype != LWDETR_F16 && dtype != LWDETR_BF16 && dtype != LWDETR_F16_E4M3)
    return fail("lwdetr_create: dtype must be LWDETR_F16, LWDETR_BF16 or LWDETR_F16_E4M3");
  if (cfg->n_taps < 1 || cfg->n_taps > 4 || cfg->n_levels < 1 || cfg->n_levels > 2 || cfg->vit_depth < 1 || cfg->vit_depth > 31)
    return fail("lwdetr_create: unsupported configuration");
  if (cfg->img_size % 64 != 0 || cfg->vit_dim % 64 != 0 || cfg->hidden_dim % 128 != 0)
    return fail("lwdetr_create: img_size % 64, vit_dim % 64 and hidden_dim % 128 must be 0");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail("lwdetr_create: no CUDA device (there is no CPU fallback)");
  if (cfg->num_classes < 1 || cfg->num_classes > 4096) return fail("lwdetr_create: num_classes must be in [1, 4096]");
  lwdetr_handle* h = new (std::nothrow) lwdetr_handle;
  if (!h) return fail("lwdetr_create: out of memory");
  h->eng = new (std::nothrow) lwb::Engine(*cfg, dtype);
  if (!h->eng) { delete h; return fail("lwdetr_create: out of memory"); }
  *out = h;
  return 0;
}

void lwdetr_destroy(lwdetr_handle* h) {
  if (!h) return;
  delete h->eng;
  delete h;
}

int lwdetr_load_weights(lwdetr_handle* h, int n, const char* const* names, const float* const* data, const int64_t* numel) {
  if (!h || !names || !data || !numel) return fail("lwdetr_load_weights: null pointer");
  std::map<std::string, lwb::HostTensor> m;
  for (int i = 0; i < n; ++i) m[names[i]] = lwb::HostTensor{data[i], numel[i]};
  std::string err;
  if (h->eng->load_weights(m, &err)) return fail("lwdetr_load_weights: " + err);
  return 0;
}

static int forward_input(const char* fn, lwdetr_handle* h, const lwdetr_input* input, int B, int height, int width, float* pred_logits,
                         float* pred_boxes, const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream) {
  if (!h || !input || !input->images) return fail(std::string(fn) + ": null pointer");
  if (input->format != LWDETR_IN_F32_NCHW && input->format != LWDETR_IN_16_NCHW && input->format != LWDETR_IN_U8_NHWC)
    return fail(std::string(fn) + ": format must be LWDETR_IN_F32_NCHW, LWDETR_IN_16_NCHW or LWDETR_IN_U8_NHWC");
  lwb::ForwardIn in;
  in.images = input->images; in.kind = input->format; in.mask = input->padding_mask;
  for (int c = 0; c < 3; ++c) {
    in.mean[c] = input->mean[c]; in.stdv[c] = input->std[c];
    if (input->format == LWDETR_IN_U8_NHWC && !(input->std[c] > 0.f)) return fail(std::string(fn) + ": std must be positive");
  }
  std::string err;
  if (h->eng->forward(in, B, height, width, pred_logits, pred_boxes, aux, topk_override, static_cast<cudaStream_t>(stream), &err)) return fail(err);
  return 0;
}

int lwdetr_forward(lwdetr_handle* h, const void* images, int images_fp32, int B, float* pred_logits, float* pred_boxes,
                   const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream) {
  if (!h || !images) return fail("lwdetr_forward: null pointer");
  const lwdetr_input input = {images, images_fp32 ? LWDETR_IN_F32_NCHW : LWDETR_IN_16_NCHW, nullptr, {0.f, 0.f, 0.f}, {1.f, 1.f, 1.f}};
  const int S = h->eng->config().img_size;
  return forward_input("lwdetr_forward", h, &input, B, S, S, pred_logits, pred_boxes, aux, topk_override, stream);
}

int lwdetr_forward_ex(lwdetr_handle* h, const lwdetr_input* input, int B, float* pred_logits, float* pred_boxes,
                      const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream) {
  if (!h) return fail("lwdetr_forward_ex: null pointer");
  const int S = h->eng->config().img_size;
  return forward_input("lwdetr_forward_ex", h, input, B, S, S, pred_logits, pred_boxes, aux, topk_override, stream);
}

int lwdetr_forward_hw(lwdetr_handle* h, const lwdetr_input* input, int B, int height, int width, float* pred_logits, float* pred_boxes,
                      const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream) {
  return forward_input("lwdetr_forward_hw", h, input, B, height, width, pred_logits, pred_boxes, aux, topk_override, stream);
}

}  // extern "C"

// the frame entry points of both source formats (lwdetr_frame, lwdetr_frame_nv12)
template <typename F>
static int forward_frames(const char* fn, lwdetr_handle* h, const F* frames, const float mean[3], const float std[3], int B, int height,
                          int width, float* pred_logits, float* pred_boxes, const lwdetr_aux_out* aux, const int32_t* topk_override,
                          void* stream) {
  if (!h || !frames || !mean || !std) return fail(std::string(fn) + ": null pointer");
  if (B <= 0) return fail(std::string(fn) + ": batch must be positive");
  lwb::ForwardIn in;
  if constexpr (std::is_same<F, lwdetr_frame_nv12>::value) { in.kind = lwb::IN_FRAMES_NV12; in.frames_nv12 = frames; }
  else { in.kind = lwb::IN_FRAMES; in.frames = frames; }
  for (int c = 0; c < 3; ++c) {
    in.mean[c] = mean[c]; in.stdv[c] = std[c];
    if (!(std[c] > 0.f)) return fail(std::string(fn) + ": std must be positive");
  }
  std::string err;
  if (lwb::frames_check(frames, B, height, width, &err)) return fail(std::string(fn) + ": " + err);
  if (h->eng->forward(in, B, height, width, pred_logits, pred_boxes, aux, topk_override, static_cast<cudaStream_t>(stream), &err)) return fail(err);
  return 0;
}

template <typename F>
static int resize_patches(const char* fn, int dtype, const F* frames, int B, int height, int width, const float mean[3], const float std[3],
                          void* A, uint8_t* mask, void* stream) {
  const std::string f(fn);
  if (!frames || !mean || !std || !A) return fail(f + ": null pointer");
  if (dtype != LWDETR_F16 && dtype != LWDETR_BF16) return fail(f + ": dtype must be LWDETR_F16 or LWDETR_BF16");
  if (B <= 0 || height < 64 || width < 64 || height % 64 || width % 64) return fail(f + ": batch must be positive, height and width multiples of 64");
  for (int c = 0; c < 3; ++c)
    if (!(std[c] > 0.f)) return fail(f + ": std must be positive");
  std::string err;
  if (lwb::frames_check(frames, B, height, width, &err)) return fail(f + ": " + err);
  int e = mask ? lwb::frame_mask_launch(frames, B, height, width, mask, static_cast<cudaStream_t>(stream)) : 0;
  if (!e) e = lwb::resize_patches_launch(dtype, frames, B, height, width, mean, std, A, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, (f + " launch").c_str());
  return 0;
}

// lwdetr_annotate and lwdetr_annotate_nv12
template <typename F>
static int annotate_call(const char* fn, lwdetr_annotator* a, const F* frames, int B, const int32_t* ids, const float* scores,
                         const int32_t* labels, const float* boxes, const int32_t* counts, int k, float score_threshold, lwdetr_zones* zones,
                         const int32_t* stream_ids, const int32_t* occupancy, void* stream) {
  const std::string f(fn);
  if (!a || !frames || !scores || !labels || !boxes || (zones && !stream_ids)) return fail(f + ": null pointer");
  if (B < 1 || B > lwb::ANN_FRAMES) return fail(f + ": B must be in [1, 1024]");
  if (k < 1 || k > lwb::ANN_K) return fail(f + ": k must be in [1, 1024]");
  if (score_threshold != score_threshold) return fail(f + ": score_threshold is NaN");
  if (occupancy && !zones) return fail(f + ": occupancy needs zones");
  if (zones && zones->state.device != a->state.device) return fail(f + ": the annotator and the zones object live on different devices");
  if (zones)
    for (int b = 0; b < B; ++b)
      if (stream_ids[b] < 0 || stream_ids[b] >= zones->table.num_streams)
        return fail(f + ": stream id " + std::to_string(stream_ids[b]) + " outside [0, " + std::to_string(zones->table.num_streams) + ")");
  const uintptr_t mis = reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(scores) | reinterpret_cast<uintptr_t>(labels) |
                        reinterpret_cast<uintptr_t>(boxes) | reinterpret_cast<uintptr_t>(counts) | reinterpret_cast<uintptr_t>(occupancy);
  if (mis % 4) return fail(f + ": ids, scores, labels, boxes, counts and occupancy must be 4-byte aligned");
  std::string err;
  if (lwb::crop_frames_check(frames, B, &err)) return fail(f + ": " + err);
  lwb::AnnCall c = {};
  c.ids = ids; c.scores = scores; c.labels = labels; c.boxes = boxes; c.counts = counts; c.k = k; c.threshold = score_threshold;
  c.zones = zones ? &zones->table : nullptr;
  c.streams = stream_ids;
  c.occupancy = occupancy;
  // the kernels read the zones object's geometry and counters, so its later set / export waits for this launch too
  return a->state.launch(f, stream, [&](cudaStream_t st) { return lwb::annotate_launch(a->table, a->options, frames, B, c, st); },
                         zones ? &zones->state : nullptr);
}

// lwdetr_crops and lwdetr_crops_nv12
template <typename F>
static int crops_call(const char* fn, const F* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                      int out_h, int out_w, int filter, int normalize, const float mean[3], const float std[3], int out_dtype, void* out,
                      int8_t* valid, void* stream) {
  const std::string f(fn);
  if (!frames || !boxes || !frame_index || !out || !valid || (normalize && (!mean || !std))) return fail(f + ": null pointer");
  if (B < 1 || B > lwb::kCropMaxFrames) return fail(f + ": B must be in [1, " + std::to_string(lwb::kCropMaxFrames) + "]");
  if (N < 1 || N > lwb::kCropMaxCount) return fail(f + ": N must be in [1, " + std::to_string(lwb::kCropMaxCount) + "]");
  if (out_h < lwb::kCropMinSide || out_w < lwb::kCropMinSide || out_h > lwb::kCropMaxSide || out_w > lwb::kCropMaxSide)
    return fail(f + ": output sides must be in [" + std::to_string(lwb::kCropMinSide) + ", " + std::to_string(lwb::kCropMaxSide) + "]");
  if (filter != LWDETR_CROP_BILINEAR && filter != LWDETR_CROP_ANTIALIAS) return fail(f + ": filter must be LWDETR_CROP_BILINEAR or LWDETR_CROP_ANTIALIAS");
  if (out_dtype != LWDETR_ET_F32 && out_dtype != LWDETR_ET_F16 && out_dtype != LWDETR_ET_BF16)
    return fail(f + ": out_dtype must be LWDETR_ET_F32, _F16 or _BF16");
  if (reinterpret_cast<uintptr_t>(out) % (out_dtype == LWDETR_ET_F32 ? 4 : 2) || reinterpret_cast<uintptr_t>(boxes) % 4 ||
      reinterpret_cast<uintptr_t>(frame_index) % 4 || reinterpret_cast<uintptr_t>(count) % 4)
    return fail(f + ": out, boxes, frame_index and count must be aligned to their element size");
  lwb::CropDesc d = {};
  d.out_h = out_h; d.out_w = out_w; d.filter = filter; d.normalize = normalize ? 1 : 0; d.etype = out_dtype;
  for (int c = 0; c < 3; ++c) {
    d.mean[c] = normalize ? mean[c] : 0.f;
    d.stdv[c] = normalize ? std[c] : 1.f;
    if (!(d.stdv[c] > 0.f)) return fail(f + ": std must be positive");
  }
  std::string err;
  if (lwb::crop_frames_check(frames, B, &err)) return fail(f + ": " + err);
  const int e = lwb::crops_launch(frames, B, boxes, frame_index, N, count, d, out, valid, static_cast<cudaStream_t>(stream));
  if (e == -2) return fail(f + ": the tap tables of these frame and output sizes exceed a CTA's shared memory");
  if (e) return cuda_fail(e, (f + " launch").c_str());
  return 0;
}

extern "C" {

int lwdetr_crops(const lwdetr_frame* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count, int out_h,
                 int out_w, int filter, int normalize, const float mean[3], const float std[3], int out_dtype, void* out, int8_t* valid,
                 void* stream) {
  return crops_call("lwdetr_crops", frames, B, boxes, frame_index, N, count, out_h, out_w, filter, normalize, mean, std, out_dtype, out,
                    valid, stream);
}

int lwdetr_crops_nv12(const lwdetr_frame_nv12* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                      int out_h, int out_w, int filter, int normalize, const float mean[3], const float std[3], int out_dtype, void* out,
                      int8_t* valid, void* stream) {
  return crops_call("lwdetr_crops_nv12", frames, B, boxes, frame_index, N, count, out_h, out_w, filter, normalize, mean, std, out_dtype,
                    out, valid, stream);
}

int lwdetr_crop_select(const float* scores, const float* boxes, int B, int k, const int32_t* frame_hw, float threshold, int32_t* frame_of,
                       int32_t* entry, float* sel_boxes, int32_t* count, void* stream) {
  if (!scores || !boxes || !frame_hw || !frame_of || !entry || !sel_boxes || !count) return fail("lwdetr_crop_select: null pointer");
  if (B < 1 || B > lwb::kCropMaxFrames || k < 1) return fail("lwdetr_crop_select: need B in [1, 1024] and k >= 1");
  if (threshold != threshold) return fail("lwdetr_crop_select: threshold is NaN");
  for (int b = 0; b < B; ++b)
    if (frame_hw[2 * b] < 1 || frame_hw[2 * b + 1] < 1) return fail("lwdetr_crop_select: frame " + std::to_string(b) + " has a side below 1");
  const int e = lwb::crop_select_launch(scores, boxes, B, k, frame_hw, threshold, frame_of, entry, sel_boxes, count,
                                        static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_crop_select launch");
  return 0;
}

int lwdetr_scatter_rows(int etype, const void* rows, int ld_rows, int D, const int32_t* entry, const int32_t* count, int N, void* out,
                        int num_out, void* stream) {
  if (!rows || !entry || !out) return fail("lwdetr_scatter_rows: null pointer");
  if (etype != LWDETR_ET_F32 && etype != LWDETR_ET_F16 && etype != LWDETR_ET_BF16) return fail("lwdetr_scatter_rows: etype must be LWDETR_ET_F32, _F16 or _BF16");
  if (D < 1 || N < 1 || num_out < 1 || ld_rows < D) return fail("lwdetr_scatter_rows: need D, N and num_out >= 1 and ld_rows >= D");
  const int es = etype == LWDETR_ET_F32 ? 4 : 2;
  if (reinterpret_cast<uintptr_t>(rows) % es || reinterpret_cast<uintptr_t>(out) % es) return fail("lwdetr_scatter_rows: rows and out must be aligned to their element size");
  const int e = lwb::scatter_rows_launch(etype, rows, ld_rows, D, entry, count, N, out, num_out, static_cast<cudaStream_t>(stream));
  if (e) return cuda_fail(e, "lwdetr_scatter_rows launch");
  return 0;
}

int lwdetr_annotate(lwdetr_annotator* a, const lwdetr_frame* frames, int B, const int32_t* ids, const float* scores, const int32_t* labels,
                    const float* boxes, const int32_t* counts, int k, float score_threshold, lwdetr_zones* zones, const int32_t* stream_ids,
                    const int32_t* occupancy, void* stream) {
  return annotate_call("lwdetr_annotate", a, frames, B, ids, scores, labels, boxes, counts, k, score_threshold, zones, stream_ids, occupancy,
                       stream);
}

int lwdetr_annotate_nv12(lwdetr_annotator* a, const lwdetr_frame_nv12* frames, int B, const int32_t* ids, const float* scores,
                         const int32_t* labels, const float* boxes, const int32_t* counts, int k, float score_threshold, lwdetr_zones* zones,
                         const int32_t* stream_ids, const int32_t* occupancy, void* stream) {
  return annotate_call("lwdetr_annotate_nv12", a, frames, B, ids, scores, labels, boxes, counts, k, score_threshold, zones, stream_ids,
                       occupancy, stream);
}

int lwdetr_forward_frames(lwdetr_handle* h, const lwdetr_frame* frames, const float mean[3], const float std[3], int B, int height,
                          int width, float* pred_logits, float* pred_boxes, const lwdetr_aux_out* aux, const int32_t* topk_override,
                          void* stream) {
  return forward_frames("lwdetr_forward_frames", h, frames, mean, std, B, height, width, pred_logits, pred_boxes, aux, topk_override, stream);
}

int lwdetr_forward_frames_nv12(lwdetr_handle* h, const lwdetr_frame_nv12* frames, const float mean[3], const float std[3], int B, int height,
                               int width, float* pred_logits, float* pred_boxes, const lwdetr_aux_out* aux, const int32_t* topk_override,
                               void* stream) {
  return forward_frames("lwdetr_forward_frames_nv12", h, frames, mean, std, B, height, width, pred_logits, pred_boxes, aux, topk_override,
                        stream);
}

int lwdetr_resize_patches(int dtype, const lwdetr_frame* frames, int B, int height, int width, const float mean[3], const float std[3],
                          void* A, uint8_t* mask, void* stream) {
  return resize_patches("lwdetr_resize_patches", dtype, frames, B, height, width, mean, std, A, mask, stream);
}

int lwdetr_resize_patches_nv12(int dtype, const lwdetr_frame_nv12* frames, int B, int height, int width, const float mean[3],
                               const float std[3], void* A, uint8_t* mask, void* stream) {
  return resize_patches("lwdetr_resize_patches_nv12", dtype, frames, B, height, width, mean, std, A, mask, stream);
}

// One ncclBroadcast of the packed weight arena (SURVEY.md 8b / 8e).  NCCL is not linked: the symbol is taken from the
// libnccl the host process already loaded (torch's bundled libnccl.so.2) or dlopen'ed by soname.
int lwdetr_broadcast_weights(lwdetr_handle* h, void* nccl_comm, int root, void* stream) {
  if (!h || !nccl_comm) return fail("lwdetr_broadcast_weights: null pointer");
  if (!h->eng->weights_loaded()) return fail("lwdetr_broadcast_weights: call lwdetr_load_weights on every rank first (it fixes the arena layout)");
  typedef int (*PFN_bcast)(const void*, void*, size_t, int, int, void*, cudaStream_t);
  static PFN_bcast fn = nullptr;
  if (!fn) {
    void* sym = dlsym(RTLD_DEFAULT, "ncclBroadcast");
    if (!sym) {
      void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
      if (lib) sym = dlsym(lib, "ncclBroadcast");
    }
    if (!sym) return fail("lwdetr_broadcast_weights: ncclBroadcast not found (load libnccl.so.2 into the process first)");
    fn = reinterpret_cast<PFN_bcast>(sym);
  }
  int prev = 0;
  cudaGetDevice(&prev);
  cudaSetDevice(h->eng->device());
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // layout check: every rank must hold an arena of the root's size (same config, dtype and library version)
  unsigned long long* dsz = nullptr;
  unsigned long long mine = h->eng->arena_used(), roots = 0;
  int rc = 0;
  if (cudaMalloc(&dsz, 8) != cudaSuccess) rc = -1;
  if (!rc && cudaMemcpyAsync(dsz, &mine, 8, cudaMemcpyHostToDevice, st) != cudaSuccess) rc = -1;
  if (!rc && fn(dsz, dsz, 8, /*ncclChar*/ 0, root, nccl_comm, st) != 0) rc = -2;
  if (!rc && cudaMemcpyAsync(&roots, dsz, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) rc = -1;
  if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = -1;
  if (dsz) cudaFree(dsz);
  if (!rc && roots != mine) rc = -3;
  if (!rc && fn(h->eng->arena_ptr(), h->eng->arena_ptr(), h->eng->arena_used(), 0, root, nccl_comm, st) != 0) rc = -2;
  cudaSetDevice(prev);
  if (rc == -1) return fail(std::string("lwdetr_broadcast_weights: CUDA error: ") + cudaGetErrorString(cudaGetLastError()));
  if (rc == -2) return fail("lwdetr_broadcast_weights: ncclBroadcast failed");
  if (rc == -3) return fail("lwdetr_broadcast_weights: arena size differs from the root's (" + std::to_string(mine) + " vs " + std::to_string(roots) + " bytes): config / dtype mismatch between ranks");
  return 0;
}

int64_t lwdetr_weight_arena_bytes(lwdetr_handle* h) { return h ? static_cast<int64_t>(h->eng->arena_used()) : -1; }

int lwdetr_set_option(lwdetr_handle* h, const char* name, int value) {
  if (!h || !name) return fail("lwdetr_set_option: null pointer");
  if (h->eng->set_option(name, value)) return fail(std::string("lwdetr_set_option: unknown option ") + name);
  return 0;
}

int lwdetr_add_capture(lwdetr_handle* h, const char* label, float* dst, int64_t capacity) {
  if (!h || !label || !dst) return fail("lwdetr_add_capture: null pointer");
  h->eng->add_capture(label, dst, capacity);
  return 0;
}
int64_t lwdetr_capture_result(lwdetr_handle* h, int index) { return h ? h->eng->capture_written(index) : -1; }
void lwdetr_clear_captures(lwdetr_handle* h) { if (h) h->eng->clear_captures(); }

int lwdetr_num_ops(lwdetr_handle* h) { return h ? h->eng->num_ops() : 0; }
const char* lwdetr_op_label(lwdetr_handle* h, int i) {
  if (!h || i < 0 || i >= h->eng->num_ops()) return "";
  return h->eng->op(i).label.c_str();
}
int lwdetr_op_cost(lwdetr_handle* h, int i, double* flops, double* bytes) {
  if (!h || i < 0 || i >= h->eng->num_ops()) return fail("lwdetr_op_cost: bad index");
  if (flops) *flops = h->eng->op(i).flops;
  if (bytes) *bytes = h->eng->op(i).bytes;
  return 0;
}
int lwdetr_last_hidden(lwdetr_handle* h, void* dst, int ld_dst, void* stream) {
  if (!h || !dst) return fail("lwdetr_last_hidden: null pointer");
  std::string err;
  if (h->eng->last_hidden(dst, ld_dst, static_cast<cudaStream_t>(stream), &err)) return fail(err);
  return 0;
}

int lwdetr_profile_ops(lwdetr_handle* h, int iters, float* ms_per_op, void* stream) {
  if (!h || !ms_per_op || iters < 1) return fail("lwdetr_profile_ops: bad arguments");
  std::vector<float> ms;
  std::string err;
  if (h->eng->profile_ops(iters, &ms, static_cast<cudaStream_t>(stream), &err)) return fail(err);
  for (size_t i = 0; i < ms.size(); ++i) ms_per_op[i] = ms[i];
  return 0;
}

}  // extern "C"
