// LW-DETR forward engine: weight packing (folding, layout changes, 16-bit conversion) and the fixed
// kernel schedule for one (batch size, input height, input width).  Host-only interface; see engine.cpp.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "lwdetr_b200.h"

namespace lwb {

struct HostTensor {
  const float* data;
  long long numel;
};

struct Capture {
  std::string label;
  float* dst;
  long long capacity;   // in floats
  long long written;    // rows*cols actually written (or -1 if label not found)
};

// Element kinds of a captured view; do_capture converts each to fp32 on the host (exact for uint8 and for int32 below 2^24).
enum : int { EL_16 = 0, EL_F32 = 1, EL_I32 = 2, EL_U8 = 3 };
// What a debug capture of an op copies back: rows x cols of a [*, ld] matrix of `kind` elements (EL_16: the compute dtype).
struct OutView {
  const void* p = nullptr;
  long long rows = 0;
  int cols = 0, ld = 0, kind = EL_16;
};

struct Op {
  std::string label;
  std::function<int(cudaStream_t)> run;
  // outputs for debug captures: the primary one under `label`, any further ones under "<label>.<name>"
  OutView out;
  std::vector<std::pair<std::string, OutView>> extra;
  double flops = 0, bytes = 0;
  bool reads_input = false;   // consumes caller-owned pointers (images, mask): launched eagerly, never captured in the graph
};

// One forward's input: the image batch in one of three encodings plus the optional NestedTensor padding mask.
enum : int { IN_F32_NCHW = 0, IN_16_NCHW = 1, IN_U8_NHWC = 2, IN_FRAMES = 3, IN_FRAMES_NV12 = 4 };
struct ForwardIn {
  const void* images = nullptr;   // DEVICE [B,3,H,W] fp32 / compute dtype, or [B,H,W,3] uint8
  const lwdetr_frame* frames = nullptr;   // IN_FRAMES: HOST array of B checked descriptors (resize.h); mean / stdv apply
  const lwdetr_frame_nv12* frames_nv12 = nullptr;   // IN_FRAMES_NV12: the same for NV12 frames
  int kind = IN_F32_NCHW;
  const uint8_t* mask = nullptr;  // DEVICE bool [B,H,W] (True = padded pixel) or null
  float mean[3] = {0.f, 0.f, 0.f}, stdv[3] = {1.f, 1.f, 1.f};   // IN_U8_NHWC: (x/255 - mean) / std
};

// Switches to a device for the duration of a call (the caller's current device is restored afterwards).
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev); else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// The kernel schedule of one (batch size, height, width): its ops, their CUDA graphs and the result buffers the ops write
// (in the engine's workspace arena).  Destroying a plan destroys its graphs.
struct Plan {
  int B = 0, H = 0, W = 0;
  std::vector<Op> ops;
  // CUDA graphs: the two ops that read caller-owned memory (mask tables, patch gather) are launched eagerly on the caller's
  // stream; everything behind them only touches engine-owned buffers and is ONE executable graph per plan - whatever
  // tensor, input encoding or mask the caller passes.  (The test-only top-k override pointer is the one caller pointer left
  // inside, hence the key.)  Captured on an internal stream: the caller's stream may be the legacy default stream, which
  // cannot be captured.
  std::map<const int32_t*, cudaGraphExec_t> graphs;
  int eager_runs = 0;
  // result buffers
  float* logits = nullptr;       // [layers, B, nq, ldc]
  int ldc = 96;                  // row pitch of the class-logit buffers: num_classes rounded up to 32
  float* boxes = nullptr;        // [layers, B, nq, 4]
  float* enc_logits = nullptr;   // [B, nq, ncls]
  float* enc_boxes = nullptr;    // [B, nq, 4]
  int* topk_idx = nullptr;       // [B, nq]
  const void* hidden = nullptr;  // [layers, B, nq, hidden_dim] decoder output (after its norm), compute dtype

  Plan() = default;
  Plan(const Plan&) = delete;
  Plan& operator=(const Plan&) = delete;
  ~Plan() { clear_graphs(); }
  void clear_graphs() {
    for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
    graphs.clear();
  }
};

class Engine {
 public:
  // supported input sides (pixels, multiples of 64: 4x4 windows of 16-pixel patches)
  static constexpr int kMinSide = 128, kMaxSide = 1344;
  Engine(const lwdetr_config& cfg, int dtype);
  ~Engine();
  int load_weights(const std::map<std::string, HostTensor>& w, std::string* err);
  // input [B, 3, H, W] (or [B, H, W, 3] uint8); a (B, H, W) other than the last one re-plans and drops the graphs
  int forward(const ForwardIn& in, int B, int H, int W, float* pred_logits, float* pred_boxes,
              const lwdetr_aux_out* aux, const int32_t* topk_override, cudaStream_t st, std::string* err);
  void add_capture(const char* label, float* dst, long long cap) { captures_.push_back({label, dst, cap, -1}); }
  void clear_captures() { captures_.clear(); }
  long long capture_written(int i) const { return i < (int)captures_.size() ? captures_[i].written : -1; }
  int set_option(const char* name, int value);
  // packed weight arena (device): base pointer and bytes in use - identical layout on every rank with the same config / dtype
  void* arena_ptr() const { return warena_.p; }
  size_t arena_used() const { return woff_; }
  bool weights_loaded() const { return weights_loaded_; }
  int device() const { return device_; }
  int num_ops() const { return plan_ ? static_cast<int>(plan_->ops.size()) : 0; }
  const Op& op(int i) const { return plan_->ops[i]; }
  const lwdetr_config& config() const { return cfg_; }
  // per-op timing of the last planned batch (CUDA events, `iters` runs per op); returns ms per op
  int profile_ops(int iters, std::vector<float>* ms, cudaStream_t st, std::string* err);
  // the last forward's final-layer decoder hidden state [B * nq, hidden_dim] into dst (row stride ld elements), on st
  int last_hidden(void* dst, int ld, cudaStream_t st, std::string* err);

 private:
  struct DevBuf { void* p = nullptr; size_t bytes = 0; };
  int plan(int B, int H, int W, std::string* err);
  void* walloc(size_t bytes);      // weight arena (bump)
  std::vector<uint16_t> to16(const std::vector<float>& v) const;   // round to the compute dtype
  void* upload16(const std::vector<float>& v);
  float* upload32(const std::vector<float>& v);
  void* upload8(const std::vector<uint8_t>& v);
  int do_capture(const Op& op, cudaStream_t st);
  int copy_view(const OutView& v, Capture* c);

  lwdetr_config cfg_;
  int dtype_;
  bool e4m3_ = false;   // LWDETR_F16_E4M3: dtype_ is DT_F16; the encoder's LN->qkv and LN->fc1 run in e4m3
  int device_ = 0;    // CUDA device the engine was created on; every entry point switches to it (one handle per device)
  bool weights_loaded_ = false;
  int use_graph_ = 0;
  int fuse_ln_ = 1;   // ViT LayerNorms folded into the consuming GEMM's epilogue (option "fuse_layernorm"; no effect on the
                      // encoder in the e4m3 mode)
  std::unique_ptr<Plan> plan_;   // the current schedule, or none (dropped whenever what it was built from changes)
  cudaStream_t gstream_ = nullptr;   // graph capture and launch
  cudaEvent_t ev_in_ = nullptr, ev_out_ = nullptr;
  std::vector<Capture> captures_;
  // arenas: packed weights (bump), and the workspace every plan lays out from its base (grow-only)
  DevBuf warena_, sarena_;
  size_t woff_ = 0;
  // packed weights (device pointers), keyed by short names
  std::map<std::string, void*> W_;
  std::map<std::string, float*> F_;
  // live I/O pointers patched into the schedule at forward() time
  ForwardIn in_;
  std::vector<lwdetr_frame> frames_;   // the engine's copy of an IN_FRAMES batch's descriptors (in_.frames points here)
  std::vector<lwdetr_frame_nv12> frames_nv12_;   // the same for IN_FRAMES_NV12 (in_.frames_nv12 points here)
  bool frames_padded_ = false;         // some frame leaves part of the canvas unfilled: mask_setup takes the device-made mask
  const int32_t* in_topk_override_ = nullptr;
};

// host helpers exposed for CPU tests
void bicubic_resize_chlast(const float* src, int n_in, int C, int n_out, float* dst);   // [n_in,n_in,C] -> [n_out,n_out,C]
void bicubic_resize_chlast_hw(const float* src, int n_in, int C, int out_h, int out_w, float* dst);   // [n_in,n_in,C] -> [out_h,out_w,C]
// per row: scale = max|x| / 448 (0 -> 1), q = e4m3(x * 448 / max) round to nearest even, saturating (the e4m3 weight packing)
void host_quant_e4m3_rows(const float* src, long long rows, int K, uint8_t* q, float* scale);

}  // namespace lwb
