// wgmma + TMA GEMM family used for every linear / convolution of the LW-DETR forward.
//   out[row_map(m), n] = epilogue( sum_k A[m, k] * W[n, k] )
// A is gathered by TMA either from a plain row-major matrix, or implicitly (im2col-free) from an
// NHWC feature map for 3x3 convolutions (stride 1 and 2).  W is always [N, K] row-major, i.e. the
// nn.Linear / reordered conv weight layout, so both operands are K-major for the tensor core.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <string>

namespace lwb {

enum : int { DT_F16 = 0, DT_BF16 = 1, DT_E4M3 = 2 };   // DT_E4M3: 1-byte e4m3 operands (gemm_e4m3_build), fp16 out
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SILU = 3 };
enum : int { AMODE_PLAIN = 0, AMODE_CONV3_S1 = 1, AMODE_CONV3_S2 = 2 };
enum : int { ROWS_PLAIN = 0, ROWS_WINDOW_MAJOR = 1 };

// Device-visible arguments (passed by value to the kernel).
struct GemmArgs {
  int M, N, kblocks;        // valid rows / valid output columns / K in units of 64
  int n_tiles, m_tiles, stages;
  int a_mode;
  uint32_t a_stage_tx;      // bytes TMA delivers into the A slot per stage
  // conv geometry (output grid OH x OW per image, tile TW x TH pixels, Cin/64 channel blocks)
  int OH, OW, TW, TH, tiles_x, tiles_y, cin_blocks, lda;
  // epilogue
  const float* bias;        // [N] fp32 or null
  const float* gamma;       // [N] fp32 or null (layer-scale applied before the residual add)
  const void* resid;        // 16-bit [*, ld_resid] or null
  int ld_resid, resid_mod;  // residual row = m % resid_mod when resid_mod > 0
  int act;
  void* out;
  int ld_out, out_fp32;
  int rows_in;              // how input rows m are ordered: plain (b,y,x) or window-major (b,win,t)
  int remap_rows;           // 1: write rows in spatial (b,y,x) order (needs rows_in grid IH x IW)
  int shuffle_cout;         // >0: ConvTranspose2d(k=2,s=2) pixel shuffle, n = (dy*2+dx)*cout + co
  int IH, IW;               // token grid per image for rows_in / shuffle (40 x 40 for the ViT)
  // head-major store (the deformable-attention value tensor, msda.cu): hm_S > 0 writes element (row b*hm_S + s,
  // column slice*hm_heads*16 + head*16 + c) to out[(((b*hm_slices + slice)*hm_heads + head)*hm_S + s)*16 + c]
  int hm_S, hm_heads, hm_slices;
  const uint8_t* row_zero;  // [M] or null: rows flagged non-zero are stored as zeros (padded memory tokens, ms_deform_attn.py:114-115)
  // LayerNorm fusion (ViT blocks).  Producer side: the epilogue also emits per-row partial (sum, sum of
  // squares) of the rounded output, one float2 per (row, n_tile, column half).  Consumer side: the GEMM runs
  // on the RAW rows and applies  out = rstd*(acc - mean*colsum[n]) + bias[n]  where the LN weight is folded into
  // W, colsum[n] = sum_k W'[n,k] and bias already contains sum_k ln_b[k]*W[n,k].
  float2* stats_out;        // [M, stats_parts_out] or null
  int stats_parts_out;
  const float2* stats_in;   // [M, stats_parts_in] or null
  int stats_parts_in;
  const float* colsum;      // [N] fp32 (consumer)
  float ln_inv_c, ln_eps;   // 1/C of the normalised dimension, epsilon
  // e4m3 GEMM only: out = a_scale[m] * w_scale[n] * acc + bias[n]
  const float* a_scale;     // [M] fp32
  const float* w_scale;     // [N] fp32
};

// Host description of one GEMM.
struct GemmDesc {
  int dtype = DT_F16;
  int a_mode = AMODE_PLAIN;
  const void* A = nullptr;  // plain: [M, lda]; conv: NHWC [B, IH_in, IW_in, lda] (channel slice base)
  int lda = 0;
  int M = 0, N = 0, K = 0;  // conv: M = B*OH*OW, K = 9*Cin
  int B = 0, OH = 0, OW = 0;  // conv output grid
  const void* W = nullptr;  // [N, K]
  const float* bias = nullptr;
  const float* gamma = nullptr;
  const void* resid = nullptr;
  int ld_resid = 0, resid_mod = 0;
  int act = ACT_NONE;
  void* out = nullptr;
  int ld_out = 0;
  int out_fp32 = 0;
  int rows_in = ROWS_PLAIN, remap_rows = 0, shuffle_cout = 0, IH = 0, IW = 0;
  int hm_S = 0, hm_heads = 0, hm_slices = 0;   // head-major store (see GemmArgs)
  const uint8_t* row_zero = nullptr;
  float2* stats_out = nullptr;          // producer: buffer with room for M * 2 * n_tiles float2
  const float2* stats_in = nullptr;     // consumer
  int stats_parts_in = 0;
  const float* colsum = nullptr;
  int ln_C = 0;
  float ln_eps = 0.f;
};

struct GemmOp {
  CUtensorMap ta, tb;
  GemmArgs args;
  int dtype, bn;
  unsigned grid;
  size_t smem;
  double flops;
};

// Epilogue specialisations of gemm_tc_kernel (gemm_tc.cu): EP_GENERIC keeps every feature behind runtime flags, the others
// compile in only what the hot GEMMs use (bias; bias + activation; LayerNorm fold (+ GELU); residual / layer-scale / statistics).
enum : int { EP_GENERIC = 0, EP_BIAS = 1, EP_BIAS_ACT = 2, EP_LN = 3, EP_LN_GELU = 4, EP_RESID = 5 };

// Output tile of the implicit-GEMM 3x3 convolution over an OH x OW grid (OH, OW >= 1): TW x TH pixels, TW * TH <= 128, the
// pair that maximises the share of useful A rows.  Host only; gemm_build uses it for both strides.
void conv_tile_plan(int OH, int OW, int* tw, int* th);

// Returns 0 on success; on failure fills *err.
int gemm_build(const GemmDesc& d, GemmOp* op, std::string* err);
int gemm_launch(const GemmOp& op, cudaStream_t stream);
// The EP_* specialisation gemm_launch runs for a built 16-bit op (-1 for an e4m3 op).
int gemm_epilogue(const GemmOp& op);

// FP8 GEMM (gemm_e4m3_kernel): out[m, n] = act(a_scale[m] * w_scale[n] * sum_k A[m, k] W[n, k] + bias[n]) in fp16, A [M, lda]
// and W [N, K] e4m3 codes (both K-major), fp32 accumulation on the tensor cores.  act: ACT_NONE or ACT_GELU (the fc1
// epilogue's GELU).  K % 64 == 0; the last 128-wide k-block may be half empty (TMA fills it with zeros).
struct GemmE4m3Desc {
  const void* A = nullptr;
  int lda = 0;                          // bytes (= elements), multiple of 16
  const float* a_scale = nullptr;       // [M]
  int M = 0, N = 0, K = 0;
  const void* W = nullptr;              // [N, K]
  const float* w_scale = nullptr;       // [N]
  const float* bias = nullptr;          // [N] or null
  int act = ACT_NONE;
  void* out = nullptr;                  // fp16 [M, ld_out]
  int ld_out = 0;
};
// Fills *op for gemm_launch (op->dtype = DT_E4M3).
int gemm_e4m3_build(const GemmE4m3Desc& d, GemmOp* op, std::string* err);

// Fused ViT MLP of the 192-wide encoder (mlp.cu vit_mlp_kernel), the LayerNorm-fused fc1 GEMM and the fc2 GEMM in one kernel:
//   h = T(gelu(rstd * (x W1'^T) - rstd * mean * colsum1 + b1))        [M, 768], never stored
//   out = x + gamma * (h W2^T + b2)                                     [M, 192] in the compute dtype T
// x: the raw residual rows [M, ldx]; (mean, rstd) combined from the row partials stats_in (as the LN-fused GEMMs do); W1' the
// fc1 weight [768, 192] with the LayerNorm affine folded in, colsum1 its row sums, b1 its folded bias; W2 the fc2 weight
// [192, 768].  stats_out (optional) receives the LayerNorm partials of the rounded output rows, stats_parts_out = 2 or 6
// per row, laid out as the fc2 GEMM at BN = 192 or 64 writes them.  The result equals gemm_tc fc1 -> fc2 bit for bit.
static constexpr int MLP_C = 192;
struct MlpArgs {
  int M, m_tiles;
  const void* x;
  int ldx;
  const float2* stats_in;
  int stats_parts_in;
  float ln_inv_c, ln_eps;
  const float* b1;          // [768]
  const float* colsum1;     // [768]
  const float* b2;          // [192] or null
  const float* gamma;       // [192] or null
  void* out;
  int ld_out;
  float2* stats_out;        // [M, stats_parts_out] or null
  int stats_parts_out;
};
struct MlpDesc {
  int dtype = DT_F16;
  const void* x = nullptr;
  int ldx = 0, M = 0;
  const float2* stats_in = nullptr;
  int stats_parts_in = 0;
  float ln_eps = 0.f;
  const void* w1 = nullptr;
  const float* colsum1 = nullptr;
  const float* b1 = nullptr;
  const void* w2 = nullptr;
  const float* b2 = nullptr;
  const float* gamma = nullptr;
  void* out = nullptr;
  int ld_out = 0;
  float2* stats_out = nullptr;
  int stats_parts_out = 2;
};
struct MlpOp {
  CUtensorMap tx, tw1, tw2;
  MlpArgs args;
  int dtype;
  unsigned grid;
  size_t smem;
  double flops;
};
int vit_mlp_build(const MlpDesc& d, MlpOp* op, std::string* err);
int vit_mlp_launch(const MlpOp& op, cudaStream_t stream);

}  // namespace lwb
