// Memory-bound helper kernels (see rowops.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "gemm_tc.h"

namespace lwb {

struct LayerNormArgs {
  const void* x; int ldx;
  void* y; int ldy;
  const float* w; const float* b;
  float eps;
  long long rows; int C;
  const uint8_t* row_flag; int flag_mod; const float* override_vec;   // optional masked-row override
  const void* add_src; int ld_add; void* y2; int ldy2;                // optional y2 = y + add_src
  long long y_group, y_group_stride, y_row_off;   // y_group > 0: y row = (r / y_group) * y_group_stride + y_row_off + r % y_group
  // optional chained second LayerNorm of the ROUNDED y (decoder: hs = dec_norm(tgt), transformer.py:279-285): y3 = LN(y; w3, b3, eps3)
  const float* w3; const float* b3; float eps3; void* y3; int ldy3;
};
int layernorm_launch(int dtype, const LayerNormArgs& a, cudaStream_t st);
// rows each warp of layernorm_launch's kernel takes for this size (1 or 4)
int layernorm_rows_per_warp(long long rows, int C);
// the e4m3 mode's LayerNorm (rowops.cu layernorm_e4m3_kernel): fp16 rows [rows, C] -> e4m3 codes [rows, ldq] + fp32
// row_scale [rows]; C % 8 == 0, C <= 1024, ldx / ldq multiples of 8.  -2: bad sizes
int layernorm_e4m3_launch(const void* x, int ldx, long long rows, int C, float eps, uint8_t* q, int ldq, float* row_scale, cudaStream_t st);

// image [B,3,H,W] -> window-major patch matrix [B*(H/16)*(W/16), 768]; H, W multiples of 64
int patch_gather_launch(int dtype, const void* img, int img_is_fp32, void* A, int B, int H, int W, cudaStream_t st);
// uint8 HWC [B,H,W,3] with fused (x/255 - mean) / std
int patch_gather_u8_launch(int dtype, const void* img, const float* mean, const float* stdv, void* A, int B, int H, int W, cudaStream_t st);
// padding-mask tables of a (possibly) padded batch; mask == nullptr: no padding
int mask_setup_launch(const uint8_t* mask, int B, int Himg, int Wimg, int L, int S, const int* lvl_h, const int* lvl_w, const int* lvl_start,
                      float* proposals, uint8_t* invalid, uint8_t* pad, float* valid_ratio, cudaStream_t st);
// window-major rows of a GH x GW token grid -> row-major (b, y, x); GH, GW multiples of 4
int unwindow_launch(int dtype, const void* src, int lds, void* dst, int ldd, long long rows, int C, int GH, int GW, cudaStream_t st);
int add_rows_launch(int dtype, const void* a, int lda, long long amod, const void* b, int ldb, void* out, int ldo,
                    long long rows, int C, cudaStream_t st);
int rowmax_launch(const float* x, int ld, int n, float* out, long long rows, cudaStream_t st);
// per-image top-k indices, descending, ties to the lower index: shared-memory bitonic sort up to S = 16384, radix select
// streaming the row from global memory above (then k <= 4096)
int topk_launch(const float* score, int B, int S, int k, int* idx_out, cudaStream_t st);
// work: B * ceil(nq*ncls / 16384) * k ints
int postprocess_launch(const float* logits, const float* boxes, const float* target_sizes, int B, int nq, int ncls, int k,
                       int* work, float* scores, int* labels, float* out_boxes, cudaStream_t st);
int gather_topk_launch(int dtype, const void* feat, int ldf, const float* logits, int ldl, int ncls, const int* idx, int B, int S,
                       int k, int d, void* sel, float* enc_logits, cudaStream_t st);
int query_init_launch(int dtype, const float* delta_ts, const float* proposals, const int* idx, const float* refpoint_embed, int B,
                      int k, int d, float* box_ts, float* refpoint, void* sine, int S, int L, const float* valid_ratio, cudaStream_t st);
int final_boxes_launch(const float* delta, const float* refpoint, long long rows_per_layer, int layers, float* boxes, cudaStream_t st);

}  // namespace lwb
