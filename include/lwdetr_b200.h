/*
 * lwdetr_b200 - C ABI of the CUDA-native (sm_90a) LW-DETR inference path.
 *
 * Every entry point takes plain pointers and sizes (no torch types).  Device pointers are CUDA
 * device addresses on the current device; `stream` is a cudaStream_t passed as void* (NULL = the
 * legacy default stream).  All calls are stream-ordered and asynchronous unless stated otherwise.
 * Return value: 0 on success, non-zero on failure with a message in lwdetr_last_error()
 * (thread-local).  Nothing throws across this boundary.
 *
 * The reference interface each group replaces is cited as file:line relative to the
 * Atten4Vis/LW-DETR tree.
 */
#ifndef LWDETR_B200_H_
#define LWDETR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LWDETR_API __attribute__((visibility("default")))

/* Compute modes of lwdetr_create.  LWDETR_F16_E4M3 is LWDETR_F16 with the ViT encoder's qkv and fc1 GEMMs on the FP8
 * tensor cores (e4m3 x e4m3 -> fp32), with dynamic per-token and static per-channel scales.  Per block, for the fp16
 * residual row x, the LayerNorm (w, b, eps 1e-6) and the linear (W [N, C], bias beta; qkv: beta = [q_bias, 0, v_bias]):
 *   activations, per row m: x^ = (x - mean) * rstd in fp32 (affine not applied), a_m = max_k |x^_mk|,
 *     s_a[m] = a_m / 448, q_a = e4m3(x^ * 448 / a_m) (round to nearest even, saturating; a_m = 0: both factors 1);
 *   weights, per output channel n, packed once by lwdetr_load_weights: W' = W diag(w), s_w[n] = max_k |W'_nk| / 448
 *     (0 -> 1), q_w = e4m3(W'_nk * 448 / max_k |W'_nk|), beta'[n] = beta[n] + sum_k b_k W_nk;
 *   y = s_a[m] * s_w[n] * sum_k q_a q_w + beta'[n] (fp32 accumulation on the tensor cores, which keep fewer than 32 bits
 *     of the running sum): qkv stores y, fc1 stores gelu(y), both fp16.
 * Everything else (attention, proj, fc2, the projector, the decoder, every input path) is LWDETR_F16.  The option
 * "fuse_layernorm" has no effect on the encoder in this mode. */
enum { LWDETR_F16 = 0, LWDETR_BF16 = 1, LWDETR_F16_E4M3 = 2 };
enum { LWDETR_ACT_NONE = 0, LWDETR_ACT_RELU = 1, LWDETR_ACT_GELU = 2, LWDETR_ACT_SILU = 3 };

LWDETR_API const char* lwdetr_last_error(void);
LWDETR_API int lwdetr_abi_version(void);

/* ------------------------------------------------------------------------------------------------
 * Kernel-level entry points (unit tests, ncu captures).  They are the same kernels the model-level
 * forward schedules.
 * ---------------------------------------------------------------------------------------------- */

/* out[rowmap(m), n] = resid[m', n] + gamma[n] * act(sum_k A[m,k] W[n,k] + bias[n])
 * wgmma/TMA GEMM standing in for F.linear / 1x1 conv / ConvTranspose2d(k2,s2)
 * (models/backbone/vit.py:120-140,206-220; projector.py:85-98,165-190; transformer.py:27-39).
 *   A [M, lda] 16-bit, W [N, K] 16-bit, K % 64 == 0, bias/gamma fp32 [N] or NULL,
 *   resid 16-bit [*, ld_resid] or NULL (row m % resid_mod when resid_mod > 0),
 *   out 16-bit (out_fp32 = 0) or fp32 [*, ld_out].
 *   rows_in = 1: rows are window-major tokens (b, win 4x4, t) of an IH x IW grid (vit.py:353-358);
 *   remap_rows = 1: write rows in spatial (b, y, x) order (the un-windowing of vit.py:362-364);
 *   shuffle_cout > 0: N == 4*cout, column (dy*2+dx)*cout+co goes to pixel (2y+dy, 2x+dx), channel co. */
LWDETR_API int lwdetr_gemm(int dtype, const void* A, int lda, int M, int K, const void* W, int N,
                           const float* bias, const float* gamma, const void* resid, int ld_resid, int resid_mod,
                           int act, void* out, int ld_out, int out_fp32, int rows_in, int remap_rows,
                           int shuffle_cout, int IH, int IW, void* stream);

/* lwdetr_gemm with every epilogue feature the model schedules (same kernels, same plan as the forward builds).  dtype
 * LWDETR_F16 or LWDETR_BF16 (the e4m3 GEMM is lwdetr_gemm_e4m3).  Beyond the lwdetr_gemm arguments:
 *   LayerNorm consumer (stats_in != NULL): A holds the RAW rows [M, K = ln_C]; stats_in fp32 pairs [M, stats_parts_in] are each
 *     row's partials (sum, M2) over equal slices of its ln_C columns (ln_C % stats_parts_in == 0); colsum fp32 [N];
 *     out = act(rstd * (acc - mean * colsum[n]) + bias[n]) with mean / rstd = 1 / sqrt(var + ln_eps) combined from the
 *     partials (W and bias carry the folded LayerNorm affine);
 *   statistics producer (stats_out != NULL): also writes fp32 pairs [M, stats_parts_out], the partials (sum, M2) of each
 *     ROUNDED output row, one per (n-tile, column half); N must be a multiple of the tile width bn;
 *   head-major store (hm_S > 0): element (b*hm_S + s, (slice*hm_heads + head)*16 + c) goes to
 *     out[(((b*hm_slices + slice)*hm_heads + head)*hm_S + s)*16 + c]; N == hm_slices*hm_heads*16, M % hm_S == 0, ld_out unused;
 *   row_zero uint8 [M] or NULL: rows flagged non-zero are stored as zeros (forces the generic epilogue).
 * Reported by the call (also with dry_run != 0, which builds the plan and launches nothing): bn, the n-tile width; epilogue,
 * the LWDETR_EP_* specialisation that runs; stats_parts_out = 2 * ceil(N / bn). */
enum { LWDETR_EP_GENERIC = 0, LWDETR_EP_BIAS = 1, LWDETR_EP_BIAS_ACT = 2, LWDETR_EP_LN = 3, LWDETR_EP_LN_GELU = 4, LWDETR_EP_RESID = 5 };
typedef struct {
  int32_t dtype;
  const void* A; int32_t lda, M, K;
  const void* W; int32_t N;
  const float* bias; const float* gamma;
  const void* resid; int32_t ld_resid, resid_mod;
  int32_t act;
  void* out; int32_t ld_out, out_fp32;
  int32_t rows_in, remap_rows, shuffle_cout, IH, IW;
  const float* stats_in; int32_t stats_parts_in;
  const float* colsum; int32_t ln_C; float ln_eps;
  float* stats_out;
  int32_t hm_S, hm_heads, hm_slices;
  const uint8_t* row_zero;
  int32_t dry_run;
  int32_t bn, epilogue, stats_parts_out;   /* out */
} lwdetr_gemm_args;
LWDETR_API int lwdetr_gemm_ex(lwdetr_gemm_args* args, void* stream);

/* 3x3 convolution, padding 1, stride 1 or 2, NHWC, as an implicit GEMM (no im2col buffer):
 * X [B, stride*OH, stride*OW, ldx] (channel slice of width Cin), W [N, 9*Cin] with k = (dy*3+dx)*Cin + c,
 * out [B*OH*OW, ld_out].  Stands in for ConvX (projector.py:85-98) with BN folded into W/bias. */
LWDETR_API int lwdetr_conv3x3(int dtype, const void* X, int ldx, int B, int OH, int OW, int stride, int Cin,
                              const void* W, int N, const float* bias, int act, void* out, int ld_out,
                              void* stream);
/* Host query (no device needed): the output tile lwdetr_conv3x3 and the model's 3x3 convolutions use for an OH x OW grid,
 * either stride.  *tw x *th pixels, tw * th <= 128; the grid is covered by ceil(OW / tw) x ceil(OH / th) tiles. */
LWDETR_API int lwdetr_conv3x3_plan(int OH, int OW, int32_t* tw, int32_t* th);

/* LayerNorm over the last dimension of rows (vit.py:198,217 eps 1e-6; projector.py:21-47 on NHWC rows;
 * transformer.py norms eps 1e-5).  x/y 16-bit with leading dimensions, w/b fp32 [C], C % 8 == 0, C <= 1024. */
LWDETR_API int lwdetr_layernorm(int dtype, const void* x, int ldx, void* y, int ldy, const float* w, const float* b,
                                float eps, int64_t rows, int C, void* stream);

/* lwdetr_layernorm with the extras the decoder and the projector use (one launch, same kernel):
 *   row_flag uint8 [flag_mod] or NULL: row r with row_flag[r % flag_mod] != 0 normalises override_vec (fp32 [C]) instead of
 *     its x row (masked two-stage memory rows, transformer.py:116-123);
 *   y2 (with add_src [rows, ld_add]): y2 = round16(round16(y) + add_src), the sum as a 16-bit consumer of y would form it;
 *   y_group > 0: row r of y is written to row (r / y_group) * y_group_stride + y_row_off + r % y_group (the memory rows of one
 *     projector level inside the batch's memory);
 *   y3 (with w3, b3, eps3): the LayerNorm of the rounded y, exactly what a second call on y would write (decoder norm3 ->
 *     dec_norm); y3 and y2 rows are NOT regrouped.
 * Leading dimensions multiples of 8.  rows_per_warp (out) reports the kernel instance that ran: 1, or 4 for C <= 512 once
 * rows >= 64 * SMs. */
typedef struct {
  const void* x; int32_t ldx;
  void* y; int32_t ldy;
  const float* w; const float* b; float eps;
  int64_t rows; int32_t C;
  const uint8_t* row_flag; int32_t flag_mod; const float* override_vec;
  const void* add_src; int32_t ld_add; void* y2; int32_t ldy2;
  int64_t y_group, y_group_stride, y_row_off;
  const float* w3; const float* b3; float eps3; void* y3; int32_t ldy3;
  int32_t rows_per_warp;   /* out */
} lwdetr_layernorm_args;
LWDETR_API int lwdetr_layernorm_ex(int dtype, lwdetr_layernorm_args* args, void* stream);

/* softmax(Q K^T * scale) V for `nseq` independent sequences of `seqlen` tokens and `heads` heads of
 * width dh in {16, 32, 64}; token (s, t) is matrix row s*seqlen + t, head h occupies columns
 * [h*dh, (h+1)*dh).  Window attention: nseq = 16*B, seqlen = 100; global: nseq = B, seqlen = 1600
 * (vit.py:120-140, 195-222); decoder self-attention: nseq = B, seqlen = nq (attention.py:563-606).
 * dtype LWDETR_F16 or LWDETR_BF16.  Refused before anything is launched, with an error naming the limit: q, k, v or out
 * not 16-byte aligned; a leading dimension that is not a multiple of 8 or is below heads * dh; dh outside {16, 32, 64};
 * nseq, seqlen or heads not positive; nseq or heads above 65535 (the grid of the chosen kernel); and on the packed path
 * nseq * seqlen of 2^31 or more.
 * Kernels: a PACKED q / k / v (k = q + heads*dh, v = q + 2*heads*dh elements, one leading dimension, the ViT's qkv matrix)
 * runs on the wgmma / TMA kernel (LWDETR_ATTN_WG) at every length.  Anything else (the decoder's q / k column slices of
 * one matrix and a separate v) runs on mma.sync kernels: LWDETR_ATTN_MMA_SHORT (persistent CTAs over (sequence, head)
 * items) up to 112 tokens, LWDETR_ATTN_MMA with 4 warps per CTA below 1024 tokens and with 8 from there.  The environment
 * variable LWDETR_B200_ATTN_POLY (read once per process) moves part of the exponentials of the mma.sync kernels at head
 * dims 16 and 32 to a polynomial on the FMA pipe: 1 = n-tiles 2 and 5 of every 8 (mask 0x24), 2 = n-tiles 0, 3 and 6
 * (0x49); LWDETR_ATTN_MMA takes it with 8 warps only. */
LWDETR_API int lwdetr_attention(int dtype, const void* q, int ldq, const void* k, int ldk, const void* v, int ldv,
                                void* out, int ldo, int nseq, int seqlen, int heads, int dh, float scale,
                                void* stream);

/* lwdetr_attention with the arguments in a struct, reporting the kernel instance it chose (the same choice a launch
 * makes, under the same checks).  dry_run != 0: check and choose only, with no CUDA call at all (no launch, no device
 * query), so the pointers are never dereferenced and it runs without a device.
 *   kernel     LWDETR_ATTN_WG, LWDETR_ATTN_MMA or LWDETR_ATTN_MMA_SHORT;
 *   warps      4 or 8 for LWDETR_ATTN_MMA, 0 otherwise;
 *   poly_mask  0, 0x24 or 0x49: bit i set = n-tile i of each 64-key chunk takes the polynomial exp2. */
enum { LWDETR_ATTN_WG = 0, LWDETR_ATTN_MMA = 1, LWDETR_ATTN_MMA_SHORT = 2 };
typedef struct {
  int32_t dtype;
  const void* q; int32_t ldq;
  const void* k; int32_t ldk;
  const void* v; int32_t ldv;
  void* out; int32_t ldo;
  int32_t nseq, seqlen, heads, dh;
  float scale;
  int32_t dry_run;
  int32_t kernel, warps, poly_mask;   /* out */
} lwdetr_attention_args;
LWDETR_API int lwdetr_attention_ex(lwdetr_attention_args* args, void* stream);

/* Multi-scale deformable attention forward with the REFERENCE OPERATOR'S OWN INTERFACE:
 *   MultiScaleDeformableAttention.ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc,
 *   attn_weight, im2col_step) -> [B, Lq, M*D]
 *   (models/ops/src/ms_deform_attn.h:19-35, vision.cpp:13-16, cuda/ms_deform_attn_cuda.cu:20-80,
 *   cuda/ms_deform_im2col_cuda.cuh:33-84,237-299; Python caller functions/ms_deform_attn_func.py:28-38).
 * All pointers DEVICE, contiguous, as the reference asserts (ms_deform_attn_cuda.cu:28-38):
 *   value [B, S, M, D], sampling_loc [B, Lq, M, L, P, 2] (x, y normalised), attn_weight [B, Lq, M, L, P] and
 *   out [B, Lq, M*D] share one element type `etype` (LWDETR_ET_F32 / _F16 / _BF16 - the reference compiles float and
 *   double only, ms_deform_attn_cuda.cu:64); spatial_shapes int64 [L, 2] (H, W) and level_start_index int64 [L] are
 *   DEVICE tensors exactly as the reference receives them.  Any D; D % 4 == 0 (fp32) / D % 8 == 0 (16-bit) with
 *   16-byte aligned value / out takes the vectorised kernel, everything else a one-thread-per-channel kernel.
 * Differences from the reference: the caller owns `out` (the reference allocates at::zeros, :54); every element of out
 * is written, so it need not be zeroed; there is no im2col_step batching loop, but the reference's precondition
 * B % min(B, im2col_step) == 0 (:50-52) is still checked so that the error behaviour matches. */
enum { LWDETR_ET_F32 = 0, LWDETR_ET_F16 = 1, LWDETR_ET_BF16 = 2 };
LWDETR_API int lwdetr_ms_deform_attn_forward(int etype, const void* value, const int64_t* spatial_shapes,
                                             const int64_t* level_start_index, const void* sampling_loc,
                                             const void* attn_weight, void* out, int B, int S, int M, int D, int Lq,
                                             int L, int P, int im2col_step, void* stream);

/* Backward of the same operator, fp32 (ms_deform_attn.h:37-60, ms_deform_attn_cuda.cu:83-154, cuh:301-920):
 *   MSDA.ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
 *   im2col_step) -> [grad_value, grad_sampling_loc, grad_attn_weight].
 * grad_output [B, Lq, M*D]; grad_value [B, S, M, D] is zeroed by the call (the reference returns at::zeros_like, :120) and
 * accumulated with atomicAdd as in the reference; grad_sampling_loc [B, Lq, M, L, P, 2] and grad_attn_weight
 * [B, Lq, M, L, P] are written once per element.  Caller-owned, stream-ordered. */
LWDETR_API int lwdetr_ms_deform_attn_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                              const float* sampling_loc, const float* attn_weight, const float* grad_output,
                                              float* grad_value, float* grad_sampling_loc, float* grad_attn_weight, int B, int S,
                                              int M, int D, int Lq, int L, int P, int im2col_step, void* stream);

/* The fused form the model schedules (same arithmetic, fewer bytes): the softmax over the L*P attention logits and the
 * sampling-location arithmetic of MSDeformAttn.forward (ops/modules/ms_deform_attn.py:118-131, 4-d reference boxes) run
 * inside the kernel, which therefore takes the RAW projections, and the value tensor is HEAD-MAJOR so that everything one
 * (image, head) can sample is one contiguous slab streamed through shared memory (csrc/msda.cu):
 *   value_hm     16-bit, element (b, m, s, c) at b*v_image_stride + (m*S + s)*16 + c   (D = 16)
 *   offs_logits  16-bit [B*Lq, ld_ol] = [M*L*P*2 sampling offsets | M*L*P attention logits]
 *   ref          fp32   [B*Lq, 4]     reference boxes (cx, cy, w, h)
 *   valid_ratio  fp32   [B, L, 2] (w, h) or NULL: per-level valid ratios of a padded batch
 *                (transformer.py:189-196, 352-353)
 *   spatial_shapes int32 [L, 2] (H, W) and level_start_index int32 [L] on the HOST
 *   out          16-bit [B*Lq, ld_out] */
LWDETR_API int lwdetr_msda_forward(int dtype, const void* value_hm, int64_t v_image_stride, const void* offs_logits,
                                   int ld_ol, const float* ref, const float* valid_ratio, void* out, int ld_out, int B,
                                   int S, int Lq, int M, int L, int P, const int32_t* spatial_shapes_host,
                                   const int32_t* level_start_host, void* stream);
/* Host query (no device needed): the plan lwdetr_msda_forward builds for a level table (same arguments, same validation and
 * error message).  *nbands = 0: the direct-gather kernel runs.  Otherwise the staged kernel streams *nbands bands (at most
 * LWDETR_MSDA_MAX_BANDS) of each (image, head) slab; bands, int32 [LWDETR_MSDA_MAX_BANDS, 6], receives one row per band:
 *   level, row0 (first staged row), own0, own1 (the band samples every location whose floor(y) lies in [own0, own1]),
 *   tok0 (first staged token inside the slab), bytes (staged bytes, rows * W * 32). */
enum { LWDETR_MSDA_MAX_BANDS = 16 };
LWDETR_API int lwdetr_msda_plan(int L, const int32_t* spatial_shapes_host, const int32_t* level_start_host, int S, int32_t* nbands,
                                int32_t* bands);

/* torch.topk(score, k, dim=1)[1] for fp32 score [B, S] -> int32 idx [B, k], sorted, ties -> lower index
 * (transformer.py:246).  Any S >= k; above S = 16384 (large inputs) a radix select that streams the row, with k <= 4096. */
LWDETR_API int lwdetr_topk(const float* score, int B, int S, int k, int32_t* idx, void* stream);

/* PostProcess.forward (lwdetr.py:515-544) fused on the device: per image the top `num_select` of
 * sigmoid(pred_logits) over the nq*num_classes (query, class) pairs, sorted descending (ties -> lower flat index, as
 * torch.topk), labels = flat % num_classes, boxes = pred_boxes[flat / num_classes] converted cxcywh -> xyxy and scaled
 * by target_sizes [B,2] = (height, width).  All pointers DEVICE: pred_logits fp32 [B,nq,num_classes], pred_boxes fp32
 * [B,nq,4], target_sizes fp32 [B,2], work int32 [B * ceil(nq*num_classes/16384) * num_select] scratch,
 * scores fp32 [B,num_select], labels int32 [B,num_select], boxes fp32 [B,num_select,4]. */
LWDETR_API int lwdetr_postprocess(const float* pred_logits, const float* pred_boxes, const float* target_sizes, int B, int nq,
                                  int num_classes, int num_select, int32_t* work, float* scores, int32_t* labels, float* boxes,
                                  void* stream);

/* Tiled (sliced) detection of high-resolution frames: the detector runs on overlapping full-resolution crops of each frame
 * plus one downscaled view of the whole frame, and the per-view detections are merged per frame.  Three calls:
 *   1. lwdetr_forward_frames (or _nv12) on the V crop views, all on one run size H x W (a crop is an lwdetr_frame: device
 *      pointer of its first pixel, its size, the surface's pitch; NV12 crops need even offsets);
 *   2. lwdetr_postprocess with k = num_select and target_sizes = each view's crop size (ch, cw): boxes in crop pixels;
 *   3. lwdetr_tile_merge.
 * The views (b200.config.tile_views; a host in another language reproduces them from this rule).  Per axis, with n the
 * frame's side, t the tile side (default: the run side), H the run side, overlap in [0, 0.5]:
 *   stride s = t - (int)(overlap * t + 0.5);
 *   starts: [0] if n <= t, else p = 0, s, 2s, ... while p + t < n, then n - t; every start rounded down to even (NV12
 *     chroma covers 2x2 pixels), duplicates dropped.  When n - t is odd the last tile ends one pixel short of the edge;
 *   crop side c = min(t, n); destination side H when c == t, else (2 * c * H + t) / (2 * t) (integer division, i.e.
 *     c * H / t rounded half up) clamped to [1, H], placed top-left on the padded, masked canvas;
 *   views: per frame the tiles in row-major order, then (optionally) the whole frame stretched to H x W; frames in order.
 *   every crop side at most 16 times its destination side (the resize's downscale limit): t <= 16 H, and a partial tile's
 *     rounded destination checked too.
 * lwdetr_tile_merge: scores fp32 [V, k], labels int32 [V, k], boxes fp32 [V, k, 4] (xyxy in view crop pixels, 16-byte
 * aligned), all DEVICE, as lwdetr_postprocess writes them; views a HOST array of V {frame, x0, y0} (frames non-decreasing in
 * [0, num_frames), so each frame's views are contiguous; the caller may reuse it on return).  Per frame:
 *   candidates: every (view, rank) with score >= score_threshold, box moved to frame pixels by one fp32 add of
 *     (x0, y0, x0, y0);
 *   order: score descending, ties to the lower flat index view * k + rank;
 *   greedy class-aware NMS: a candidate is dropped when an earlier KEPT candidate with the same label overlaps it beyond
 *     iou_threshold (in [0, 1]).  fp32, each operation rounded on its own (no fused multiply-add):
 *       ix = max(0, min(ax2, bx2) - max(ax1, bx1)), iy likewise, inter = ix * iy, area = max(0, x2 - x1) * max(0, y2 - y1);
 *       LWDETR_TILE_IOU: inter > thr * ((area_a + area_b) - inter);  LWDETR_TILE_IOS: inter > thr * min(area_a, area_b).
 *     A box whose area is not > 0 never suppresses and is never suppressed.  IoS (intersection over the smaller box) is the
 *     usual choice here: a box cut off at a tile border lies inside the whole-object box of the neighbouring tile or the
 *     full view, while its IoU with that box can stay below 0.5;
 *   output: the first max_det kept candidates in that order: out_scores fp32 [num_frames, max_det], out_labels int32,
 *     out_boxes fp32 [num_frames, max_det, 4] (frame pixels, 16-byte aligned), counts int32 [num_frames]; unused slots get
 *     score 0, label -1 and a zero box.
 * Limits: at most 16384 candidates (views * k) and 2048 views per frame, max_det in [1, 1024].  Asynchronous, nothing
 * allocated per call, no device scratch. */
enum { LWDETR_TILE_IOU = 0, LWDETR_TILE_IOS = 1 };
typedef struct {
  int32_t frame, x0, y0;
} lwdetr_tile_view;
LWDETR_API int lwdetr_tile_merge(const float* scores, const int32_t* labels, const float* boxes, int V, int k,
                                 const lwdetr_tile_view* views, int num_frames, float score_threshold, float iou_threshold,
                                 int metric, int max_det, float* out_scores, int32_t* out_labels, float* out_boxes,
                                 int32_t* counts, void* stream);

/* Multi-object tracking of video streams: ByteTrack (BYTETracker.update of the YOLOX tracker, non-MOT20 settings) per
 * camera stream on the device.  The usual C composition per batch of frames, one frame per stream:
 *   1. lwdetr_forward_frames (or _nv12) on the frames;
 *   2. lwdetr_query_best: one entry per query (its best class), in query order - LW-DETR is NMS-free and lwdetr_postprocess
 *      ranks (query, class) pairs, so one query can appear there several times with one box; a tracker fed with those makes
 *      duplicate tracks;
 *   3. lwdetr_track with k = nq.  Any per-frame entry list works (lwdetr_tile_merge output, with k = max_det, too).
 * Calls on one tracker must be ordered on one CUDA stream (lwdetr_track reads and writes the tracker's device table).
 *
 * lwdetr_query_best: per query, score = max over classes of the fp32 sigmoid of pred_logits (ties to the lower class),
 * label = that class, box = pred_boxes converted and scaled exactly as lwdetr_postprocess does, so each entry has the bits
 * lwdetr_postprocess gives the same (query, class) pair.  pred_logits fp32 [B, nq, num_classes], pred_boxes fp32 [B, nq, 4],
 * target_sizes fp32 [B, 2] (height, width) -> scores fp32 [B, nq], labels int32 [B, nq], boxes fp32 [B, nq, 4]; DEVICE,
 * boxes 16-byte aligned.
 *
 * The tracker contract (tools/track_spec.py is this restatement in numpy).  Parameters (lwdetr_track_params_default fills
 * ByteTrack's defaults): thresholds are fp32; max_time_lost = (int)(frame_rate / 30.0 * track_buffer).
 * Entries of a frame: k of them (score fp32, label int32, xyxy fp32 in frame pixels), in input order.  An entry with a
 * non-finite coordinate, or whose width x2 - x1 or height y2 - y1 (float64) is not > 0, is ignored (ByteTrack would
 * produce NaN).  High: score > track_thresh; low: low_thresh < score < track_thresh.
 * Everything below is float64 with every operation rounded on its own (no fused multiply-add), in the order written.
 * Motion: constant-velocity Kalman filter in xyah.  Its covariance stays four independent 2x2 blocks, so per coordinate
 * q in (cx, cy, a, h) the state is position p, velocity v and (P, C, V): position variance, covariance, velocity variance.
 * With wp = 1.0 / 20, wv = 1.0 / 160 and std(w, h, f) = (w * h, w * h, f, w * h) (f for the coordinate a):
 *   measurement of an entry: w = x2 - x1, h = y2 - y1, z = (x1 + w / 2, y1 + h / 2, w / h, h);
 *   initiate from z: p = z, v = 0, P = sp * sp with sp = std(2 * wp, z_h, 1e-2), C = 0, V = sv * sv with
 *     sv = std(10 * wv, z_h, 1e-5);
 *   predict (h = p_h before the step; a track not in state Tracked first has v_h = 0):
 *     p = p + v; P = ((P + (C + C)) + V) + sp * sp; C = C + V; V = V + sv * sv, sp = std(wp, h, 1e-2), sv = std(wv, h, 1e-5);
 *   update with z (h = p_h before the update): S = P + sr * sr, sr = std(wp, h, 1e-1); Kp = P / S; Kv = C / S;
 *     y = z - p; p = p + Kp * y; v = v + Kv * y; P = P - (Kp * Kp) * S; C = C - (Kp * Kv) * S; V = V - (Kv * Kv) * S;
 *   box of a track: w = a * h, x1 = cx - w / 2, y1 = cy - h / 2, x2 = x1 + w, y2 = y1 + h.
 * IoU (no +1 pixel term): ix = max(0, min(ax2, bx2) - max(ax1, bx1)), iy likewise, inter = ix * iy,
 *   area = max(0, x2 - x1) * max(0, y2 - y1), union = (area_a + area_b) - inter; iou = inter / union, 0 when either area
 *   or the union is not > 0.  Entry boxes are widened from fp32.
 * Cost: 1 - iou, or with score fusion 1 - iou * score (score widened).  A pair is admissible iff cost < L (the association's
 *   threshold, widened) and, with class_aware, the labels agree.
 * Assignment (rows: tracks in list order, columns: entries in input order): the shortest-augmenting-path Hungarian method
 *   (classic potentials formulation) on the n x (m + n) matrix [cost | D], inadmissible pairs +inf, D[i][i] = L and +inf
 *   elsewhere; rows processed in order; each Dijkstra step takes the unused column of least slack, lowest column on ties;
 *   row i ending on column m + i is unmatched.  This maximises the sum of (L - cost) over matched pairs, which is what
 *   lap.lapjv(cost, extend_cost=True, cost_limit=L) returns up to ties.
 * One frame of one stream (frame counts from 1; lists keep ByteTrack's order):
 *   1. the tracked list splits into unconfirmed (not activated) and confirmed tracks; pool = confirmed, then the lost
 *      list; the pool is predicted (unconfirmed tracks are not);
 *   2. pool x high entries at match_thresh, fused if fuse_score: a matched track is updated (a Lost one is re-activated:
 *      same id and start frame, into the "refound" list);
 *   3. the pool's unmatched tracks in state Tracked x low entries at second_thresh, never fused: matched ones are updated,
 *      the others become Lost;
 *   4. unconfirmed tracks x the high entries left at unconfirmed_thresh, fused if fuse_score: matched ones are updated,
 *      the others removed;
 *   5. ageing: a track of the lost list (as it was before this frame) that was not refound and has
 *      frame - end_frame > max_time_lost is removed;
 *   6. births: every high entry left with score >= new_track_thresh, in input order, starts a track (initiate; id = the
 *      stream's next id, from 1; activated at once only on frame 1).  A birth that would take the stream past `capacity`
 *      tracks (tracked + lost after steps 2-5) is refused and counted in the stream's overflow count; it takes no id;
 *   7. tracked = previous tracked still Tracked, births, refound; lost = previous lost minus refound and removed, then the
 *      new lost tracks.  Removed tracks are dropped (ByteTrack keeps them forever);
 *   8. duplicates: for every (tracked, lost) pair with 1 - iou < duplicate_thresh (and equal labels under class_aware), the
 *      track with the smaller end_frame - start_frame is dropped, the tracked one on a tie;
 *   9. output: the activated tracks of the tracked list, in order: id, score and label of the entry that updated or started
 *      it this frame, xyxy of its state rounded to fp32, and that entry's index.
 * "Updated" sets the Kalman update with the entry's measurement, state Tracked, activated, end_frame = frame, and the
 * entry's score, label and index.
 *
 * lwdetr_tracker_create: num_streams >= 1 independent streams, params validated (thresholds in [0, 1], the three
 *   association thresholds in (0, 1], capacity in [1, 1024], track_buffer >= 0, frame_rate >= 1); allocates the device
 *   table (num_streams * capacity * 2 records) on the current device, every stream at frame 1.  Synchronous, on a
 *   stream of the tracker's own.
 * lwdetr_tracker_reset: the n streams listed (HOST array; ids distinct and in [0, num_streams), else an error and nothing
 *   happens) back to frame 1, next id 1, empty lists, overflow 0.
 * lwdetr_track: one frame for each of B streams (stream_ids, HOST; ids distinct and in [0, num_streams), else an error and
 *   nothing happens; a stream absent from a call does not advance):
 *   scores fp32 [B, k], labels int32 [B, k], boxes fp32 [B, k, 4] (16-byte aligned), k <= 1024; outputs [B, max_out]:
 *   out_ids int32, out_scores fp32, out_labels int32, out_boxes fp32 [B, max_out, 4] (16-byte aligned), out_index int32;
 *   counts int32 [B] = min(output tracks, max_out); unused slots id 0, score 0, label -1, zero box, index -1.  All DEVICE;
 *   asynchronous, nothing allocated or copied per call, safe to capture in a CUDA graph.
 * lwdetr_tracker_export: the list state of one stream, synchronous: it waits for the tracker's last lwdetr_track /
 *   lwdetr_tracker_reset launch (also when that launch was replayed from a CUDA graph) and for nothing else on the device,
 *   then copies up to cap records (tracked list, then lost list) into host; *count = the stream's record count,
 *   frame_next_overflow = (frame, next id, overflow). */
enum { LWDETR_TRACK_TRACKED = 1, LWDETR_TRACK_LOST = 2 };
typedef struct {
  float track_thresh, low_thresh, new_track_thresh, match_thresh, second_thresh, unconfirmed_thresh, duplicate_thresh;
  int32_t track_buffer, frame_rate, fuse_score, class_aware, capacity;
} lwdetr_track_params;
typedef struct {
  int32_t id, state, activated, start_frame, end_frame, label;
  float score;
  int32_t index;        /* entry that last updated the track */
  double mean[8];       /* p (cx, cy, a, h), then v */
  double cov[12];       /* P[4], C[4], V[4] */
} lwdetr_track_record;
typedef struct lwdetr_tracker lwdetr_tracker;
LWDETR_API void lwdetr_track_params_default(lwdetr_track_params* p);
LWDETR_API int lwdetr_tracker_create(int num_streams, const lwdetr_track_params* params, lwdetr_tracker** out);
LWDETR_API void lwdetr_tracker_destroy(lwdetr_tracker* t);
LWDETR_API int lwdetr_tracker_reset(lwdetr_tracker* t, const int32_t* streams, int n, void* stream);
LWDETR_API int lwdetr_track(lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes, int B, int k,
                            const int32_t* stream_ids, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels,
                            float* out_boxes, int32_t* out_index, int32_t* counts, void* stream);
LWDETR_API int lwdetr_tracker_export(lwdetr_tracker* t, int stream_id, lwdetr_track_record* host, int cap, int32_t* count,
                                     int32_t frame_next_overflow[3]);
LWDETR_API int lwdetr_query_best(const float* pred_logits, const float* pred_boxes, const float* target_sizes, int B, int nq, int num_classes,
                                 float* scores, int32_t* labels, float* boxes, void* stream);

/* lwdetr_track_ex: lwdetr_track with the camera motion of each frame (lwdetr_gmc_estimate's output), for moving cameras.
 * motion: DEVICE float64 [B, 4] (a, b, tx, ty), 8-byte aligned, the similarity x' = a x - b y + tx, y' = b x + a y + ty from
 * the stream's previous frame to this one in frame pixels; NULL is lwdetr_track, bit for bit.  With a motion, step 1 of the
 * contract above gains a warp (BoT-SORT's multi_gmc): after the pool is predicted, every record of the stream (confirmed,
 * lost and unconfirmed) is warped, each operation rounded on its own, with s2 = a * a + b * b and s = sqrt(s2):
 *   cx' = (a * cx - b * cy) + tx;  cy' = (b * cx + a * cy) + ty;  vx' = a * vx - b * vy;  vy' = b * vx + a * vy;
 *   h' = s * h;  vh' = s * vh;  a (aspect) and va unchanged;
 *   P, C and V of x, y and h multiplied by s2; those of the aspect unchanged.
 * This is exact, not an approximation: ByteTrack's x and y noise are both std(., h), so the x and y blocks of the covariance
 * are always equal (P_x = P_y, C_x = C_y, V_x = V_y) and a rotation by R = s Q maps sigma^2 I to s^2 sigma^2 I; the block
 * structure of the state survives.  (BoT-SORT's kron(I4, R) would also rotate the (aspect, h) pair, which has no meaning
 * in the xyah state; the aspect is left alone and h scales with the frame.) */
LWDETR_API int lwdetr_track_ex(lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes, const double* motion,
                               int B, int k, const int32_t* stream_ids, int max_out, int32_t* out_ids, float* out_scores,
                               int32_t* out_labels, float* out_boxes, int32_t* out_index, int32_t* counts, void* stream);

/* Tracking by appearance: BoT-SORT's re-identification cost (the with_reid path of BoTSORT.update, its defaults) on top of
 * the contract above, with an embedding per entry - the decoder's last hidden state of each query (lwdetr_last_hidden; the
 * C composition is lwdetr_forward_frames -> lwdetr_last_hidden -> lwdetr_query_best -> lwdetr_track_reid) or any ReID
 * model's.  The restatement in numpy is tools/track_spec.py (Stream with reid_params()).
 * Parameters (lwdetr_reid_params_default: D = 256 and BoT-SORT's 0.5 / 0.25 / 0.9): embedding_dim D in [1, 2048],
 * proximity_thresh in [0, 1), appearance_thresh in [0, 1], ema_alpha in [0, 1]; all fp32, widened.
 * Fixed order: the sum of D float64 terms is taken as 32 partial sums from 0, partial j adding terms j, j + 32, ... in
 * ascending order, combined by the xor butterfly 16, 8, 4, 2, 1 (partial j + partial j ^ o); norm |x| = sqrt(sum x_i * x_i),
 * dot(x, y) = sum x_i * y_i, every operation rounded on its own.
 * Entry embedding e (D values widened exactly to float64): ne = |e|; an entry whose ne is not finite or not > 0 has no
 * appearance.  Only high entries are looked at.
 * Track embedding t, fp32: a birth from an entry with appearance sets t = e / ne (each element rounded to fp32); an update
 * by a high entry with appearance (steps 2 and 4) sets t = e / ne when the track has none, else s = alpha * t + (1 - alpha)
 * * (e / ne) per element and t = s / |s| rounded to fp32 (BoT-SORT's update_features; t unchanged when |s| is not finite
 * or not > 0).  A low entry (step 3) leaves t as it is; a track born from an entry without appearance has none until an
 * update gives it one.
 * Cost in steps 2 (pool x high) and 4 (unconfirmed x high left) only; step 3 stays IoU only.  With the track's box as in
 * the contract: emb = max(0, 1 - dot(t, e) / ne) / 2; emb' = emb when (1 - iou) <= proximity_thresh and
 * emb <= appearance_thresh, else 1 (also 1 when either side has no appearance); cost = min(the IoU cost above, fused with
 * the score if fuse_score, emb'); admissible iff cost < L and the class gate passes.  emb' < 1 needs iou >= 1 -
 * proximity_thresh > 0, so an admissible pair still overlaps.
 * Deviations from BoT-SORT: the track embedding is stored in fp32; the distance does not normalise t and e again (BoT-SORT's
 * cdist(..., "cosine") divides by both norms); a non-finite or zero embedding means no appearance (BoT-SORT gives NaN);
 * lwdetr_tile_merge's entries carry no embeddings.
 *
 * lwdetr_tracker_create_reid: lwdetr_tracker_create plus the appearance state: the embedding table (num_streams *
 *   capacity * D * 4 bytes: one slot per track a stream can hold; a track keeps its slot for life, so nothing moves per
 *   frame), a slot per record and a per-stream scratch of 8192 proximity pairs (12 bytes each) per frame, in one
 *   allocation with the table.  Synchronous, on a stream of the tracker's own.
 * lwdetr_track_reid: lwdetr_track_ex with embeddings DEVICE [B, k, D], row stride ld_emb >= D elements, of type emb_dtype
 *   (LWDETR_ET_F32, _F16 or _BF16: the engine's 16-bit rows need no conversion), aligned to their element size.  NULL
 *   embeddings, or a tracker made by lwdetr_tracker_create, give lwdetr_track_ex's bits.  Asynchronous, nothing allocated
 *   per call, safe to capture in a CUDA graph.  lwdetr_track and lwdetr_track_ex on a tracker made by
 *   lwdetr_tracker_create_reid are lwdetr_track_reid with NULL embeddings: the same bits, and the tracks keep their
 *   embeddings, so the calls can be mixed on one tracker.
 * lwdetr_tracker_export_embeddings: synchronous like lwdetr_tracker_export; the D floats of each record in that function's
 *   order into host [cap][D], has[i] = 1 when record i has an embedding (its row is then valid), *count = the record count.
 * lwdetr_tracker_reset also forgets the streams' embeddings. */
typedef struct {
  int32_t embedding_dim;
  float proximity_thresh, appearance_thresh, ema_alpha;
} lwdetr_reid_params;
LWDETR_API void lwdetr_reid_params_default(lwdetr_reid_params* p);
LWDETR_API int lwdetr_tracker_create_reid(int num_streams, const lwdetr_track_params* params, const lwdetr_reid_params* reid,
                                          lwdetr_tracker** out);
LWDETR_API int lwdetr_track_reid(lwdetr_tracker* t, const float* scores, const int32_t* labels, const float* boxes, const double* motion,
                                 const void* embeddings, int emb_dtype, int ld_emb, int B, int k, const int32_t* stream_ids, int max_out,
                                 int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes, int32_t* out_index,
                                 int32_t* counts, void* stream);
LWDETR_API int lwdetr_tracker_export_embeddings(lwdetr_tracker* t, int stream_id, float* host, int cap, int32_t* count, int8_t* has);

/* Camera-motion estimation (global motion compensation, BoT-SORT's sparseOptFlow with the deviations stated here) per video
 * stream on the device, for lwdetr_track_ex.  The C composition per batch of frames, one frame per stream:
 * lwdetr_forward_frames (or _nv12) -> lwdetr_query_best -> lwdetr_gmc_estimate (or _nv12) on the same frame descriptors ->
 * lwdetr_track_ex with its motion.  Calls on one estimator must be ordered on one CUDA stream.
 * The contract (tools/gmc_spec.py restates it in numpy), d = downscale:
 *   1. grey and downscale: RGB grey g = (9798 R + 19235 G + 3735 B + 16384) >> 15 (cv2.COLOR_RGB2GRAY, bit for bit); NV12: the
 *      luma byte.  Level 0 is (floor(h / d), floor(w / d)); pixel (y, x) = (S + d*d / 2) / (d*d) in integers, S the sum of
 *      the d x d block of grey at (d y, d x) (for d = 2 that is cv2.resize's INTER_LINEAR / INTER_AREA halving).
 *   2. pyramid: level l from level l - 1 as cv2.pyrDown, bit for bit: ((w + 1) / 2, (h + 1) / 2), the 5-tap [1 4 6 4 1]
 *      kernel in both axes, BORDER_REFLECT_101, (sum + 128) >> 8.  Levels used: the largest L <= levels with both sides of
 *      level L > window (cv2.buildOpticalFlowPyramid's rule).
 *   3. corners on level 0: Sobel 3x3 derivatives dx, dy (BORDER_REFLECT_101), their products summed over the 3x3 block
 *      (BORDER_REFLECT_101 on the products), exact in integers: Sxx, Sxy, Syy.  Response R = (Sxx + Syy) - sqrt((Sxx - Syy)^2
 *      + 4 Sxy^2) in float64, the integer under the root exact, the root and the subtraction rounded once each: that is
 *      cv2.cornerMinEigenVal(blockSize 3, ksize 3) times 2 * 3060^2.  The frame is cut into c x c cells, c the smallest side
 *      with ceil(w0 / c) * ceil(h0 / c) <= max_points (row-major cells); each cell keeps its best pixel (largest R, lowest
 *      pixel index y * w0 + x on ties) when R > 0 and R >= (double)quality * max R over the frame.  The corners, in cell
 *      order, are kept for the stream's next frame.  (goodFeaturesToTrack's global top list is replaced on purpose: no sort,
 *      deterministic, points spread over the frame for the robust fit.)
 *   4. pyramidal Lucas-Kanade of the previous frame's corners into this frame: cv2.calcOpticalFlowPyrLK's iteration
 *      (window x window, the levels of 2., iterations, eps, min_eig; Scharr derivatives of the previous level with
 *      BORDER_REFLECT_101, 0 outside the image; images BORDER_REFLECT_101; 14-bit bilinear weights), except that the window
 *      sums are exact int64 before their scaling to float.  A corner is matched when level 0 ends with status 1.
 *   5. fit: each matched pair maps to frame pixels, x_f = d * (x + 0.5) - 0.5 (both axes, both frames), in float64.  With n
 *      pairs (n >= min_inliers, else status LWDETR_GMC_FEW_POINTS), hypothesis h in [0, hypotheses) takes pairs
 *      i = H(2h) mod n and j = H(2h + 1) mod (n - 1), plus 1 when >= i, with H(k) = mix(k * 0x9e3779b9 + 0x7f4a7c15) (uint32
 *      arithmetic) and mix(x): x ^= x >> 16; x *= 0x7feb352d; x ^= x >> 15; x *= 0x846ca68b; x ^= x >> 16.  Its similarity
 *      (dp = p_j - p_i, dq = q_j - q_i, n2 = dpx dpx + dpy dpy, skipped unless n2 > 0): a = (dqx dpx + dqy dpy) / n2,
 *      b = (dqy dpx - dqx dpy) / n2, tx = qx_i - (a px_i - b py_i), ty = qy_i - (b px_i + a py_i).  Its inliers: pairs with
 *      ex^2 + ey^2 <= (ransac_thresh * d)^2, ex = ((a px - b py) + tx) - qx, ey = ((b px + a py) + ty) - qy; every operation
 *      of this step is float64 rounded on its own.  The most inliers wins, the lowest h on ties; fewer than min_inliers:
 *      LWDETR_GMC_FEW_INLIERS.  Then 3 rounds: the inliers of the current model refit it by least squares (centred sums,
 *      a = sum(px' qx' + py' qy') / sum(px'^2 + py'^2), b = sum(px' qy' - py' qx') / sum(px'^2 + py'^2), t from the means),
 *      summed in a fixed order, so a call is bit-reproducible; the final model's inlier count is returned (fewer than
 *      min_inliers: LWDETR_GMC_FEW_INLIERS).
 *   6. outputs per frame: motion float64 [B, 4] (a, b, tx, ty) from the stream's previous frame to this one, frame pixels;
 *      status int32 [B]; inliers int32 [B].  Every status but LWDETR_GMC_OK gives the identity (1, 0, 0, 0).  A stream's first
 *      frame (after create or reset) and a frame whose size differs from the stream's previous one (re)start the stream.
 * lwdetr_gmc_params_default: downscale 2, max_points 1024, quality 0.01, levels 3, window 21, iterations 30, eps 0.01,
 *   min_eig 1e-4, ransac_thresh 3 (level-0 pixels), hypotheses 1024, min_inliers 10, max_height 2160, max_width 3840.
 * lwdetr_gmc_create: params validated (downscale in [1, 8], max_points in [16, 4096], quality in (0, 1], levels in [0, 5],
 *   window odd in [5, 31], iterations in [1, 100], eps > 0, min_eig >= 0, ransac_thresh > 0, hypotheses in [1, 4096],
 *   min_inliers in [2, max_points], max sides in [16 d, 8192]); allocates the device table (two pyramids and corner lists
 *   per stream, sized by the largest frame) on the current device.  Synchronous, on a stream of the estimator's own.
 * lwdetr_gmc_reset: the n streams listed (HOST; ids distinct and in [0, num_streams), else an error and nothing happens)
 *   start again at their next frame.
 * lwdetr_gmc_estimate / _nv12: one frame for each of B streams (stream_ids HOST; ids distinct and in [0, num_streams), else
 *   an error and nothing happens); frames as lwdetr_forward_frames takes them (dst_h, dst_w and colorspace are not read;
 *   NV12: the luma plane only), sides at least 16 d and at most the table's largest frame.  motion 8-byte aligned; all
 *   DEVICE; asynchronous, nothing allocated or copied per call, safe to capture in a CUDA graph. */
enum { LWDETR_GMC_OK = 0, LWDETR_GMC_FIRST_FRAME = 1, LWDETR_GMC_SIZE_CHANGED = 2, LWDETR_GMC_FEW_POINTS = 3, LWDETR_GMC_FEW_INLIERS = 4 };
typedef struct {
  int32_t downscale, max_points;
  float quality;
  int32_t levels, window, iterations;
  float eps, min_eig, ransac_thresh;
  int32_t hypotheses, min_inliers, max_height, max_width;
} lwdetr_gmc_params;
typedef struct lwdetr_gmc lwdetr_gmc;
LWDETR_API void lwdetr_gmc_params_default(lwdetr_gmc_params* p);
LWDETR_API int lwdetr_gmc_create(int num_streams, const lwdetr_gmc_params* params, lwdetr_gmc** out);
LWDETR_API void lwdetr_gmc_destroy(lwdetr_gmc* g);
LWDETR_API int lwdetr_gmc_reset(lwdetr_gmc* g, const int32_t* streams, int n, void* stream);
/* Inspection (tests), synchronous: it waits for the estimator's last lwdetr_gmc_estimate / _nv12 / lwdetr_gmc_reset launch
 * (also when that launch was replayed from a CUDA graph) and for nothing else on the device, then copies one stream's state
 * after its last frame.  levels: that frame's pyramid, levels 0..info[3] one after another, each dense at its size
 * (levels_bytes must hold them); corners float [max_points, 2]: its corners (info[4] of them); flow float [max_points, 4]
 * (from x, y, to x, y, level-0 pixels) and found int8 [max_points]: the last call's Lucas-Kanade results for the previous
 * frame's info[5] corners (meaningful when that call had a previous frame of the same size).  info = (has a last frame, its
 * height, its width, levels used or -1, corners, corners of the previous frame). */
LWDETR_API int lwdetr_gmc_export(lwdetr_gmc* g, int stream_id, uint8_t* levels, int64_t levels_bytes, float* corners, float* flow,
                                 int8_t* found, int32_t info[6]);

/* Tracking between detections: the detector runs on every N-th frame of a stream and the frames between are tracked by
 * per-object optical flow on the device - the Median Flow tracker (Kalal et al., 2010; OpenCV's TrackerMedianFlow) for
 * every track of every stream, on the camera-motion estimator's pyramids.  The C composition per call: the streams whose
 * frame is a keyframe go lwdetr_forward_frames (or _nv12) -> lwdetr_query_best -> lwdetr_track (or _ex with
 * lwdetr_gmc_estimate); the others go lwdetr_gmc_observe (or lwdetr_gmc_estimate, with a moving camera) ->
 * lwdetr_track_flow; both then -> lwdetr_zones_update.  tools/flow_spec.py restates the flow in numpy and
 * tools/track_spec.py (Stream.update_flow) the tracker step.
 * lwdetr_gmc_observe / _nv12 (declared after the frame descriptors): lwdetr_gmc_estimate's steps 1-3 only (grey, pyramid,
 *   corners); no Lucas-Kanade, no fit, no outputs.  The stream's chain of pyramids and corners stays current at a lower
 *   cost, so an estimate or a flow may follow on its next frame.
 * The flow of one stream, d = the estimator's downscale, every float64 operation rounded on its own:
 *   1. tracks: the activated records of the tracked list (state Tracked), in list order, as the tracker holds them after the
 *      stream's previous frame; track j >= max_tracks gets LWDETR_FLOW_SKIPPED.  When the estimator has no previous frame of
 *      the same size for the stream (its last two frames must be this one and the one before, through estimate or observe),
 *      every track gets LWDETR_FLOW_NO_PREVIOUS.
 *   2. seeds: box (x1, y1, w, h) of the track's state (w = a h, x1 = cx - w / 2, y1 = cy - h / 2); seed (i, k) of the
 *      grid x grid lattice, q = k grid + i: x_f = x1 + ((i + 0.5) w) / grid, y_f = y1 + ((k + 0.5) h) / grid, to level 0 by
 *      x_0 = (x_f + 0.5) / d - 0.5, rounded to fp32.
 *   3. forward Lucas-Kanade of each seed from the previous pyramid into the current one, then backward from the forward
 *      point, with lwdetr_gmc_estimate's step-4 iteration (the estimator's levels; the flow's window, iterations, eps and
 *      min_eig).  A seed is valid when both end with status 1.
 *   4. per valid seed, in frame pixels (x_f = d (x_0 + 0.5) - 0.5 of the fp32 points): FB = |p - p_back|; NCC of the
 *      ncc_window^2 patches of level 0 around round(p) in the previous frame and round(p_fwd) in the current one (round half
 *      to even, BORDER_REFLECT_101), from exact int64 sums: (n S_ab - S_a S_b) / sqrt((double)(n S_aa - S_a^2) * (double)(n
 *      S_bb - S_b^2)), -1 when either variance is 0.  OpenCV samples the patches at sub-pixel positions (getRectSubPix); the
 *      rounding is a deviation.
 *   5. "median" is the lower median: element (n - 1) / 2 of the ascending order.  Selected: the valid seeds with FB <=
 *      median(FB) and NCC >= median(NCC), both medians over the valid seeds.
 *   6. status, in this order: fewer than min_points selected: LWDETR_FLOW_FEW_POINTS; median FB > fb_max: LWDETR_FLOW_FB.
 *      Else dx, dy = the medians of the selected displacements p_fwd - p; s = the median over the selected pairs i < j (seed
 *      order) with |p_i - p_j| > 0 of |q_i - q_j| / |p_i - p_j| (each norm sqrt(ex * ex + ey * ey)); no such pair, or s not
 *      in [scale_min, scale_max]: LWDETR_FLOW_SCALE.  Else the measurement z = (cx + dx, cy + dy, a, h * s) of the state
 *      (cx, cy, a, h): centre moved, size scaled; a box under 2 level-0 pixels on a side (a (h s) or h s < 2 d):
 *      LWDETR_FLOW_SMALL.  Else LWDETR_FLOW_OK.
 *   Deviations from OpenCV's TrackerMedianFlow: the seeds are the state's box, not the last measured one; the scale is the
 *   lower median of the ratios (OpenCV: the median of the sorted vector's middle element); the status rules are the ones
 *   above.
 *   Limits, measured on rendered textured sprites (tests/test_flow_cpu.py, cv2's Lucas-Kanade on this contract): a sprite
 *   that nothing covers is measured to within 1.1 px on every side, not 0.5 px (the worst of three scenes is 0.96 px off;
 *   80-100 % of its frames are within 0.5 px); the cause was not isolated (leaving out the outer ring of seeds, whose windows
 *   see the background, does not remove it).  The failure statuses do not catch every bad measurement: a texture-less
 *   object on a textured background is measured from the seeds near its outline, and an object partly covered by a flat
 *   bar or by another textured object from the seeds on the cover; both can get LWDETR_FLOW_OK with a box 1-14 px off.
 *   Through the tracker (32 streams of rendered 1080p sprites, detections every 4th frame): no identity changes for
 *   uncovered sprites; the output box (the Kalman state after the flow's update) has IoU >= 0.9 with the truth on 99.7 % of
 *   the flow frames and 0.88 at worst.
 * lwdetr_flow_params_default: grid 10 (in [2, 16]), window 15 (odd, [5, 31]), iterations 30, eps 0.01, min_eig 1e-4 (the
 *   estimator's defaults), ncc_window 11 (odd, [3, 31]), min_points 8 (in [1, grid^2]), fb_max 10 frame pixels (> 0),
 *   scale_min 0.5, scale_max 2 (0 < scale_min <= 1 <= scale_max), max_tracks 256 per stream (in [1, 1024]).
 * lwdetr_flow_create: a flow bound to the estimator gmc (which must outlive it) with its stream count; one device allocation
 *   of num_streams * max_tracks * grid^2 seeds (about 41 bytes each) on the estimator's device.  Synchronous.
 * lwdetr_track_flow: one flow frame for each of B streams (stream_ids HOST, distinct, in [0, num_streams) of both the
 *   tracker and the flow's estimator); outputs as lwdetr_track's.  Per stream, float64 as the tracker contract:
 *   1. the pool (confirmed tracks, then lost) is predicted as in step 1; with motion (DEVICE [B, 4], or NULL) every record
 *      is then warped as lwdetr_track_ex does: the flow already carries the camera motion of the tracks it measures, the
 *      warp keeps the lost tracks aligned for the next keyframe;
 *   2. the flow above runs on the records as they were before this step (so on the states after the previous frame);
 *   3. a confirmed Tracked track whose status is LWDETR_FLOW_OK is updated with the Kalman update by z; it keeps its score
 *      and label, takes index -1 and end_frame = frame.  A confirmed Tracked track with any other status becomes Lost;
 *   4. unconfirmed tracks are carried unchanged: not updated, not removed, not output;
 *   5. ageing (step 5), the new lists (tracked = previous tracked still Tracked; lost = previous lost not removed, then the
 *      new lost), duplicates (step 8) and the output (step 9, index -1) as the contract.  No births; the frame counter
 *      advances.
 *   Asynchronous, nothing allocated or copied per call, safe to capture in a CUDA graph.  A tracker with appearance keeps its
 *   embeddings: a flow frame neither updates nor moves them.
 * lwdetr_flow_export (tests), synchronous: waits for the flow's last lwdetr_track_flow; one stream's last call.
 *   info = (tracks found by step 1, tracks measured = min(that, max_tracks), grid); per measured track j and seed q (index
 *   j * grid^2 + q): seeds, fwd, bwd float [.., 2] (level 0), valid int8, fb, ncc float64 (NaN where not valid); per track:
 *   status int32 and meas float64 [.., 8] = (dx, dy, s, z[4], unused), NaN where the status came before them.  cap: the
 *   room in tracks; the arrays hold min(cap, info[1]) tracks. */
enum { LWDETR_FLOW_OK = 0, LWDETR_FLOW_FEW_POINTS = 1, LWDETR_FLOW_FB = 2, LWDETR_FLOW_SCALE = 3, LWDETR_FLOW_SMALL = 4,
       LWDETR_FLOW_SKIPPED = 5, LWDETR_FLOW_NO_PREVIOUS = 6 };
typedef struct {
  int32_t grid, window, iterations;
  float eps, min_eig;
  int32_t ncc_window, min_points;
  float fb_max, scale_min, scale_max;
  int32_t max_tracks;
} lwdetr_flow_params;
typedef struct lwdetr_flow lwdetr_flow;
LWDETR_API void lwdetr_flow_params_default(lwdetr_flow_params* p);
LWDETR_API int lwdetr_flow_create(lwdetr_gmc* gmc, const lwdetr_flow_params* params, lwdetr_flow** out);
LWDETR_API void lwdetr_flow_destroy(lwdetr_flow* f);
LWDETR_API int lwdetr_track_flow(lwdetr_tracker* t, lwdetr_flow* flow, const double* motion, int B, const int32_t* stream_ids, int max_out,
                                 int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes, int32_t* out_index,
                                 int32_t* counts, void* stream);
LWDETR_API int lwdetr_flow_export(lwdetr_flow* f, int stream_id, int cap, float* seeds, float* fwd, float* bwd, int8_t* valid, double* fb,
                                  double* ncc, int32_t* status, double* meas, int32_t info[3]);

/* Line crossings and zone occupancy per camera stream, on the tracker's outputs (what DeepStream's nvdsanalytics and
 * supervision's LineZone / PolygonZone compute after a tracker).  The C composition per batch of frames: ... ->
 * lwdetr_track (or _ex / _reid) -> lwdetr_zones_update on its out_ids, out_labels, out_boxes and counts with the same
 * stream_ids, on the same CUDA stream; nothing is read back in between, so the pair can be captured in one CUDA graph.
 * Calls on one zones object must be ordered on one CUDA stream.  tools/zone_spec.py restates this contract in numpy.
 * Geometry per stream, float64 frame pixels: up to 32 lines (ax, ay, bx, by) of non-zero length and up to 32 polygons of 3
 *   to 256 vertices, at most 2048 vertices in all; any polygon (concave, self-intersecting).  Zones are fixed in frame
 *   pixels: with a moving camera (lwdetr_track_ex) they stay image regions, not world regions.
 * Parameters (lwdetr_zones_params_default): num_classes in [1, 1024] (default 91, LW-DETR's COCO head); capacity, the
 *   records per stream, in [1, 4096] (default 1024); forget_after >= 0 (default 30, ByteTrack's max_time_lost at its
 *   defaults); zone_anchor in [0, 9) (default LWDETR_ANCHOR_BOTTOM_CENTER, as PolygonZone); line_anchors a non-zero mask
 *   of anchor bits below 1 << 9 (default the four corners, as LineZone).
 * Anchors of an fp32 xyxy box widened to float64: anchor 3 * row + column, rows y1, (y1 + y2) * 0.5, y2 and columns x1,
 *   (x1 + x2) * 0.5, x2.  Everything is float64 with each operation rounded on its own (no FMA), in the order written.
 * Line side: dx = bx - ax, dy = by - ay, L2 = dx * dx + dy * dy; per anchor t = (px - ax) * dx + (py - ay) * dy and
 *   c = dx * (py - ay) - dy * (px - ax).  The frame's decision is +1 when every selected anchor has 0 <= t <= L2 and c > 0,
 *   -1 when every one has 0 <= t <= L2 and c < 0, else 0.  Each (track, line) keeps its last non-zero side s; a decision
 *   d != 0 with s != 0 and d != s is a crossing, LWDETR_ZONE_LINE_IN for d = +1 and _LINE_OUT for d = -1, counted in
 *   line_counts[line][label][in = 0 | out = 1]; then s = d.  A track's first decision only records its side.  In image
 *   coordinates (y down), for a line drawn left to right "in" is downward; swapping the endpoints swaps in and out.
 * Zone membership of the zone anchor: the crossing-number (even-odd) rule, for i = 0..n-1 and j = (i + n - 1) % n:
 *   if ((yi > py) != (yj > py)) && (px < (xj - xi) * (py - yi) / (yj - yi) + xi) inside = !inside.
 *   Points on edges and vertices get what this half-open rule gives (a horizontal edge never flips).
 * A frame of a stream (frames count its update calls from 1; a stream absent from a call does not advance):
 *   - entries at index >= min(counts[b], max_out), with id <= 0 or a non-finite box are absent; a repeated id's later
 *     entries are ignored too (the tracker never repeats one).  An absent track keeps its record as it is;
 *   - present tracks in input order: inside = the mask of the zones holding its anchor; occupancy[zone] counts them.  A
 *     track without a record takes one if the stream holds fewer than capacity records (else it is not recorded, makes no
 *     event and adds 1 to the stream's overflow); then lines ascending (crossings as above), then zones ascending: turning
 *     inside is LWDETR_ZONE_ENTER (entry frame = frame, entries[zone][label] += 1), turning outside is LWDETR_ZONE_EXIT with
 *     dwell = frame - entry frame (entry frame back to 0).  The record takes the frame as last_seen and the entry's label;
 *   - then every record with frame - last_seen > forget_after, in ascending id, is dropped, and for each zone it was
 *     inside (ascending) makes LWDETR_ZONE_FORGET with its last label and dwell = last_seen - entry frame.  So every enter
 *     is matched by exactly one exit or forget.
 *   A label outside [0, num_classes) counts in the extra column num_classes.  Events are (id, kind, index (line or zone),
 *   label (as given), dwell (0 for line and enter events)).
 * lwdetr_zones_create: num_streams >= 1, params validated; one device allocation (geometry, records, counters) on the
 *   current device, every stream at frame 1 without geometry.  Synchronous, on a stream of the object's own.
 * lwdetr_zones_set: one stream's geometry from HOST arrays, lines [n_lines][4], polygons' vertex counts [n_polygons] and
 *   vertices [sum of counts][2]; replaces the geometry and clears the stream's records, counters and overflow (the frame
 *   count goes on).  A limit overrun, a non-finite coordinate or a zero-length line is an error and nothing changes.
 *   Synchronous: it waits for the object's last launch (an lwdetr_zones_update, _reset, or an lwdetr_annotate that read the
 *   object) and nothing else on the device; not callable during a stream capture.
 * lwdetr_zones_reset: the n streams listed (HOST; ids distinct and in [0, num_streams), else an error and nothing happens)
 *   back to frame 1 with no records, zero counters and overflow; their geometry is kept.  Stream-ordered.
 * lwdetr_zones_update: one frame for each of B streams (stream_ids HOST, distinct and in [0, num_streams)); ids, labels int32
 *   [B, max_out], boxes fp32 [B, max_out, 4] (16-byte aligned), counts int32 [B]: exactly lwdetr_track's outputs;
 *   max_out in [1, 1024].  Outputs: inside uint32 [B, max_out] (0 for absent entries), occupancy int32 [B, 32] (0 past the
 *   stream's polygons), events int32 [B, max_events, 5] (the first max_events of the frame's events in order, unused rows
 *   zero; may be NULL when max_events = 0) and event_counts int32 [B], the true number.  The counters count every event.
 *   All DEVICE; asynchronous, nothing allocated or copied per call, safe to capture in a CUDA graph.
 * lwdetr_zones_export: one stream, synchronous: it waits for the object's last launch (as lwdetr_zones_set) and nothing else
 *   on the device.
 *   frame_overflow = (frame, overflow); line_counts int32 [n_lines][num_classes + 1][2] and entries int32
 *   [n_polygons][num_classes + 1] (n_* of the stream's geometry: info = (n_lines, n_polygons, records)); then up to cap
 *   records in ascending id: lwdetr_zone_record with sides[l] in {-1, 0, +1} and entry[z] the entry frame (0 when
 *   outside). */
enum {
  LWDETR_ANCHOR_TOP_LEFT = 0, LWDETR_ANCHOR_TOP_CENTER = 1, LWDETR_ANCHOR_TOP_RIGHT = 2, LWDETR_ANCHOR_CENTER_LEFT = 3,
  LWDETR_ANCHOR_CENTER = 4, LWDETR_ANCHOR_CENTER_RIGHT = 5, LWDETR_ANCHOR_BOTTOM_LEFT = 6, LWDETR_ANCHOR_BOTTOM_CENTER = 7,
  LWDETR_ANCHOR_BOTTOM_RIGHT = 8
};
enum { LWDETR_ZONE_LINE_IN = 1, LWDETR_ZONE_LINE_OUT = 2, LWDETR_ZONE_ENTER = 3, LWDETR_ZONE_EXIT = 4, LWDETR_ZONE_FORGET = 5 };
typedef struct {
  int32_t num_classes, capacity, forget_after, zone_anchor, line_anchors;
} lwdetr_zones_params;
typedef struct {
  int32_t id, last_seen, label;
  uint32_t inside;
  int8_t sides[32];
  int32_t entry[32];
} lwdetr_zone_record;
typedef struct lwdetr_zones lwdetr_zones;
LWDETR_API void lwdetr_zones_params_default(lwdetr_zones_params* p);
LWDETR_API int lwdetr_zones_create(int num_streams, const lwdetr_zones_params* params, lwdetr_zones** out);
LWDETR_API void lwdetr_zones_destroy(lwdetr_zones* z);
LWDETR_API int lwdetr_zones_set(lwdetr_zones* z, int stream_id, const double* lines, int n_lines, const int32_t* polygon_sizes,
                                int n_polygons, const double* vertices);
LWDETR_API int lwdetr_zones_reset(lwdetr_zones* z, const int32_t* streams, int n, void* stream);
LWDETR_API int lwdetr_zones_update(lwdetr_zones* z, const int32_t* ids, const int32_t* labels, const float* boxes, const int32_t* counts,
                                   int B, int max_out, const int32_t* stream_ids, uint32_t* inside, int32_t* occupancy, int32_t* events,
                                   int max_events, int32_t* event_counts, void* stream);
LWDETR_API int lwdetr_zones_export(lwdetr_zones* z, int stream_id, int32_t frame_overflow[2], int32_t info[3], int32_t* line_counts,
                                   int32_t* entries, lwdetr_zone_record* records, int cap);

/* Ground-plane position, velocity and speed of each track per camera stream, on the tracker's outputs (what supervision's
 * speed-estimation example and the road-analytics stages of DeepStream-style pipelines compute after a tracker).  The C
 * composition per batch of frames: ... -> lwdetr_track (or _ex / _reid / lwdetr_track_flow) -> lwdetr_zones_update ->
 * lwdetr_speed_update on the same out_ids, out_boxes and counts with the same stream_ids, on the same CUDA stream; nothing
 * is read back in between, so the chain can be captured in one CUDA graph.  Calls on one speed object must be ordered on
 * one CUDA stream.  tools/speed_spec.py restates this contract in numpy.
 * Per stream: a 3x3 float64 homography H (row-major, h0..h8) from frame pixels to ground units (default the identity:
 *   pixels and pixels per second); a frame counter from 1; the last timestamp t_last (-inf at first); overflow and
 *   clock-error counters; up to capacity records, one per track id, each a ring of its last `window` samples (t, x, y),
 *   x and y the track's anchor in frame PIXELS (float64).  The ring keeps pixels, so lwdetr_speed_set can replace H
 *   without dropping any history: every estimate projects the ring with the current H.  H is fixed: it describes a still
 *   camera over a ground plane (with lwdetr_track_ex's moving cameras it has no meaning).
 * Parameters (lwdetr_speed_create): capacity in [1, 4096] (default 1024), window in [2, 64] (default 30: one second at
 *   30 fps), min_samples in [2, window] (default 15), forget_after >= 0 (default 30), anchor in [0, 9) (default
 *   LWDETR_ANCHOR_BOTTOM_CENTER, the ground-contact point; the zones' anchor rule), frame_rate finite and > 0 (default 30).
 * Everything is float64 with each operation rounded on its own (no FMA), in the order written; outputs are rounded to
 *   fp32 once at the end.
 * Projection of (x, y): w = (h6 * x + h7 * y) + h8, X = ((h0 * x + h1 * y) + h2) / w, Y = ((h3 * x + h4 * y) + h5) / w.
 *   The point is valid iff w > 0 and X and Y are finite: points on or beyond the horizon are invalid, so H must give
 *   w > 0 on the ground (capi.homography normalises the sign).
 * Time: timestamps DEVICE float64 [B] in seconds, or NULL: then t = frame / frame_rate, frame the stream's own update
 *   count, so a stream whose caller skips real frames runs slow.  A frame whose t is not finite or not greater than the
 *   stream's t_last adds no samples; it is otherwise a normal frame, and adds 1 to the stream's clock errors.  Else
 *   t_last = t.
 * A frame of a stream (a stream absent from a call does not advance):
 *   - entries at index >= min(counts[b], max_out), with id <= 0 or a non-finite box are absent; a repeated id's later
 *     entries are ignored (the zones' rule);
 *   - present tracks in input order: a track without a record takes one if the stream holds fewer than capacity records
 *     (else it is not recorded and adds 1 to the overflow).  A recorded track appends (t, anchor) to its ring (unless the
 *     clock is bad), dropping the oldest sample once the ring holds `window`; its record takes the frame as last_seen;
 *   - the fit runs over the ring's samples whose projection is valid (n of them), oldest first, with tau_i = t_i - t of
 *     the newest of them: mt = (sum tau_i) / n, mX = (sum X_i) / n, mY likewise, each sum left to right from 0.0;
 *     Stt = sum (tau_i - mt) * (tau_i - mt), StX = sum (tau_i - mt) * (X_i - mX), StY likewise; vX = StX / Stt,
 *     vY = StY / Stt, speed = sqrt(vX * vX + vY * vY).  There is an estimate iff n >= min_samples and Stt > 0;
 *   - then every record with frame - last_seen > forget_after is dropped.
 * Outputs per entry [B, max_out]: kin fp32 [B, max_out, 5] = (X, Y, vX, vY, speed): X, Y this frame's anchor projected
 *   (NaN when invalid or absent), vX, vY, speed NaN without an estimate; samples int32 = n for a recorded present track,
 *   else 0.
 * lwdetr_speed_create: num_streams >= 1, parameters validated; one device allocation on the current device (the rings
 *   take num_streams * capacity * window * 24 bytes), every stream at frame 1 with H the identity.  Synchronous.
 * lwdetr_speed_destroy: frees the object.
 * lwdetr_speed_set: one stream's H from a HOST [9] array; a non-finite H or a singular one (its determinant
 *   h0 (h4 h8 - h5 h7) - h1 (h3 h8 - h5 h6) + h2 (h3 h7 - h4 h6) is 0 or not finite) is an error and nothing changes.
 *   The history is kept.  Synchronous: it waits for the object's last launch and nothing else on the device; not callable
 *   during a stream capture.
 * lwdetr_speed_reset: the n streams listed (HOST; distinct and in [0, num_streams), else an error and nothing happens)
 *   back to frame 1, no records, zero counters, t_last = -inf; H is kept.  Stream-ordered.
 * lwdetr_speed_update: one frame for each of B streams (stream_ids HOST, distinct and in [0, num_streams)); ids int32
 *   [B, max_out], boxes fp32 [B, max_out, 4] (16-byte aligned), counts int32 [B]: lwdetr_track's outputs; max_out in
 *   [1, 1024]; timestamps as above.  All DEVICE; asynchronous, nothing allocated or copied per call, safe to capture in a
 *   CUDA graph.
 * lwdetr_speed_export: one stream, synchronous: it waits for the object's last launch and nothing else on the device.
 *   head = (frame, records, overflow, clock_errors), last_t, homography [9]; then up to cap records in ascending id:
 *   ids, last_seen, counts (samples in the ring) int32 [cap] and samples float64 [cap][window][3] (t, x, y), oldest
 *   first, the rest of each record's rows untouched. */
typedef struct lwdetr_speed lwdetr_speed;
LWDETR_API int lwdetr_speed_create(int num_streams, int capacity, int window, int min_samples, int forget_after, int anchor,
                                   double frame_rate, lwdetr_speed** out);
LWDETR_API void lwdetr_speed_destroy(lwdetr_speed* s);
LWDETR_API int lwdetr_speed_set(lwdetr_speed* s, int stream_id, const double* homography);
LWDETR_API int lwdetr_speed_reset(lwdetr_speed* s, const int32_t* streams, int n, void* stream);
LWDETR_API int lwdetr_speed_update(lwdetr_speed* s, const int32_t* ids, const float* boxes, const int32_t* counts, int B, int max_out,
                                   const int32_t* stream_ids, const double* timestamps, float* kin, int32_t* samples, void* stream);
LWDETR_API int lwdetr_speed_export(lwdetr_speed* s, int stream_id, int32_t head[4], double* last_t, double* homography, int32_t* ids,
                                   int32_t* last_seen, int32_t* counts, double* samples, int cap);

/* The LWDETR_F16_E4M3 mode's two kernels.
 * lwdetr_layernorm_e4m3: fp16 rows x [rows, ldx] -> e4m3 codes q [rows, ldq] (uint8) and fp32 row_scale [rows], as the mode's
 *   activation contract above (x^ without the LayerNorm affine, eps as given).  C % 8 == 0, C <= 1024, ldx and ldq
 *   multiples of 8.
 * lwdetr_gemm_e4m3: out[m, n] = act(a_scale[m] * w_scale[n] * sum_k A[m,k] W[n,k] + bias[n]) in fp16; A e4m3 [M, lda]
 *   (lda bytes, a multiple of 16), W e4m3 [N, K], a_scale fp32 [M], w_scale fp32 [N], bias fp32 [N] or NULL,
 *   act LWDETR_ACT_NONE or LWDETR_ACT_GELU (exact-erf GELU, as the fp16 fc1), out fp16 [M, ld_out].  K % 64 == 0. */
LWDETR_API int lwdetr_layernorm_e4m3(const void* x, int ldx, int64_t rows, int C, float eps, uint8_t* q, int ldq, float* row_scale,
                                     void* stream);
LWDETR_API int lwdetr_gemm_e4m3(const void* A, int lda, const float* a_scale, int M, int K, const void* W, const float* w_scale, int N,
                                const float* bias, int act, void* out, int ld_out, void* stream);
/* The fused ViT MLP of the 192-wide encoder (tiny, small), one kernel in place of the LayerNorm-fused fc1 GEMM and the fc2 GEMM:
 *   h   = round16(gelu(rstd*(x W1^T) - rstd*mean*colsum1 + b1))    [M, 768], kept on chip
 *   out = x + gamma * (h W2^T + b2)                                 [M, 192]
 * dtype LWDETR_F16 / LWDETR_BF16.  x 16-bit [M, ldx] (the raw residual rows, C = 192); stats_in fp32 pairs [M, stats_parts]
 * with each row's LayerNorm partials (sum, M2) over equal slices of the 192 columns (stats_parts divides 192); W1 16-bit
 * [768, 192] (the LayerNorm affine folded in), colsum1 / b1 fp32 [768]; W2 16-bit [192, 768], b2 / gamma fp32 [192] or NULL;
 * out 16-bit [M, ld_out]; stats_out fp32 pairs [M, stats_parts_out] (2 or 6) or NULL: the partials of the rounded output
 * rows.  ldx and ld_out multiples of 16, x and out 32-byte aligned.  Bit-identical to the two GEMMs it replaces. */
LWDETR_API int lwdetr_vit_mlp(int dtype, const void* x, int ldx, int M, const float* stats_in, int stats_parts, float eps,
                              const void* W1, const float* colsum1, const float* b1, const void* W2, const float* b2,
                              const float* gamma, void* out, int ld_out, float* stats_out, int stats_parts_out, void* stream);
/* Host helper (no GPU): the weight quantiser lwdetr_load_weights uses in the LWDETR_F16_E4M3 mode.  Per row r of src
 * fp32 [rows, K]: scale[r] = max_k |src[r,k]| / 448 (0 -> 1) and q[r,k] = e4m3(src[r,k] * 448 / max_k |src[r,k]|) as a
 * uint8 code (round to nearest even, saturating to +-448). */
LWDETR_API int lwdetr_host_quant_e4m3_rows(const float* src, int64_t rows, int K, uint8_t* q, float* scale);

/* Host helper (no GPU): bicubic, align_corners=False resize of a channels-last [n_in, n_in, C] fp32 grid
 * to [n_out, n_out, C] - the absolute position embedding resize of vit.py:26-54, done once at load. */
LWDETR_API int lwdetr_host_bicubic(const float* src, int n_in, int C, int n_out, float* dst);
/* The same resize to a non-square [out_h, out_w, C] grid: the position table of a non-square input (vit.py:26-54 with
 * hw = (H/16, W/16)). */
LWDETR_API int lwdetr_host_bicubic_hw(const float* src, int n_in, int C, int out_h, int out_w, float* dst);

/* ------------------------------------------------------------------------------------------------
 * Model-level API: what models.lwdetr.LWDETR.forward (lwdetr.py:111-174) binds to.
 * ---------------------------------------------------------------------------------------------- */
typedef struct lwdetr_handle lwdetr_handle;

typedef struct {
  int32_t vit_dim, vit_depth, vit_heads;
  int32_t window_block_mask;     /* bit i set: block i uses window attention (vit.py:195-222) */
  int32_t n_taps, taps[4];       /* out_feature_indexes, ascending (vit.py:311-316) */
  int32_t n_levels, level_scale_log2[2]; /* projector levels: +1 = P3 (x2), 0 = P4, -1 = P5 (/2) */
  int32_t hidden_dim, sa_heads, ca_heads, dec_points, num_queries, dec_layers, dim_feedforward;
  int32_t num_classes, group_detr, img_size;
} lwdetr_config;

typedef struct {
  float* aux_logits;   /* [dec_layers-1, B, nq, num_classes] or NULL */
  float* aux_boxes;    /* [dec_layers-1, B, nq, 4] or NULL */
  float* enc_logits;   /* [B, nq, num_classes] or NULL */
  float* enc_boxes;    /* [B, nq, 4] or NULL */
  int32_t* topk_index; /* [B, nq] two-stage selection (token index per query slot) or NULL */
} lwdetr_aux_out;

/* dtype: LWDETR_F16, LWDETR_BF16 or LWDETR_F16_E4M3 (see above).
 * One handle per (device, config, compute dtype); not thread-safe per handle.  The handle binds to the CUDA device
 * that is current at creation; every later call switches to that device for its duration. */
LWDETR_API int lwdetr_create(const lwdetr_config* cfg, int dtype, lwdetr_handle** out);
LWDETR_API void lwdetr_destroy(lwdetr_handle* h);

/* Pack the checkpoint: `n` named fp32 HOST tensors with the reference's state_dict names
 * (SURVEY.md 8b).  Folds BatchNorm into the convolutions, merges q/v biases, concatenates the
 * deformable-attention projections, resizes the position embedding, converts to the compute dtype
 * and uploads.  Synchronous.  May be called again after the weights change. */
LWDETR_API int lwdetr_load_weights(lwdetr_handle* h, int n, const char* const* names, const float* const* data,
                                   const int64_t* numel);

/* images: DEVICE [B, 3, S, S], fp32 (images_fp32 = 1) or the compute dtype; outputs: DEVICE fp32
 * pred_logits [B, nq, num_classes], pred_boxes [B, nq, 4]; aux may be NULL.  topk_override: DEVICE
 * int32 [B, nq] or NULL - test hook that forces the two-stage selection (SURVEY.md 8c tier T2).  Every index must lie in
 * [0, S), S the memory length of this input size; the C entry points do not check that (b200.capi.Engine does, before
 * the call), and an index outside it makes the forward read outside its buffers. */
LWDETR_API int lwdetr_forward(lwdetr_handle* h, const void* images, int images_fp32, int B, float* pred_logits,
                              float* pred_boxes, const lwdetr_aux_out* aux, const int32_t* topk_override,
                              void* stream);

/* The same forward with the two input forms the callers on either side of the path use (SURVEY.md 8f):
 *   format LWDETR_IN_U8_NHWC: images is DEVICE uint8 [B, S, S, 3] - the output of an image decoder + resize.  ToTensor's /255
 *     and Normalize(mean, std) (demo/demo.py:146-159, datasets/transforms.py:223-252) are fused into the patch gather:
 *     (x/255 - mean[c]) / std[c]; the fp32 NCHW image never exists (4x fewer input bytes over PCIe and HBM).
 *   padding_mask: DEVICE bool [B, S, S] (True = padded pixel), the NestedTensor mask of a padded / mixed-size batch
 *     (util/misc.py:317-339), or NULL.  Implements backbone.py:153-158 (nearest resize per level), transformer.py:
 *     86-89,112-123 (per-image proposals, masked memory rows), :189-196,352-355 (valid ratios on the reference boxes) and
 *     ops/modules/ms_deform_attn.py:114-115 (masked value rows).  The ViT itself takes no mask (backbone.py:145). */
enum { LWDETR_IN_F32_NCHW = 0, LWDETR_IN_16_NCHW = 1, LWDETR_IN_U8_NHWC = 2 };
typedef struct {
  const void* images;
  int32_t format;
  const uint8_t* padding_mask;
  float mean[3], std[3];        /* LWDETR_IN_U8_NHWC only */
} lwdetr_input;
LWDETR_API int lwdetr_forward_ex(lwdetr_handle* h, const lwdetr_input* input, int B, float* pred_logits, float* pred_boxes,
                                 const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream);

/* lwdetr_forward_ex at any supported input size: images [B, 3, height, width] (fp32 / compute dtype) or [B, height, width, 3]
 * (uint8), padding_mask [B, height, width].  height and width are multiples of 64 in [128, 1344] (4x4 windows of 16-pixel
 * patches, vit.py:353-358); the position embedding is resized to the (height/16, width/16) token grid (vit.py:26-54) and
 * every feature level takes its shape from that grid.  The memory length (tokens over all levels) must be at least
 * num_queries.  lwdetr_forward_ex is this call with height = width = img_size.  A (B, height, width) different from the
 * previous call re-plans the schedule and drops its CUDA graphs (one plan is kept at a time). */
LWDETR_API int lwdetr_forward_hw(lwdetr_handle* h, const lwdetr_input* input, int B, int height, int width, float* pred_logits,
                                 float* pred_boxes, const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream);

/* Raw camera / decoder frames of any size (SURVEY.md 8f rank 2: the resize in front of the uint8 path).  One frame is a
 * DEVICE uint8 HWC RGB image of height x width pixels, rows pitch_bytes >= 3 * width apart; `data` and `pitch_bytes` need
 * no alignment (decoder surfaces, crops of a larger surface).  The frame is resized on the device to dst_h x dst_w by
 * antialiased bilinear interpolation - the separable triangle filter of PIL.Image.resize(BILINEAR) and
 * F.interpolate(mode="bilinear", antialias=True): per axis scale = n_in / n_out, support = max(scale, 1), output o has
 * centre c = (o + 0.5) * scale, taps x in [max(int(c - support + 0.5), 0), min(int(c + support + 0.5), n_in)), weight
 * max(0, 1 - |x - c + 0.5| / support) over the sum of the weights; horizontal then vertical in fp32, rounded half up to an
 * integer level and clamped to [0, 255] - so the result is the uint8 image a host resize hands to LWDETR_IN_U8_NHWC, within
 * one level of PIL (which also rounds between the passes).  Then (v / 255 - mean[c]) / std[c] as for LWDETR_IN_U8_NHWC.
 * Limits: source sides in [8, 8192]; n_in / dst <= 16 per axis; any upscale; dst sides in [1, run side]. */
typedef struct {
  const uint8_t* data;
  int32_t height, width;
  int64_t pitch_bytes;
  int32_t dst_h, dst_w;
} lwdetr_frame;

/* lwdetr_forward_hw on B frames, each with its own size: frame b is resized to its (dst_h, dst_w) and placed top-left on
 * the height x width canvas the batch runs at (height, width as lwdetr_forward_hw requires).  The rest of the canvas is 0
 * after normalisation and, when any frame leaves some, carries a padding mask made on the device (as util/misc.py:317-339
 * builds it).  The resize is fused into the patch gather: no resized and no fp32 image exists in device memory.  `frames`
 * is a HOST array of B descriptors with DEVICE data pointers; the caller may reuse it as soon as the call returns.  Same
 * outputs and stream ordering as lwdetr_forward_hw; asynchronous; nothing is allocated per call.  Source sizes, pointers
 * and dst sizes are not part of the plan: only a change of (B, height, width) re-plans. */
LWDETR_API int lwdetr_forward_frames(lwdetr_handle* h, const lwdetr_frame* frames, const float mean[3], const float std[3], int B,
                                     int height, int width, float* pred_logits, float* pred_boxes, const lwdetr_aux_out* aux,
                                     const int32_t* topk_override, void* stream);

/* The kernel behind it, without a model: frames -> A, the 16-bit window-major patch matrix [B * (height/16) * (width/16), 768]
 * (k = c*256 + py*16 + px) that the patch-embedding GEMM reads, and (mask != NULL) the padding mask uint8 [B, height, width],
 * 1 = outside the frame.  height and width multiples of 64. */
LWDETR_API int lwdetr_resize_patches(int dtype, const lwdetr_frame* frames, int B, int height, int width, const float mean[3],
                                     const float std[3], void* A, uint8_t* mask, void* stream);

/* NV12 (YUV 4:2:0) frames, the output of video decoders and camera pipelines: a luma plane of height rows of width bytes,
 * rows luma_pitch >= width apart, and an interleaved chroma plane of ceil(height/2) rows of ceil(width/2) (U, V) byte pairs,
 * rows chroma_pitch >= 2 * ceil(width/2) apart.  No pointer or pitch needs any alignment; odd sizes are allowed.
 * Each source pixel (y, x) is converted to an RGB uint8 triple from Y at (y, x) and the chroma pair at (y >> 1, x >> 1)
 * (replicated, not filtered), and from there on the frame is exactly an lwdetr_frame of that RGB image: the same resize,
 * rounding, normalisation, gather, padding and mask.  The conversion is int32 and exact (>> is an arithmetic shift):
 *   u = U - 128, v = V - 128;  y' = max(Y - 16, 0) * cY (the _LIMITED rows)  or  Y * cY (the _FULL rows)
 *   R = clamp((y' + cRv * v + 2^19) >> 20, 0, 255)
 *   G = clamp((y' + cGu * u + cGv * v + 2^19) >> 20, 0, 255)
 *   B = clamp((y' + cBu * u + 2^19) >> 20, 0, 255)
 *   colorspace               cY        cRv       cGu       cGv       cBu
 *   LWDETR_CSC_BT601_LIMITED 1220542   1673527   -409993   -852492   2116026   (bit-identical to OpenCV's COLOR_YUV2RGB_NV12)
 *   LWDETR_CSC_BT709_LIMITED 1220945   1879825   -223607   -558796   2215014
 *   LWDETR_CSC_BT601_FULL    1048576   1470104   -360853   -748826   1858077
 *   LWDETR_CSC_BT709_FULL    1048576   1651297   -196424   -490864   1945738
 * The first row is OpenCV's 3-decimal table times 2^20; the others are round(2^20 c) of the exact BT.601 / BT.709
 * coefficients, with 255/219 luma and 255/224 chroma scaling for limited range.  Every row is within one level of the
 * float64 conversion.  Limits as lwdetr_frame. */
enum { LWDETR_CSC_BT601_LIMITED = 0, LWDETR_CSC_BT709_LIMITED = 1, LWDETR_CSC_BT601_FULL = 2, LWDETR_CSC_BT709_FULL = 3 };
typedef struct {
  const uint8_t* luma;   int64_t luma_pitch;    /* height rows of width bytes */
  const uint8_t* chroma; int64_t chroma_pitch;  /* ceil(height/2) rows of ceil(width/2) (U, V) byte pairs */
  int32_t height, width, dst_h, dst_w;
  int32_t colorspace;                           /* per frame: cameras of one batch may differ */
} lwdetr_frame_nv12;

/* lwdetr_forward_frames on NV12 frames.  RGB and NV12 batches of one (B, height, width) share the plan and its CUDA graphs. */
LWDETR_API int lwdetr_forward_frames_nv12(lwdetr_handle* h, const lwdetr_frame_nv12* frames, const float mean[3], const float std[3],
                                          int B, int height, int width, float* pred_logits, float* pred_boxes,
                                          const lwdetr_aux_out* aux, const int32_t* topk_override, void* stream);
/* lwdetr_resize_patches on NV12 frames. */
LWDETR_API int lwdetr_resize_patches_nv12(int dtype, const lwdetr_frame_nv12* frames, int B, int height, int width,
                                          const float mean[3], const float std[3], void* A, uint8_t* mask, void* stream);

/* Camera motion of B frames (lwdetr_gmc_create above; declared here, after the frame descriptors). */
LWDETR_API int lwdetr_gmc_estimate(lwdetr_gmc* g, const lwdetr_frame* frames, int B, const int32_t* stream_ids, double* motion,
                                   int32_t* status, int32_t* inliers, void* stream);
LWDETR_API int lwdetr_gmc_estimate_nv12(lwdetr_gmc* g, const lwdetr_frame_nv12* frames, int B, const int32_t* stream_ids,
                                        double* motion, int32_t* status, int32_t* inliers, void* stream);
/* Pyramids and corners only (lwdetr_gmc_observe above), for the frames tracked by flow. */
LWDETR_API int lwdetr_gmc_observe(lwdetr_gmc* g, const lwdetr_frame* frames, int B, const int32_t* stream_ids, void* stream);
LWDETR_API int lwdetr_gmc_observe_nv12(lwdetr_gmc* g, const lwdetr_frame_nv12* frames, int B, const int32_t* stream_ids, void* stream);

/* Detection crops for second-stage networks (ReID, attribute, vehicle-type or plate models, a second detector pass): each
 * box cut out of its frame on the device and resized to one out_h x out_w size, so no frame leaves the device and no host
 * resize runs.  The C composition of tracking by a crop-based ReID network (BoT-SORT's FastReID configuration), with no
 * synchronisation, so that it can be captured in one CUDA graph:
 *   lwdetr_forward_frames (or _nv12) -> lwdetr_query_best -> lwdetr_crop_select (threshold = track_thresh: the high entries,
 *   the only ones lwdetr_track_reid looks at) -> lwdetr_crops with N = B * k and the selection's device count -> the host's
 *   own fixed-batch ReID engine on the N crops (rows past the count are left as they were) -> lwdetr_scatter_rows with the
 *   same count -> lwdetr_track_reid.  tools/crop_spec.py restates this contract in numpy.
 * Crop rectangle of a box (x1, y1, x2, y2), fp32 xyxy in the pixels of an h x w frame: cx0 = clamp(floor(x1), 0, w),
 *   cx1 = clamp(floor(x2), 0, w), cy0 / cy1 likewise with h; the crop is rows [cy0, cy1) and columns [cx0, cx1).  It is
 *   valid when cx1 > cx0, cy1 > cy0 and all four coordinates are finite.  This is the truncation of BoT-SORT's
 *   tlbr.astype(int) slicing for boxes inside the frame; deviations: BoT-SORT clamps the end to w - 1 (here w: the last
 *   column and row stay reachable), and an empty slice makes it fail (here: an invalid crop).
 * Filters, per axis n_in (crop side) -> n_out, scale = n_in / n_out in fp32; horizontal pass, then vertical, both in fp32;
 *   the result is rounded half up (floor(v + 0.5)) to a level and clamped to [0, 255]:
 *   LWDETR_CROP_BILINEAR, cv2.resize(INTER_LINEAR) as BoT-SORT / FastReID use it: f = (o + 0.5) * scale - 0.5 (fp32, each
 *     operation rounded), s = floor(f), t = f - s; s < 0 gives s = 0, t = 0; s >= n_in - 1 gives the one tap n_in - 1;
 *     otherwise taps s, s + 1 with weights 1 - t, t.  No antialiasing.  Within one level of cv2, not equal to it: cv2 uses
 *     11-bit fixed-point weights (on random crops some 12 % of values differ by one level).
 *   LWDETR_CROP_ANTIALIAS: the triangle filter of lwdetr_frame (PIL / F.interpolate(antialias=True), the torchreid-style
 *     pipelines), at ANY downscale: boxes are device data, so nothing can be refused per crop, and a whole 8192-pixel frame
 *     to an 8-pixel side is computed exactly.  (The frame path's limit of 16x per axis does not apply here.)
 * Values: normalize != 0: (v / 255 - mean[c]) / std[c] as for lwdetr_frame; normalize = 0: the level v itself (FastReID
 *   normalises inside the model and takes 0..255).  RGB channel order.  NV12 frames: every source pixel converted as
 *   lwdetr_frame_nv12 states, chroma at (y >> 1, x >> 1) of the WHOLE frame, so crops at odd offsets are exact: the result
 *   is the RGB result of the converted frame.
 * lwdetr_crops / _nv12: frames a HOST array of B descriptors (B in [1, 1024]; dst_h / dst_w are not read; the caller may
 *   reuse it as soon as the call returns), sources as lwdetr_frame allows (sides in [8, 8192], any pitch and alignment);
 *   boxes fp32 [N, 4] and frame_index int32 [N] (the frame of each box; one outside [0, B) makes an invalid crop), N in
 *   [1, 65536]; count int32 [1] or NULL: crops at or past *count are not written (nor their flags); out [N, 3, out_h, out_w]
 *   NCHW of out_dtype (LWDETR_ET_F32, _F16 or _BF16), out sides in [8, 1024]; valid int8 [N]: 1 for a valid crop, 0 for an
 *   invalid one, whose output is zeros.  All DEVICE.  Asynchronous, nothing allocated or copied per call, safe to capture in
 *   a CUDA graph; stream-ordered like lwdetr_forward_frames.
 * lwdetr_crop_select: entries scores fp32 [B, k] and xyxy boxes fp32 [B, k, 4] (lwdetr_query_best's or lwdetr_tile_merge's
 *   output), frame_hw a HOST int32 [B][2] array of each frame's (height, width).  Keeps every entry with score > threshold
 *   whose crop is valid, in (frame, entry) order (an ordered compaction: deterministic): frame_of int32, entry int32 (the
 *   flat index b * k + j) and sel_boxes fp32 [., 4] of each, and *count, all DEVICE with room for B * k rows; rows past the
 *   count are not written.  B in [1, 1024], k >= 1.  Asynchronous, graph-safe.
 * lwdetr_scatter_rows: rows [N, D] of etype (LWDETR_ET_F32, _F16 or _BF16; row stride ld_rows >= D elements) -> out
 *   [num_out, D] dense of the same type: row i < *count (count NULL: i < N) goes to row entry[i], every other row is zeros
 *   (a zero embedding is "no appearance" for lwdetr_track_reid).  All DEVICE.  Asynchronous, graph-safe. */
enum { LWDETR_CROP_BILINEAR = 0, LWDETR_CROP_ANTIALIAS = 1 };
LWDETR_API int lwdetr_crops(const lwdetr_frame* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                            int out_h, int out_w, int filter, int normalize, const float mean[3], const float std[3], int out_dtype,
                            void* out, int8_t* valid, void* stream);
LWDETR_API int lwdetr_crops_nv12(const lwdetr_frame_nv12* frames, int B, const float* boxes, const int32_t* frame_index, int N,
                                 const int32_t* count, int out_h, int out_w, int filter, int normalize, const float mean[3],
                                 const float std[3], int out_dtype, void* out, int8_t* valid, void* stream);
LWDETR_API int lwdetr_crop_select(const float* scores, const float* boxes, int B, int k, const int32_t* frame_hw, float threshold,
                                  int32_t* frame_of, int32_t* entry, float* sel_boxes, int32_t* count, void* stream);
LWDETR_API int lwdetr_scatter_rows(int etype, const void* rows, int ld_rows, int D, const int32_t* entry, const int32_t* count, int N,
                                   void* out, int num_out, void* stream);

/* Drawing into the frames on the device (what DeepStream's nvdsosd and supervision's box, label, zone and pixelate annotators
 * do): boxes, labels, zones and their counts, and privacy pixelation, written IN PLACE into RGB or NV12 frames, so that
 * lwdetr_forward_frames -> lwdetr_query_best -> lwdetr_track -> lwdetr_zones_update -> lwdetr_annotate stays one chain with
 * no read-back, capturable in one CUDA graph.  tools/annotate_spec.py restates this contract in numpy.
 * lwdetr_annotate WRITES the pixels of the frames it is given, through the `data` (RGB) or `luma` / `chroma` (NV12) pointers
 * of the descriptors: their `const` is the promise of the readers (the forward, crops, motion), not of this call.  dst_h and
 * dst_w are ignored.  A byte that no primitive below covers is never written: not the pitch padding, not the rest of a
 * larger surface around a frame.
 * The object: lwdetr_annotator_create(num_classes in [1, 1024]) makes one device allocation on the current device (palette,
 *   class names, privacy mask and a fixed scratch for 32 frames of 1024 entries, reused group after group in stream order).
 *   Synchronous.  lwdetr_annotator_set_option (name, value), validated, takes effect at the next lwdetr_annotate (a CUDA
 *   graph keeps the options it was captured with):
 *     "thickness" [1, 32], default 2; "text_scale" [1, 8], default 2; "box_fill_alpha" [0, 256], default 0;
 *     "label" mask of LWDETR_LABEL_NAME | _ID | _SCORE, default all (0: no labels); "zone_fill_alpha" [0, 256], default 64;
 *     "zone_thickness" [1, 32], default 2; "privacy_block" 2, 4, 8, 16, 32 or 64, default 16.
 *   lwdetr_annotator_set_names: '\n'-separated class names for classes 0, 1, ... (at most num_classes, each at most 31
 *   characters; more is an error); a class without a name (or an empty one) is named by its id in decimal, the default for
 *   all.  lwdetr_annotator_set_palette: n in [1, 256] RGB triples.  Default palette (n = 16): (230,25,75) (60,180,75)
 *   (255,225,25) (0,130,200) (245,130,48) (145,30,180) (70,240,240) (240,50,230) (210,245,60) (250,190,212) (0,128,128)
 *   (220,190,255) (170,110,40) (255,250,200) (128,0,0) (170,255,195).  lwdetr_annotator_set_privacy: the labels in
 *   [0, num_classes) whose boxes are pixelated instead of drawn (n = 0: none, the default).  The three setters replace the
 *   table, synchronously: they wait for the object's last lwdetr_annotate and nothing else; not during a stream capture.
 *   Replays of a captured graph read the tables as they are.
 * lwdetr_annotate / _nv12: frames a HOST array of B descriptors, B in [1, 1024], sides in [8, 8192], any pitch and alignment,
 *   odd sizes allowed (the caller may reuse the array on return).  Entries [B, k], k in [1, 1024], DEVICE: scores fp32,
 *   labels int32, boxes fp32 xyxy [B, k, 4] in frame pixels; ids int32 or NULL; counts int32 [B] or NULL (k each).
 *   lwdetr_track's outputs as they are (k = max_out); with ids NULL, lwdetr_query_best / lwdetr_postprocess /
 *   lwdetr_tile_merge output.  zones (may be NULL) with stream_ids (HOST, one per frame, in [0, zones' num_streams)): each
 *   frame also gets its stream's lines and polygons, the line totals read from the zones object's device counters, and with
 *   occupancy (DEVICE int32 [B, 32], lwdetr_zones_update's output; may be NULL: no occupancy text) each polygon's count.
 *   The zones object must live on the annotator's device, and its calls must be ordered on the annotator's CUDA stream;
 *   lwdetr_zones_set and _export wait for the call, which reads the object.  Calls on one annotator must be ordered on one
 *   CUDA stream.  Asynchronous, nothing allocated or copied per call, safe to
 *   capture in a CUDA graph.
 * The drawing contract, per frame (h x w); float64 operations are rounded each on its own, in the order written:
 *   entry j is drawn when j < count, score >= score_threshold and its rectangle is valid: lwdetr_crops' rule,
 *     [clamp(floor(x1), 0, w), clamp(floor(x2), 0, w)) x [.. y ..), non-empty and from finite coordinates.
 *   colour: palette[i mod n] (non-negative remainder) with i = id, or the label when ids is NULL, or the line / polygon index.
 *   primitives, each with a colour, an alpha a in [0, 256] and a set of covered pixels (those in the frame only):
 *     rect fill: the rectangle; outline: the rectangle's pixels with x < x0 + t, x >= x1 - t, y < y0 + t or y >= y1 - t
 *       (t = thickness);
 *     segment A-B, radius r = t / 2 (t = zone_thickness), pixel centre (cx, cy) = (x + 0.5, y + 0.5): dx = bx - ax,
 *       dy = by - ay, L2 = dx * dx + dy * dy, qx = cx - ax, qy = cy - ay, u = qx * dx + qy * dy; d2 = qx * qx + qy * qy when
 *       u <= 0, else (cx - bx)^2 + (cy - by)^2 (each square a product) when u >= L2, else c * c / L2 with
 *       c = dx * qy - dy * qx; covered when d2 <= r * r;
 *     polygon fill: pixel centres inside by lwdetr_zones' even-odd rule, exactly (what is drawn inside is what Zones counts);
 *     text at origin (ox, oy), scale s: character i of the string occupies the cell [ox + 6 s i, ox + 6 s (i + 1)) x
 *       [oy, oy + 8 s); pixel (x, y) of it is glyph pixel (gx, gy) = ((x - ox) / s - 6 i, (y - oy) / s) of the 5x7 font of
 *       csrc/font5x7.cuh (characters outside 0x20..0x7E drawn as '?'); a text background is the rect fill of all cells.
 *   blending of colour c: RGB, per channel, out = (src * (256 - a) + c * a + 128) >> 8.  NV12: c is converted to Y'CbCr by
 *     the frame's colorspace, Y = clamp(((kYR R + kYG G + kYB B + 2^15) >> 16) + o, 0, 255) with o = 16 (limited range) or
 *     0 (full), Cb and Cr likewise with their rows and o = 128:
 *       colorspace               kYR    kYG    kYB    kUR     kUG     kUB    kVR    kVG     kVB
 *       LWDETR_CSC_BT601_LIMITED 16840  33058  6405   -9713   -19068  28781  28781  -24110  -4671
 *       LWDETR_CSC_BT709_LIMITED 11966  40254  4064   -6596   -22189  28784  28784  -26145  -2639
 *       LWDETR_CSC_BT601_FULL    19595  38470  7471   -11058  -21710  32768  32768  -27439  -5329
 *       LWDETR_CSC_BT709_FULL    13933  46871  4732   -7509   -25259  32768  32768  -29763  -3005
 *     (round(2^16 m) of the inverse m of each lwdetr_frame_nv12 row).  Luma is blended per covered pixel; a chroma sample with
 *     n > 0 of its in-frame 2x2 luma pixels covered by the primitive is blended with a' = (a * n + 2) >> 2, per primitive.
 *   privacy: the covered set is the union of the rectangles of the drawn entries whose label is in the privacy set; with
 *     P = privacy_block, the blocks of P x P pixels on the frame's grid (cut by its edges); each covered pixel takes the
 *     rounded mean (sum + cnt / 2) / cnt of its block's cnt covered pixels, per channel; NV12 luma the same, chroma on the
 *     chroma grid with blocks of P / 2 samples, a sample covered when its top-left luma pixel is.  Those entries get no box
 *     and no label.
 *   labels (option "label" != 0): the parts name (or the class id in decimal), "#id" (with ids) and the score as "0.xx" /
 *     "1.00" from p = clamp(floor(score * 100 + 0.5), 0, 100) in fp32, in that order, joined by one space.  A text of n
 *     characters at scale s is 6 s n x 8 s; its origin is (x0, y0 - 8 s) above the rectangle's top-left corner, or (x0, y0)
 *     just inside the top edge when y0 - 8 s < 0.  Background: the colour, opaque; text: black when the colour's grey
 *     (9798 R + 19235 G + 3735 B + 16384) >> 15 is at least 128, else white, opaque.
 *   zone texts: "in N out M" of each line (N, M its in and out totals over all classes) with its origin at
 *     (floor((ax + bx) * 0.5), floor((ay + by) * 0.5)); the occupancy of each polygon in decimal at (floor(x0), floor(y0)) of
 *     its first vertex (origins clamped to [-2^20, 2^20]); background and text as the labels', with the line's or polygon's colour.
 *   painter's order: 1. privacy; 2. polygon fills (zone_fill_alpha) in polygon order; 3. polygon outlines (each edge i ->
 *     i + 1 a segment of its own, in order), then lines (opaque); 4. box fills (box_fill_alpha; none at 0) in entry order,
 *     then box outlines (opaque) in entry order; 5. labels in entry order (background, then text); 6. line texts, then
 *     polygon texts. */
enum { LWDETR_LABEL_NAME = 1, LWDETR_LABEL_ID = 2, LWDETR_LABEL_SCORE = 4 };
typedef struct lwdetr_annotator lwdetr_annotator;
LWDETR_API int lwdetr_annotator_create(int num_classes, lwdetr_annotator** out);
LWDETR_API void lwdetr_annotator_destroy(lwdetr_annotator* a);
LWDETR_API int lwdetr_annotator_set_option(lwdetr_annotator* a, const char* name, int value);
LWDETR_API int lwdetr_annotator_set_names(lwdetr_annotator* a, const char* names);
LWDETR_API int lwdetr_annotator_set_palette(lwdetr_annotator* a, const uint8_t* rgb, int n);
LWDETR_API int lwdetr_annotator_set_privacy(lwdetr_annotator* a, const int32_t* classes, int n);
LWDETR_API int lwdetr_annotate(lwdetr_annotator* a, const lwdetr_frame* frames, int B, const int32_t* ids, const float* scores,
                               const int32_t* labels, const float* boxes, const int32_t* counts, int k, float score_threshold,
                               lwdetr_zones* zones, const int32_t* stream_ids, const int32_t* occupancy, void* stream);
LWDETR_API int lwdetr_annotate_nv12(lwdetr_annotator* a, const lwdetr_frame_nv12* frames, int B, const int32_t* ids, const float* scores,
                                    const int32_t* labels, const float* boxes, const int32_t* counts, int k, float score_threshold,
                                    lwdetr_zones* zones, const int32_t* stream_ids, const int32_t* occupancy, void* stream);

/* Multi-GPU init (SURVEY.md 8e): ONE ncclBroadcast of the packed weight arena from rank `root`, stream-ordered on
 * `stream`; the only collective of the path (images shard across ranks as independent replicas, nothing on the hot path).
 * Every rank first calls lwdetr_load_weights with tensors of the right shapes (any values on the non-root ranks): that
 * fixes the arena layout, which is a function of (config, dtype) only; the call verifies that the arena sizes agree.
 * The arena holds the raw pos_embed too, so position tables planned for other input sizes follow the root's weights.
 * `nccl_comm` is an ncclComm_t of a communicator the caller created (one rank per GPU); NCCL is resolved at run time
 * from the libnccl already loaded in the process (or dlopen("libnccl.so.2")), the library does not link it. */
LWDETR_API int lwdetr_broadcast_weights(lwdetr_handle* h, void* nccl_comm, int root, void* stream);
LWDETR_API int64_t lwdetr_weight_arena_bytes(lwdetr_handle* h);

/* options: "cuda_graph" (0/1, default 0: the caller opts in after warm-up), "fuse_layernorm" (0/1, default 1), "pdl" (0/1, default 1: programmatic dependent
 * launch of every kernel; process-wide) */
LWDETR_API int lwdetr_set_option(lwdetr_handle* h, const char* name, int value);

/* Debug captures (tests): after the op labelled `label` runs in the next forward, its output is copied to
 * the HOST buffer dst as fp32 (row-major, dense).  lwdetr_capture_result returns the element count (-1: no such output,
 * -2: larger than capacity).  Ops that write more than one buffer expose the others as "<label>.<name>":
 *   mask_setup              proposals [B*S, 4];  mask_setup.invalid, mask_setup.pad [B*S] (0 / 1);  mask_setup.valid_ratio [B*L, 2] (w, h)
 *   topk                    the selected memory rows [B*nq] (int32, exact in fp32)
 *   gather_topk             the selected encoder rows [B*nq, hidden_dim];  gather_topk.enc_logits [B*nq, num_classes]
 *   query_init              the decoder reference boxes [B*nq, 4];  query_init.box_ts [B*nq, 4] (enc_outputs boxes);
 *                           query_init.sine [B*nq, 2*hidden_dim] (the sine embedding of the reference, compute dtype)
 * Captures run the forward eagerly and synchronise after every captured op; without any, nothing of this is done. */
LWDETR_API int lwdetr_add_capture(lwdetr_handle* h, const char* label, float* dst, int64_t capacity);
LWDETR_API int64_t lwdetr_capture_result(lwdetr_handle* h, int index);
LWDETR_API void lwdetr_clear_captures(lwdetr_handle* h);

/* lwdetr_last_hidden: the last forward's final-layer decoder hidden state (after the decoder's output norm: the rows
 * class_embed and bbox_embed read), [B, num_queries, hidden_dim] in the compute dtype (fp16 in the e4m3 mode), into DEVICE
 * dst with a row stride of ld_dst >= hidden_dim elements.  Ordered on `stream` like the forward's own result copies, so
 * call it on the forward's stream; the source is valid until the next forward.  It adds nothing to the forward's schedule
 * or its CUDA graphs.  Row q of frame b is the feature of query q, i.e. of lwdetr_query_best's entry q: the built-in
 * appearance embedding for lwdetr_track_reid (emb_dtype LWDETR_ET_F16 or _BF16). */
LWDETR_API int lwdetr_last_hidden(lwdetr_handle* h, void* dst, int ld_dst, void* stream);

/* Schedule introspection / per-op timing of the last planned batch size. */
LWDETR_API int lwdetr_num_ops(lwdetr_handle* h);
LWDETR_API const char* lwdetr_op_label(lwdetr_handle* h, int i);
LWDETR_API int lwdetr_op_cost(lwdetr_handle* h, int i, double* flops, double* bytes);
LWDETR_API int lwdetr_profile_ops(lwdetr_handle* h, int iters, float* ms_per_op, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LWDETR_B200_H_ */
