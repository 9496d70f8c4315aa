// Multi-scale deformable attention forward (see msda.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "gemm_tc.h"

namespace lwb {

static constexpr int MSDA_MAX_LEVELS = 4;
static constexpr int MSDA_MAX_BANDS = 16;
static constexpr int MSDA_D = 16;             // channels per head on the model path (d / ca_heads for every released config)

// ---- model path: fused softmax + location math + gather over a HEAD-MAJOR value tensor staged through shared memory
struct MsdaBand {
  int level;        // feature level of the band
  int row0;         // first image row held in shared memory
  int own0, own1;   // the band handles the samples whose floor(y) lies in [own0, own1] (rows floor(y), floor(y)+1 are both staged)
  int tok0;         // first token of the band inside the (image, head) slab
  int bytes;        // bytes staged (rows * W * 32)
};

struct MsdaArgs {
  const void* value;        // 16-bit head-major [B][v_b_stride]: (image b, head m, token s, channel c) at b*v_b_stride + m*S*16 + s*16 + c
  long long v_b_stride;     // elements between images (= slices * M * S * 16 when several layers' values share one buffer)
  const void* offs_logits;  // 16-bit [B*nq, ld_ol]: [M*L*P*2 sampling offsets | M*L*P attention logits]
  int ld_ol;
  const float* ref;         // fp32 [B*nq, 4] reference boxes (cx, cy, w, h), un-sigmoided space
  const float* valid_ratio; // fp32 [B, L, 2] (w, h) valid ratios of a padded batch (transformer.py:189-196, 352-353) or null (= 1)
  void* out;                // 16-bit [B*nq, ld_out]
  int ld_out;
  int batch, nq, heads, levels, points, S;
  int lvl_h[MSDA_MAX_LEVELS], lvl_w[MSDA_MAX_LEVELS], lvl_start[MSDA_MAX_LEVELS];
  int nbands;
  MsdaBand bands[MSDA_MAX_BANDS];
};

// fills nbands / bands from the level table; nbands = 0 when a level cannot be staged (row wider than half a stage, more
// than 8192 tokens, more than MSDA_MAX_BANDS bands): msda_launch then takes the direct-gather kernel.  Returns -2 for an
// invalid level table.
int msda_plan(MsdaArgs* a);
int msda_launch(int dtype, const MsdaArgs& a, cudaStream_t st);

// ---- operator boundary: the reference op's own signature (ms_deform_attn.h:19-35), token-major value, explicit
// sampling locations and attention weights; element type fp32 / fp16 / bf16 for value, loc, weight and out alike.
enum : int { MSDA_ET_F32 = 0, MSDA_ET_F16 = 1, MSDA_ET_BF16 = 2 };
struct MsdaOpArgs {
  const void* value;                 // [B, S, M, D]
  const int64_t* spatial_shapes;     // DEVICE [L, 2] (H, W)
  const int64_t* level_start_index;  // DEVICE [L]
  const void* sampling_loc;          // [B, Lq, M, L, P, 2] normalised (x, y)
  const void* attn_weight;           // [B, Lq, M, L, P]
  void* out;                         // [B, Lq, M*D]
  int B, S, M, D, Lq, L, P;
};
int msda_op_launch(int etype, const MsdaOpArgs& a, cudaStream_t st);
// fp32 backward of the operator: grad_value [B,S,M,D] (zeroed here), grad_loc [B,Lq,M,L,P,2], grad_aw [B,Lq,M,L,P]
int msda_op_backward_launch(const MsdaOpArgs& a, const float* grad_out, float* grad_value, float* grad_loc, float* grad_aw, cudaStream_t st);

}  // namespace lwb
