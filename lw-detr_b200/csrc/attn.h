// Fused attention core (see attn.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "gemm_tc.h"   // DT_* codes

namespace lwb {

struct AttnArgs {
  const void* q; const void* k; const void* v;   // 16-bit row-major, head h at columns [h*dh, (h+1)*dh)
  int ldq, ldk, ldv;
  void* o; int ldo;
  int seqlen;        // tokens per sequence (100 window / 1600 global / nq decoder)
  int nseq;          // number of sequences; token (s, t) is matrix row s*seqlen + t
  int heads;
  float scale_log2;  // softmax scale * log2(e)
};

// The kernel instance attention_launch runs for a set of arguments (codes as LWDETR_ATTN_* of include/lwdetr_b200.h).
enum { ATTN_WG = 0, ATTN_MMA = 1, ATTN_MMA_SHORT = 2 };
struct AttnPlan {
  int kernel = ATTN_WG;
  int warps = 0;            // attn_kernel's warps per CTA (4 or 8), 0 for the other kernels
  uint32_t poly_mask = 0;   // the n-tiles whose exponentials take the polynomial exp2 (the kernel's PM argument)
  int C = 0;                // packed path: column offset of k in the qkv matrix (heads * dh)
};

// Checks the arguments and chooses the kernel, calling no CUDA API: 0, or -2 with *err naming the violated limit.
int attention_plan(int dtype, const AttnArgs& a, int dh, AttnPlan* plan, std::string* err);
// Launches the planned kernel; a plan that attention_plan did not accept for these arguments is undefined.
int attention_run(int dtype, const AttnArgs& a, int dh, const AttnPlan& plan, cudaStream_t st);
// attention_plan + attention_run (-2: arguments refused).
int attention_launch(int dtype, const AttnArgs& a, int dh, cudaStream_t st);

}  // namespace lwb
