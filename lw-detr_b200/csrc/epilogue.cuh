// Device helpers shared by the GEMM epilogues (gemm_tc.cu) and the fused ViT MLP (mlp.cu), so that both compute the
// LayerNorm fold, the GELU and the row statistics with the same instructions in the same order.
#pragma once
#include "ptx.cuh"

namespace lwb {

// Exact (erf) GELU, nn.GELU() default used by timm's Mlp (vit.py:184).  gelu(x) = x*Phi(x) with
// Phi(-|x|) = 0.5*erfc(|x|/sqrt2) from Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7):
//   gelu(x) = max(x, 0) - |x| * [0.5 * poly(t) * exp(-x^2/2)],  t = 1 / (1 + p|x|/sqrt2)
// 14 instructions incl. 2 MUFU instead of ~30 for erff(); max abs deviation from the erff form 2.2e-7.
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.2316418882f, ax, 1.0f)));       // 0.3275911 / sqrt(2)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * -0.72134752044448170f));        // exp(-x^2/2)
  float p = fmaf(0.5307027145f, t, -0.7265760135f);                                          // 0.5 * A&S coefficients
  p = fmaf(p, t, 0.7107068705f);
  p = fmaf(p, t, -0.142248368f);
  p = fmaf(p, t, 0.127414796f);
  return fmaf(-ax * t, p * e, fmaxf(x, 0.f));
}

// The same exact-erf GELU for a PAIR of values (ptx.cuh f2_*), without the MUFU: gelu(x) = x * (0.5 + xc * q(xc^2)), xc = x
// clamped to [-4.5, 4.5], q a degree-9 polynomial fitted to erf(x/sqrt2) / (2x) (weighted least squares at Chebyshev nodes;
// fp32 Horner: max |error| 7.4e-5 at |x| ~ 4.46 where gelu ~ 4.46, < 1e-5 for |x| < 3 (tests/test_numerics_cpu.py); beyond the clamp Phi(-4.5) = 3.4e-6
// multiplies x).  FMA pipe only, where gelu_erf spends two MUFU operations per element.
__device__ __forceinline__ uint64_t gelu_erf2(uint64_t x2) {
  float x0, x1;
  f2_unpack(x2, x0, x1);
  const uint64_t xc = f2_pack(fminf(fmaxf(x0, -4.5f), 4.5f), fminf(fmaxf(x1, -4.5f), 4.5f));
  const uint64_t u = f2_mul(xc, xc);
#define LWB_K2(v) f2_pack(v, v)
  uint64_t q = f2_fma(LWB_K2(-1.3369040159e-12f), u, LWB_K2(1.6336444415e-10f));
  q = f2_fma(q, u, LWB_K2(-8.9213697499e-09f));
  q = f2_fma(q, u, LWB_K2(2.8944761772e-07f));
  q = f2_fma(q, u, LWB_K2(-6.2733902842e-06f));
  q = f2_fma(q, u, LWB_K2(9.7063541348e-05f));
  q = f2_fma(q, u, LWB_K2(-1.1183810776e-03f));
  q = f2_fma(q, u, LWB_K2(9.8202145566e-03f));
  q = f2_fma(q, u, LWB_K2(-6.6317755718e-02f));
  q = f2_fma(q, u, LWB_K2(3.9887377948e-01f));
  const uint64_t t = f2_fma(xc, q, LWB_K2(0.5f));
#undef LWB_K2
  return f2_mul(x2, t);
}

// keeps the compiler from moving uses of the accumulators across the asynchronous MMAs' wait
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ float4 lds128(const float* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(smem_u32(p)));
  return v;
}

// LayerNorm statistics of one row from its equal-width partials (sum_p, M2_p), one float2 per partial, as written by a
// statistics producer (gemm_tc.cu EP_RESID): mean = sum(sum_p) / C, var = [sum(M2_p) + n_p * sum((sum_p / n_p - mean)^2)] / C
// (Chan et al.); part_n = n_p = C / parts, part_inv_n = 1 / n_p.
__device__ __forceinline__ void ln_row_stats(const float2* q_row, int parts, float part_n, float part_inv_n, float inv_c, float eps,
                                             float& mean, float& rstd) {
  float s1 = 0.f, m2 = 0.f;
  for (int i = 0; i < parts; ++i) s1 += __ldg(q_row + i).x;
  mean = s1 * inv_c;
  for (int i = 0; i < parts; ++i) {
    const float2 q = __ldg(q_row + i);
    const float dm = q.x * part_inv_n - mean;
    m2 += q.y + part_n * dm * dm;
  }
  rstd = rsqrtf(m2 * inv_c + eps);
}

}  // namespace lwb
