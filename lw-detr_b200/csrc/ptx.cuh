// Thin inline-PTX wrappers for the sm_90a features the LW-DETR kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma shared-memory descriptors (the MMAs themselves are in wgmma.cuh)
// and wide global accesses.  Everything here is device-only and header-only.
#pragma once
#include <cuda.h>          // CUtensorMap (types only, libcuda is never linked)
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace lwb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe: has the phase with this parity completed?
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug must surface as a trap (CUDA error), never as a hung GPU.  The spin loop is kept
// to try_wait + counter + branch (try_wait itself suspends the thread for a while): waiting warps share issue
// slots with the working ones, so a clock read / 64-bit compare per iteration would be a large share of what a waiting
// kernel executes.  The clock is only consulted every 4096 failed tries.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 4095u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000LL) __trap();   // ~2 s at 2 GHz
    }
  }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, "
      "%7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}

// 1-D bulk copy global -> shared (no tensor map): `bytes` % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}


// ----------------------------------------------------------------------------- wgmma operands
// Shared-memory matrix descriptor of a 16-bit tile whose rows are `pitch` bytes (32 / 64 / 128) written by TMA with the
// swizzle of the same span: 8-row groups `8 * pitch` bytes apart (stride byte offset), leading byte offset unused (one
// swizzle span covers the whole row).  The same descriptor serves a K-major operand (rows = M or N) and an MN-major
// one (rows = K, transposed by the tensor core).  Advancing 16 elements along a K-major row adds 32 bytes (+2).
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t pitch) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((8 * pitch) >> 4) << 32;
  d |= static_cast<uint64_t>(pitch == 128 ? 1 : (pitch == 64 ? 2 : 3)) << 62;   // SWIZZLE_128B / 64B / 32B
  return d;
}
template <int N> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ----------------------------------------------------------------------------- fp32 pairs
// Two fp32 values carried in a 64-bit register pair (epilogues and softmax loops work on adjacent columns); sm_90 has no
// packed fp32x2 arithmetic, so every operation is two scalar instructions.
__device__ __forceinline__ uint64_t f2_pack(float a, float b) {
  uint64_t r;
  asm("mov.b64 %0, {%1,%2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ void f2_unpack(uint64_t v, float& a, float& b) { asm("mov.b64 {%0,%1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  f2_unpack(c, c0, c1);
  return f2_pack(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ uint64_t f2_add(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(a0 + b0, a1 + b1);
}
__device__ __forceinline__ uint64_t f2_mul(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(a0 * b0, a1 * b1);
}


// 2^(s*c - m) for a PAIR of scores without the MUFU (the exp-bound attention kernels can move a fraction of their exponentials
// to the FMA pipe): y = s*c - m by one FMA per score (the argument the MUFU path feeds ex2), t = round(y) + 1.5*2^23 by one
// add, the fraction f = y - round(y) in [-0.5, 0.5] by two more, a degree-3 polynomial for 2^f (max relative error 7.5e-5 on
// [-0.5, 0.5], an order of magnitude below the 16-bit rounding of P) and the integer part added into the exponent field.
// y is formed before the magic add: 1.5*2^23 - m rounded to fp32 (ulp 1 there) would drop the fraction of m and leave f in
// [-1, 1], where the polynomial is off by up to 1.2e-2.  The raw scores are clamped at smin = (m - 125)/c first: below
// that 2^x is 0 for every purpose here, and an unclamped argument would wrap the exponent field.
__device__ __forceinline__ void exp2_poly2(float s0, float s1, float smin, uint64_t c2, uint64_t negm2, float& e0, float& e1) {
  constexpr float kMagic = 12582912.f;   // 1.5 * 2^23
  const uint64_t s2 = f2_pack(fmaxf(s0, smin), fmaxf(s1, smin));
  const uint64_t y2 = f2_fma(s2, c2, negm2);
  const uint64_t t2 = f2_add(y2, f2_pack(kMagic, kMagic));
  const uint64_t r2 = f2_add(t2, f2_pack(-kMagic, -kMagic));
  const uint64_t f2 = f2_fma(r2, f2_pack(-1.f, -1.f), y2);
  uint64_t p2 = f2_fma(f2, f2_pack(0.05517164617776871f, 0.05517164617776871f), f2_pack(0.2426111251115799f, 0.2426111251115799f));
  p2 = f2_fma(p2, f2, f2_pack(0.6932609677314758f, 0.6932609677314758f));
  p2 = f2_fma(p2, f2, f2_pack(0.9999280571937561f, 0.9999280571937561f));
  float p0, p1, t0, t1;
  f2_unpack(p2, p0, p1);
  f2_unpack(t2, t0, t1);
  e0 = __int_as_float(__float_as_int(p0) + (__float_as_int(t0) << 23));
  e1 = __int_as_float(__float_as_int(p1) + (__float_as_int(t1) << 23));
}

// ----------------------------------------------------------------------------- 16/32-byte global access
struct __align__(16) U4 { uint32_t x, y, z, w; };
struct __align__(32) U8 { uint32_t v[8]; };

// 32 bytes as two 16-byte accesses (sm_90 has no 256-bit global load / store)
__device__ __forceinline__ U8 ldg256(const void* p) {
  U8 r;
  asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]) : "l"(p));
  asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%4+16];" : "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7]) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg256(void* p, const U8& r) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(r.v[0]), "r"(r.v[1]), "r"(r.v[2]), "r"(r.v[3]) : "memory");
  asm volatile("st.global.v4.b32 [%0+16], {%1,%2,%3,%4};" ::"l"(p), "r"(r.v[4]), "r"(r.v[5]), "r"(r.v[6]), "r"(r.v[7]) : "memory");
}


// ----------------------------------------------------------------------------- 16-bit conversions
template <typename T> struct Cvt;
template <> struct Cvt<__half> {
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack(uint32_t u) {
    return __half22float2(*reinterpret_cast<__half2*>(&u));
  }
  static __device__ __forceinline__ float to_f(__half h) { return __half2float(h); }
  static __device__ __forceinline__ __half from_f(float f) { return __float2half_rn(f); }
  static constexpr bool is_bf16 = false;
};
template <> struct Cvt<__nv_bfloat16> {
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static __device__ __forceinline__ float2 unpack(uint32_t u) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  }
  static __device__ __forceinline__ float to_f(__nv_bfloat16 h) { return __bfloat162float(h); }
  static __device__ __forceinline__ __nv_bfloat16 from_f(float f) { return __float2bfloat16_rn(f); }
  static constexpr bool is_bf16 = true;
};

}  // namespace lwb
