// Memory-bound helper kernels of the LW-DETR forward: LayerNorm, patch gathering, row max, per-image
// top-k, gathers, box re-parameterisation and the sine query embedding.  All are HBM-bound; they use
// 16/32-byte accesses, one warp per row where a row reduction is needed, and fp32 math throughout.
#include "rowops.h"
#include "launch.h"
#include "postproc.cuh"
#include "ptx.cuh"

#include <math_constants.h>

namespace lwb {

// ----------------------------------------------------------------------------------- LayerNorm
// y = (x - mean) / sqrt(var + eps) * w + b per row (biased variance), one warp per row, row in
// registers.  Serves nn.LayerNorm in the ViT (eps 1e-6, vit.py:198,217), the channel-first
// LayerNorm of the projector on NHWC rows (projector.py:21-47) and the decoder norms (eps 1e-5).
// Optional: rows flagged in `row_flag` take `override_vec` as input (masked two-stage memory rows,
// transformer.py:116-123); optional second output y2 = y + add_src (decoder: tgt + query_pos).
template <typename T, int CHUNKS, int RPW>   // CHUNKS = ceil(C / 256): 8-element chunks per lane; RPW rows per warp, loaded together
__global__ void __launch_bounds__(256) layernorm_kernel(const LayerNormArgs p) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row0 = (static_cast<long long>(blockIdx.x) * 8 + warp) * RPW;
  if (row0 >= p.rows) return;
  const int nchunk = p.C >> 3;
  float v[RPW][CHUNKS][8];
  bool live[RPW];
  // ---- every load of the warp's RPW rows is in flight before the first reduction (memory-level parallelism: the kernel
  // is latency-bound, one 16-byte load per lane and row otherwise)
#pragma unroll
  for (int r = 0; r < RPW; ++r) {
    const long long row = row0 + r;
    live[r] = row < p.rows;
    const bool ovr = live[r] && p.row_flag != nullptr && p.row_flag[row % p.flag_mod] != 0;
    const T* x = reinterpret_cast<const T*>(p.x) + (live[r] ? row : row0) * p.ldx;
#pragma unroll
    for (int i = 0; i < CHUNKS; ++i) {
      const int c = lane + i * 32;
      if (c < nchunk) {
        if (ovr) {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[r][i][j] = p.override_vec[c * 8 + j];
        } else {
          const U4 u = *reinterpret_cast<const U4*>(x + c * 8);
          const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = Cvt<T>::unpack(w4[j]);
            v[r][i][2 * j] = f.x;
            v[r][i][2 * j + 1] = f.y;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[r][i][j] = 0.f;
      }
    }
  }
  float wv[CHUNKS][8], bv[CHUNKS][8];
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c = lane + i * 32;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      wv[i][j] = c < nchunk ? __ldg(p.w + c * 8 + j) : 0.f;
      bv[i][j] = c < nchunk ? __ldg(p.b + c * 8 + j) : 0.f;
    }
  }
#pragma unroll
  for (int r = 0; r < RPW; ++r) {
    if (!live[r]) continue;
    const long long row = row0 + r;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < CHUNKS; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[r][i][j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / p.C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < CHUNKS; ++i) {
      if (lane + i * 32 < nchunk) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[r][i][j] - mean;
          q += d * d;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / p.C + p.eps);
    const long long yrow = p.y_group > 0 ? (row / p.y_group) * p.y_group_stride + p.y_row_off + row % p.y_group : row;
    T* y = reinterpret_cast<T*>(p.y) + yrow * p.ldy;
#pragma unroll
    for (int i = 0; i < CHUNKS; ++i) {
      const int c = lane + i * 32;
      if (c < nchunk) {
        float o8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o8[j] = (v[r][i][j] - mean) * rstd * wv[i][j] + bv[i][j];
        U4 o;
        o.x = Cvt<T>::pack(o8[0], o8[1]); o.y = Cvt<T>::pack(o8[2], o8[3]);
        o.z = Cvt<T>::pack(o8[4], o8[5]); o.w = Cvt<T>::pack(o8[6], o8[7]);
        *reinterpret_cast<U4*>(y + c * 8) = o;
        if (p.y3 != nullptr) {                      // keep the rounded y for the chained LayerNorm below
          const uint32_t w4[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = Cvt<T>::unpack(w4[j]);
            v[r][i][2 * j] = f.x;
            v[r][i][2 * j + 1] = f.y;
          }
        }
        if (p.y2 != nullptr) {
          const T* a = reinterpret_cast<const T*>(p.add_src) + row * p.ld_add + c * 8;
          const U4 u = *reinterpret_cast<const U4*>(a);
          const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
          uint32_t o2[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = Cvt<T>::unpack(w4[j]);
            // add to the ROUNDED y so that y2 == y + add exactly as a 16-bit consumer would compute it
            const float2 yr = Cvt<T>::unpack(j == 0 ? o.x : j == 1 ? o.y : j == 2 ? o.z : o.w);
            o2[j] = Cvt<T>::pack(yr.x + f.x, yr.y + f.y);
          }
          U4 oo; oo.x = o2[0]; oo.y = o2[1]; oo.z = o2[2]; oo.w = o2[3];
          *reinterpret_cast<U4*>(reinterpret_cast<T*>(p.y2) + row * p.ldy2 + c * 8) = oo;
        }
      }
    }
    if (p.y3 != nullptr) {
      // chained LayerNorm of the rounded y (exactly what a separate launch reading y would compute)
      float s3 = 0.f;
#pragma unroll
      for (int i = 0; i < CHUNKS; ++i)
        if (lane + i * 32 < nchunk) {
#pragma unroll
          for (int j = 0; j < 8; ++j) s3 += v[r][i][j];
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s3 += __shfl_xor_sync(0xffffffffu, s3, o);
      const float mean3 = s3 / p.C;
      float q3 = 0.f;
#pragma unroll
      for (int i = 0; i < CHUNKS; ++i)
        if (lane + i * 32 < nchunk) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float dd = v[r][i][j] - mean3;
            q3 += dd * dd;
          }
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q3 += __shfl_xor_sync(0xffffffffu, q3, o);
      const float rstd3 = rsqrtf(q3 / p.C + p.eps3);
      T* y3 = reinterpret_cast<T*>(p.y3) + row * p.ldy3;
#pragma unroll
      for (int i = 0; i < CHUNKS; ++i) {
        const int c = lane + i * 32;
        if (c < nchunk) {
          float o8[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) o8[j] = (v[r][i][j] - mean3) * rstd3 * __ldg(p.w3 + c * 8 + j) + __ldg(p.b3 + c * 8 + j);
          U4 o;
          o.x = Cvt<T>::pack(o8[0], o8[1]); o.y = Cvt<T>::pack(o8[2], o8[3]);
          o.z = Cvt<T>::pack(o8[4], o8[5]); o.w = Cvt<T>::pack(o8[6], o8[7]);
          *reinterpret_cast<U4*>(y3 + c * 8) = o;
        }
      }
    }
  }
}

// rows per warp: 4 when there are enough rows to keep every SM busy with a quarter of the warps (and C <= 512), else 1
int layernorm_rows_per_warp(long long rows, int C) {
  return (C + 255) / 256 <= 2 && rows >= 8LL * 4 * 2 * current_device_sms() ? 4 : 1;
}

template <typename T>
static int ln_dispatch(const LayerNormArgs& a, cudaStream_t st) {
  const int chunks = (a.C + 255) / 256;
  const bool many = layernorm_rows_per_warp(a.rows, a.C) == 4;
  const unsigned grid4 = static_cast<unsigned>((a.rows + 31) / 32), grid1 = static_cast<unsigned>((a.rows + 7) / 8);
  if (chunks == 1) { if (many) launch_k(layernorm_kernel<T, 1, 4>, dim3(grid4), dim3(256), 0, st, a); else launch_k(layernorm_kernel<T, 1, 1>, dim3(grid1), dim3(256), 0, st, a); }
  else if (chunks == 2) { if (many) launch_k(layernorm_kernel<T, 2, 4>, dim3(grid4), dim3(256), 0, st, a); else launch_k(layernorm_kernel<T, 2, 1>, dim3(grid1), dim3(256), 0, st, a); }
  else if (chunks == 3) launch_k(layernorm_kernel<T, 3, 1>, dim3(grid1), dim3(256), 0, st, a);
  else if (chunks == 4) launch_k(layernorm_kernel<T, 4, 1>, dim3(grid1), dim3(256), 0, st, a);
  else return -2;
  return static_cast<int>(cudaGetLastError());
}
int layernorm_launch(int dtype, const LayerNormArgs& a, cudaStream_t st) {
  if (a.C % 8 != 0 || a.C > 1024) return -2;
  return dtype == DT_BF16 ? ln_dispatch<__nv_bfloat16>(a, st) : ln_dispatch<__half>(a, st);
}

// ----------------------------------------------------------------------------------- LayerNorm -> e4m3
// The e4m3 mode's LayerNorm in front of qkv / fc1: per row x^ = (x - mean) * rstd in fp32 with the affine NOT applied (it is
// folded into the e4m3 weights at load), a = max|x^|, q = e4m3(x^ * (448 / a)) (round to nearest even, saturating) and
// row_scale = a / 448 (a = 0: both factors 1).  One warp per row, row in registers.  The row is summed SHIFTED by its first
// value (x - x0 is exact in fp32 for 16-bit x), so a row whose mean is large against its spread keeps its x^ accurate.
template <int CHUNKS>
__global__ void __launch_bounds__(256) layernorm_e4m3_kernel(const void* __restrict__ xp, int ldx, long long rows, int C, float eps,
                                                             uint8_t* __restrict__ q, int ldq, float* __restrict__ row_scale) {
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * 8 + warp;
  if (row >= rows) return;
  const int nchunk = C >> 3;
  const __half* x = reinterpret_cast<const __half*>(xp) + row * ldx;
  const float x0 = __half2float(x[0]);
  float v[CHUNKS][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c = lane + i * 32;
    if (c < nchunk) {
      const U4 u = *reinterpret_cast<const U4*>(x + c * 8);
      const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = Cvt<__half>::unpack(w4[j]);
        v[i][2 * j] = f.x - x0;
        v[i][2 * j + 1] = f.y - x0;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float dm = s / C;                      // mean - x0
  float m2 = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i)
    if (lane + i * 32 < nchunk) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[i][j] -= dm;
        m2 = fmaf(v[i][j], v[i][j], m2);
      }
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m2 += __shfl_xor_sync(0xffffffffu, m2, o);
  const float rstd = 1.f / sqrtf(m2 / C + eps);
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i)
    if (lane + i * 32 < nchunk) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        v[i][j] *= rstd;
        amax = fmaxf(amax, fabsf(v[i][j]));
      }
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float inv = amax > 0.f ? 448.f / amax : 1.f;
  if (lane == 0) row_scale[row] = amax > 0.f ? amax / 448.f : 1.f;
  uint8_t* qrow = q + row * ldq;
#pragma unroll
  for (int i = 0; i < CHUNKS; ++i) {
    const int c = lane + i * 32;
    if (c < nchunk) {
      uint32_t w2[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint16_t lo, hi;
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(v[i][4 * h + 1] * inv), "f"(v[i][4 * h] * inv));
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(v[i][4 * h + 3] * inv), "f"(v[i][4 * h + 2] * inv));
        w2[h] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
      }
      *reinterpret_cast<uint2*>(qrow + c * 8) = make_uint2(w2[0], w2[1]);
    }
  }
}

int layernorm_e4m3_launch(const void* x, int ldx, long long rows, int C, float eps, uint8_t* q, int ldq, float* row_scale, cudaStream_t st) {
  if (C % 8 != 0 || C < 8 || C > 1024 || ldx % 8 != 0 || ldq % 8 != 0 || ldx < C || ldq < C || rows < 1) return -2;
  const int chunks = (C + 255) / 256;
  const dim3 grid(static_cast<unsigned>((rows + 7) / 8));
  if (chunks == 1) launch_k(layernorm_e4m3_kernel<1>, grid, dim3(256), 0, st, x, ldx, rows, C, eps, q, ldq, row_scale);
  else if (chunks == 2) launch_k(layernorm_e4m3_kernel<2>, grid, dim3(256), 0, st, x, ldx, rows, C, eps, q, ldq, row_scale);
  else if (chunks == 3) launch_k(layernorm_e4m3_kernel<3>, grid, dim3(256), 0, st, x, ldx, rows, C, eps, q, ldq, row_scale);
  else launch_k(layernorm_e4m3_kernel<4>, grid, dim3(256), 0, st, x, ldx, rows, C, eps, q, ldq, row_scale);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- patch gather
// Image [B,3,H,W] (fp32 or 16-bit, NCHW) -> A [B*GH*GW, 3*256] 16-bit with rows in WINDOW-MAJOR token
// order and k = c*256 + py*16 + px, so that the 16x16/s16 patch-embedding conv (vit.py:79-83)
// becomes one wgmma GEMM whose output is already in the layout of vit.py:353-358: 4x4 windows of
// (GH/4) x (GW/4) tokens, windows enumerated row-major.
__device__ __forceinline__ void window_token_yx(int rem, int GH, int GW, int* Y, int* X) {
  const int wh = GH / 4, ww = GW / 4, wsz = wh * ww;
  const int win = rem / wsz, t = rem % wsz;
  *Y = (win >> 2) * wh + t / ww;
  *X = (win & 3) * ww + t % ww;
}

template <typename T, typename TIn>
__global__ void __launch_bounds__(256) patch_gather_kernel(const TIn* __restrict__ img, T* __restrict__ A, int B, int H, int W) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const int GH = H / 16, GW = W / 16, T_ = GH * GW;
  const long long total = static_cast<long long>(B) * T_ * 48;      // (row, c, py)
  const long long id = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const long long rows = static_cast<long long>(B) * T_;
  const long long r = id % rows;
  const int cp = static_cast<int>(id / rows);
  const int c = cp / 16, py = cp % 16;
  const int b = static_cast<int>(r / T_), rem = static_cast<int>(r % T_);
  int Y, X;
  window_token_yx(rem, GH, GW, &Y, &X);
  const TIn* src = img + ((static_cast<long long>(b) * 3 + c) * H + (Y * 16 + py)) * W + X * 16;
  float f[16];
  if constexpr (sizeof(TIn) == 4) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(src) + j);
      f[4 * j] = q.x; f[4 * j + 1] = q.y; f[4 * j + 2] = q.z; f[4 * j + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) f[j] = Cvt<T>::to_f(reinterpret_cast<const T*>(src)[j]);
  }
  U8 o;
#pragma unroll
  for (int j = 0; j < 8; ++j) o.v[j] = Cvt<T>::pack(f[2 * j], f[2 * j + 1]);
  stg256(A + r * 768 + c * 256 + py * 16, o);
}

int patch_gather_launch(int dtype, const void* img, int img_is_fp32, void* A, int B, int H, int W, cudaStream_t st) {
  if (H % 64 != 0 || W % 64 != 0 || H < 64 || W < 64) return -2;
  const long long total = static_cast<long long>(B) * (H / 16) * (W / 16) * 48;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (dtype == DT_BF16) {
    if (img_is_fp32) launch_k(patch_gather_kernel<__nv_bfloat16, float>, dim3(grid), dim3(256), 0, st, static_cast<const float*>(img), static_cast<__nv_bfloat16*>(A), B, H, W);
    else launch_k(patch_gather_kernel<__nv_bfloat16, __nv_bfloat16>, dim3(grid), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(img), static_cast<__nv_bfloat16*>(A), B, H, W);
  } else {
    if (img_is_fp32) launch_k(patch_gather_kernel<__half, float>, dim3(grid), dim3(256), 0, st, static_cast<const float*>(img), static_cast<__half*>(A), B, H, W);
    else launch_k(patch_gather_kernel<__half, __half>, dim3(grid), dim3(256), 0, st, static_cast<const __half*>(img), static_cast<__half*>(A), B, H, W);
  }
  return static_cast<int>(cudaGetLastError());
}

// uint8 HWC image [B, S, S, 3] (what an image decoder + resize produce; demo/demo.py:146-159 then runs ToTensor -> /255 and
// Normalize(mean, std), datasets/transforms.py:223-252) -> the same 16-bit patch matrix.  The normalisation is fused
// into the gather: the fp32 NCHW image of the reference (4.9 MB per image) never exists.  One thread = the 16 pixels
// of one patch row, all three channels: three 16-byte loads, three 32-byte stores.
struct NormParams {
  float mean[3], stdv[3];
};
template <typename T>
__global__ void __launch_bounds__(256) patch_gather_u8_kernel(const uint8_t* __restrict__ img, T* __restrict__ A, int B, int H, int W, const NormParams np) {
  pdl_sync();
  const int GH = H / 16, GW = W / 16, T_ = GH * GW;
  const long long rows = static_cast<long long>(B) * T_;
  const long long id = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;      // (py, row): row fastest
  if (id >= rows * 16) return;
  const long long r = id % rows;
  const int py = static_cast<int>(id / rows);
  const int b = static_cast<int>(r / T_), rem = static_cast<int>(r % T_);
  int Y, X;
  window_token_yx(rem, GH, GW, &Y, &X);
  const uint8_t* src = img + ((static_cast<long long>(b) * H + (Y * 16 + py)) * W + X * 16) * 3;
  uint32_t w[12];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(src) + j);
    w[4 * j] = q.x; w[4 * j + 1] = q.y; w[4 * j + 2] = q.z; w[4 * j + 3] = q.w;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float f[16];
#pragma unroll
    for (int px = 0; px < 16; ++px) {
      const int byte = px * 3 + c;
      const float u = static_cast<float>((w[byte >> 2] >> ((byte & 3) * 8)) & 0xffu);
      f[px] = (u / 255.f - np.mean[c]) / np.stdv[c];             // ToTensor (/255) then Normalize, IEEE divisions as torch
    }
    U8 o;
#pragma unroll
    for (int j = 0; j < 8; ++j) o.v[j] = Cvt<T>::pack(f[2 * j], f[2 * j + 1]);
    stg256(A + r * 768 + c * 256 + py * 16, o);
  }
}

int patch_gather_u8_launch(int dtype, const void* img, const float* mean, const float* stdv, void* A, int B, int H, int W, cudaStream_t st) {
  if (H % 64 != 0 || W % 64 != 0 || H < 64 || W < 64) return -2;
  NormParams np;
  for (int c = 0; c < 3; ++c) { np.mean[c] = mean[c]; np.stdv[c] = stdv[c]; }
  const long long total = static_cast<long long>(B) * (H / 16) * (W / 16) * 16;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (dtype == DT_BF16) launch_k(patch_gather_u8_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, static_cast<const uint8_t*>(img), static_cast<__nv_bfloat16*>(A), B, H, W, np);
  else launch_k(patch_gather_u8_kernel<__half>, dim3(grid), dim3(256), 0, st, static_cast<const uint8_t*>(img), static_cast<__half*>(A), B, H, W, np);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- padding-mask tables (padded / mixed-size batches)
// From the NestedTensor mask [B, Himg, Wimg] (True = padded pixel, util/misc.py:317-339) build, per image and level:
//   the level mask by nearest resize (backbone.py:153-158), valid_H / valid_W and the valid ratios (transformer.py:
//   189-196), the encoder proposals ((j+.5)/valid_W, (i+.5)/valid_H, .05*2^lvl, .05*2^lvl), the rows whose memory /
//   proposal are zeroed (padding or a component outside (0.01, 0.99); transformer.py:71-125) and the rows whose VALUE is
//   zeroed (padding only; ms_deform_attn.py:114-115).  mask == nullptr means "no padding": the tables then equal the
//   per-config constants.  One CTA per (image, level).
struct MaskSetupArgs {
  const uint8_t* mask;
  int B, Himg, Wimg, L, S;
  int lvl_h[4], lvl_w[4], lvl_start[4];
  float* proposals;    // [B, S, 4]
  uint8_t* invalid;    // [B, S]
  uint8_t* pad;        // [B, S]
  float* valid_ratio;  // [B, L, 2] (w, h)
};
__global__ void __launch_bounds__(256) mask_setup_kernel(const MaskSetupArgs p) {
  pdl_sync();
  const int b = blockIdx.x / p.L, l = blockIdx.x % p.L;
  const int H = p.lvl_h[l], W = p.lvl_w[l];
  const float sy = static_cast<float>(p.Himg) / H, sx = static_cast<float>(p.Wimg) / W;     // F.interpolate(mode="nearest") source index
  auto padded = [&](int i, int j) -> bool {
    if (p.mask == nullptr) return false;
    const int yi = min(static_cast<int>(floorf(i * sy)), p.Himg - 1), xi = min(static_cast<int>(floorf(j * sx)), p.Wimg - 1);
    return p.mask[(static_cast<long long>(b) * p.Himg + yi) * p.Wimg + xi] != 0;
  };
  __shared__ int vh, vw;
  if (threadIdx.x == 0) { vh = 0; vw = 0; }
  __syncthreads();
  for (int i = threadIdx.x; i < H; i += blockDim.x) if (!padded(i, 0)) atomicAdd(&vh, 1);     // transformer.py:87-88
  for (int j = threadIdx.x; j < W; j += blockDim.x) if (!padded(0, j)) atomicAdd(&vw, 1);
  __syncthreads();
  const float valid_h = static_cast<float>(vh), valid_w = static_cast<float>(vw);
  if (threadIdx.x == 0) {
    p.valid_ratio[(b * p.L + l) * 2] = valid_w / W;                                           // transformer.py:189-196
    p.valid_ratio[(b * p.L + l) * 2 + 1] = valid_h / H;
  }
  const float whv = 0.05f * exp2f(static_cast<float>(l));
  for (int t = threadIdx.x; t < H * W; t += blockDim.x) {
    const int i = t / W, j = t - i * W;
    const bool pd = padded(i, j);
    const float v[4] = {(j + 0.5f) / valid_w, (i + 0.5f) / valid_h, whv, whv};
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 4; ++c) ok = ok && (v[c] > 0.01f) && (v[c] < 0.99f);
    const long long row = static_cast<long long>(b) * p.S + p.lvl_start[l] + t;
    const bool keep = ok && !pd;
    reinterpret_cast<float4*>(p.proposals)[row] = keep ? make_float4(v[0], v[1], v[2], v[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
    p.invalid[row] = keep ? 0 : 1;
    p.pad[row] = pd ? 1 : 0;
  }
}
int mask_setup_launch(const uint8_t* mask, int B, int Himg, int Wimg, int L, int S, const int* lvl_h, const int* lvl_w, const int* lvl_start,
                      float* proposals, uint8_t* invalid, uint8_t* pad, float* valid_ratio, cudaStream_t st) {
  if (L < 1 || L > 4) return -2;
  MaskSetupArgs a;
  a.mask = mask; a.B = B; a.Himg = Himg; a.Wimg = Wimg; a.L = L; a.S = S;
  for (int l = 0; l < 4; ++l) { a.lvl_h[l] = l < L ? lvl_h[l] : 0; a.lvl_w[l] = l < L ? lvl_w[l] : 0; a.lvl_start[l] = l < L ? lvl_start[l] : 0; }
  a.proposals = proposals; a.invalid = invalid; a.pad = pad; a.valid_ratio = valid_ratio;
  launch_k(mask_setup_kernel, dim3(static_cast<unsigned>(B * L)), dim3(256), 0, st, a);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- window-major -> spatial copy
// rows of a GH x GW token grid per image, window-major (vit.py:353-358) -> row-major (b, y, x)
template <typename T>
__global__ void __launch_bounds__(256) unwindow_kernel(const T* __restrict__ src, int lds, T* __restrict__ dst, int ldd,
                                                       long long rows, int C, int GH, int GW) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const int cpr = C / 8;
  const long long id = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (id >= rows * cpr) return;
  const long long r = id / cpr;
  const int c = static_cast<int>(id % cpr);
  const int T_ = GH * GW;
  const long long b = r / T_;
  int y, x;
  window_token_yx(static_cast<int>(r % T_), GH, GW, &y, &x);
  const U4 v = *reinterpret_cast<const U4*>(src + r * lds + c * 8);
  *reinterpret_cast<U4*>(dst + (b * T_ + y * GW + x) * ldd + c * 8) = v;
}
int unwindow_launch(int dtype, const void* src, int lds, void* dst, int ldd, long long rows, int C, int GH, int GW, cudaStream_t st) {
  if (GH % 4 != 0 || GW % 4 != 0 || GH < 4 || GW < 4 || C % 8 != 0 || rows % (static_cast<long long>(GH) * GW) != 0) return -2;
  const long long n = rows * (C / 8);
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  if (dtype == DT_BF16) launch_k(unwindow_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(src), lds, static_cast<__nv_bfloat16*>(dst), ldd, rows, C, GH, GW);
  else launch_k(unwindow_kernel<__half>, dim3(grid), dim3(256), 0, st, static_cast<const __half*>(src), lds, static_cast<__half*>(dst), ldd, rows, C, GH, GW);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- out = a[r % amod] + b[r]
template <typename T>
__global__ void __launch_bounds__(256) add_rows_kernel(const T* __restrict__ a, int lda, long long amod, const T* __restrict__ b,
                                                       int ldb, T* __restrict__ out, int ldo, long long rows, int C) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const int cpr = C / 8;
  const long long id = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (id >= rows * cpr) return;
  const long long r = id / cpr;
  const int c = static_cast<int>(id % cpr) * 8;
  const U4 ua = *reinterpret_cast<const U4*>(a + (amod > 0 ? r % amod : r) * lda + c);
  uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wb[4] = {0, 0, 0, 0};
  if (b != nullptr) {
    const U4 ub = *reinterpret_cast<const U4*>(b + r * ldb + c);
    wb[0] = ub.x; wb[1] = ub.y; wb[2] = ub.z; wb[3] = ub.w;
  }
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 fa = Cvt<T>::unpack(wa[j]);
    float2 fb = make_float2(0.f, 0.f);
    if (b != nullptr) fb = Cvt<T>::unpack(wb[j]);
    o[j] = Cvt<T>::pack(fa.x + fb.x, fa.y + fb.y);
  }
  U4 oo; oo.x = o[0]; oo.y = o[1]; oo.z = o[2]; oo.w = o[3];
  *reinterpret_cast<U4*>(out + r * ldo + c) = oo;
}
int add_rows_launch(int dtype, const void* a, int lda, long long amod, const void* b, int ldb, void* out, int ldo,
                    long long rows, int C, cudaStream_t st) {
  const long long n = rows * (C / 8);
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  if (dtype == DT_BF16) launch_k(add_rows_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(a), lda, amod, static_cast<const __nv_bfloat16*>(b), ldb, static_cast<__nv_bfloat16*>(out), ldo, rows, C);
  else launch_k(add_rows_kernel<__half>, dim3(grid), dim3(256), 0, st, static_cast<const __half*>(a), lda, amod, static_cast<const __half*>(b), ldb, static_cast<__half*>(out), ldo, rows, C);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- row max over classes (fp32)
__global__ void __launch_bounds__(256) rowmax_kernel(const float* __restrict__ x, int ld, int n, float* __restrict__ out, long long rows) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float m = -CUDART_INF_F;
  for (int i = lane; i < n; i += 32) m = fmaxf(m, x[row * ld + i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) out[row] = m;
}
int rowmax_launch(const float* x, int ld, int n, float* out, long long rows, cudaStream_t st) {
  launch_k(rowmax_kernel, dim3(static_cast<unsigned>((rows + 7) / 8)), dim3(256), 0, st, x, ld, n, out, rows);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- per-image top-k (sorted, descending)
// torch.topk(score, nq, dim=1) (transformer.py:246): one CTA per image, bitonic sort of (score, index)
// in shared memory; ties broken towards the lower index.
// Descending bitonic sort of np2 (key, index) pairs in shared memory; ties go to the lower index (= torch.topk on
// distinct positions).  All threads of the CTA call it.
__device__ __forceinline__ void bitonic_sort_desc(float* key, int* val, int np2) {
  for (int size = 2; size <= np2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < np2 / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);          // first half of each `size` block sorted descending
        const float ka = key[lo], kb = key[hi];
        const int va = val[lo], vb = val[hi];
        const bool a_first = (ka > kb) || (ka == kb && va < vb);   // "a ranks before b"
        if (a_first != desc) {
          key[lo] = kb; key[hi] = ka;
          val[lo] = vb; val[hi] = va;
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(1024) topk_kernel(const float* __restrict__ score, int S, int np2, int k, int* __restrict__ idx_out) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  extern __shared__ uint8_t sm_topk[];
  float* key = reinterpret_cast<float*>(sm_topk);
  int* val = reinterpret_cast<int*>(key + np2);
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    key[i] = i < S ? score[static_cast<long long>(b) * S + i] : -CUDART_INF_F;
    val[i] = i;
  }
  __syncthreads();
  bitonic_sort_desc(key, val, np2);
  for (int i = threadIdx.x; i < k; i += blockDim.x) idx_out[static_cast<long long>(b) * k + i] = val[i];
}
// Rows longer than a shared-memory sort holds (S > 16384: the P3 level of the two-level configs from 1024x1024 on).
// One CTA per image; the score row is streamed from global memory / L2 and never held on chip:
//   1. radix select on order-preserving uint32 keys, 8 bits per pass (four passes, a 256-bin shared histogram each):
//      finds the k-th largest key `thr` and how many of the k winners equal it (`need`);
//   2. one ordered pass compacts the <= k winners: every key > thr (any slot order) and the `need` LOWEST indices whose
//      key equals thr (a block-wide prefix count over index order) - torch.topk's tie rule;
//   3. the k survivors are sorted by (score desc, index asc) in shared memory.
// Same result as topk_kernel (and torch.topk): descending, ties to the lower index.  -0.0 counts as +0.0, as a float
// comparison does.
__device__ __forceinline__ uint32_t topk_key(float f) {
  const uint32_t u = f == 0.f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(1024) topk_radix_kernel(const float* __restrict__ score, int S, int k, int np2k, int* __restrict__ idx_out) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  extern __shared__ uint8_t sm_topk[];
  float* ckey = reinterpret_cast<float*>(sm_topk);
  int* cval = reinterpret_cast<int*>(ckey + np2k);
  __shared__ int hist[256];
  __shared__ int warp_excl[32];
  __shared__ uint32_t s_prefix;
  __shared__ int s_need, s_gt, s_eq_base, s_eq_tile;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const float* row = score + static_cast<long long>(b) * S;
  if (tid == 0) { s_prefix = 0u; s_need = k; s_gt = 0; s_eq_base = 0; }
  uint32_t mask = 0u;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix;
    for (int i = tid; i < S; i += blockDim.x) {
      const uint32_t key = topk_key(__ldg(row + i));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1);
    }
    __syncthreads();
    if (tid == 0) {                     // the bin holding the need-th largest key of the candidates
      int cum = 0, need = s_need, bin = 255;
      for (; bin > 0; --bin) {
        if (cum + hist[bin] >= need) break;
        cum += hist[bin];
      }
      s_need = need - cum;
      s_prefix = prefix | (static_cast<uint32_t>(bin) << shift);
    }
    mask |= 255u << shift;
    __syncthreads();
  }
  const uint32_t thr = s_prefix;
  const int need = s_need, n_gt = k - need;
  // ---- ordered compaction, one tile of blockDim indices at a time
  for (int base = 0; base < S; base += blockDim.x) {
    const int i = base + tid;
    const float f = i < S ? __ldg(row + i) : 0.f;
    const uint32_t key = i < S ? topk_key(f) : 0u;
    const bool gt = i < S && key > thr, eq = i < S && key == thr;
    if (gt) {
      const int slot = atomicAdd(&s_gt, 1);
      ckey[slot] = f;
      cval[slot] = i;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, eq);
    if (lane == 0) warp_excl[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {
      const int v = lane < nwarps ? warp_excl[lane] : 0;
      int incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      if (lane < nwarps) warp_excl[lane] = incl - v;
      if (lane == 31) s_eq_tile = incl;
    }
    __syncthreads();
    const int rank = s_eq_base + warp_excl[warp] + __popc(bal & ((1u << lane) - 1u));
    if (eq && rank < need) {
      ckey[n_gt + rank] = f;
      cval[n_gt + rank] = i;
    }
    __syncthreads();
    if (tid == 0) s_eq_base += s_eq_tile;
  }
  for (int i = k + tid; i < np2k; i += blockDim.x) {
    ckey[i] = -CUDART_INF_F;
    cval[i] = 0x7fffffff;
  }
  __syncthreads();
  bitonic_sort_desc(ckey, cval, np2k);
  for (int i = tid; i < k; i += blockDim.x) idx_out[static_cast<long long>(b) * k + i] = cval[i];
}

int topk_launch(const float* score, int B, int S, int k, int* idx_out, cudaStream_t st) {
  if (k > S) return -2;
  int np2 = 1;
  while (np2 < S) np2 <<= 1;
  if (np2 <= 16384) {
    const size_t smem = static_cast<size_t>(np2) * 8;
    if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(topk_kernel), 16384 * 8)) return e;
    launch_k(topk_kernel, dim3(B), dim3(1024), smem, st, score, S, np2, k, idx_out);
    return static_cast<int>(cudaGetLastError());
  }
  if (k < 1) return 0;
  int np2k = 1;
  while (np2k < k) np2k <<= 1;
  if (np2k > 4096) return -2;
  const size_t smem = static_cast<size_t>(np2k) * 8;
  launch_k(topk_radix_kernel, dim3(B), dim3(1024), smem, st, score, S, k, np2k, idx_out);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- gather of the selected rows
// sel[b,j,:] = feat[b, idx[b,j], :] (16-bit), enc_logits[b,j,:] = logits[b, idx[b,j], :] (fp32).
template <typename T>
__global__ void __launch_bounds__(128) gather_topk_kernel(const T* __restrict__ feat, int ldf, const float* __restrict__ logits, int ldl,
                                                          int ncls, const int* __restrict__ idx, int S, int k, int d,
                                                          T* __restrict__ sel, float* __restrict__ enc_logits) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const long long bj = blockIdx.x;
  const long long b = bj / k;
  const long long src = b * S + idx[bj];
  for (int c = threadIdx.x; c < d / 8; c += blockDim.x)
    *reinterpret_cast<U4*>(sel + bj * d + c * 8) = *reinterpret_cast<const U4*>(feat + src * ldf + c * 8);
  if (enc_logits != nullptr)
    for (int c = threadIdx.x; c < ncls; c += blockDim.x) enc_logits[bj * ncls + c] = logits[src * ldl + c];
}
int gather_topk_launch(int dtype, const void* feat, int ldf, const float* logits, int ldl, int ncls, const int* idx, int B, int S,
                       int k, int d, void* sel, float* enc_logits, cudaStream_t st) {
  const unsigned grid = static_cast<unsigned>(B) * k;
  if (dtype == DT_BF16) launch_k(gather_topk_kernel<__nv_bfloat16>, dim3(grid), dim3(128), 0, st, static_cast<const __nv_bfloat16*>(feat), ldf, logits, ldl, ncls, idx, S, k, d, static_cast<__nv_bfloat16*>(sel), enc_logits);
  else launch_k(gather_topk_kernel<__half>, dim3(grid), dim3(128), 0, st, static_cast<const __half*>(feat), ldf, logits, ldl, ncls, idx, S, k, d, static_cast<__half*>(sel), enc_logits);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- two-stage boxes + query reference + sine embedding
// For each selected token (transformer.py:234-240, 266-276, 42-68, 344-357):
//   box_ts   = reparam(delta_ts, proposal[idx])             -> enc_outputs.pred_boxes
//   refpoint = reparam(refpoint_embed[j], box_ts)           -> decoder reference (kept fp32)
//   sine     = [sin/cos embedding of (y, x, w, h)], 4*(d/2) = 2d values, 16-bit
template <typename T>
__global__ void __launch_bounds__(256) query_init_kernel(const float* __restrict__ delta_ts, const float* __restrict__ proposals,
                                                         const int* __restrict__ idx, const float* __restrict__ refpoint_embed,
                                                         int k, int d, long long rows, float* __restrict__ box_ts,
                                                         float* __restrict__ refpoint, T* __restrict__ sine, int S, int L,
                                                         const float* __restrict__ valid_ratio) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const long long row = blockIdx.x;
  if (row >= rows) return;
  const int j = static_cast<int>(row % k);
  __shared__ float rp[4];
  if (threadIdx.x < 4) {
    const int c = threadIdx.x;
    const float* pr = proposals + (static_cast<long long>(row / k) * S + idx[row]) * 4;       // per-image proposal table [B, S, 4]
    const float* dl = delta_ts + row * 4;
    const float bx = c < 2 ? dl[c] * pr[c + 2] + pr[c] : expf(dl[c]) * pr[c];
    box_ts[row * 4 + c] = bx;
    // refpoint needs box_ts of both halves: recompute the partner instead of syncing twice
    const float bxy = c < 2 ? bx : dl[c - 2] * pr[c] + pr[c - 2];
    const float bwh = c < 2 ? expf(dl[c + 2]) * pr[c + 2] : bx;
    const float e = refpoint_embed[j * 4 + c];
    const float r = c < 2 ? e * bwh + bxy : expf(e) * bwh;
    refpoint[row * 4 + c] = r;
    // the sine embedding sees the level-0 reference box scaled by the valid ratio (transformer.py:352-355; 1 when unpadded)
    rp[c] = r * valid_ratio[(row / k) * L * 2 + (c & 1)];
  }
  __syncthreads();
  const int dim = d / 2;                        // per-coordinate embedding width
  const float two_pi = 6.283185307179586f;
  for (int i = threadIdx.x; i < 2 * d; i += blockDim.x) {
    const int coord_slot = i / dim;             // output order (y, x, w, h)
    const int e = i % dim;
    const float c = rp[coord_slot == 0 ? 1 : (coord_slot == 1 ? 0 : coord_slot)];
    // 1 / dim_t = 10000^(-2*(e/2)/dim) by exp2 (13.2877 = log2 1e4).  |v| is not bounded: the reference's width is
    // exp(refpoint_embed) times the encoder box's, so |v| = 2*pi*|rp| can reach hundreds.  The fast sin/cos stay within
    // 2^-21.41 plus the argument's own fp32 error there: tests/test_query_select_gpu.py holds every element of the embedding
    // to that plus half a 16-bit ulp for |v| up to ~560, and the 16-bit rounding dominates
    const float inv_dim_t = exp2f(-13.287712379549449f * static_cast<float>(2 * (e / 2)) / static_cast<float>(dim));
    const float v = c * two_pi * inv_dim_t;
    sine[row * (2 * d) + i] = Cvt<T>::from_f((e & 1) ? __cosf(v) : __sinf(v));
  }
}
int query_init_launch(int dtype, const float* delta_ts, const float* proposals, const int* idx, const float* refpoint_embed, int B,
                      int k, int d, float* box_ts, float* refpoint, void* sine, int S, int L, const float* valid_ratio, cudaStream_t st) {
  const long long rows = static_cast<long long>(B) * k;
  if (dtype == DT_BF16) launch_k(query_init_kernel<__nv_bfloat16>, dim3(static_cast<unsigned>(rows)), dim3(256), 0, st, delta_ts, proposals, idx, refpoint_embed, k, d, rows, box_ts, refpoint, static_cast<__nv_bfloat16*>(sine), S, L, valid_ratio);
  else launch_k(query_init_kernel<__half>, dim3(static_cast<unsigned>(rows)), dim3(256), 0, st, delta_ts, proposals, idx, refpoint_embed, k, d, rows, box_ts, refpoint, static_cast<__half*>(sine), S, L, valid_ratio);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- final boxes (lwdetr.py:149-155)
__global__ void __launch_bounds__(256) final_boxes_kernel(const float* __restrict__ delta, const float* __restrict__ refpoint,
                                                          long long rows_per_layer, long long total, float* __restrict__ boxes) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  const long long id = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (id >= total) return;
  const long long row = id >> 2;
  const int c = static_cast<int>(id & 3);
  const float* rf = refpoint + (row % rows_per_layer) * 4;
  const float dl = delta[id];
  boxes[id] = c < 2 ? dl * rf[c + 2] + rf[c] : expf(dl) * rf[c];
}
int final_boxes_launch(const float* delta, const float* refpoint, long long rows_per_layer, int layers, float* boxes, cudaStream_t st) {
  const long long total = rows_per_layer * layers * 4;
  launch_k(final_boxes_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, st, delta, refpoint, rows_per_layer, total, boxes);
  return static_cast<int>(cudaGetLastError());
}

// ----------------------------------------------------------------------------------- PostProcess (lwdetr.py:515-544)
// sigmoid -> top num_select over the nq*ncls (query, class) scores of an image -> labels, boxes in absolute xyxy.
// Two launches: (1) every image's score list is cut into `parts` slices of <= 16384 entries, one CTA sorts a slice
// (sigmoid computed while loading) and keeps its k best flat indices; (2) one CTA per image merges the parts*k
// candidates, sorts them again and writes scores / labels / scaled boxes - only [B, k, 6] numbers leave the GPU.
__global__ void __launch_bounds__(1024) postprocess_part_kernel(const float* __restrict__ logits, int S, int parts, int part_len,
                                                                 int np2, int k, int* __restrict__ cand) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  extern __shared__ uint8_t sm_topk[];
  float* key = reinterpret_cast<float*>(sm_topk);
  int* val = reinterpret_cast<int*>(key + np2);
  const int b = blockIdx.x / parts, part = blockIdx.x % parts;
  const int base = part * part_len;
  const int n = min(part_len, S - base);
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    key[i] = i < n ? sigmoid_f32(logits[static_cast<long long>(b) * S + base + i]) : -CUDART_INF_F;
    val[i] = i < n ? base + i : -1;
  }
  __syncthreads();
  bitonic_sort_desc(key, val, np2);
  for (int i = threadIdx.x; i < k; i += blockDim.x) cand[(static_cast<long long>(b) * parts + part) * k + i] = val[i];
}

__global__ void __launch_bounds__(1024) postprocess_merge_kernel(const float* __restrict__ logits, const float* __restrict__ boxes,
                                                                  const float* __restrict__ target_sizes, const int* __restrict__ cand,
                                                                  int S, int ncand, int np2, int ncls, int k, float* __restrict__ scores,
                                                                  int* __restrict__ labels, float* __restrict__ out_boxes) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  extern __shared__ uint8_t sm_topk[];
  float* key = reinterpret_cast<float*>(sm_topk);
  int* val = reinterpret_cast<int*>(key + np2);
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    const int c = i < ncand ? cand[static_cast<long long>(b) * ncand + i] : -1;
    key[i] = c >= 0 ? sigmoid_f32(logits[static_cast<long long>(b) * S + c]) : -CUDART_INF_F;
    val[i] = c >= 0 ? c : 0x7fffffff;
  }
  __syncthreads();
  bitonic_sort_desc(key, val, np2);
  const float img_h = target_sizes[2 * b], img_w = target_sizes[2 * b + 1];
  const int nq = S / ncls;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    const int flat = val[i];
    const int q = flat / ncls;
    const float4 bx = *reinterpret_cast<const float4*>(boxes + (static_cast<long long>(b) * nq + q) * 4);   // cx, cy, w, h
    const long long o = static_cast<long long>(b) * k + i;
    scores[o] = key[i];
    labels[o] = flat - q * ncls;
    *reinterpret_cast<float4*>(out_boxes + o * 4) = box_cxcywh_to_xyxy(bx, img_h, img_w);
  }
}

int postprocess_launch(const float* logits, const float* boxes, const float* target_sizes, int B, int nq, int ncls, int k,
                       int* work, float* scores, int* labels, float* out_boxes, cudaStream_t st) {
  const int S = nq * ncls;
  const int parts = (S + 16383) / 16384;
  const int part_len = (S + parts - 1) / parts;
  int np2 = 1;
  while (np2 < part_len) np2 <<= 1;
  const int ncand = parts * k;
  int np2m = 1;
  while (np2m < ncand) np2m <<= 1;
  if (k > part_len || np2m > 16384 || B < 1) return -2;
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(postprocess_part_kernel), 16384 * 8)) return e;
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(postprocess_merge_kernel), 16384 * 8)) return e;
  launch_k(postprocess_part_kernel, dim3(B * parts), dim3(1024), static_cast<size_t>(np2) * 8, st, logits, S, parts, part_len, np2, k, work);
  launch_k(postprocess_merge_kernel, dim3(B), dim3(1024), static_cast<size_t>(np2m) * 8, st, logits, boxes, target_sizes,
           static_cast<const int*>(work), S, ncand, np2m, ncls, k, scores, labels, out_boxes);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace lwb
