// Fused ViT MLP for the 192-wide encoder (vit_tiny: the tiny and small configs), see gemm_tc.h MlpDesc:
//   out = x + gamma * (fc2(gelu(fc1(LN(x)))) + b2)
// in one persistent, warp-specialised wgmma + TMA kernel, so the [M, 768] hidden activation never leaves the SM.
//   warp 0 (of the producer warpgroup): TMA producer (one elected lane): the tile's raw rows X [128 x 192] once (three
//              128B-swizzled 64-column k-blocks, one buffer), then per 64-column hidden chunk the fc1 weight slice
//              W1'[chunk] [64 x 192] and the fc2 weight slice W2[:, chunk] [192 x 64] into two rings of two stages each
//   warps 4-11: two consumer warpgroups, 64 rows each.  Per chunk c (12 of them, in increasing order):
//                S = X W1'[c]^T (fp32, 64 x 64, both operands in shared memory); the LayerNorm fold + exact-erf GELU on the
//                accumulator fragments (the expressions of gemm_tc.cu's EP_LN_GELU epilogue), rounded to 16 bits and packed
//                straight into the register A fragments of  O += H W2[:, c]^T  (O: 64 x 192 fp32, 96 registers).  The MMAs
//                of chunk c + 1's fc1 are issued before chunk c's GELU, so the tensor core works while the GELU is issued.
//              After the last chunk: out = resid + gamma * (O + b2) and the LayerNorm partials of the rounded rows, through
//              the same per-warp staging and chunk order as gemm_tc.cu's EP_RESID epilogue (fc2 at BN = 192 or 64).
// Summation orders are those of the two-GEMM path (fc1 over k = 0..191, fc2 over k = 0..767 in steps of 16, the hidden
// values rounded to the compute dtype in between), so the result is that of fc1 -> fc2 bit for bit.
#include "epilogue.cuh"
#include "gemm_tc.h"
#include "launch.h"
#include "ptx.cuh"
#include "tma_util.h"
#include "wgmma.cuh"

#include <algorithm>
#include <cstring>

namespace lwb {
namespace mlp {

static constexpr int C = MLP_C;                       // model width
static constexpr int HID = 4 * C;                     // 768 hidden columns
static constexpr int BM = 128;                        // rows per tile
static constexpr int HC = 64;                         // hidden columns per chunk
static constexpr int NCH = HID / HC;                  // 12 chunks
static constexpr int KB = C / 64;                     // fc1 k-blocks (128-byte swizzle rows)
static constexpr int THREADS = 128 + 256;             // producer warpgroup + two consumer warpgroups
static constexpr int X_KB_BYTES = BM * 64 * 2;        // 16 KB per k-block of X
static constexpr int X_BYTES = KB * X_KB_BYTES;       // 48 KB
static constexpr int W1_KB_BYTES = HC * 64 * 2;       // 8 KB
static constexpr int W1_STAGE = KB * W1_KB_BYTES;     // 24 KB
static constexpr int W2_STAGE = C * HC * 2;           // 24 KB
static constexpr int STAGES = 2;
static constexpr int STG_LD = 68;                     // floats per staged accumulator row (as gemm_tc.cu)
static constexpr int STG_BYTES = 8 * 16 * STG_LD * 4;
static constexpr int VEC_FLOATS = 2 * HID + 2 * C;    // b1' | colsum | b2 | gamma
static constexpr size_t SMEM = 1024 + X_BYTES + STAGES * (W1_STAGE + W2_STAGE) + 256 + STG_BYTES + VEC_FLOATS * 4;

template <typename T>
__global__ void __launch_bounds__(THREADS, 1)
vit_mlp_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW1,
               const __grid_constant__ CUtensorMap tmW2, const MlpArgs p) {
  constexpr bool BF = Cvt<T>::is_bf16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sX = smem;
  uint8_t* sW1 = sX + X_BYTES;
  uint8_t* sW2 = sW1 + STAGES * W1_STAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sW2 + STAGES * W2_STAGE);
  uint64_t* x_full = bars;
  uint64_t* x_empty = bars + 1;
  uint64_t* w1_full = bars + 2;
  uint64_t* w1_empty = w1_full + STAGES;
  uint64_t* w2_full = w1_empty + STAGES;
  uint64_t* w2_empty = w2_full + STAGES;
  float* s_stage = reinterpret_cast<float*>(bars + 32);
  float* s_b1 = s_stage + 8 * 16 * STG_LD;
  float* s_cs1 = s_b1 + HID;
  float* s_b2 = s_cs1 + HID;
  float* s_g2 = s_b2 + C;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW1);
    tma_prefetch_desc(&tmW2);
    mbar_init(x_full, 1);
    mbar_init(x_empty, 8);                 // one elected arrival per consumer warp
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&w1_full[s], 1);
      mbar_init(&w1_empty[s], 8);
      mbar_init(&w2_full[s], 1);
      mbar_init(&w2_empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();   // the prologue above touched no global data; everything below may read the predecessor's output

  if (warp < 4) {
    reg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------------------------------------------ TMA producer
      uint32_t it = 0, ch = 0;
      for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++it) {
        mbar_wait(x_empty, (it & 1) ^ 1);
        mbar_arrive_expect_tx(x_full, X_BYTES);
        for (int kb = 0; kb < KB; ++kb) tma_load_2d(sX + kb * X_KB_BYTES, &tmX, x_full, kb * 64, tile * BM);
        for (int c = 0; c < NCH; ++c, ++ch) {
          const int s = ch % STAGES;
          const uint32_t ph = ((ch / STAGES) & 1) ^ 1;
          mbar_wait(&w1_empty[s], ph);
          mbar_arrive_expect_tx(&w1_full[s], W1_STAGE);
          for (int kb = 0; kb < KB; ++kb) tma_load_2d(sW1 + s * W1_STAGE + kb * W1_KB_BYTES, &tmW1, &w1_full[s], kb * 64, c * HC);
          mbar_wait(&w2_empty[s], ph);
          mbar_arrive_expect_tx(&w2_full[s], W2_STAGE);
          tma_load_2d(sW2 + s * W2_STAGE, &tmW2, &w2_full[s], c * HC, 0);
        }
      }
    }
    return;
  }

  reg_inc<232>();
  // ---------------------------------------------------------------------- consumers
  const int cw = warp - 4;                    // consumer warp: rows [16*cw, 16*cw + 16) of the tile
  const int wg = cw >> 2;                     // its warpgroup: rows [64*wg, 64*wg + 64)
  const int g = lane >> 2, t4 = lane & 3;     // fragment rows 16*cw + g (+8), columns 8j + 2*t4 (+1)
  const int chalf = lane & 1;                 // final epilogue: two threads per row (as gemm_tc.cu)
  const int r = cw * 16 + (lane >> 1);
  float* stg = s_stage + cw * 16 * STG_LD;
  for (int i = threadIdx.x - 128; i < HID; i += 256) {
    s_b1[i] = __ldg(p.b1 + i);
    s_cs1[i] = __ldg(p.colsum1 + i);
  }
  for (int i = threadIdx.x - 128; i < C; i += 256) {
    s_b2[i] = p.b2 != nullptr ? __ldg(p.b2 + i) : 0.f;
    s_g2[i] = p.gamma != nullptr ? __ldg(p.gamma + i) : 1.f;
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  const float part_n = 1.f / (p.ln_inv_c * p.stats_parts_in), part_inv_n = 1.f / part_n;
  const bool do_stats = p.stats_out != nullptr;
  const int parts_per_pass = p.stats_parts_out / 2;   // 1: one 192-wide slice per row half; 3: one per 64-column pass

  const uint32_t x_addr = smem_u32(sX) + wg * (64 * 128);
  const uint32_t w1_addr = smem_u32(sW1), w2_addr = smem_u32(sW2);
  uint32_t it = 0, ch = 0;
  for (int tile = blockIdx.x; tile < p.m_tiles; tile += gridDim.x, ++it) {
    // LayerNorm of the fragment rows (the loads overlap the first MMAs)
    uint64_t ln_a[2], ln_b[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = tile * BM + cw * 16 + g + 8 * h;
      float mean = 0.f, rstd = 1.f;
      if (m < p.M) ln_row_stats(p.stats_in + static_cast<long long>(m) * p.stats_parts_in, p.stats_parts_in, part_n, part_inv_n,
                                p.ln_inv_c, p.ln_eps, mean, rstd);
      // rstd*(acc - mean*colsum) + bias  ==  a*acc + (b*colsum + bias),  a = rstd, b = -rstd*mean  (gemm_tc.cu finish_chunk)
      ln_a[h] = f2_pack(rstd, rstd);
      ln_b[h] = f2_pack(-rstd * mean, -rstd * mean);
    }

    auto issue_fc1 = [&](float (&s)[HC / 2], uint32_t gc) {
      const int st = gc % STAGES;
      mbar_wait(&w1_full[st], (gc / STAGES) & 1);
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        const uint64_t adesc = wgmma_desc(x_addr + kb * X_KB_BYTES, 128);
        const uint64_t bdesc = wgmma_desc(w1_addr + st * W1_STAGE + kb * W1_KB_BYTES, 128);
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<BF, HC>::ss(s, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
    };

    float o[C / 2];
    float sa[HC / 2], sb[HC / 2];
    mbar_wait(x_full, it & 1);
    issue_fc1(sa, ch);

    // one chunk: fc1 of the next chunk in flight, then the GELU of this one, then its fc2 MMAs
    auto step = [&](int c, float (&cur)[HC / 2], float (&nxt)[HC / 2]) {
      const uint32_t gc = ch + c;
      if (c + 1 < NCH) {
        issue_fc1(nxt, gc + 1);
        wgmma_wait<1>();                       // fc1(c) and fc2(c - 1) done, fc1(c + 1) may run on
      } else {
        wgmma_wait<0>();
      }
      fence_regs(cur);
      if (lane == 0) {
        mbar_arrive(&w1_empty[gc % STAGES]);
        if (c > 0) mbar_arrive(&w2_empty[(gc - 1) % STAGES]);
        if (c == NCH - 1) mbar_arrive(x_empty);  // every fc1 MMA of the tile has read X
      }
      uint32_t hf[HC / 16][4];                   // C fragments of n-groups (2k, 2k+1) form the A fragment of k-step k
      const float* b1 = s_b1 + c * HC;
      const float* cs1 = s_cs1 + c * HC;
#pragma unroll
      for (int j = 0; j < HC / 8; ++j) {
        const float2 bb = *reinterpret_cast<const float2*>(b1 + 8 * j + 2 * t4);
        const float2 cc = *reinterpret_cast<const float2*>(cs1 + 8 * j + 2 * t4);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint64_t w = f2_pack(cur[4 * j + 2 * h], cur[4 * j + 2 * h + 1]);
          w = f2_fma(ln_a[h], w, f2_fma(ln_b[h], f2_pack(cc.x, cc.y), f2_pack(bb.x, bb.y)));
          w = gelu_erf2(w);
          float v0, v1;
          f2_unpack(w, v0, v1);
          hf[j >> 1][(j & 1) * 2 + h] = Cvt<T>::pack(v0, v1);
        }
      }
      const int st = gc % STAGES;
      mbar_wait(&w2_full[st], (gc / STAGES) & 1);
      wgmma_fence();
      const uint64_t bdesc = wgmma_desc(w2_addr + st * W2_STAGE, 128);
#pragma unroll
      for (int k = 0; k < HC / 16; ++k) Wgmma<BF, C>::rs(o, hf[k], bdesc + 2 * k, (c | k) != 0 ? 1u : 0u);
      wgmma_commit();
    };
#pragma unroll 1
    for (int c = 0; c < NCH; c += 2) {
      step(c, sa, sb);
      step(c + 1, sb, sa);
    }
    wgmma_wait<0>();
    fence_regs(o);
    if (lane == 0) mbar_arrive(&w2_empty[(ch + NCH - 1) % STAGES]);
    ch += NCH;

    // ------------------------------------------------------------------ epilogue: out = resid + gamma * (O + b2)
    const int m = tile * BM + r;
    const bool valid = m < p.M;
    const T* resid_row = reinterpret_cast<const T*>(p.x) + static_cast<long long>(m) * p.ldx;
    T* out_row = reinterpret_cast<T*>(p.out) + static_cast<long long>(m) * p.ld_out;
    float st_sum = 0.f, st_sq = 0.f, st_K = 0.f;
    bool st_have = false;
    int st_n = 0;
#pragma unroll
    for (int pc = 0; pc < C / 64; ++pc) {
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int a0 = 4 * (8 * pc + j), col = 8 * j + 2 * t4;
        *reinterpret_cast<float2*>(stg + g * STG_LD + col) = make_float2(o[a0], o[a0 + 1]);
        *reinterpret_cast<float2*>(stg + (g + 8) * STG_LD + col) = make_float2(o[a0 + 2], o[a0 + 3]);
      }
      __syncwarp();
      if (valid) {
#pragma unroll 1
        for (int i = 0; i < 2; ++i) {
          const int cl = 2 * chalf + i, n = (4 * pc + cl) * 16;
          const U8 rr = ldg256(resid_row + n);
          const float* src = stg + (lane >> 1) * STG_LD + cl * 16;
          uint64_t w[8];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 f = lds128(src + 4 * q);
            w[2 * q] = f2_pack(f.x, f.y);
            w[2 * q + 1] = f2_pack(f.z, f.w);
          }
          // (acc + b2) * gamma + resid with every operation rounded on its own, as the fc2 GEMM's epilogue computes it:
          // the explicit _rn forms keep the compiler from contracting the multiply and the residual add into one FMA
          U8 ov;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 b4 = lds128(s_b2 + n + 4 * q), g4 = lds128(s_g2 + n + 4 * q);
            const float bv[4] = {b4.x, b4.y, b4.z, b4.w}, gv[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              float v0, v1;
              f2_unpack(w[2 * q + hh], v0, v1);
              const float2 f = Cvt<T>::unpack(rr.v[2 * q + hh]);
              v0 = __fadd_rn(__fmul_rn(__fadd_rn(v0, bv[2 * hh]), gv[2 * hh]), f.x);
              v1 = __fadd_rn(__fmul_rn(__fadd_rn(v1, bv[2 * hh + 1]), gv[2 * hh + 1]), f.y);
              ov.v[2 * q + hh] = Cvt<T>::pack(v0, v1);
            }
          }
          stg256(out_row + n, ov);
          if (do_stats) {                          // statistics of the ROUNDED values the next LayerNorm will read
            st_n += 16;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float2 f = Cvt<T>::unpack(ov.v[j]);
              if (!st_have) {
                st_K = f.x;
                st_have = true;
              }
              const float d0 = f.x - st_K, d1 = f.y - st_K;
              st_sum += d0 + d1;
              st_sq = fmaf(d0, d0, fmaf(d1, d1, st_sq));
            }
          }
        }
        // one partial per (slice, column half): a slice is the whole row (2 partials) or one 64-column pass (6 partials)
        if (do_stats && (parts_per_pass == 3 || pc == C / 64 - 1)) {
          const float nn = static_cast<float>(st_n > 0 ? st_n : 1);
          const float part_sum = fmaf(nn, st_K, st_sum), part_m2 = fmaxf(st_sq - st_sum * st_sum / nn, 0.f);
          const int slice = parts_per_pass == 3 ? pc : 0;
          p.stats_out[static_cast<long long>(m) * p.stats_parts_out + slice * 2 + chalf] = make_float2(part_sum, part_m2);
          st_sum = st_sq = st_K = 0.f;
          st_have = false;
          st_n = 0;
        }
      }
    }
  }
}

}  // namespace mlp

// ------------------------------------------------------------------------------------------- host
int vit_mlp_build(const MlpDesc& d, MlpOp* op, std::string* err) {
  std::memset(op, 0, sizeof(*op));
  if (d.dtype != DT_F16 && d.dtype != DT_BF16) { *err = "vit_mlp: dtype must be fp16 or bf16"; return -1; }
  if (!d.x || !d.stats_in || !d.w1 || !d.colsum1 || !d.b1 || !d.w2 || !d.out) { *err = "vit_mlp: null pointer"; return -1; }
  if (d.M < 1) { *err = "vit_mlp: M must be positive"; return -1; }
  if (d.stats_parts_in < 1 || MLP_C % d.stats_parts_in != 0) { *err = "vit_mlp: the input partial count must divide 192"; return -1; }
  if (d.stats_out && d.stats_parts_out != 2 && d.stats_parts_out != 6) { *err = "vit_mlp: stats_parts_out must be 2 or 6"; return -1; }
  // every 16-column chunk of a row is one 32-byte access (residual and output)
  if (d.ldx < MLP_C || d.ldx % 16 != 0 || d.ld_out < MLP_C || d.ld_out % 16 != 0 ||
      (reinterpret_cast<uintptr_t>(d.x) & 31) != 0 || (reinterpret_cast<uintptr_t>(d.out) & 31) != 0) {
    *err = "vit_mlp: ldx and ld_out must be >= 192 and multiples of 16, x and out 32-byte aligned";
    return -1;
  }
  MlpArgs& a = op->args;
  a.M = d.M;
  a.m_tiles = (d.M + mlp::BM - 1) / mlp::BM;
  a.x = d.x; a.ldx = d.ldx;
  a.stats_in = d.stats_in; a.stats_parts_in = d.stats_parts_in;
  a.ln_inv_c = 1.f / MLP_C; a.ln_eps = d.ln_eps;
  a.b1 = d.b1; a.colsum1 = d.colsum1; a.b2 = d.b2; a.gamma = d.gamma;
  a.out = d.out; a.ld_out = d.ld_out;
  a.stats_out = d.stats_out; a.stats_parts_out = d.stats_out ? d.stats_parts_out : 2;
  op->dtype = d.dtype;
  {
    const cuuint64_t dims[2] = {MLP_C, static_cast<cuuint64_t>(d.M)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.ldx) * 2};
    const cuuint32_t box[2] = {64, mlp::BM};
    if (tma_encode(&op->tx, d.dtype, 2, d.x, dims, strides, box, 128, err)) return -1;
  }
  {
    const cuuint64_t dims[2] = {MLP_C, 4 * MLP_C};
    const cuuint64_t strides[1] = {MLP_C * 2};
    const cuuint32_t box[2] = {64, mlp::HC};
    if (tma_encode(&op->tw1, d.dtype, 2, d.w1, dims, strides, box, 128, err)) return -1;
  }
  {
    const cuuint64_t dims[2] = {4 * MLP_C, MLP_C};
    const cuuint64_t strides[1] = {4 * MLP_C * 2};
    const cuuint32_t box[2] = {64, MLP_C};
    if (tma_encode(&op->tw2, d.dtype, 2, d.w2, dims, strides, box, 128, err)) return -1;
  }
  op->smem = mlp::SMEM;
  op->grid = static_cast<unsigned>(std::min(a.m_tiles, current_device_sms()));
  op->flops = 2.0 * 2.0 * d.M * static_cast<double>(4 * MLP_C) * MLP_C;
  return 0;
}

template <typename T>
static int launch_mlp(const MlpOp& op, cudaStream_t st) {
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(mlp::vit_mlp_kernel<T>), static_cast<int>(mlp::SMEM))) return e;
  launch_k(mlp::vit_mlp_kernel<T>, dim3(op.grid), dim3(mlp::THREADS), op.smem, st, op.tx, op.tw1, op.tw2, op.args);
  return static_cast<int>(cudaGetLastError());
}

int vit_mlp_launch(const MlpOp& op, cudaStream_t st) {
  return op.dtype == DT_BF16 ? launch_mlp<__nv_bfloat16>(op, st) : launch_mlp<__half>(op, st);
}

}  // namespace lwb
