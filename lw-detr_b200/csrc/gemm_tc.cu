// wgmma / TMA GEMM family (see gemm_tc.h).  Persistent CTAs (one per SM) walk 128 x BN output tiles:
//   warp 0 (of the producer warpgroup): TMA producer (one elected lane): the 128 x 64 A tile and the BN x 64 W tile per
//              k-block into a ring of shared-memory stages (full / empty mbarriers); the warpgroup gives its registers
//              to the consumers (setmaxnreg)
//   warps 4-11: two consumer warpgroups, 64 rows each: wgmma.mma_async m64nBNk16 straight out of the swizzled stages,
//              fp32 accumulators in registers, one k-block of MMAs in flight while the next stage is awaited; then the
//              epilogue of their own rows: the accumulators pass through a per-warp shared-memory staging area, 64 columns
//              at a time, so that every row is finished by two threads on 16-column chunks - LayerNorm-fold / bias /
//              activation / layer-scale / residual -> 16-bit (or fp32) rows to global, optional row re-ordering / pixel
//              shuffle, optional per-row (sum, M2) statistics for the next LayerNorm-fused GEMM.  The producer keeps
//              filling the ring with the next tile's stages while the epilogue runs.
// Replaces, on the LW-DETR path, every F.linear / nn.Conv2d / nn.ConvTranspose2d call listed in
// SURVEY.md appendix B (reference: models/backbone/vit.py:120-140,206-220, projector.py:85-132,
// transformer.py:27-39,466-517, ops/modules/ms_deform_attn.py:112-143, lwdetr.py:149-159).
#include "gemm_tc.h"
#include "epilogue.cuh"
#include "launch.h"
#include "ptx.cuh"
#include "tma_util.h"
#include "wgmma.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace lwb {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int A_STAGE_BYTES = BM * BK * 2;
static constexpr int MMA_WARPS = 8;                       // two consumer warpgroups of 64 rows; warp w owns rows 16w .. 16w+15
static constexpr int GEMM_THREADS = 128 + 32 * MMA_WARPS; // producer warpgroup + consumers
static constexpr int MAX_STAGES = 8;
static constexpr int STG_LD = 68;                         // floats per staged accumulator row: 64 columns + 4 (bank spread)
static constexpr int STG_BYTES = MMA_WARPS * 16 * STG_LD * 4;


struct TileCoord {
  int m_tile, n_tile, n0, cb, cy0, cx0;
};
// tile index -> (m_tile, n_tile); n fastest, so CTAs running at the same time share the A rows in L2
__device__ __forceinline__ TileCoord decode_tile(const GemmArgs& p, int tile, int BN) {
  TileCoord t;
  t.n_tile = tile % p.n_tiles;
  t.m_tile = tile / p.n_tiles;
  t.n0 = t.n_tile * BN;
  t.cb = t.cy0 = t.cx0 = 0;
  if (p.a_mode != AMODE_PLAIN) {
    const int per_img = p.tiles_x * p.tiles_y;
    t.cb = t.m_tile / per_img;
    const int r = t.m_tile % per_img;
    t.cy0 = (r / p.tiles_x) * p.TH;
    t.cx0 = (r % p.tiles_x) * p.TW;
  }
  return t;
}

// EP (epilogue specialisation): EP_GENERIC keeps every feature behind runtime flags; the others compile the
// features of the hot GEMMs in or out so the per-element instruction count stays minimal:
//   EP_BIAS      out = acc + bias                     (16-bit out, plain rows, no LN / residual / activation)
//   EP_BIAS_ACT  out = act(acc + bias)                (activation still a runtime switch, hoisted per chunk)
//   EP_LN        out = LN-fold(acc) + bias            (qkv)
//   EP_LN_GELU   out = gelu(LN-fold(acc) + bias)      (fc1)
//   EP_RESID     out = resid + gamma*(acc + bias), optional row statistics (proj, fc2, patch embed, decoder)
// (the enum is in gemm_tc.h)

template <typename T, int BN, int EP>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmArgs p) {
  constexpr int B_STAGE_BYTES = BN * BK * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stages = p.stages;
  uint8_t* sA = smem;
  uint8_t* sB = smem + stages * A_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sB + stages * B_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  float* s_stage = reinterpret_cast<float*>(full_bar + 32);   // 256 B of barriers, then the accumulator staging [warp][16][STG_LD]
  float* s_vec = s_stage + MMA_WARPS * 16 * STG_LD;           // then {bias | gamma | colsum}[n_tiles * BN]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);                   // the producer's arrive.expect_tx
      mbar_init(&empty_bar[s], MMA_WARPS);          // one elected arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();   // the prologue above touched no global data; everything below reads the predecessor's output

  if (warp < 4) {
    reg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------------------------------------------ TMA producer
      uint32_t ring = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord tc = decode_tile(p, tile, BN);
        for (int kb = 0; kb < p.kblocks; ++kb, ++ring) {
          const int s = ring % stages;
          const uint32_t ph = (ring / stages) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], p.a_stage_tx + B_STAGE_BYTES);
          uint8_t* a_dst = sA + s * A_STAGE_BYTES;
          if (p.a_mode == AMODE_PLAIN) {
            tma_load_2d(a_dst, &tmA, &full_bar[s], kb * BK, tc.m_tile * BM);
          } else {
            const int tap = kb / p.cin_blocks;
            const int c0 = (kb % p.cin_blocks) * BK;
            const int dy = tap / 3, dx = tap % 3;
            if (p.a_mode == AMODE_CONV3_S1) {
              tma_load_4d(a_dst, &tmA, &full_bar[s], c0, tc.cx0 + dx - 1, tc.cy0 + dy - 1, tc.cb);
            } else {
              // input row iy = 2*oy + dy - 1 = 2*(oy + yoff) + py ; same for columns
              const int py = (dy == 1) ? 0 : 1, yoff = (dy == 0) ? -1 : 0;
              const int px = (dx == 1) ? 0 : 1, xoff = (dx == 0) ? -1 : 0;
              tma_load_5d(a_dst, &tmA, &full_bar[s], px * p.lda + c0, tc.cx0 + xoff, py, tc.cy0 + yoff, tc.cb);
            }
          }
          tma_load_2d(sB + s * B_STAGE_BYTES, &tmB, &full_bar[s], kb * BK, tc.n0);
        }
      }
    }
  } else {
    reg_inc<232>();
    // -------------------------------------------------------------------- MMA + epilogue (two warpgroups)
    const int cw = warp - 4;                    // consumer warp: rows [16*cw, 16*cw + 16) of the tile
    const int wg = cw >> 2;                     // its warpgroup: rows [64*wg, 64*wg + 64)
    const int g = lane >> 2, t4 = lane & 3;     // accumulator fragment: rows 16*cw + g (+8), columns 8j + 2*t4 (+1)
    const int chalf = lane & 1;                 // epilogue: two threads per row, this one takes chunks 4i + 2*chalf, +1
    const int r = cw * 16 + (lane >> 1);        // row inside the 128-row tile (epilogue)
    float* stg = s_stage + cw * 16 * STG_LD;
    constexpr bool GEN = EP == EP_GENERIC;
    const bool has_gamma = (GEN || EP == EP_RESID) && p.gamma != nullptr;
    const bool ln_in = GEN ? (p.stats_in != nullptr) : (EP == EP_LN || EP == EP_LN_GELU);
    const int act = GEN || EP == EP_BIAS_ACT ? p.act : (EP == EP_LN_GELU ? ACT_GELU : ACT_NONE);
    const bool has_resid = (GEN || EP == EP_RESID) && p.resid != nullptr;
    const bool do_stats = (GEN || EP == EP_RESID) && p.stats_out != nullptr;
    const bool plain_out = !GEN;                 // 16-bit, rows in place, no pixel shuffle
    // Stage the bias / layer-scale / LayerNorm column-sum vectors of ALL n-tiles once per CTA (consumer warps only,
    // while the producer already streams the first tile): the per-tile epilogue then has no dependent global loads
    // except the residual and the per-row LayerNorm statistics.
    {
      const int npad_all = p.n_tiles * BN;
      for (int i = threadIdx.x - 128; i < npad_all; i += 32 * MMA_WARPS) {
        const bool in = i < p.N;
        s_vec[i] = (p.bias != nullptr && in) ? __ldg(p.bias + i) : 0.f;
        s_vec[npad_all + i] = (p.gamma != nullptr && in) ? __ldg(p.gamma + i) : 1.f;
        s_vec[2 * npad_all + i] = (p.colsum != nullptr && in) ? __ldg(p.colsum + i) : 0.f;
      }
      asm volatile("bar.sync 1, %0;" ::"n"(32 * MMA_WARPS) : "memory");
    }
    // combine equal-width partials (sum_p, M2_p): mean = sum(sum_p) / C, var = [sum(M2_p) + n_p * sum((sum_p / n_p - mean)^2)] / C
    const float part_n = p.stats_parts_in > 0 ? 1.f / (p.ln_inv_c * p.stats_parts_in) : 1.f, part_inv_n = 1.f / part_n;

    auto stats_of = [&](long long mrow, float& mean, float& rstd) {
      ln_row_stats(p.stats_in + mrow * p.stats_parts_in, p.stats_parts_in, part_n, part_inv_n, p.ln_inv_c, p.ln_eps, mean, rstd);
    };
    uint32_t ring = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord tc = decode_tile(p, tile, BN);
      const int n0 = tc.n0;
      int m, b = 0, y = 0, x = 0;
      bool valid;
      if (p.a_mode == AMODE_PLAIN) {
        m = tc.m_tile * BM + r;
        valid = m < p.M;
        if (GEN && (p.remap_rows || p.shuffle_cout)) {
          const int per = p.IH * p.IW;
          b = m / per;
          const int rem = m - b * per;
          if (p.rows_in == ROWS_WINDOW_MAJOR) {
            const int wh = p.IH >> 2, ww = p.IW >> 2, wsz = wh * ww;
            const int win = rem / wsz, t = rem - win * wsz;
            y = (win >> 2) * wh + t / ww;
            x = (win & 3) * ww + t % ww;
          } else {
            y = rem / p.IW;
            x = rem - y * p.IW;
          }
        }
      } else {
        const int ry = r / p.TW;
        y = tc.cy0 + ry;
        x = tc.cx0 + (r - ry * p.TW);
        b = tc.cb;
        valid = (tc.m_tile < p.m_tiles) && (r < p.TW * p.TH) && (y < p.OH) && (x < p.OW);
        m = (b * p.OH + y) * p.OW + x;
      }
      long long out_row = m;
      if (GEN && p.remap_rows) out_row = (static_cast<long long>(b) * p.IH + y) * p.IW + x;
      const long long res_row = p.resid_mod > 0 ? (m % p.resid_mod) : m;
      const bool zero_row = GEN && p.row_zero != nullptr && valid && __ldg(p.row_zero + m) != 0;

      const int npad = p.n_tiles * BN;
      const float* s_bias = s_vec + n0;
      const float* s_gamma = s_vec + npad + n0;
      const float* s_csum = s_vec + 2 * npad + n0;
      // fused LayerNorm (consumer): combine the producer's partial sums of this row; the loads overlap the MMAs below
      float ln_mean = 0.f, ln_rstd = 1.f;
      if (ln_in && valid) stats_of(m, ln_mean, ln_rstd);

      // ------------------------------------------------------------------ main loop: this warpgroup's 64 x BN accumulator
      float acc[BN / 2];
      for (int kb = 0; kb < p.kblocks; ++kb, ++ring) {
        const int s = ring % stages;
        mbar_wait(&full_bar[s], (ring / stages) & 1);
        const uint64_t adesc = wgmma_desc(smem_u32(sA + s * A_STAGE_BYTES + wg * (64 * BK * 2)), 128);
        const uint64_t bdesc = wgmma_desc(smem_u32(sB + s * B_STAGE_BYTES), 128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)     // 16 elements (32 B) along K inside the 128 B swizzle row: +2 in 16-byte units
          Wgmma<Cvt<T>::is_bf16, BN>::ss(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        if (kb > 0) {                          // the previous k-block's MMAs are done: hand its stage back
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[(ring - 1) % stages]);
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[(ring - 1) % stages]);
      // Row statistics for the fused LayerNorm of the consumer, SHIFTED by the first value of the slice: sums of (x - K) and
      // (x - K)^2 do not cancel when the row mean is large against its spread (real checkpoints; E[x^2] - mean^2 would).
      float st_sum = 0.f, st_sq = 0.f, st_K = 0.f;
      bool st_have = false;
      int st_n = 0;
      const T* resid_row = has_resid ? reinterpret_cast<const T*>(p.resid) + res_row * p.ld_resid : nullptr;

      // one 16-column chunk: LN-fold / bias / activation / layer-scale / residual / store
      auto finish_chunk = [&](int c, float (&v)[16], const U8& rr, bool rvec) {
        const int n = n0 + c * 16;
        const int nrem = p.N - n;                     // may be <= 0 for the padded tail of the last n-tile
        if (!valid || nrem <= 0) return;
        const bool full = nrem >= 16;
        // fp32 pairs from here on (ptx.cuh f2_*: adjacent columns travel together)
        uint64_t w[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = f2_pack(v[2 * j], v[2 * j + 1]);
        {
          const float4* sb = reinterpret_cast<const float4*>(s_bias + c * 16);
          if (ln_in) {
            // rstd*(acc - mean*colsum) + bias  ==  a*acc + (b*colsum + bias),  a = rstd, b = -rstd*mean
            const uint64_t a2 = f2_pack(ln_rstd, ln_rstd), b2 = f2_pack(-ln_rstd * ln_mean, -ln_rstd * ln_mean);
            const float4* sc = reinterpret_cast<const float4*>(s_csum + c * 16);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 c4 = lds128(reinterpret_cast<const float*>(sc + j));
              const float4 b4 = lds128(reinterpret_cast<const float*>(sb + j));
              w[2 * j] = f2_fma(a2, w[2 * j], f2_fma(b2, f2_pack(c4.x, c4.y), f2_pack(b4.x, b4.y)));
              w[2 * j + 1] = f2_fma(a2, w[2 * j + 1], f2_fma(b2, f2_pack(c4.z, c4.w), f2_pack(b4.z, b4.w)));
            }
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 b4 = lds128(reinterpret_cast<const float*>(sb + j));
              w[2 * j] = f2_add(w[2 * j], f2_pack(b4.x, b4.y));
              w[2 * j + 1] = f2_add(w[2 * j + 1], f2_pack(b4.z, b4.w));
            }
          }
        }
        if (act == ACT_GELU) {
#pragma unroll
          for (int j = 0; j < 8; ++j) w[j] = gelu_erf2(w[j]);
        } else if (act == ACT_RELU) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float a, b;
            f2_unpack(w[j], a, b);
            w[j] = f2_pack(fmaxf(a, 0.f), fmaxf(b, 0.f));
          }
        } else if (act == ACT_SILU) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float a, b;
            f2_unpack(w[j], a, b);
            w[j] = f2_pack(__fdividef(a, 1.f + __expf(-a)), __fdividef(b, 1.f + __expf(-b)));
          }
        }
        if (has_gamma) {
          const float4* sg = reinterpret_cast<const float4*>(s_gamma + c * 16);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 g4 = lds128(reinterpret_cast<const float*>(sg + j));
            w[2 * j] = f2_mul(w[2 * j], f2_pack(g4.x, g4.y));
            w[2 * j + 1] = f2_mul(w[2 * j + 1], f2_pack(g4.z, g4.w));
          }
        }
        if (rvec) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 f = Cvt<T>::unpack(rr.v[j]);
            w[j] = f2_add(w[j], f2_pack(f.x, f.y));
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) f2_unpack(w[j], v[2 * j], v[2 * j + 1]);
        if (!rvec && (GEN || EP == EP_RESID) && resid_row != nullptr) {
          for (int j = 0; j < 16; ++j)
            if (j < nrem) v[j] += Cvt<T>::to_f(resid_row[n + j]);
        }
        if (GEN && zero_row) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = 0.f;
        }
        // destination
        long long orow = out_row;
        int ocol = n;
        if (GEN && p.hm_S > 0) {                      // head-major: one 16-column chunk = one (slice, head), ld_out == 16
          const int dd = p.hm_heads * 16;
          const int slice = n / dd, head = (n - slice * dd) >> 4;
          const int bb = m / p.hm_S, ss = m - bb * p.hm_S;
          orow = ((static_cast<long long>(bb) * p.hm_slices + slice) * p.hm_heads + head) * p.hm_S + ss;
          ocol = 0;
        }
        if (GEN && p.shuffle_cout > 0) {
          const int q = n / p.shuffle_cout;
          ocol = n - q * p.shuffle_cout;
          orow = (static_cast<long long>(b) * (2 * p.IH) + 2 * y + (q >> 1)) * (2 * p.IW) + 2 * x + (q & 1);
        }
        if (!plain_out && p.out_fp32) {
          float* op = reinterpret_cast<float*>(p.out) + orow * p.ld_out + ocol;
          if (full && (reinterpret_cast<uintptr_t>(op) & 15) == 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              reinterpret_cast<float4*>(op)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          } else {
            for (int j = 0; j < 16; ++j)
              if (j < nrem) op[j] = v[j];
          }
        } else {
          T* op = reinterpret_cast<T*>(p.out) + orow * p.ld_out + ocol;
          if (full && (reinterpret_cast<uintptr_t>(op) & 31) == 0) {
            U8 o;
#pragma unroll
            for (int j = 0; j < 8; ++j) o.v[j] = Cvt<T>::pack(v[2 * j], v[2 * j + 1]);
            stg256(op, o);
            if (do_stats) {                           // statistics of the ROUNDED values the consumer will read
              st_n += 16;
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float2 f = Cvt<T>::unpack(o.v[j]);
                if (!st_have) {
                  st_K = f.x;
                  st_have = true;
                }
                const float d0 = f.x - st_K, d1 = f.y - st_K;
                st_sum += d0 + d1;
                st_sq = fmaf(d0, d0, fmaf(d1, d1, st_sq));
              }
            }
          } else {
            for (int j = 0; j < 16; ++j)
              if (j < nrem) {
                const T h = Cvt<T>::from_f(v[j]);
                op[j] = h;
                if (do_stats) {
                  const float f = Cvt<T>::to_f(h);
                  if (!st_have) {
                    st_K = f;
                    st_have = true;
                  }
                  const float d0 = f - st_K;
                  ++st_n;
                  st_sum += d0;
                  st_sq = fmaf(d0, d0, st_sq);
                }
              }
          }
        }
      };
      // residual prefetch for a chunk (independent of the accumulator)
      auto resid_prefetch = [&](int c, U8& rr) -> bool {
        const int n = n0 + c * 16;
        if ((GEN || EP == EP_RESID) && valid && (p.N - n) >= 16 && resid_row != nullptr && (reinterpret_cast<uintptr_t>(resid_row + n) & 31) == 0) {
          rr = ldg256(resid_row + n);
          return true;
        }
        return false;
      };

      // ------------------------------------------------------------------ epilogue, 64 columns per pass
#pragma unroll
      for (int pc = 0; pc < BN / 64; ++pc) {
        __syncwarp();                                  // the previous pass has been read
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int a0 = 4 * (8 * pc + j), col = 8 * j + 2 * t4;
          *reinterpret_cast<float2*>(stg + g * STG_LD + col) = make_float2(acc[a0], acc[a0 + 1]);
          *reinterpret_cast<float2*>(stg + (g + 8) * STG_LD + col) = make_float2(acc[a0 + 2], acc[a0 + 3]);
        }
        __syncwarp();
#pragma unroll 1                                       // one copy of the (large) chunk code per pass
        for (int i = 0; i < 2; ++i) {
          const int cl = 2 * chalf + i, c = 4 * pc + cl;
          U8 rr;
          const bool rv = resid_prefetch(c, rr);
          float v[16];
          const float* src = stg + (lane >> 1) * STG_LD + cl * 16;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 f = lds128(src + 4 * q);
            v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
          }
          finish_chunk(c, v, rr, rv);
        }
      }
      if (do_stats && valid) {
        // partial = (sum of the slice, sum of squared deviations from the slice's own mean); every slice has the same width
        // (gemm_build checks N % BN == 0 for producers), which is all the consumer needs to combine them (Chan et al.)
        const float nn = static_cast<float>(st_n > 0 ? st_n : 1);
        const float part_sum = fmaf(nn, st_K, st_sum), part_m2 = fmaxf(st_sq - st_sum * st_sum / nn, 0.f);
        p.stats_out[static_cast<long long>(m) * p.stats_parts_out + tc.n_tile * 2 + chalf] = make_float2(part_sum, part_m2);
      }
    }
  }
}



// ------------------------------------------------------------------------------------------- FP8 (e4m3) GEMM
// The encoder's qkv and fc1 in the e4m3 compute mode (gemm_tc.h GemmE4m3Desc).  Same tile walk, producer / consumer split,
// stage ring and accumulator staging as gemm_tc_kernel, with 1-byte operands: a k-block is one 128-byte swizzle row, i.e.
// 128 elements, and the MMA is m64nBNk32 e4m3 x e4m3 -> fp32.  A k-block past K (K = 192: the second one is half empty)
// is zero-filled by TMA.  Epilogue: out = act(a_scale[m] * w_scale[n] * acc + bias[n]) -> fp16; no residual, LayerNorm
// fold, row statistics or row remap.
static constexpr int BK8 = 128;
static constexpr int A8_STAGE_BYTES = BM * BK8;

template <int BN, bool GELU>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_e4m3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmArgs p) {
  constexpr int B_STAGE_BYTES = BN * BK8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stages = p.stages;
  uint8_t* sA = smem;
  uint8_t* sB = smem + stages * A8_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sB + stages * B_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  float* s_stage = reinterpret_cast<float*>(full_bar + 32);
  float* s_vec = s_stage + MMA_WARPS * 16 * STG_LD;           // {w_scale | bias}[n_tiles * BN]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], MMA_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();

  if (warp < 4) {
    reg_dec<40>();
    if (warp == 0 && lane == 0) {
      uint32_t ring = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord tc = decode_tile(p, tile, BN);
        for (int kb = 0; kb < p.kblocks; ++kb, ++ring) {
          const int s = ring % stages;
          mbar_wait(&empty_bar[s], ((ring / stages) & 1) ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], A8_STAGE_BYTES + B_STAGE_BYTES);
          tma_load_2d(sA + s * A8_STAGE_BYTES, &tmA, &full_bar[s], kb * BK8, tc.m_tile * BM);
          tma_load_2d(sB + s * B_STAGE_BYTES, &tmB, &full_bar[s], kb * BK8, tc.n0);
        }
      }
    }
  } else {
    reg_inc<232>();
    const int cw = warp - 4, wg = cw >> 2;
    const int g = lane >> 2, t4 = lane & 3;
    const int chalf = lane & 1;
    const int r = cw * 16 + (lane >> 1);
    float* stg = s_stage + cw * 16 * STG_LD;
    const int npad = p.n_tiles * BN;
    for (int i = threadIdx.x - 128; i < npad; i += 32 * MMA_WARPS) {
      const bool in = i < p.N;
      s_vec[i] = in ? __ldg(p.w_scale + i) : 0.f;
      s_vec[npad + i] = (p.bias != nullptr && in) ? __ldg(p.bias + i) : 0.f;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(32 * MMA_WARPS) : "memory");

    uint32_t ring = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const TileCoord tc = decode_tile(p, tile, BN);
      const int n0 = tc.n0;
      const int m = tc.m_tile * BM + r;
      const bool valid = m < p.M;
      const float sa = valid ? __ldg(p.a_scale + m) : 0.f;   // the load overlaps the MMAs below

      float acc[BN / 2];
      for (int kb = 0; kb < p.kblocks; ++kb, ++ring) {
        const int s = ring % stages;
        mbar_wait(&full_bar[s], (ring / stages) & 1);
        const uint64_t adesc = wgmma_desc(smem_u32(sA + s * A8_STAGE_BYTES + wg * (64 * BK8)), 128);
        const uint64_t bdesc = wgmma_desc(smem_u32(sB + s * B_STAGE_BYTES), 128);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK8 / 32; ++k)     // 32 elements (32 B) along K inside the 128 B swizzle row: +2 in 16-byte units
          WgmmaE4m3<BN>::ss(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[(ring - 1) % stages]);
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (lane == 0) mbar_arrive(&empty_bar[(ring - 1) % stages]);

      __half* out_row = reinterpret_cast<__half*>(p.out) + static_cast<long long>(m) * p.ld_out;
      const uint64_t sa2 = f2_pack(sa, sa);
#pragma unroll
      for (int pc = 0; pc < BN / 64; ++pc) {
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int a0 = 4 * (8 * pc + j), col = 8 * j + 2 * t4;
          *reinterpret_cast<float2*>(stg + g * STG_LD + col) = make_float2(acc[a0], acc[a0 + 1]);
          *reinterpret_cast<float2*>(stg + (g + 8) * STG_LD + col) = make_float2(acc[a0 + 2], acc[a0 + 3]);
        }
        __syncwarp();
#pragma unroll 1
        for (int i = 0; i < 2; ++i) {
          const int c = 4 * pc + 2 * chalf + i;
          const int n = n0 + c * 16, nrem = p.N - n;
          if (!valid || nrem <= 0) continue;
          const float* src = stg + (lane >> 1) * STG_LD + (2 * chalf + i) * 16;
          const float* sw = s_vec + n;
          const float* sb = s_vec + npad + n;
          uint64_t w[8];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 f = lds128(src + 4 * q), w4 = lds128(sw + 4 * q), b4 = lds128(sb + 4 * q);
            w[2 * q] = f2_fma(f2_mul(sa2, f2_pack(w4.x, w4.y)), f2_pack(f.x, f.y), f2_pack(b4.x, b4.y));
            w[2 * q + 1] = f2_fma(f2_mul(sa2, f2_pack(w4.z, w4.w)), f2_pack(f.z, f.w), f2_pack(b4.z, b4.w));
          }
          if (GELU) {
#pragma unroll
            for (int j = 0; j < 8; ++j) w[j] = gelu_erf2(w[j]);
          }
          __half* op = out_row + n;
          if (nrem >= 16 && (reinterpret_cast<uintptr_t>(op) & 31) == 0) {
            U8 o;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float a, b;
              f2_unpack(w[j], a, b);
              o.v[j] = Cvt<__half>::pack(a, b);
            }
            stg256(op, o);
          } else {
            for (int j = 0; j < 8; ++j) {
              float a, b;
              f2_unpack(w[j], a, b);
              if (2 * j < nrem) op[2 * j] = __float2half_rn(a);
              if (2 * j + 1 < nrem) op[2 * j + 1] = __float2half_rn(b);
            }
          }
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------- host
static int encode(CUtensorMap* tm, int dtype, int rank, const void* base, const cuuint64_t* dims,
                  const cuuint64_t* strides_bytes, const cuuint32_t* box, std::string* err) {
  return tma_encode(tm, dtype, rank, base, dims, strides_bytes, box, 128, err);
}

static int num_sms() { return current_device_sms(); }

static int pick_bn(int N, int m_tiles) {
  int bn;
  if (N <= 64) bn = 64;
  else if (N <= 128) bn = 128;
  else {
    const int cand[3] = {256, 192, 128};
    int best = 256, best_waste = 1 << 30;
    for (int c : cand) {
      const int waste = ((N + c - 1) / c) * c - N;
      if (waste < best_waste) { best_waste = waste; best = c; }
    }
    bn = best;
  }
  // Small problems: prefer more CTAs over wider tiles so that every SM gets work.
  auto tiles = [&](int b) { return static_cast<long long>(m_tiles) * ((N + b - 1) / b); };
  while (bn > 64 && tiles(bn) < num_sms()) {
    const int nb = bn == 256 ? 128 : (bn == 192 ? 64 : 64);
    if (((N + nb - 1) / nb) * nb - N > ((N + bn - 1) / bn) * bn - N + 32) break;
    bn = nb;
  }
  return bn;
}

void conv_tile_plan(int OH, int OW, int* tw_out, int* th_out) {
  // tile = TW x TH output pixels (<= 128): maximise useful rows
  int best_tw = 1, best_th = 1; double best_u = -1;
  for (int tw = 1; tw <= std::min(OW, 128); ++tw) {
    const int th = std::min(128 / tw, OH);
    const long long tiles = static_cast<long long>((OW + tw - 1) / tw) * ((OH + th - 1) / th);
    const double u = static_cast<double>(OW) * OH / (tiles * 128.0);
    if (u > best_u + 1e-9) { best_u = u; best_tw = tw; best_th = th; }
  }
  *tw_out = best_tw; *th_out = best_th;
}

int gemm_build(const GemmDesc& d, GemmOp* op, std::string* err) {
  std::memset(op, 0, sizeof(*op));
  if (d.dtype != DT_F16 && d.dtype != DT_BF16) { *err = "gemm: dtype must be fp16 or bf16"; return -1; }
  if (d.K % BK != 0 || d.K <= 0) { *err = "gemm: K must be a positive multiple of 64"; return -1; }
  if (!d.out_fp32 && (d.ld_out % 8) != 0) { *err = "gemm: 16-bit ld_out must be a multiple of 8"; return -1; }
  if ((d.lda % 8) != 0) { *err = "gemm: lda must be a multiple of 8"; return -1; }
  GemmArgs& a = op->args;
  a.M = d.M; a.N = d.N; a.kblocks = d.K / BK; a.a_mode = d.a_mode; a.lda = d.lda;
  a.bias = d.bias; a.gamma = d.gamma; a.resid = d.resid; a.ld_resid = d.ld_resid; a.resid_mod = d.resid_mod;
  a.act = d.act; a.out = d.out; a.ld_out = d.ld_out; a.out_fp32 = d.out_fp32;
  a.rows_in = d.rows_in; a.remap_rows = d.remap_rows; a.shuffle_cout = d.shuffle_cout; a.IH = d.IH; a.IW = d.IW;
  a.hm_S = d.hm_S; a.hm_heads = d.hm_heads; a.hm_slices = d.hm_slices; a.row_zero = d.row_zero;
  if (d.hm_S > 0) {
    if (d.a_mode != AMODE_PLAIN || d.remap_rows || d.shuffle_cout || d.out_fp32 || d.hm_heads < 1 || d.hm_slices < 1 ||
        d.N != d.hm_slices * d.hm_heads * 16 || d.M % d.hm_S != 0) { *err = "gemm: head-major store needs a plain 16-bit GEMM with N == slices*heads*16 and M % S == 0"; return -1; }
    a.ld_out = 16;
  }
  if (d.out_fp32 && d.ld_out < d.N) { *err = "gemm: fp32 ld_out must be >= N"; return -1; }
  a.stats_out = d.stats_out; a.stats_in = d.stats_in; a.stats_parts_in = d.stats_parts_in; a.colsum = d.colsum;
  a.ln_inv_c = d.ln_C > 0 ? 1.f / d.ln_C : 0.f; a.ln_eps = d.ln_eps;
  if ((d.stats_out || d.stats_in) && (d.a_mode != AMODE_PLAIN || d.remap_rows || d.shuffle_cout || d.out_fp32)) { *err = "gemm: LN fusion needs a plain 16-bit GEMM"; return -1; }
  if (d.stats_in && (!d.colsum || d.stats_parts_in <= 0 || d.ln_C <= 0 || d.ln_C % d.stats_parts_in != 0)) { *err = "gemm: LN consumer needs colsum / parts / C (C a multiple of the partial count)"; return -1; }
  op->dtype = d.dtype;
  if ((d.remap_rows || d.shuffle_cout) && (d.IH <= 0 || d.IW <= 0 || d.M % (d.IH * d.IW) != 0)) {
    *err = "gemm: row remap needs IH/IW with M a multiple of IH*IW"; return -1;
  }
  if (d.rows_in == ROWS_WINDOW_MAJOR && ((d.IH % 4) || (d.IW % 4))) { *err = "gemm: window grid needs IH,IW % 4 == 0"; return -1; }
  if (d.shuffle_cout > 0 && (d.shuffle_cout % 16 != 0 || d.N != 4 * d.shuffle_cout)) {
    *err = "gemm: pixel-shuffle needs N == 4*cout, cout % 16 == 0"; return -1;
  }

  int m_tiles;
  if (d.a_mode == AMODE_PLAIN) {
    m_tiles = (d.M + BM - 1) / BM;
    a.a_stage_tx = A_STAGE_BYTES;
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.K), static_cast<cuuint64_t>(d.M)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.lda) * 2};
    const cuuint32_t box[2] = {BK, BM};
    if (encode(&op->ta, d.dtype, 2, d.A, dims, strides, box, err)) return -1;
  } else {
    if (d.K % 9 != 0 || (d.K / 9) % BK != 0) { *err = "gemm: conv needs K = 9*Cin, Cin % 64 == 0"; return -1; }
    if (d.M != d.B * d.OH * d.OW) { *err = "gemm: conv needs M == B*OH*OW"; return -1; }
    const int cin = d.K / 9;
    a.cin_blocks = cin / BK;
    a.OH = d.OH; a.OW = d.OW;
    conv_tile_plan(d.OH, d.OW, &a.TW, &a.TH);
    a.tiles_x = (d.OW + a.TW - 1) / a.TW;
    a.tiles_y = (d.OH + a.TH - 1) / a.TH;
    m_tiles = d.B * a.tiles_x * a.tiles_y;
    a.a_stage_tx = static_cast<uint32_t>(a.TW * a.TH * BK * 2);
    if (d.a_mode == AMODE_CONV3_S1) {
      const cuuint64_t dims[4] = {static_cast<cuuint64_t>(cin), static_cast<cuuint64_t>(d.OW),
                                  static_cast<cuuint64_t>(d.OH), static_cast<cuuint64_t>(d.B)};
      const cuuint64_t strides[3] = {static_cast<cuuint64_t>(d.lda) * 2, static_cast<cuuint64_t>(d.OW) * d.lda * 2,
                                     static_cast<cuuint64_t>(d.OH) * d.OW * d.lda * 2};
      const cuuint32_t box[4] = {BK, static_cast<cuuint32_t>(a.TW), static_cast<cuuint32_t>(a.TH), 1};
      if (encode(&op->ta, d.dtype, 4, d.A, dims, strides, box, err)) return -1;
    } else {
      // input grid is (2*OH) x (2*OW); view it as [B, OH, 2, OW, (2, lda)] so that a stride-2 tap is a dense box
      const int IWin = 2 * d.OW, IHin = 2 * d.OH;
      const cuuint64_t dims[5] = {static_cast<cuuint64_t>(2) * d.lda, static_cast<cuuint64_t>(d.OW), 2,
                                  static_cast<cuuint64_t>(d.OH), static_cast<cuuint64_t>(d.B)};
      const cuuint64_t strides[4] = {static_cast<cuuint64_t>(2) * d.lda * 2, static_cast<cuuint64_t>(IWin) * d.lda * 2,
                                     static_cast<cuuint64_t>(2) * IWin * d.lda * 2,
                                     static_cast<cuuint64_t>(IHin) * IWin * d.lda * 2};
      const cuuint32_t box[5] = {BK, static_cast<cuuint32_t>(a.TW), 1, static_cast<cuuint32_t>(a.TH), 1};
      if (encode(&op->ta, d.dtype, 5, d.A, dims, strides, box, err)) return -1;
    }
  }

  const int bn = pick_bn(d.N, m_tiles);
  if (d.stats_out && d.N % bn != 0) { *err = "gemm: a LayerNorm-statistics producer needs N to be a multiple of its n-tile (equal-width partials)"; return -1; }
  op->bn = bn;
  a.n_tiles = (d.N + bn - 1) / bn;
  {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.K), static_cast<cuuint64_t>(d.N)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.K) * 2};
    const cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(bn)};
    if (encode(&op->tb, d.dtype, 2, d.W, dims, strides, box, err)) return -1;
  }
  const int stage_bytes = A_STAGE_BYTES + bn * BK * 2;
  const size_t vec_bytes = 3 * 4 * static_cast<size_t>(a.n_tiles) * bn;     // bias | gamma | colsum for all n-tiles
  int stages = static_cast<int>((225 * 1024 - STG_BYTES - vec_bytes) / stage_bytes);
  stages = std::min(stages, MAX_STAGES);
  stages = std::max(2, std::min(stages, std::max(2, 2 * a.kblocks)));
  a.stages = stages;
  a.m_tiles = m_tiles;
  op->smem = 1024 + static_cast<size_t>(stages) * stage_bytes + 256 + STG_BYTES + vec_bytes;
  const long long tiles = static_cast<long long>(m_tiles) * a.n_tiles;
  op->grid = static_cast<unsigned>(std::min<long long>(tiles, num_sms()));
  a.stats_parts_out = a.n_tiles * 2;     // the LayerNorm partials a producer writes per row: one per (n-tile, column half)
  op->flops = 2.0 * d.M * static_cast<double>(d.N) * d.K;
  return 0;
}

template <typename T, int BN, int EP>
static int launch_inst(const GemmOp& op, cudaStream_t st) {
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(gemm_tc_kernel<T, BN, EP>), 227 * 1024)) return e;
  launch_k(gemm_tc_kernel<T, BN, EP>, dim3(op.grid), dim3(GEMM_THREADS), op.smem, st, op.ta, op.tb, op.args);
  return static_cast<int>(cudaGetLastError());
}

static int pick_ep(const GemmArgs& a) {
  const bool special_rows = a.out_fp32 || a.remap_rows || a.shuffle_cout > 0 || a.hm_S > 0 || a.row_zero != nullptr;
  if (special_rows) return EP_GENERIC;
  if (a.stats_in) {
    if (a.gamma || a.resid || a.stats_out) return EP_GENERIC;
    if (a.act == ACT_NONE) return EP_LN;
    if (a.act == ACT_GELU) return EP_LN_GELU;
    return EP_GENERIC;
  }
  if (a.gamma || a.resid || a.stats_out) return a.act == ACT_NONE ? EP_RESID : EP_GENERIC;
  return a.act == ACT_NONE ? EP_BIAS : EP_BIAS_ACT;
}

int gemm_epilogue(const GemmOp& op) { return op.dtype == DT_E4M3 ? -1 : pick_ep(op.args); }

template <typename T, int BN>
static int launch_ep(const GemmOp& op, cudaStream_t st) {
  switch (pick_ep(op.args)) {
    case EP_BIAS: return launch_inst<T, BN, EP_BIAS>(op, st);
    case EP_BIAS_ACT: return launch_inst<T, BN, EP_BIAS_ACT>(op, st);
    case EP_LN: return launch_inst<T, BN, EP_LN>(op, st);
    case EP_LN_GELU: return launch_inst<T, BN, EP_LN_GELU>(op, st);
    case EP_RESID: return launch_inst<T, BN, EP_RESID>(op, st);
    default: return launch_inst<T, BN, EP_GENERIC>(op, st);
  }
}

int gemm_e4m3_build(const GemmE4m3Desc& d, GemmOp* op, std::string* err) {
  std::memset(op, 0, sizeof(*op));
  if (!d.A || !d.W || !d.a_scale || !d.w_scale || !d.out) { *err = "gemm_e4m3: null pointer"; return -1; }
  if (d.M < 1 || d.N < 1 || d.K <= 0 || d.K % 64 != 0) { *err = "gemm_e4m3: M, N must be positive and K a positive multiple of 64"; return -1; }
  if (d.lda < d.K || d.lda % 16 != 0) { *err = "gemm_e4m3: lda must be >= K and a multiple of 16 bytes"; return -1; }
  if (d.ld_out < d.N || d.ld_out % 8 != 0) { *err = "gemm_e4m3: ld_out must be >= N and a multiple of 8"; return -1; }
  if (d.act != ACT_NONE && d.act != ACT_GELU) { *err = "gemm_e4m3: act must be NONE or GELU"; return -1; }
  GemmArgs& a = op->args;
  a.M = d.M; a.N = d.N; a.kblocks = (d.K + BK8 - 1) / BK8; a.a_mode = AMODE_PLAIN; a.lda = d.lda;
  a.bias = d.bias; a.act = d.act; a.out = d.out; a.ld_out = d.ld_out;
  a.a_scale = d.a_scale; a.w_scale = d.w_scale;
  op->dtype = DT_E4M3;
  const int m_tiles = (d.M + BM - 1) / BM;
  {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.K), static_cast<cuuint64_t>(d.M)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.lda)};
    const cuuint32_t box[2] = {BK8, BM};
    if (encode(&op->ta, DT_E4M3, 2, d.A, dims, strides, box, err)) return -1;
  }
  const int bn = pick_bn(d.N, m_tiles);
  op->bn = bn;
  a.n_tiles = (d.N + bn - 1) / bn;
  {
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(d.K), static_cast<cuuint64_t>(d.N)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(d.K)};
    const cuuint32_t box[2] = {BK8, static_cast<cuuint32_t>(bn)};
    if (encode(&op->tb, DT_E4M3, 2, d.W, dims, strides, box, err)) return -1;
  }
  const int stage_bytes = A8_STAGE_BYTES + bn * BK8;
  const size_t vec_bytes = 2 * 4 * static_cast<size_t>(a.n_tiles) * bn;     // w_scale | bias for all n-tiles
  int stages = static_cast<int>((225 * 1024 - STG_BYTES - vec_bytes) / stage_bytes);
  stages = std::min(stages, MAX_STAGES);
  stages = std::max(2, std::min(stages, std::max(2, 2 * a.kblocks)));
  a.stages = stages;
  a.m_tiles = m_tiles;
  op->smem = 1024 + static_cast<size_t>(stages) * stage_bytes + 256 + STG_BYTES + vec_bytes;
  op->grid = static_cast<unsigned>(std::min<long long>(static_cast<long long>(m_tiles) * a.n_tiles, num_sms()));
  op->flops = 2.0 * d.M * static_cast<double>(d.N) * d.K;
  return 0;
}

template <int BN, bool GELU>
static int launch_e4m3(const GemmOp& op, cudaStream_t st) {
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(gemm_e4m3_kernel<BN, GELU>), 227 * 1024)) return e;
  launch_k(gemm_e4m3_kernel<BN, GELU>, dim3(op.grid), dim3(GEMM_THREADS), op.smem, st, op.ta, op.tb, op.args);
  return static_cast<int>(cudaGetLastError());
}

static int gemm_e4m3_launch(const GemmOp& op, cudaStream_t st) {
  const bool gelu = op.args.act == ACT_GELU;
  switch (op.bn) {
    case 64: return gelu ? launch_e4m3<64, true>(op, st) : launch_e4m3<64, false>(op, st);
    case 128: return gelu ? launch_e4m3<128, true>(op, st) : launch_e4m3<128, false>(op, st);
    case 192: return gelu ? launch_e4m3<192, true>(op, st) : launch_e4m3<192, false>(op, st);
    case 256: return gelu ? launch_e4m3<256, true>(op, st) : launch_e4m3<256, false>(op, st);
    default: return -1;
  }
}

int gemm_launch(const GemmOp& op, cudaStream_t st) {
  if (op.dtype == DT_E4M3) return gemm_e4m3_launch(op, st);
#define LWB_BN_SWITCH(T)                                     \
  switch (op.bn) {                                           \
    case 64: return launch_ep<T, 64>(op, st);                \
    case 128: return launch_ep<T, 128>(op, st);              \
    case 192: return launch_ep<T, 192>(op, st);              \
    case 256: return launch_ep<T, 256>(op, st);              \
    default: return -1;                                      \
  }
  if (op.dtype == DT_BF16) { LWB_BN_SWITCH(__nv_bfloat16) } else { LWB_BN_SWITCH(__half) }
#undef LWB_BN_SWITCH
}

}  // namespace lwb