// wgmma / TMA flash attention for the packed qkv matrix - the ViT window attention (vit.py:130-137 with B' = 16B, N = 100)
// and the ViT global attention (vit.py:201-204), head dims 16 / 32 / 64.
//
// One CTA owns one 128-row query tile of one (sequence, head).  Q, K and V tiles are fetched by TMA straight out of the
// packed [rows, 3C] matrix (box = rows x dh columns at column  part*C + head*dh, hardware swizzle matching the dh*2-byte
// row pitch), K / V in chunks of 64 keys through a ring of stages (full / empty mbarriers):
//   warps 0-7 : two consumer warpgroups, 64 query rows each.  S = Q K^T is one wgmma m64n64k16 chain with both operands
//               in shared memory; the online softmax runs on the accumulator fragments in registers (row maxima and sums
//               across the four threads of a row by shuffles, exp2 against the running maximum of the raw scores); P goes
//               back to the tensor core as the REGISTER A operand of O += P V, whose B operand is the V chunk as it lies
//               in shared memory (MN-major, transposed by the tensor core).  O never leaves the registers until the end.
//               A warpgroup whose 64 rows lie beyond the sequence (100-token windows use 100 of 128 rows, the last tile
//               of a 1600-token sequence 64) exits at once.
//   warp 8    : TMA producer (one elected lane).
// The kernel keeps no cross-chunk overlap inside a warpgroup; latency is hidden by the second warpgroup and by the other
// resident CTAs of the SM: 3 at head dim 16 (at most 72 registers), 2 at 32 and 64.  The last chunk of a sequence masks the keys
// beyond its end; one of at most 40 keys (the second chunk of a 100-token window) computes only 5 of the 8 n-tiles.
#include "attn.h"
#include "launch.h"
#include "ptx.cuh"
#include "tma_util.h"
#include "wgmma.cuh"

#include <string>

namespace lwb {
namespace wg {

static constexpr int BM = 128;                 // query rows per CTA
static constexpr int BK = 64;                  // keys per chunk
static constexpr int STAGES = 4;
static constexpr int THREADS = 32 * 9;

template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Keys [kbase, kbase + 8 NT) of one K / V stage for the warpgroup's 64 query rows: S = Q K^T, online softmax on the
// fragments, O += P V.
//   NT   : 8-key n-tiles computed - 8 = the whole stage; 5 = keys 0..39 of it (the second stage of a 100-token window:
//          no scores, exponentials or P V steps are spent on keys that cannot exist).
//   MASK : keys at or beyond seqlen become -inf (the sequence's last stage).
template <typename T, int DH, int NT, bool MASK>
__device__ __forceinline__ void attend_chunk(uint64_t qdesc, uint64_t kdesc, uint64_t vdesc, int kbase, int seqlen, float c, int t4,
                                             float (&m_run)[2], float (&lsum)[2], float (&o)[DH / 2]) {
  constexpr bool BF = Cvt<T>::is_bf16;
  constexpr uint32_t PITCH = DH * 2;
  constexpr int NTP = (NT + 1) & ~1;                             // P V runs 16 keys per step
  float sc[NT * 4];
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < DH / 16; ++kk) Wgmma<BF, NT * 8>::ss(sc, qdesc + 2 * kk, kdesc + 2 * kk, kk != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(sc);
  if (MASK) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (kbase + nt * 8 + t4 * 2 + (e & 1) >= seqlen) sc[4 * nt + e] = -INFINITY;
  }
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    mx[0] = fmaxf(mx[0], fmaxf(sc[4 * nt], sc[4 * nt + 1]));
    mx[1] = fmaxf(mx[1], fmaxf(sc[4 * nt + 2], sc[4 * nt + 3]));
  }
  float alpha[2], msc[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float m_new = fmaxf(m_run[h], mx[h]);                  // running max of the RAW scores (finite: key kbase is valid)
    alpha[h] = ex2((m_run[h] - m_new) * c);
    m_run[h] = m_new;
    msc[h] = m_new * c;
    lsum[h] *= alpha[h];
  }
  uint32_t pf[NTP / 2][4];                                       // C fragments of n-tiles (2k, 2k+1) form the A fragment of key-step k
#pragma unroll
  for (int nt = 0; nt < NTP; ++nt) {
    if (nt >= NT) {                                              // padding half of the last 16-key step
      pf[nt >> 1][(nt & 1) * 2 + 0] = 0u;
      pf[nt >> 1][(nt & 1) * 2 + 1] = 0u;
      continue;
    }
    const float p0 = ex2(fmaf(sc[4 * nt], c, -msc[0])), p1 = ex2(fmaf(sc[4 * nt + 1], c, -msc[0]));
    const float p2 = ex2(fmaf(sc[4 * nt + 2], c, -msc[1])), p3 = ex2(fmaf(sc[4 * nt + 3], c, -msc[1]));
    lsum[0] += p0 + p1;
    lsum[1] += p2 + p3;
    pf[nt >> 1][(nt & 1) * 2 + 0] = Cvt<T>::pack(p0, p1);
    pf[nt >> 1][(nt & 1) * 2 + 1] = Cvt<T>::pack(p2, p3);
  }
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    o[4 * dt] *= alpha[0];
    o[4 * dt + 1] *= alpha[0];
    o[4 * dt + 2] *= alpha[1];
    o[4 * dt + 3] *= alpha[1];
  }
  // ---- O += P V: 16 keys per MMA, B advances 16 rows of the MN-major V chunk
  fence_regs(o);
  wgmma_fence();
#pragma unroll
  for (int kt = 0; kt < NTP / 2; ++kt) Wgmma<BF, DH>::rs_tb(o, pf[kt], vdesc + ((16 * PITCH) >> 4) * kt, 1u);
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(o);
}

// Resident CTAs per SM the register budget is cut for.  Each warpgroup runs S -> softmax -> P V one after another, so
// only the other warpgroups on the SM cover its MMA round trips: at head dim 16 the kernel is cut to 72 registers for 3
// CTAs (small's global attention: 427 us with 2, 380 us with 3, on an H100 80GB HBM3 at 700 W).  At 32, 72 registers
// would spill; 64 is held to 2 by shared memory.
template <int DH> constexpr int kMinCtas = DH == 16 ? 3 : 2;

template <typename T, int DH>
__global__ void __launch_bounds__(THREADS, kMinCtas<DH>) attn_wg_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                                                                          const AttnArgs p, int C) {
  constexpr uint32_t PITCH = DH * 2;                           // bytes per row = swizzle span
  constexpr int Q_BYTES = BM * DH * 2, KV_BYTES = BK * DH * 2;
  extern __shared__ uint8_t wg_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(wg_smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + Q_BYTES;                                 // [stage][K | V]
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sKV + STAGES * 2 * KV_BYTES);
  uint64_t* kv_full = q_full + 1;
  uint64_t* kv_empty = kv_full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int head = blockIdx.y, seq = blockIdx.z;
  const int q0 = blockIdx.x * BM;
  const int row0 = seq * p.seqlen;                              // first matrix row of this sequence
  const int nchunks = (p.seqlen + BK - 1) / BK;
  const int active_wgs = q0 + 64 < p.seqlen ? 2 : 1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    mbar_init(q_full, 1);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 4 * active_wgs);                  // one elected arrival per working consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_sync();   // the prologue above touched no global data; everything below reads the predecessor's output

  if (warp == 8) {
    if (lane == 0) {
      // ------------------------------------------------------------------ TMA producer
      mbar_arrive_expect_tx(q_full, Q_BYTES);
      tma_load_2d(sQ, &tmQ, q_full, head * DH, row0 + q0);
      for (int j = 0; j < nchunks; ++j) {
        const int s = j % STAGES;
        mbar_wait(&kv_empty[s], ((j / STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * KV_BYTES);
        tma_load_2d(sKV + s * 2 * KV_BYTES, &tmKV, &kv_full[s], C + head * DH, row0 + j * BK);
        tma_load_2d(sKV + s * 2 * KV_BYTES + KV_BYTES, &tmKV, &kv_full[s], 2 * C + head * DH, row0 + j * BK);
      }
    }
    return;
  }
  // ---------------------------------------------------------------------- consumers: S, softmax, P V for 64 query rows
  const int wgi = warp >> 2;
  if (wgi >= active_wgs) return;
  const int g = lane >> 2, t4 = lane & 3;                        // fragment rows 16*(warp % 4) + g (+8), columns 8n + 2*t4 (+1)
  const float c = p.scale_log2;
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
  const uint64_t qdesc = wgmma_desc(smem_u32(sQ + wgi * 64 * PITCH), PITCH);
  mbar_wait(q_full, 0);
  for (int j = 0; j < nchunks; ++j) {
    const int s = j % STAGES;
    mbar_wait(&kv_full[s], (j / STAGES) & 1);
    const uint64_t kdesc = wgmma_desc(smem_u32(sKV + s * 2 * KV_BYTES), PITCH);
    const uint64_t vdesc = wgmma_desc(smem_u32(sKV + s * 2 * KV_BYTES + KV_BYTES), PITCH);
    // keys beyond the sequence (the next sequence's rows / zero fill) are masked in the last chunk
    const int rem = p.seqlen - j * BK;
    if (rem >= BK) attend_chunk<T, DH, BK / 8, false>(qdesc, kdesc, vdesc, j * BK, p.seqlen, c, t4, m_run, lsum, o);
    else if (rem <= 40) attend_chunk<T, DH, 5, true>(qdesc, kdesc, vdesc, j * BK, p.seqlen, c, t4, m_run, lsum, o);
    else attend_chunk<T, DH, BK / 8, true>(qdesc, kdesc, vdesc, j * BK, p.seqlen, c, t4, m_run, lsum, o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }
  // ---- finalise: divide by the row sums, stage through this warp's own Q rows, 16-byte coalesced stores
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lsum[h] += __shfl_xor_sync(0xffffffffu, lsum[h], 1);
    lsum[h] += __shfl_xor_sync(0xffffffffu, lsum[h], 2);
  }
  const float inv[2] = {1.f / lsum[0], 1.f / lsum[1]};
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wgi) : "memory");   // every warp of the warpgroup is done with the Q tile
  T* sO = reinterpret_cast<T*>(sQ) + warp * 16 * DH;
#pragma unroll
  for (int dt = 0; dt < DH / 8; ++dt) {
    *reinterpret_cast<uint32_t*>(sO + g * DH + dt * 8 + t4 * 2) = Cvt<T>::pack(o[4 * dt] * inv[0], o[4 * dt + 1] * inv[0]);
    *reinterpret_cast<uint32_t*>(sO + (g + 8) * DH + dt * 8 + t4 * 2) = Cvt<T>::pack(o[4 * dt + 2] * inv[1], o[4 * dt + 3] * inv[1]);
  }
  __syncwarp();
  constexpr int CPR = DH / 8;                                    // 16-byte pieces per row
  T* go = reinterpret_cast<T*>(p.o) + head * DH;
  for (int i = lane; i < 16 * CPR; i += 32) {
    const int r = i / CPR, cc = i % CPR;
    const int qrow = q0 + warp * 16 + r;
    if (qrow < p.seqlen)
      *reinterpret_cast<U4*>(go + (static_cast<long long>(row0) + qrow) * p.ldo + cc * 8) = *reinterpret_cast<const U4*>(sO + r * DH + cc * 8);
  }
}

template <typename T, int DH>
static int launch(const AttnArgs& a, int C, cudaStream_t st) {
  CUtensorMap tq, tkv;
  std::string err;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(a.ldq), static_cast<cuuint64_t>(a.nseq) * a.seqlen};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(a.ldq) * 2};
  const cuuint32_t boxq[2] = {DH, BM}, boxkv[2] = {DH, BK};
  const int dt = Cvt<T>::is_bf16 ? DT_BF16 : DT_F16;
  if (tma_encode(&tq, dt, 2, a.q, dims, strides, boxq, DH * 2, &err)) return -3;
  if (tma_encode(&tkv, dt, 2, a.q, dims, strides, boxkv, DH * 2, &err)) return -3;
  const size_t smem = 1024 + static_cast<size_t>(BM + STAGES * 2 * BK) * DH * 2 + 128;
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(attn_wg_kernel<T, DH>), 100 * 1024)) return e;
  dim3 grid((a.seqlen + BM - 1) / BM, a.heads, a.nseq);
  launch_k(attn_wg_kernel<T, DH>, grid, dim3(THREADS), smem, st, tq, tkv, a, C);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace wg

// Packed-qkv path: q, k, v are the column blocks [0,C), [C,2C), [2C,3C) of one 16-bit matrix.
int attention_wg_launch(int dtype, const AttnArgs& a, int dh, int C, cudaStream_t st) {
  if (dtype == DT_BF16) {
    if (dh == 16) return wg::launch<__nv_bfloat16, 16>(a, C, st);
    if (dh == 32) return wg::launch<__nv_bfloat16, 32>(a, C, st);
    if (dh == 64) return wg::launch<__nv_bfloat16, 64>(a, C, st);
  } else {
    if (dh == 16) return wg::launch<__half, 16>(a, C, st);
    if (dh == 32) return wg::launch<__half, 32>(a, C, st);
    if (dh == 64) return wg::launch<__half, 64>(a, C, st);
  }
  return -2;
}

}  // namespace lwb
