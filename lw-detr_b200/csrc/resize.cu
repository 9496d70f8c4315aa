// Raw camera / decoder frames -> patch matrix: antialiased bilinear resize, /255, Normalize and the window-major patch
// gather in one kernel.  Replaces the host-side transforms.Resize (PIL, antialiased bilinear) of demo/demo.py:146-159 and
// datasets/transforms.py:97-134,223-252 in front of the existing uint8 path: neither the resized uint8 image nor an fp32
// image ever exists in HBM.
//
// The filter is the separable triangle filter of PIL.Image.resize(BILINEAR) and F.interpolate(mode="bilinear",
// antialias=True).  Per axis n_in -> n_out: scale = n_in / n_out, support = max(scale, 1); output o has centre
// c = (o + 0.5) * scale, taps x in [max(int(c - support + 0.5), 0), min(int(c + support + 0.5), n_in)) with weight
// max(0, 1 - |x - c + 0.5| / support) divided by the sum of the weights.  Horizontal pass, then vertical, fp32; the result
// is rounded half up to an integer level (floor(v + 0.5) in fp32) and clamped to [0, 255], i.e. it is the uint8 frame a
// host resize would have produced, and then takes the arithmetic of patch_gather_u8_kernel: (v / 255 - mean) / std with
// IEEE divisions.  At n_in == n_out every tap weight is exactly 1 or 0 and the output equals patch_gather_u8_kernel's bit
// for bit.  tools/resize_spec.py restates the filter for the tests.
//
// One CTA = 16 x 64 output pixels (one token row, four tokens).  The tap tables of the tile's 64 columns and 16 rows are
// computed from the frame's sizes in shared memory (frames of a batch differ: there is no per-plan table).  The source
// rows the tile touches are walked in chunks of R rows, R as many as fit the CTA's shared memory: the chunk's byte span
// is staged (16-byte loads where the global address allows, single bytes at an unaligned head / tail: the base pointer
// and the row pitch carry no alignment), the horizontal pass writes R x 3 x 64 fp32 values to shared memory, and the
// vertical pass accumulates them into 16 registers per thread (thread = one (token, channel, patch row), the unit of a
// 32-byte store).  Frames up to ~4x downscale take one chunk.
//
// NV12 frames (lwdetr_frame_nv12) take the same kernel: per chunk the luma span and the chroma pairs under it are staged the
// same way and converted once per CTA into the interleaved RGB rows the horizontal pass reads, so the NV12 result is the RGB
// result of the converted frame by construction.  tools/yuv_spec.py restates the conversion.
#include "resize.h"
#include "frame.cuh"
#include "gemm_tc.h"
#include "launch.h"
#include "ptx.cuh"

#include <algorithm>
#include <type_traits>

namespace lwb {

namespace {
constexpr int TILE_H = 16, TILE_W = 64, NTHREADS = 192;      // 192 = 4 tokens x 3 channels x 16 patch rows
constexpr int HROW = 3 * TILE_W;                              // fp32 values of one horizontally filtered source row
constexpr int GROUP = 64;                                     // frames per launch (descriptors are kernel parameters)
constexpr int SMEM_BUDGET = 64 * 1024;                        // dynamic shared memory of one CTA, at most

template <typename F>
struct FrameGroup {
  F f[GROUP];
};
// the padding mask depends on the dst sizes only: one kernel for every source format
struct DstGroup {
  int h[GROUP], w[GROUP];
};
struct ResizeNorm {
  float mean[3], stdv[3];
};
static_assert(sizeof(FrameGroup<lwdetr_frame_nv12>) + sizeof(ResizeNorm) + 64 <= 4096, "NV12 group exceeds 4 KB of kernel parameters");

// bytes of one staged source row: the 16-byte aligned global span covering `nbytes` from any start address
__host__ __device__ inline int staged_row_bytes(int nbytes) { return ((nbytes + 15) & ~15) + 16; }
// shared bytes per source row of a chunk that spans `ncols` source columns.  RGB: the staged row, then the horizontal pass's
// fp32 row.  NV12: the converted RGB row, the staged luma row, one staged chroma row (a chunk of R luma rows touches at most
// R chroma rows) and the fp32 row.
__host__ __device__ inline int rgb_row_bytes(int ncols) { return staged_row_bytes(ncols * 3) + HROW * 4; }
__host__ __device__ inline int nv12_row_bytes(int ncols, int nchroma_bytes) {
  return ((ncols * 3 + 15) & ~15) + staged_row_bytes(ncols) + staged_row_bytes(nchroma_bytes) + HROW * 4;
}

// upper bound of the source extent that `n_tile` outputs of an axis touch
inline int extent_bound(int n_tile, int n_in, int n_out) {
  const double scale = static_cast<double>(n_in) / n_out, support = std::max(scale, 1.0);
  return std::min(n_in, static_cast<int>(n_tile * scale + 2.0 * support) + 3);
}
// dynamic shared memory that lets a frame's tiles run in one chunk, capped at the budget (then they take several)
template <typename F>
inline int frame_smem(const F& f) {
  const int rows = extent_bound(TILE_H, f.height, f.dst_h), cols = extent_bound(TILE_W, f.width, f.dst_w);
  const long long per_row = std::is_same<F, lwdetr_frame_nv12>::value ? nv12_row_bytes(cols, cols + 2) : rgb_row_bytes(cols);
  return static_cast<int>(std::min<long long>(SMEM_BUDGET, per_row * rows));
}

// stage source rows [y0, y0 + nrows) of a byte span (row y: `nbytes` from col0 + y * pitch) into shared rows `rb` bytes apart.
// The shared row mirrors the 16-byte aligned global span, so data byte i of row y sits at ((col0 + y * pitch) & 15) + i:
// 16-byte loads where the global address allows, single bytes at an unaligned head / tail (neither base pointers nor pitches
// carry alignment)
__device__ __forceinline__ void stage_rows(uint8_t* raw, int rb, const uint8_t* col0, int y0, long long pitch, int nrows, int nbytes, int tid) {
  const int nchunk16 = rb >> 4;
  for (int idx = tid; idx < nrows * nchunk16; idx += NTHREADS) {
    const int row = idx / nchunk16, j = idx - row * nchunk16;
    const uint8_t* g = col0 + static_cast<long long>(y0 + row) * pitch;
    const int lo_b = j * 16 - static_cast<int>(reinterpret_cast<uintptr_t>(g) & 15), hi_b = lo_b + 16;
    if (lo_b >= nbytes) continue;
    uint8_t* s = raw + row * rb + j * 16;
    if (lo_b >= 0 && hi_b <= nbytes) {
      *reinterpret_cast<uint4*>(s) = __ldg(reinterpret_cast<const uint4*>(g + lo_b));
    } else {
      for (int k = max(lo_b, 0); k < min(hi_b, nbytes); ++k) s[k - lo_b] = __ldg(g + k);
    }
  }
}
// the first staged byte of source column x and the row pitch of the plane the horizontal pass reads from (NV12: luma)
__device__ __forceinline__ const uint8_t* src_col(const lwdetr_frame& f, int x) { return f.data + static_cast<long long>(x) * 3; }
__device__ __forceinline__ const uint8_t* src_col(const lwdetr_frame_nv12& f, int x) { return f.luma + x; }
__device__ __forceinline__ long long src_pitch(const lwdetr_frame& f) { return f.pitch_bytes; }
__device__ __forceinline__ long long src_pitch(const lwdetr_frame_nv12& f) { return f.luma_pitch; }
}  // namespace

// F: the source format, lwdetr_frame (packed RGB) or lwdetr_frame_nv12.  Only the staging of a chunk's source rows differs:
// NV12 stages the luma span and the chroma pairs under it and converts each staged pixel once into the interleaved RGB row the
// horizontal pass reads, so everything from the tap tables on is the same code for both, and an NV12 frame gives exactly the
// bits of its converted RGB frame.
template <typename T, typename F>
__global__ void __launch_bounds__(NTHREADS) resize_patches_kernel(const __grid_constant__ FrameGroup<F> fg, int b0, T* __restrict__ A, int H, int W,
                                                                  const ResizeNorm np, int smem_bytes) {
  constexpr bool kNV12 = std::is_same<F, lwdetr_frame_nv12>::value;
  pdl_sync();
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ float s_wx[TILE_W * kResizeMaxTaps], s_wy[TILE_H * kResizeMaxTaps];
  __shared__ int s_xlo[TILE_W], s_xn[TILE_W], s_ylo[TILE_H], s_yn[TILE_H];
  const F& f = fg.f[blockIdx.z];
  const int tid = threadIdx.x;
  const int oy0 = blockIdx.y * TILE_H, ox0 = blockIdx.x * TILE_W;
  // this thread's output: token t of the tile, channel c, patch row py -> 16 pixels, one 32-byte store
  const int t = tid / 48, c = (tid >> 4) % 3, py = tid & 15;
  const int GH = H / 16, GW = W / 16, wh = GH / 4, ww = GW / 4;
  const int Y = blockIdx.y, X = blockIdx.x * 4 + t;
  const int rem = ((Y / wh) * 4 + X / ww) * (wh * ww) + (Y % wh) * ww + X % ww;      // window-major row (vit.py:353-358)
  T* dst = A + (static_cast<long long>(b0 + blockIdx.z) * (GH * GW) + rem) * 768 + c * 256 + py * 16;
  const int nvy = min(TILE_H, f.dst_h - oy0), nvx = min(TILE_W, f.dst_w - ox0);     // the part of the tile inside the resized frame
  if (nvy <= 0 || nvx <= 0) {                                                        // padding only: zeros after normalisation
    U8 z;
#pragma unroll
    for (int j = 0; j < 8; ++j) z.v[j] = 0u;
    stg256(dst, z);
    return;
  }
  // ---- tap tables of the tile's columns and rows
  for (int i = tid; i < TILE_W + TILE_H; i += NTHREADS) {
    const bool isx = i < TILE_W;
    const int ol = isx ? i : i - TILE_W;
    const int n_in = isx ? f.width : f.height, n_out = isx ? f.dst_w : f.dst_h;
    const float scale = static_cast<float>(n_in) / static_cast<float>(n_out), support = fmaxf(scale, 1.f);
    const float ctr = __fmul_rn(static_cast<float>((isx ? ox0 : oy0) + ol) + 0.5f, scale);
    const int lo = max(static_cast<int>(ctr - support + 0.5f), 0), hi = min(static_cast<int>(ctr + support + 0.5f), n_in);
    const int n = ol < (isx ? nvx : nvy) ? min(hi - lo, kResizeMaxTaps) : 0;
    float* w = (isx ? s_wx : s_wy) + ol * kResizeMaxTaps;
    float sum = 0.f;
    for (int k = 0; k < n; ++k) {
      w[k] = fmaxf(0.f, 1.f - fabsf(static_cast<float>(lo + k) - ctr + 0.5f) / support);
      sum += w[k];
    }
    for (int k = 0; k < n; ++k) w[k] = w[k] / sum;
    (isx ? s_xlo : s_ylo)[ol] = lo;
    (isx ? s_xn : s_yn)[ol] = n;
  }
  __syncthreads();
  // ---- source footprint of the tile (tap ranges are monotone in the output index)
  const int xb0 = s_xlo[0], xb1 = s_xlo[nvx - 1] + s_xn[nvx - 1];
  const int yb0 = s_ylo[0], yb1 = s_ylo[nvy - 1] + s_yn[nvy - 1];
  const int ncols = xb1 - xb0, xc0 = xb0 >> 1, nchroma = 2 * (((xb1 + 1) >> 1) - xc0);   // chroma: the pairs under [xb0, xb1)
  // raw: the rows the horizontal pass reads, rb bytes apart (RGB: the staged rows; NV12: the converted rows)
  const int rb = kNV12 ? (ncols * 3 + 15) & ~15 : staged_row_bytes(ncols * 3);
  const int R = max(1, min(yb1 - yb0, smem_bytes / (kNV12 ? nv12_row_bytes(ncols, nchroma) : rgb_row_bytes(ncols))));
  uint8_t* raw = smem;
  const int rbY = staged_row_bytes(ncols), rbC = staged_row_bytes(nchroma);
  uint8_t* rawY = smem + static_cast<size_t>(R) * rb;                   // NV12 only: staged luma rows,
  uint8_t* rawC = rawY + static_cast<size_t>(R) * rbY;                  // staged chroma rows
  float* hbuf = reinterpret_cast<float*>(kNV12 ? rawC + static_cast<size_t>(R) * rbC : smem + static_cast<size_t>(R) * rb);
  const int my_ylo = py < nvy ? s_ylo[py] : 0, my_yhi = py < nvy ? my_ylo + s_yn[py] : 0;
  const uint8_t* col0 = src_col(f, xb0);
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  for (int yc = yb0; yc < yb1; yc += R) {
    const int rc = min(R, yb1 - yc);
    if constexpr (kNV12) {
      // luma rows [yc, yc + rc) and the chroma rows under them (a chroma row serves two luma rows and may straddle chunks)
      const int cy0 = yc >> 1, ncr = ((yc + rc - 1) >> 1) - cy0 + 1;
      const uint8_t* ccol0 = f.chroma + 2 * xc0;
      stage_rows(rawY, rbY, col0, yc, f.luma_pitch, rc, ncols, tid);
      stage_rows(rawC, rbC, ccol0, cy0, f.chroma_pitch, ncr, nchroma, tid);
      __syncthreads();
      const int* k = kCsc[f.colorspace];
      const int cY = k[0], cRv = k[1], cGu = k[2], cGv = k[3], cBu = k[4];
      const bool limited = f.colorspace < 2;
      for (int row = 0; row < rc; ++row) {                                // once per staged pixel, row by row
        const int y = yc + row, cr = y >> 1;
        const uint8_t* ys = rawY + row * rbY + static_cast<int>(reinterpret_cast<uintptr_t>(col0 + static_cast<long long>(y) * f.luma_pitch) & 15);
        const uint8_t* uvs = rawC + (cr - cy0) * rbC +
                             static_cast<int>(reinterpret_cast<uintptr_t>(ccol0 + static_cast<long long>(cr) * f.chroma_pitch) & 15) - 2 * xc0;
        uint8_t* o = raw + row * rb;
        for (int i = tid; i < ncols; i += NTHREADS) {
          const uint8_t* uv = uvs + 2 * ((xb0 + i) >> 1);
          const int Y = ys[i], u = uv[0] - 128, v = uv[1] - 128;
          const int yp = (limited ? max(Y - 16, 0) : Y) * cY;
          o[3 * i] = static_cast<uint8_t>(shift20(yp + cRv * v));
          o[3 * i + 1] = static_cast<uint8_t>(shift20(yp + cGu * u + cGv * v));
          o[3 * i + 2] = static_cast<uint8_t>(shift20(yp + cBu * u));
        }
      }
    } else {
      // stage rows [yc, yc + rc), bytes [xb0 * 3, xb1 * 3)
      stage_rows(raw, rb, col0, yc, f.pitch_bytes, rc, ncols * 3, tid);
    }
    __syncthreads();
    // horizontal pass: hbuf[row][channel][ox]
    for (int idx = tid; idx < rc * HROW; idx += NTHREADS) {
      const int row = idx / HROW, j = idx - row * HROW, cc = j >> 6, ox = j & 63;
      float v = 0.f;
      if (ox < nvx) {
        const int sh = kNV12 ? 0 : static_cast<int>(reinterpret_cast<uintptr_t>(col0 + static_cast<long long>(yc + row) * src_pitch(f)) & 15);
        const uint8_t* s = raw + row * rb + sh + (s_xlo[ox] - xb0) * 3 + cc;
        const float* w = s_wx + ox * kResizeMaxTaps;
        const int n = s_xn[ox];
        for (int k = 0; k < n; ++k) v += w[k] * static_cast<float>(s[k * 3]);
      }
      hbuf[idx] = v;
    }
    __syncthreads();
    // vertical pass over the chunk's rows that are taps of this thread's output row
    for (int y = max(yc, my_ylo); y < min(yc + rc, my_yhi); ++y) {
      const float wv = s_wy[py * kResizeMaxTaps + y - my_ylo];
      const float4* h = reinterpret_cast<const float4*>(hbuf + (y - yc) * HROW + c * TILE_W + t * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 hv = h[q];
        acc[4 * q] += wv * hv.x; acc[4 * q + 1] += wv * hv.y; acc[4 * q + 2] += wv * hv.z; acc[4 * q + 3] += wv * hv.w;
      }
    }
    __syncthreads();
  }
  float o[16];
#pragma unroll
  for (int px = 0; px < 16; ++px) {
    const float u = fminf(fmaxf(floorf(acc[px] + 0.5f), 0.f), 255.f);          // the uint8 level a host resize would store
    const bool inside = py < nvy && t * 16 + px < nvx;
    o[px] = inside ? (u / 255.f - np.mean[c]) / np.stdv[c] : 0.f;              // ToTensor, Normalize; padding is 0 AFTER normalisation
  }
  U8 pk;
#pragma unroll
  for (int j = 0; j < 8; ++j) pk.v[j] = Cvt<T>::pack(o[2 * j], o[2 * j + 1]);
  stg256(dst, pk);
}

// mask[b, y, x] = 1 outside the frame's dst_h x dst_w (the NestedTensor mask of util/misc.py:317-339), four pixels per thread
__global__ void __launch_bounds__(256) frame_mask_kernel(const __grid_constant__ DstGroup dg, int b0, uint8_t* __restrict__ mask, int H, int W) {
  pdl_sync();
  const int dst_h = dg.h[blockIdx.y], dst_w = dg.w[blockIdx.y];
  const int wq = W / 4, idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * wq) return;
  const int y = idx / wq, x = (idx - y * wq) * 4;
  uint32_t v = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) v |= (y >= dst_h || x + k >= dst_w) ? (1u << (8 * k)) : 0u;
  reinterpret_cast<uint32_t*>(mask + static_cast<long long>(b0 + blockIdx.y) * H * W)[idx] = v;
}

namespace {
template <typename F>
int frames_check_impl(const F* frames, int B, int H, int W, std::string* err) {
  for (int b = 0; b < B; ++b) {
    const F& f = frames[b];
    const std::string who = "frame " + std::to_string(b) + " (" + std::to_string(f.height) + "x" + std::to_string(f.width) + " -> " +
                            std::to_string(f.dst_h) + "x" + std::to_string(f.dst_w) + ")";
    if (const std::string e = pointers_error(f); !e.empty()) { *err = who + ": " + e; return -1; }
    if (f.height < kFrameMinSide || f.width < kFrameMinSide || f.height > kFrameMaxSide || f.width > kFrameMaxSide) {
      *err = who + ": source sides must be in [" + std::to_string(kFrameMinSide) + ", " + std::to_string(kFrameMaxSide) + "]";
      return -1;
    }
    if (const std::string e = layout_error(f); !e.empty()) { *err = who + ": " + e; return -1; }
    if (f.dst_h < 1 || f.dst_w < 1 || f.dst_h > H || f.dst_w > W) {
      *err = who + ": resized sides must be in [1, run size " + std::to_string(H) + "x" + std::to_string(W) + "]";
      return -1;
    }
    if (f.height > static_cast<long long>(kResizeMaxFactor) * f.dst_h || f.width > static_cast<long long>(kResizeMaxFactor) * f.dst_w) {
      *err = who + ": downscale factor above " + std::to_string(kResizeMaxFactor) + " per axis is not supported";
      return -1;
    }
  }
  return 0;
}

template <typename F>
bool frames_padded_impl(const F* frames, int B, int H, int W) {
  for (int b = 0; b < B; ++b)
    if (frames[b].dst_h < H || frames[b].dst_w < W) return true;
  return false;
}

template <typename T, typename F>
int resize_launch(const F* frames, int B, int H, int W, const ResizeNorm& np, T* A, cudaStream_t st) {
  if (const int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(resize_patches_kernel<T, F>), SMEM_BUDGET)) return e;
  for (int b0 = 0; b0 < B; b0 += GROUP) {
    const int nb = std::min(GROUP, B - b0);
    FrameGroup<F> fg = {};
    int smem = 0;
    for (int i = 0; i < nb; ++i) { fg.f[i] = frames[b0 + i]; smem = std::max(smem, frame_smem(frames[b0 + i])); }
    launch_k(resize_patches_kernel<T, F>, dim3(W / TILE_W, H / TILE_H, nb), dim3(NTHREADS), smem, st, fg, b0, A, H, W, np, smem);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  return 0;
}

template <typename F>
int resize_patches_impl(int dtype, const F* frames, int B, int H, int W, const float* mean, const float* stdv, void* A, cudaStream_t st) {
  if (H % 64 != 0 || W % 64 != 0 || H < 64 || W < 64) return -2;
  ResizeNorm np;
  for (int c = 0; c < 3; ++c) { np.mean[c] = mean[c]; np.stdv[c] = stdv[c]; }
  if (dtype == DT_BF16) return resize_launch(frames, B, H, W, np, static_cast<__nv_bfloat16*>(A), st);
  return resize_launch(frames, B, H, W, np, static_cast<__half*>(A), st);
}

template <typename F>
int frame_mask_impl(const F* frames, int B, int H, int W, uint8_t* mask, cudaStream_t st) {
  if (W % 4 != 0) return -2;
  for (int b0 = 0; b0 < B; b0 += GROUP) {
    const int nb = std::min(GROUP, B - b0);
    DstGroup dg = {};
    for (int i = 0; i < nb; ++i) { dg.h[i] = frames[b0 + i].dst_h; dg.w[i] = frames[b0 + i].dst_w; }
    launch_k(frame_mask_kernel, dim3((H * (W / 4) + 255) / 256, nb), dim3(256), 0, st, dg, b0, mask, H, W);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  return 0;
}
}  // namespace

int frames_check(const lwdetr_frame* frames, int B, int H, int W, std::string* err) { return frames_check_impl(frames, B, H, W, err); }
int frames_check(const lwdetr_frame_nv12* frames, int B, int H, int W, std::string* err) { return frames_check_impl(frames, B, H, W, err); }
bool frames_padded(const lwdetr_frame* frames, int B, int H, int W) { return frames_padded_impl(frames, B, H, W); }
bool frames_padded(const lwdetr_frame_nv12* frames, int B, int H, int W) { return frames_padded_impl(frames, B, H, W); }
int resize_patches_launch(int dtype, const lwdetr_frame* frames, int B, int H, int W, const float* mean, const float* stdv, void* A, cudaStream_t st) {
  return resize_patches_impl(dtype, frames, B, H, W, mean, stdv, A, st);
}
int resize_patches_launch(int dtype, const lwdetr_frame_nv12* frames, int B, int H, int W, const float* mean, const float* stdv, void* A,
                          cudaStream_t st) {
  return resize_patches_impl(dtype, frames, B, H, W, mean, stdv, A, st);
}
int frame_mask_launch(const lwdetr_frame* frames, int B, int H, int W, uint8_t* mask, cudaStream_t st) {
  return frame_mask_impl(frames, B, H, W, mask, st);
}
int frame_mask_launch(const lwdetr_frame_nv12* frames, int B, int H, int W, uint8_t* mask, cudaStream_t st) {
  return frame_mask_impl(frames, B, H, W, mask, st);
}

}  // namespace lwb
