// Crops of detections out of raw RGB / NV12 frames, resized to a fixed size for a second-stage network (ReID, attribute or
// plate models), and the two kernels around them: an ordered selection of the entries to crop and the scatter of the
// network's rows back to the entries.  The contract is in include/lwdetr_b200.h; tools/crop_spec.py restates it.
//
// One CTA = one crop x one band of TH output rows (TH * out_w <= 1024: four (row, column) pairs per thread, three channels
// each, in registers).  The crop's rectangle is read from the device box, so nothing about it is known at launch: the tap
// tables of the band's rows and of all out_w columns are built in shared memory from it, at a stride per output (capx /
// capy taps) the host bounds from the largest frame of the launch group, so any downscale fits.  The source rows the band
// touches are walked in chunks: the horizontal pass reads the taps straight from the frame (bytes through the read-only
// cache; NV12 converted per tap, chroma at (y >> 1, x >> 1) of the whole frame) into R x 3 x out_w fp32 values in shared
// memory, and the vertical pass accumulates them.  Frame descriptors travel as kernel parameters, 64 per launch: a launch
// exits at once on the crops of other groups.
#include "crops.h"
#include "frame.cuh"
#include "launch.h"
#include "resize.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

namespace lwb {

namespace {
constexpr int NT = 256;                       // threads of a crop CTA
constexpr int PAIRS = 4;                      // (output row, column) pairs per thread: TH * out_w <= NT * PAIRS
constexpr int GROUP = 64;                     // frames per launch
constexpr int HBUF_BYTES = 24 * 1024;         // horizontal pass rows of one chunk
constexpr int SMEM_MAX = 227 * 1024;          // dynamic shared memory of one CTA on sm_90

template <typename F>
struct CropFrames {
  F f[GROUP];
};
struct CropArgs {
  int B, f0, nb;                              // frames of the call, first frame and count of this launch's group
  int out_h, out_w, th, capx, capy, rows;     // output, band rows, tap strides, source rows per chunk
  int filter, normalize;
  float mean[3], stdv[3];
};
static_assert(sizeof(CropFrames<lwdetr_frame_nv12>) + sizeof(CropArgs) + 64 <= 4096, "crop launch exceeds 4 KB of kernel parameters");

// the integer crop rectangle (cx0, cy0, cx1, cy1) of an xyxy box in an h x w frame; false when the crop is invalid
__device__ __forceinline__ bool crop_rect(float x1, float y1, float x2, float y2, int h, int w, int r[4]) {
  if (!(isfinite(x1) && isfinite(y1) && isfinite(x2) && isfinite(y2))) return false;
  const float fw = static_cast<float>(w), fh = static_cast<float>(h);
  r[0] = static_cast<int>(fminf(fmaxf(floorf(x1), 0.f), fw));
  r[1] = static_cast<int>(fminf(fmaxf(floorf(y1), 0.f), fh));
  r[2] = static_cast<int>(fminf(fmaxf(floorf(x2), 0.f), fw));
  r[3] = static_cast<int>(fminf(fmaxf(floorf(y2), 0.f), fh));
  return r[2] > r[0] && r[3] > r[1];
}

// taps of output o of an axis n_in -> n_out: first source index *lo, normalised weights into w, count returned
__device__ int axis_taps(int filter, int o, int n_in, int n_out, int* lo, float* w) {
  const float scale = static_cast<float>(n_in) / static_cast<float>(n_out);
  if (filter == LWDETR_CROP_BILINEAR) {                         // cv2.resize(INTER_LINEAR)
    const float f = __fsub_rn(__fmul_rn(static_cast<float>(o) + 0.5f, scale), 0.5f);
    int s = static_cast<int>(floorf(f));
    float t = f - floorf(f);
    if (s < 0) { s = 0; t = 0.f; }
    if (s >= n_in - 1) { *lo = n_in - 1; w[0] = 1.f; return 1; }
    *lo = s; w[0] = 1.f - t; w[1] = t;
    return 2;
  }
  const float support = fmaxf(scale, 1.f);                       // the triangle filter of resize.cu, without its tap cap
  const float ctr = __fmul_rn(static_cast<float>(o) + 0.5f, scale);
  const int l = max(static_cast<int>(ctr - support + 0.5f), 0), n = min(static_cast<int>(ctr + support + 0.5f), n_in) - l;
  float sum = 0.f;
  for (int k = 0; k < n; ++k) {
    w[k] = fmaxf(0.f, 1.f - fabsf(static_cast<float>(l + k) - ctr + 0.5f) / support);
    sum += w[k];
  }
  for (int k = 0; k < n; ++k) w[k] = w[k] / sum;
  *lo = l;
  return n;
}

template <typename T> __device__ __forceinline__ T to_out(float v);
template <> __device__ __forceinline__ float to_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __half to_out<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 to_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename T, typename F>
__global__ void __launch_bounds__(NT) crop_kernel(const __grid_constant__ CropFrames<F> fg, const __grid_constant__ CropArgs a,
                                                  const float* __restrict__ boxes, const int32_t* __restrict__ frame_index,
                                                  const int32_t* __restrict__ count, T* __restrict__ out, int8_t* __restrict__ valid) {
  constexpr bool kNV12 = std::is_same<F, lwdetr_frame_nv12>::value;
  pdl_sync();
  extern __shared__ __align__(16) uint8_t smem[];
  const int i = blockIdx.x, tid = threadIdx.x;
  if (count && i >= __ldg(count)) return;
  const int fi = __ldg(frame_index + i);
  const bool known = fi >= 0 && fi < a.B;
  if (known ? (fi < a.f0 || fi >= a.f0 + a.nb) : a.f0 != 0) return;      // another launch's crop (unknown frames: the first)
  const int oy0 = blockIdx.y * a.th, th = min(a.th, a.out_h - oy0), W = a.out_w;
  const long long plane = static_cast<long long>(a.out_h) * W;
  T* dst = out + static_cast<long long>(i) * 3 * plane + static_cast<long long>(oy0) * W;
  const F& f = fg.f[known ? fi - a.f0 : 0];
  int r[4];
  const float* b = boxes + 4LL * i;
  const bool ok = known && crop_rect(__ldg(b), __ldg(b + 1), __ldg(b + 2), __ldg(b + 3), f.height, f.width, r);
  if (blockIdx.y == 0 && tid == 0) valid[i] = ok ? 1 : 0;
  if (!ok) {
    for (int p = tid; p < th * W; p += NT)
      for (int c = 0; c < 3; ++c) dst[c * plane + p] = to_out<T>(0.f);
    return;
  }
  const int cw = r[2] - r[0], ch = r[3] - r[1];
  float* wx = reinterpret_cast<float*>(smem);
  float* wy = wx + W * a.capx;
  int* xlo = reinterpret_cast<int*>(wy + a.th * a.capy);
  int* xn = xlo + W;
  int* ylo = xn + W;
  int* yn = ylo + a.th;
  float* hbuf = reinterpret_cast<float*>(yn + a.th);
  for (int o = tid; o < W + th; o += NT) {
    if (o < W) xn[o] = axis_taps(a.filter, o, cw, W, xlo + o, wx + o * a.capx);
    else yn[o - W] = axis_taps(a.filter, oy0 + o - W, ch, a.out_h, ylo + o - W, wy + (o - W) * a.capy);
  }
  __syncthreads();
  const int yb0 = ylo[0], yb1 = ylo[th - 1] + yn[th - 1];            // tap ranges are monotone in the output index
  int csc[5] = {0, 0, 0, 0, 0};
  bool limited = false;
  if constexpr (kNV12) {
#pragma unroll
    for (int j = 0; j < 5; ++j) csc[j] = kCsc[f.colorspace][j];
    limited = f.colorspace < 2;
  }
  float acc[PAIRS][3];
#pragma unroll
  for (int j = 0; j < PAIRS; ++j) acc[j][0] = acc[j][1] = acc[j][2] = 0.f;
  for (int yc = yb0; yc < yb1; yc += a.rows) {
    const int rc = min(a.rows, yb1 - yc);
    // horizontal pass: hbuf[row][channel][ox]
    for (int idx = tid; idx < rc * W; idx += NT) {
      const int row = idx / W, ox = idx - row * W;
      const int y = r[1] + yc + row, x0 = r[0] + xlo[ox], n = xn[ox];
      const float* w = wx + ox * a.capx;
      float v0 = 0.f, v1 = 0.f, v2 = 0.f;
      if constexpr (kNV12) {
        const uint8_t* ys = f.luma + static_cast<long long>(y) * f.luma_pitch;
        const uint8_t* uvs = f.chroma + static_cast<long long>(y >> 1) * f.chroma_pitch;
        for (int k = 0; k < n; ++k) {
          const int x = x0 + k;
          const int Y = __ldg(ys + x), u = __ldg(uvs + 2 * (x >> 1)) - 128, v = __ldg(uvs + 2 * (x >> 1) + 1) - 128;
          const int yp = (limited ? max(Y - 16, 0) : Y) * csc[0];
          v0 += w[k] * static_cast<float>(shift20(yp + csc[1] * v));
          v1 += w[k] * static_cast<float>(shift20(yp + csc[2] * u + csc[3] * v));
          v2 += w[k] * static_cast<float>(shift20(yp + csc[4] * u));
        }
      } else {
        const uint8_t* s = f.data + static_cast<long long>(y) * f.pitch_bytes + 3LL * x0;
        for (int k = 0; k < n; ++k) {
          v0 += w[k] * static_cast<float>(__ldg(s + 3 * k));
          v1 += w[k] * static_cast<float>(__ldg(s + 3 * k + 1));
          v2 += w[k] * static_cast<float>(__ldg(s + 3 * k + 2));
        }
      }
      float* h = hbuf + row * 3 * W + ox;
      h[0] = v0; h[W] = v1; h[2 * W] = v2;
    }
    __syncthreads();
    // vertical pass over the chunk's rows that are taps of each pair's output row
#pragma unroll
    for (int j = 0; j < PAIRS; ++j) {
      const int p = tid + j * NT;
      if (p < th * W) {
        const int ry = p / W, ox = p - ry * W, lo = ylo[ry], hi = lo + yn[ry];
        for (int y = max(yc, lo); y < min(yc + rc, hi); ++y) {
          const float wv = wy[ry * a.capy + y - lo];
          const float* h = hbuf + (y - yc) * 3 * W + ox;
          acc[j][0] += wv * h[0]; acc[j][1] += wv * h[W]; acc[j][2] += wv * h[2 * W];
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < PAIRS; ++j) {
    const int p = tid + j * NT;
    if (p < th * W) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float u = fminf(fmaxf(floorf(acc[j][c] + 0.5f), 0.f), 255.f);     // the uint8 level
        dst[c * plane + p] = to_out<T>(a.normalize ? (u / 255.f - a.mean[c]) / a.stdv[c] : u);
      }
    }
  }
}

struct SizeGroup {
  int h[GROUP], w[GROUP];
};

// ordered compaction of the entries of frames [f0, f0 + nb) with score > threshold and a valid crop, appended after the
// entries the previous group's launch kept (its count)
__global__ void __launch_bounds__(1024) crop_select_kernel(const __grid_constant__ SizeGroup sg, int f0, int nb, int k,
                                                           const float* __restrict__ scores, const float* __restrict__ boxes, float thr,
                                                           int32_t* __restrict__ frame_of, int32_t* __restrict__ entry,
                                                           float* __restrict__ sel_boxes, int32_t* __restrict__ count) {
  pdl_sync();
  __shared__ int warp_incl[32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int base = f0 == 0 ? 0 : *count;
  const long long n = static_cast<long long>(nb) * k, e0 = static_cast<long long>(f0) * k;
  for (long long c0 = 0; c0 < n; c0 += 1024) {
    const long long j = c0 + tid;
    bool keep = false;
    float bx[4] = {0.f, 0.f, 0.f, 0.f};
    int fl = 0;
    if (j < n) {
      fl = static_cast<int>(j / k);
      if (scores[e0 + j] > thr) {
        for (int q = 0; q < 4; ++q) bx[q] = boxes[(e0 + j) * 4 + q];
        int r[4];
        keep = crop_rect(bx[0], bx[1], bx[2], bx[3], sg.h[fl], sg.w[fl], r);
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_incl[wid] = __popc(m);
    __syncthreads();
    if (wid == 0) {
      int v = warp_incl[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
      }
      warp_incl[lane] = v;
    }
    __syncthreads();
    if (keep) {
      const int at = base + (wid ? warp_incl[wid - 1] : 0) + __popc(m & ((1u << lane) - 1u));
      frame_of[at] = f0 + fl;
      entry[at] = static_cast<int32_t>(e0 + j);
      for (int q = 0; q < 4; ++q) sel_boxes[4LL * at + q] = bx[q];
    }
    base += warp_incl[31];
    __syncthreads();
  }
  if (tid == 0) *count = base;
}

// row i of `rows` (i < count) to row entry[i] of out; out was zeroed before
template <typename E>
__global__ void __launch_bounds__(128) scatter_rows_kernel(const E* __restrict__ rows, int ld, int D, const int32_t* __restrict__ entry,
                                                           const int32_t* __restrict__ count, E* __restrict__ out, int num_out) {
  pdl_sync();
  const int i = blockIdx.x;
  if (count && i >= __ldg(count)) return;
  const int e = __ldg(entry + i);
  if (e < 0 || e >= num_out) return;
  for (int d = threadIdx.x; d < D; d += blockDim.x) out[static_cast<long long>(e) * D + d] = rows[static_cast<long long>(i) * ld + d];
}

template <typename T, typename F>
int crops_impl(const F* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count, const CropDesc& d,
               T* out, int8_t* valid, cudaStream_t st) {
  auto kern = crop_kernel<T, F>;
  if (const int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(kern), SMEM_MAX)) return e;
  CropArgs a = {};
  a.B = B;
  a.out_h = d.out_h; a.out_w = d.out_w; a.filter = d.filter; a.normalize = d.normalize;
  for (int c = 0; c < 3; ++c) { a.mean[c] = d.mean[c]; a.stdv[c] = d.stdv[c]; }
  a.th = std::min(d.out_h, std::max(1, NT * PAIRS / d.out_w));
  a.rows = std::max(1, HBUF_BYTES / (12 * d.out_w));
  const dim3 grid(N, (d.out_h + a.th - 1) / a.th);
  for (int f0 = 0; f0 < B; f0 += GROUP) {
    CropFrames<F> fg = {};
    a.f0 = f0;
    a.nb = std::min(GROUP, B - f0);
    int hmax = 1, wmax = 1;
    for (int j = 0; j < a.nb; ++j) {
      fg.f[j] = frames[f0 + j];
      hmax = std::max(hmax, frames[f0 + j].height);
      wmax = std::max(wmax, frames[f0 + j].width);
    }
    // taps per output: 2 (bilinear), at most 2 * support + 2 (triangle; +1 for the fp32 scale's rounding)
    a.capx = d.filter == LWDETR_CROP_BILINEAR ? 2 : static_cast<int>(2.0 * std::max(1.0, static_cast<double>(wmax) / d.out_w)) + 3;
    a.capy = d.filter == LWDETR_CROP_BILINEAR ? 2 : static_cast<int>(2.0 * std::max(1.0, static_cast<double>(hmax) / d.out_h)) + 3;
    const long long smem = 4LL * (static_cast<long long>(d.out_w) * a.capx + static_cast<long long>(a.th) * a.capy + 2 * d.out_w + 2 * a.th +
                                  3LL * a.rows * d.out_w);
    if (smem > SMEM_MAX) return -2;
    launch_k(kern, grid, dim3(NT), static_cast<size_t>(smem), st, fg, a, boxes, frame_index, count, out, valid);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  return 0;
}

template <typename F>
int frames_check_impl(const F* frames, int B, std::string* err) {
  for (int b = 0; b < B; ++b) {
    const F& f = frames[b];
    const std::string who = "frame " + std::to_string(b) + " (" + std::to_string(f.height) + "x" + std::to_string(f.width) + ")";
    if (const std::string e = pointers_error(f); !e.empty()) { *err = who + ": " + e; return -1; }
    if (f.height < kFrameMinSide || f.width < kFrameMinSide || f.height > kFrameMaxSide || f.width > kFrameMaxSide) {
      *err = who + ": sides must be in [" + std::to_string(kFrameMinSide) + ", " + std::to_string(kFrameMaxSide) + "]";
      return -1;
    }
    if (const std::string e = layout_error(f); !e.empty()) { *err = who + ": " + e; return -1; }
  }
  return 0;
}

template <typename F>
int crops_dispatch(const F* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count, const CropDesc& d,
                   void* out, int8_t* valid, cudaStream_t st) {
  if (d.etype == LWDETR_ET_F16) return crops_impl(frames, B, boxes, frame_index, N, count, d, static_cast<__half*>(out), valid, st);
  if (d.etype == LWDETR_ET_BF16) return crops_impl(frames, B, boxes, frame_index, N, count, d, static_cast<__nv_bfloat16*>(out), valid, st);
  return crops_impl(frames, B, boxes, frame_index, N, count, d, static_cast<float*>(out), valid, st);
}
}  // namespace

int crop_frames_check(const lwdetr_frame* frames, int B, std::string* err) { return frames_check_impl(frames, B, err); }
int crop_frames_check(const lwdetr_frame_nv12* frames, int B, std::string* err) { return frames_check_impl(frames, B, err); }
int crops_launch(const lwdetr_frame* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                 const CropDesc& d, void* out, int8_t* valid, cudaStream_t st) {
  return crops_dispatch(frames, B, boxes, frame_index, N, count, d, out, valid, st);
}
int crops_launch(const lwdetr_frame_nv12* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                 const CropDesc& d, void* out, int8_t* valid, cudaStream_t st) {
  return crops_dispatch(frames, B, boxes, frame_index, N, count, d, out, valid, st);
}

int crop_select_launch(const float* scores, const float* boxes, int B, int k, const int32_t* sizes, float threshold, int32_t* frame_of,
                       int32_t* entry, float* sel_boxes, int32_t* count, cudaStream_t st) {
  for (int f0 = 0; f0 < B; f0 += GROUP) {
    SizeGroup sg = {};
    const int nb = std::min(GROUP, B - f0);
    for (int j = 0; j < nb; ++j) { sg.h[j] = sizes[2 * (f0 + j)]; sg.w[j] = sizes[2 * (f0 + j) + 1]; }
    launch_k(crop_select_kernel, dim3(1), dim3(1024), 0, st, sg, f0, nb, k, scores, boxes, threshold, frame_of, entry, sel_boxes, count);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  return 0;
}

int scatter_rows_launch(int etype, const void* rows, int ld_rows, int D, const int32_t* entry, const int32_t* count, int N, void* out,
                        int num_out, cudaStream_t st) {
  const size_t esize = etype == LWDETR_ET_F32 ? 4 : 2;
  cudaError_t e = cudaMemsetAsync(out, 0, esize * D * static_cast<size_t>(num_out), st);
  if (e != cudaSuccess) return static_cast<int>(e);
  if (esize == 4)
    launch_k(scatter_rows_kernel<uint32_t>, dim3(N), dim3(128), 0, st, static_cast<const uint32_t*>(rows), ld_rows, D, entry, count,
             static_cast<uint32_t*>(out), num_out);
  else
    launch_k(scatter_rows_kernel<uint16_t>, dim3(N), dim3(128), 0, st, static_cast<const uint16_t*>(rows), ld_rows, D, entry, count,
             static_cast<uint16_t*>(out), num_out);
  e = cudaGetLastError();
  return e == cudaSuccess ? 0 : static_cast<int>(e);
}

}  // namespace lwb
