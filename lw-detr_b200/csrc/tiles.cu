// lwdetr_tile_merge: merge the detections of overlapping views (tiles + a full-frame view) of each frame on the device.
//
// Input: the [V, k] per-view output of lwdetr_postprocess (scores fp32, labels int32, xyxy boxes fp32 in the view's crop
// pixels) and a HOST table of V views {frame, x0, y0}, each frame's views contiguous.  One CTA per frame:
//   1. candidates: every (view, rank) with score >= score_threshold, compacted into shared memory as one 64-bit key
//      (order-preserving score bits << 32 | ~local index), so a descending sort is score descending with ties to the lower
//      flat index v*k + rank (the tie rule of lwdetr_postprocess);
//   2. bitonic sort of the keys in shared memory (16384 x 8 B = 128 KiB at the limit);
//   3. greedy class-aware NMS, walking the sorted list in blocks of 256: every candidate of a block is tested against the
//      boxes kept so far (4 threads per candidate, each a quarter of the kept list); then the 256 x 256 upper-triangular
//      suppression bitmask of the block is built (1024 threads, one 32-bit word each, twice) and one warp resolves the
//      in-block chain in order, keeping a candidate unless a kept one suppresses it.  The walk stops once max_det are
//      kept: greedy NMS's first max_det depend only on the prefix.
// The box moves into frame pixels by one fp32 add of (x0, y0, x0, y0); the overlap test is fp32 with every operation
// rounded separately (no FMA contraction), the exact arithmetic stated in include/lwdetr_b200.h.  No global scratch: the
// view table travels in the kernel's parameters (up to TILE_MAX_VIEWS per launch, so frames are launched in groups).
#include "tiles.h"

#include <algorithm>
#include <vector>

#include "launch.h"

namespace lwb {
namespace {

constexpr int THREADS = 1024;
constexpr int BLK = 256;                 // candidates per NMS step
constexpr int LAUNCH_FRAMES = 512;       // frames (CTAs) per launch

struct TileMergeArgs {
  const float* scores;
  const int32_t* labels;
  const float* boxes;
  float* out_scores;
  int32_t* out_labels;
  float* out_boxes;
  int32_t* counts;
  float score_thr, iou_thr;
  int k, metric, max_det, frame0, np2;
  int view_begin[LAUNCH_FRAMES + 1];     // index of each frame's first view (global), frame i of this launch
  int2 off[TILE_MAX_VIEWS];              // (x0, y0) of view view_begin[0] + i
};

__device__ __forceinline__ uint32_t score_key(float f) {
  const uint32_t u = f == 0.f ? 0u : __float_as_uint(f);   // -0.0 ranks as +0.0, as a float comparison does
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float box_area(float4 b) {
  return __fmul_rn(fmaxf(0.f, __fsub_rn(b.z, b.x)), fmaxf(0.f, __fsub_rn(b.w, b.y)));
}

// Does the earlier kept box a (area aa) suppress the later box b (area ab)?  A degenerate box (area not > 0) never does and
// never is suppressed.
__device__ __forceinline__ bool suppresses(float4 a, float aa, float4 b, float ab, float thr, int metric) {
  if (!(aa > 0.f) || !(ab > 0.f)) return false;
  const float ix = fmaxf(0.f, __fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)));
  const float iy = fmaxf(0.f, __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)));
  const float inter = __fmul_rn(ix, iy);
  const float den = metric == TILE_IOU ? __fsub_rn(__fadd_rn(aa, ab), inter) : fminf(aa, ab);
  return inter > __fmul_rn(thr, den);
}

__device__ __forceinline__ void bitonic_sort_desc_u64(uint64_t* key, int np2) {
  for (int size = 2; size <= np2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < np2 / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = (lo & size) == 0;
        const uint64_t a = key[lo], b = key[hi];
        if ((a > b) != desc && a != b) {
          key[lo] = b;
          key[hi] = a;
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(THREADS) tile_merge_kernel(const __grid_constant__ TileMergeArgs a) {
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  extern __shared__ __align__(16) uint8_t sm_tiles[];
  uint64_t* key = reinterpret_cast<uint64_t*>(sm_tiles);
  float4* kbox = reinterpret_cast<float4*>(key + a.np2);        // the kept list, in output order (a.np2 even: 16-byte aligned)
  int* klab = reinterpret_cast<int*>(kbox + a.max_det);
  float* karea = reinterpret_cast<float*>(klab + a.max_det);
  __shared__ float4 bbox[BLK];
  __shared__ int blab[BLK];
  __shared__ float barea[BLK], bscore[BLK];
  __shared__ int border[BLK];
  __shared__ uint32_t bmask[BLK * (BLK / 32)];
  __shared__ uint32_t bsup[BLK / 32];
  __shared__ int s_n, s_new, s_kept;

  const int tid = threadIdx.x;
  const int fl = blockIdx.x;
  const int f = a.frame0 + fl;
  const int vb = a.view_begin[fl];
  const int k = a.k;
  const int ncand = (a.view_begin[fl + 1] - vb) * k;
  const int2* off = a.off + (vb - a.view_begin[0]);
  const long long c0 = static_cast<long long>(vb) * k;          // flat index of the frame's first candidate
  const float* sc = a.scores + c0;
  const int32_t* lb = a.labels + c0;
  const float4* bx = reinterpret_cast<const float4*>(a.boxes) + c0;
  if (tid == 0) {
    s_n = 0;
    s_kept = 0;
  }
  __syncthreads();
  for (int i = tid; i < ncand; i += THREADS) {
    const float s = sc[i];
    if (s >= a.score_thr) {
      const int slot = atomicAdd(&s_n, 1);
      key[slot] = (static_cast<uint64_t>(score_key(s)) << 32) | (0xffffffffu - static_cast<uint32_t>(i));
    }
  }
  __syncthreads();
  const int n = s_n;
  int np2 = 1;
  while (np2 < n) np2 <<= 1;
  for (int i = n + tid; i < np2; i += THREADS) key[i] = 0;      // below every candidate (a real key has its top bits set)
  __syncthreads();
  bitonic_sort_desc_u64(key, np2);

  const float thr = a.iou_thr;
  const int metric = a.metric, max_det = a.max_det;
  for (int base = 0; base < n && s_kept < max_det; base += BLK) {
    const int nb = min(BLK, n - base);
    const int kept0 = s_kept;
    if (tid < nb) {
      const int i = static_cast<int>(0xffffffffu - static_cast<uint32_t>(key[base + tid]));
      const int2 o = off[i / k];
      float4 b = bx[i];
      const float x0 = static_cast<float>(o.x), y0 = static_cast<float>(o.y);
      b.x = __fadd_rn(b.x, x0);
      b.y = __fadd_rn(b.y, y0);
      b.z = __fadd_rn(b.z, x0);
      b.w = __fadd_rn(b.w, y0);
      bbox[tid] = b;
      blab[tid] = lb[i];
      barea[tid] = box_area(b);
      bscore[tid] = sc[i];
    }
    if (tid < BLK / 32) bsup[tid] = 0;
    __syncthreads();
    // (a) against the boxes kept before this block
    {
      const int c = tid & (BLK - 1);
      if (c < nb && barea[c] > 0.f) {
        const float4 b = bbox[c];
        const float ab = barea[c];
        const int l = blab[c];
        for (int j = tid / BLK; j < kept0; j += THREADS / BLK) {
          if (klab[j] == l && suppresses(kbox[j], karea[j], b, ab, thr, metric)) {
            atomicOr(&bsup[c >> 5], 1u << (c & 31));
            break;
          }
        }
      }
    }
    // (b) in-block pairs: bit j of row i set when i < j and i, if kept, suppresses j
    for (int w = tid; w < BLK * (BLK / 32); w += THREADS) {
      const int i = w >> 3, j0 = (w & 7) * 32;
      uint32_t bits = 0;
      if (i < nb && j0 + 31 > i) {
        const float4 bi = bbox[i];
        const float ai = barea[i];
        const int li = blab[i];
        for (int jj = 0; jj < 32; ++jj) {
          const int j = j0 + jj;
          if (j > i && j < nb && blab[j] == li && suppresses(bi, ai, bbox[j], barea[j], thr, metric)) bits |= 1u << jj;
        }
      }
      bmask[w] = bits;
    }
    __syncthreads();
    // (c) one warp walks the block in order
    if (tid < 32) {
      uint32_t removed = tid < BLK / 32 ? bsup[tid] : 0u;
      const int room = max_det - kept0;
      int nn = 0;
      for (int i = 0; i < nb && nn < room; ++i) {
        const uint32_t w = __shfl_sync(0xffffffffu, removed, i >> 5);
        if (!((w >> (i & 31)) & 1u)) {
          if (tid == 0) border[nn] = i;
          ++nn;
          if (tid < BLK / 32) removed |= bmask[i * (BLK / 32) + tid];
        }
      }
      if (tid == 0) s_new = nn;
    }
    __syncthreads();
    const int nn = s_new;
    for (int q = tid; q < nn; q += THREADS) {
      const int i = border[q], slot = kept0 + q;
      kbox[slot] = bbox[i];
      klab[slot] = blab[i];
      karea[slot] = barea[i];
      const long long o = static_cast<long long>(f) * max_det + slot;
      a.out_scores[o] = bscore[i];
      a.out_labels[o] = blab[i];
      reinterpret_cast<float4*>(a.out_boxes)[o] = bbox[i];
    }
    if (tid == 0) s_kept = kept0 + nn;
    __syncthreads();
  }
  const int kept = s_kept;
  for (int slot = kept + tid; slot < max_det; slot += THREADS) {
    const long long o = static_cast<long long>(f) * max_det + slot;
    a.out_scores[o] = 0.f;
    a.out_labels[o] = -1;
    reinterpret_cast<float4*>(a.out_boxes)[o] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (tid == 0) a.counts[f] = kept;
}

}  // namespace

int tile_merge_launch(const float* scores, const int32_t* labels, const float* boxes, int V, int k, const TileViewHost* views,
                      int num_frames, float score_threshold, float iou_threshold, int metric, int max_det, float* out_scores,
                      int32_t* out_labels, float* out_boxes, int32_t* counts, cudaStream_t st) {
  if (V < 1 || k < 1 || num_frames < 1 || max_det < 1 || max_det > TILE_MAX_DET) return -2;
  std::vector<int> first(static_cast<size_t>(num_frames) + 1, 0);      // first[f]: first view of frame f
  for (int v = 0; v < V; ++v) first[views[v].frame + 1] = v + 1;
  for (int f = 1; f <= num_frames; ++f) first[f] = first[f] > first[f - 1] ? first[f] : first[f - 1];
  for (int f = 0; f < num_frames; ++f) {
    const long long nv = first[f + 1] - first[f];
    if (nv > TILE_MAX_VIEWS || nv * k > TILE_MAX_CAND) return -2;
  }
  const int smem_max = TILE_MAX_CAND * 8 + TILE_MAX_DET * 24;
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(tile_merge_kernel), smem_max)) return e;
  std::vector<TileMergeArgs> hold(1);            // ~19 KB of parameters: kept off the stack
  TileMergeArgs& a = hold[0];
  a.scores = scores;
  a.labels = labels;
  a.boxes = boxes;
  a.out_scores = out_scores;
  a.out_labels = out_labels;
  a.out_boxes = out_boxes;
  a.counts = counts;
  a.score_thr = score_threshold;
  a.iou_thr = iou_threshold;
  a.k = k;
  a.metric = metric;
  a.max_det = max_det;
  for (int f = 0; f < num_frames;) {
    const int v0 = first[f];
    int nf = 0, maxc = 1;
    while (f + nf < num_frames && nf < LAUNCH_FRAMES && first[f + nf + 1] - v0 <= TILE_MAX_VIEWS) {
      maxc = std::max(maxc, (first[f + nf + 1] - first[f + nf]) * k);
      ++nf;
    }
    for (int i = 0; i <= nf; ++i) a.view_begin[i] = first[f + i];
    for (int v = v0; v < first[f + nf]; ++v) a.off[v - v0] = make_int2(views[v].x0, views[v].y0);
    int np2 = 2;                   // >= 2: the key region is a multiple of 16 bytes, so the float4 kept list after it is aligned
    while (np2 < maxc) np2 <<= 1;
    a.frame0 = f;
    a.np2 = np2;
    const size_t smem = static_cast<size_t>(np2) * 8 + static_cast<size_t>(max_det) * 24;
    launch_k(tile_merge_kernel, dim3(nf), dim3(THREADS), smem, st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
    f += nf;
  }
  return 0;
}

}  // namespace lwb
