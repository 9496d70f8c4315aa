// lwdetr_gmc_estimate: the camera motion of each stream from its previous frame to this one, the contract stated in
// include/lwdetr_b200.h and restated in tools/gmc_spec.py.  Per call, for the B streams of the call:
//   grey_kernel     one thread per level-0 pixel: grey (RGB: OpenCV's fixed-point weights; NV12: the luma byte) box-averaged
//                   over d x d, into the buffer the stream's header does not mark current;
//   pyr_kernel      level l from level l - 1, cv2.pyrDown's arithmetic (one launch per level);
//   cells_kernel    one CTA per grid cell: the Shi-Tomasi response of each pixel (exact integer sums, one float64 square
//                   root) in 32 x 32 tiles, the cell's best pixel (lowest index on ties);
//   select_kernel   one CTA per stream: the frame's largest response, the cells that pass the quality test, compacted in
//                   cell order into the buffer's corner list (used at the stream's next frame);
//   lk_kernel       one warp per corner of the previous frame: calcOpticalFlowPyrLK's iteration from the previous pyramid
//                   into this one, window sums in exact int64 (lk_point, lk.cuh);
//   fit_kernel      one CTA per stream: deterministic RANSAC over 2-point similarity hypotheses, float64 least-squares
//                   refits, the outputs; it then makes the new buffer current.
// lwdetr_gmc_observe runs grey, pyramid and corners, then commit_kernel makes the new buffer current (no LK, no fit), so
// the stream's chain of pyramids and corners stays current for the next estimate or for the per-object flow (flow.cu).
// Everything reads the current buffer from the device header, so a replayed CUDA graph advances the state.
#include "gmc.h"

#include <climits>
#include <cmath>
#include <vector>

#include "launch.h"
#include "lk.cuh"

namespace lwb {
namespace {

constexpr int LAUNCH_STREAMS = 256;      // streams per launch (the frame table travels in the parameters)
constexpr int FLAT_BLOCKS = 512;         // CTAs per stream of the per-pixel kernels (grid-stride)
constexpr int TILE = 32;
constexpr int LK_WARPS = 4;
constexpr int FIT_NT = 512;
constexpr int SEL_NT = 1024;

struct GmcFrame {
  const uint8_t* data;
  long long pitch;
  int h, w, sid, nv12, nlev, cell, ncx, ncy;
};

struct GmcArgs {
  GmcTable t;
  double* motion;
  int32_t* status;
  int32_t* inliers;
  int row0, level;
  GmcFrame f[LAUNCH_STREAMS];
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ void level_sizes(const GmcFrame& f, int d, int* lw, int* lh) {
  lw[0] = f.w / d;
  lh[0] = f.h / d;
  for (int l = 1; l <= GMC_MAX_LEVELS; ++l) {
    lw[l] = (lw[l - 1] + 1) >> 1;
    lh[l] = (lh[l - 1] + 1) >> 1;
  }
}

// ------------------------------------------------------------------------------------------------ grey and pyramid
__global__ void __launch_bounds__(256) grey_kernel(const __grid_constant__ GmcArgs a) {
  pdl_sync();
  const GmcFrame& f = a.f[blockIdx.y];
  const int d = a.t.p.downscale;
  const int ws = f.w / d, hs = f.h / d;
  uint8_t* dst = level_ptr(a.t, f.sid, a.t.head[f.sid].cur ^ 1, 0);
  const int dd = d * d;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < static_cast<long long>(ws) * hs; i += 256LL * gridDim.x) {
    const int y = static_cast<int>(i / ws), x = static_cast<int>(i - static_cast<long long>(y) * ws);
    int sum = 0;
    for (int r = 0; r < d; ++r) {
      const uint8_t* row = f.data + static_cast<long long>(y * d + r) * f.pitch;
      for (int c = 0; c < d; ++c) {
        const int xx = x * d + c;
        if (f.nv12) {
          sum += row[xx];
        } else {
          const uint8_t* px = row + 3 * xx;
          sum += (px[0] * 9798 + px[1] * 19235 + px[2] * 3735 + 16384) >> 15;
        }
      }
    }
    dst[i] = static_cast<uint8_t>((sum + dd / 2) / dd);
  }
}

__global__ void __launch_bounds__(256) pyr_kernel(const __grid_constant__ GmcArgs a) {
  pdl_sync();
  const GmcFrame& f = a.f[blockIdx.y];
  const int l = a.level;
  if (l > f.nlev) return;
  int lw[GMC_MAX_LEVELS + 1], lh[GMC_MAX_LEVELS + 1];
  level_sizes(f, a.t.p.downscale, lw, lh);
  const int buf = a.t.head[f.sid].cur ^ 1;
  const uint8_t* src = level_ptr(a.t, f.sid, buf, l - 1);
  uint8_t* dst = level_ptr(a.t, f.sid, buf, l);
  const int sw = lw[l - 1], sh = lh[l - 1], w = lw[l], h = lh[l];
  const int k[5] = {1, 4, 6, 4, 1};
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < static_cast<long long>(w) * h; i += 256LL * gridDim.x) {
    const int y = static_cast<int>(i / w), x = static_cast<int>(i - static_cast<long long>(y) * w);
    int xs[5];
    for (int j = 0; j < 5; ++j) xs[j] = refl(2 * x + j - 2, sw);
    int sum = 0;
    for (int r = 0; r < 5; ++r) {
      const uint8_t* row = src + static_cast<long long>(refl(2 * y + r - 2, sh)) * sw;
      int s = 0;
      for (int j = 0; j < 5; ++j) s += k[j] * row[xs[j]];
      sum += k[r] * s;
    }
    dst[i] = static_cast<uint8_t>((sum + 128) >> 8);
  }
}

// ------------------------------------------------------------------------------------------------ corners
// Shi-Tomasi response of a pixel from the 3x3 sums of the Sobel products (exact integers):
// R = (Sxx + Syy) - sqrt((Sxx - Syy)^2 + 4 Sxy^2), float64, the square root and the subtraction rounded once each.
__device__ __forceinline__ double response(int sxx, int sxy, int syy) {
  const long long df = static_cast<long long>(sxx) - syy;
  const long long disc = df * df + 4LL * sxy * static_cast<long long>(sxy);
  return dsub(static_cast<double>(sxx + syy), __dsqrt_rn(static_cast<double>(disc)));
}

__global__ void __launch_bounds__(256) cells_kernel(const __grid_constant__ GmcArgs a) {
  pdl_sync();
  __shared__ int pxx[TILE + 2][TILE + 2], pxy[TILE + 2][TILE + 2], pyy[TILE + 2][TILE + 2];
  __shared__ double rbest[256];
  __shared__ int ibest[256];
  const GmcFrame& f = a.f[blockIdx.y];
  const int cid = blockIdx.x;
  if (cid >= f.ncx * f.ncy) return;
  const int d = a.t.p.downscale;
  const int w = f.w / d, h = f.h / d;
  const uint8_t* img = level_ptr(a.t, f.sid, a.t.head[f.sid].cur ^ 1, 0);
  const int cy = cid / f.ncx, cx = cid - cy * f.ncx;
  const int x0 = cx * f.cell, y0 = cy * f.cell, x1 = min(x0 + f.cell, w), y1 = min(y0 + f.cell, h);
  double best = -1.0;
  int bi = -1;
  const auto px = [&](int y, int x) { return static_cast<int>(img[static_cast<long long>(refl(y, h)) * w + refl(x, w)]); };
  for (int ty0 = y0; ty0 < y1; ty0 += TILE) {
    for (int tx0 = x0; tx0 < x1; tx0 += TILE) {
      for (int q = threadIdx.x; q < (TILE + 2) * (TILE + 2); q += 256) {
        const int qy = q / (TILE + 2), qx = q - qy * (TILE + 2);
        const int y = refl(ty0 - 1 + qy, h), x = refl(tx0 - 1 + qx, w);
        if (ty0 - 1 + qy > y1 || tx0 - 1 + qx > x1) continue;          // outside this tile's halo
        const int dx = (px(y - 1, x + 1) - px(y - 1, x - 1)) + 2 * (px(y, x + 1) - px(y, x - 1)) + (px(y + 1, x + 1) - px(y + 1, x - 1));
        const int dy = (px(y + 1, x - 1) - px(y - 1, x - 1)) + 2 * (px(y + 1, x) - px(y - 1, x)) + (px(y + 1, x + 1) - px(y - 1, x + 1));
        pxx[qy][qx] = dx * dx;
        pxy[qy][qx] = dx * dy;
        pyy[qy][qx] = dy * dy;
      }
      __syncthreads();
      for (int q = threadIdx.x; q < TILE * TILE; q += 256) {
        const int qy = q / TILE, qx = q - qy * TILE;
        const int y = ty0 + qy, x = tx0 + qx;
        if (y >= y1 || x >= x1) continue;
        int sxx = 0, sxy = 0, syy = 0;
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) {
            sxx += pxx[qy + r][qx + c];
            sxy += pxy[qy + r][qx + c];
            syy += pyy[qy + r][qx + c];
          }
        const double R = response(sxx, sxy, syy);
        const int idx = y * w + x;
        if (R > best || (R == best && idx < bi)) {
          best = R;
          bi = idx;
        }
      }
      __syncthreads();
    }
  }
  rbest[threadIdx.x] = best;
  ibest[threadIdx.x] = bi;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const double r2 = rbest[threadIdx.x + s];
      const int i2 = ibest[threadIdx.x + s];
      if (i2 >= 0 && (ibest[threadIdx.x] < 0 || r2 > rbest[threadIdx.x] || (r2 == rbest[threadIdx.x] && i2 < ibest[threadIdx.x]))) {
        rbest[threadIdx.x] = r2;
        ibest[threadIdx.x] = i2;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const long long o = static_cast<long long>(f.sid) * a.t.p.max_points + cid;
    a.t.cell_r[o] = rbest[0];
    a.t.cell_i[o] = ibest[0];
  }
}

// Ordered compaction of flags over [0, n) by the whole block (blockDim.x == NT): returns each flagged index's rank via emit.
template <int NT, typename Pred, typename Emit>
__device__ int ordered_scan(int* wsum, int n, Pred pred, Emit emit) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += NT) {
    const int i = i0 + threadIdx.x;
    const bool fl = i < n && pred(i);
    const unsigned bal = __ballot_sync(0xffffffffu, fl);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
    for (int q = 0; q < NT / 32; ++q) {
      const int c = wsum[q];
      off += q < w ? c : 0;
      tot += c;
    }
    if (fl) emit(i, base + off + __popc(bal & ((1u << lane) - 1u)));
    base += tot;
    __syncthreads();
  }
  return base;
}

__global__ void __launch_bounds__(SEL_NT) select_kernel(const __grid_constant__ GmcArgs a) {
  pdl_sync();
  __shared__ double red[SEL_NT / 32];
  __shared__ int wsum[SEL_NT / 32];
  const GmcFrame& f = a.f[blockIdx.x];
  const int n = f.ncx * f.ncy, w = f.w / a.t.p.downscale;
  const long long o = static_cast<long long>(f.sid) * a.t.p.max_points;
  const double* cr = a.t.cell_r + o;
  const int* ci = a.t.cell_i + o;
  double m = -1.0;
  for (int i = threadIdx.x; i < n; i += SEL_NT) m = fmax(m, cr[i]);
  for (int s = 16; s > 0; s >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, s));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int q = 1; q < SEL_NT / 32; ++q) m = fmax(m, red[q]);
  const double thr = dmul(static_cast<double>(a.t.p.quality), m);
  GmcHead& hd = a.t.head[f.sid];
  const int buf = hd.cur ^ 1;
  float2* pts = a.t.pts + (static_cast<long long>(f.sid) * 2 + buf) * a.t.p.max_points;
  const int np = ordered_scan<SEL_NT>(wsum, n, [&](int i) { return ci[i] >= 0 && cr[i] > 0.0 && cr[i] >= thr; }, [&](int i, int r) {
    const int y = ci[i] / w;
    pts[r] = make_float2(static_cast<float>(ci[i] - y * w), static_cast<float>(y));
  });
  if (threadIdx.x == 0) hd.npts[buf] = np;
}

// ------------------------------------------------------------------------------------------------ Lucas-Kanade
__global__ void __launch_bounds__(LK_WARPS * 32) lk_kernel(const __grid_constant__ GmcArgs a) {
  pdl_sync();
  __shared__ LkWarp sw[LK_WARPS];
  const GmcFrame& f = a.f[blockIdx.y];
  const GmcHead hd = a.t.head[f.sid];
  if (!hd.valid || hd.h != f.h || hd.w != f.w) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int pi = blockIdx.x * LK_WARPS + wid;
  if (pi >= hd.npts[hd.cur]) return;
  const lwdetr_gmc_params& p = a.t.p;
  int lw[GMC_MAX_LEVELS + 1], lh[GMC_MAX_LEVELS + 1];
  level_sizes(f, p.downscale, lw, lh);
  const float2 p0 = a.t.pts[(static_cast<long long>(f.sid) * 2 + hd.cur) * p.max_points + pi];
  float2 nxt;
  const bool ok = lk_point(sw[wid], a.t, f.sid, hd.cur, hd.cur ^ 1, lw, lh, f.nlev, p0, p.window, p.iterations, p.eps * p.eps, p.min_eig, &nxt);
  if (lane == 0) {
    const long long o = static_cast<long long>(f.sid) * p.max_points + pi;
    a.t.flow[o] = make_float4(p0.x, p0.y, nxt.x, nxt.y);
    a.t.found[o] = ok ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------------ robust fit
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t hyp_hash(uint32_t k) { return mix32(k * 0x9e3779b9u + 0x7f4a7c15u); }

struct Sim {
  double a, b, tx, ty;
};

// squared transfer error of pair i under m, each operation rounded on its own
__device__ __forceinline__ double err2(const double4& q, const Sim& m) {
  const double ex = dsub(dadd(dsub(dmul(m.a, q.x), dmul(m.b, q.y)), m.tx), q.z);
  const double ey = dsub(dadd(dadd(dmul(m.b, q.x), dmul(m.a, q.y)), m.ty), q.w);
  return dadd(dmul(ex, ex), dmul(ey, ey));
}

// Block sum of K doubles in a fixed order: each thread's strided terms in index order, then a fixed tree.
template <int K>
__device__ void block_sum(double (*red)[FIT_NT], double* v) {
  for (int k = 0; k < K; ++k) red[k][threadIdx.x] = v[k];
  __syncthreads();
  for (int s = FIT_NT / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int k = 0; k < K; ++k) red[k][threadIdx.x] = dadd(red[k][threadIdx.x], red[k][threadIdx.x + s]);
    __syncthreads();
  }
  for (int k = 0; k < K; ++k) v[k] = red[k][0];
  __syncthreads();
}

__global__ void __launch_bounds__(FIT_NT) fit_kernel(const __grid_constant__ GmcArgs a) {
  pdl_sync();
  extern __shared__ __align__(16) uint8_t sm_fit[];
  double4* pr = reinterpret_cast<double4*>(sm_fit);                  // (x, y) previous, (x, y) current, frame pixels
  __shared__ double red[5][FIT_NT];
  __shared__ int wsum[FIT_NT / 32];
  __shared__ int cnt[FIT_NT], cidx[FIT_NT];
  const GmcFrame& f = a.f[blockIdx.x];
  const long long row = a.row0 + blockIdx.x;
  GmcHead* hp = a.t.head + f.sid;
  const GmcHead hd = *hp;
  const lwdetr_gmc_params& p = a.t.p;
  int st = LWDETR_GMC_OK;
  if (!hd.valid) st = LWDETR_GMC_FIRST_FRAME;
  else if (hd.h != f.h || hd.w != f.w) st = LWDETR_GMC_SIZE_CHANGED;
  Sim m = {1.0, 0.0, 0.0, 0.0};
  int ninl = 0;
  if (st == LWDETR_GMC_OK) {
    const long long o = static_cast<long long>(f.sid) * p.max_points;
    const double d = p.downscale;
    const int n = ordered_scan<FIT_NT>(wsum, hd.npts[hd.cur], [&](int i) { return a.t.found[o + i] != 0; }, [&](int i, int r) {
      const float4 fl = a.t.flow[o + i];
      pr[r] = make_double4(dsub(dmul(d, dadd(fl.x, 0.5)), 0.5), dsub(dmul(d, dadd(fl.y, 0.5)), 0.5),
                           dsub(dmul(d, dadd(fl.z, 0.5)), 0.5), dsub(dmul(d, dadd(fl.w, 0.5)), 0.5));
    });
    if (n < p.min_inliers) {
      st = LWDETR_GMC_FEW_POINTS;
    } else {
      const double thr = dmul(static_cast<double>(p.ransac_thresh), d);
      const double thr2 = dmul(thr, thr);
      int bc = -1, bh = INT_MAX;
      for (int h = threadIdx.x; h < p.hypotheses; h += FIT_NT) {
        const int i = static_cast<int>(hyp_hash(2u * h) % static_cast<uint32_t>(n));
        int j = static_cast<int>(hyp_hash(2u * h + 1u) % static_cast<uint32_t>(n - 1));
        j += j >= i;
        const double4 u = pr[i], v = pr[j];
        const double dpx = dsub(v.x, u.x), dpy = dsub(v.y, u.y), dqx = dsub(v.z, u.z), dqy = dsub(v.w, u.w);
        const double n2 = dadd(dmul(dpx, dpx), dmul(dpy, dpy));
        if (!(n2 > 0.0)) continue;
        Sim hm;
        hm.a = ddiv(dadd(dmul(dqx, dpx), dmul(dqy, dpy)), n2);
        hm.b = ddiv(dsub(dmul(dqy, dpx), dmul(dqx, dpy)), n2);
        hm.tx = dsub(u.z, dsub(dmul(hm.a, u.x), dmul(hm.b, u.y)));
        hm.ty = dsub(u.w, dadd(dmul(hm.b, u.x), dmul(hm.a, u.y)));
        int c = 0;
        for (int q = 0; q < n; ++q) c += err2(pr[q], hm) <= thr2;
        if (c > bc) {                     // h ascends per thread: the first of equal counts is kept
          bc = c;
          bh = h;
        }
      }
      cnt[threadIdx.x] = bc;
      cidx[threadIdx.x] = bh;
      __syncthreads();
      for (int s = FIT_NT / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
          const int c2 = cnt[threadIdx.x + s], h2 = cidx[threadIdx.x + s];
          if (c2 > cnt[threadIdx.x] || (c2 == cnt[threadIdx.x] && h2 < cidx[threadIdx.x])) {
            cnt[threadIdx.x] = c2;
            cidx[threadIdx.x] = h2;
          }
        }
        __syncthreads();
      }
      const int best = cidx[0];
      if (cnt[0] < p.min_inliers) {
        st = LWDETR_GMC_FEW_INLIERS;
      } else {
        {
          const int i = static_cast<int>(hyp_hash(2u * best) % static_cast<uint32_t>(n));
          int j = static_cast<int>(hyp_hash(2u * best + 1u) % static_cast<uint32_t>(n - 1));
          j += j >= i;
          const double4 u = pr[i], v = pr[j];
          const double dpx = dsub(v.x, u.x), dpy = dsub(v.y, u.y), dqx = dsub(v.z, u.z), dqy = dsub(v.w, u.w);
          const double n2 = dadd(dmul(dpx, dpx), dmul(dpy, dpy));
          m.a = ddiv(dadd(dmul(dqx, dpx), dmul(dqy, dpy)), n2);
          m.b = ddiv(dsub(dmul(dqy, dpx), dmul(dqx, dpy)), n2);
          m.tx = dsub(u.z, dsub(dmul(m.a, u.x), dmul(m.b, u.y)));
          m.ty = dsub(u.w, dadd(dmul(m.b, u.x), dmul(m.a, u.y)));
        }
        // least-squares refits on the inliers of the current model: centred sums, closed form
        for (int round = 0; round < GMC_REFITS; ++round) {
          double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
          for (int q = threadIdx.x; q < n; q += FIT_NT) {
            const double4 e = pr[q];
            if (err2(e, m) <= thr2) {
              s[0] = dadd(s[0], 1.0);
              s[1] = dadd(s[1], e.x);
              s[2] = dadd(s[2], e.y);
              s[3] = dadd(s[3], e.z);
              s[4] = dadd(s[4], e.w);
            }
          }
          block_sum<5>(red, s);
          if (s[0] < 2.0) break;
          const double mx = ddiv(s[1], s[0]), my = ddiv(s[2], s[0]), mu = ddiv(s[3], s[0]), mv = ddiv(s[4], s[0]);
          double t[3] = {0.0, 0.0, 0.0};
          for (int q = threadIdx.x; q < n; q += FIT_NT) {
            const double4 e = pr[q];
            if (err2(e, m) <= thr2) {
              const double px = dsub(e.x, mx), py = dsub(e.y, my), qx = dsub(e.z, mu), qy = dsub(e.w, mv);
              t[0] = dadd(t[0], dadd(dmul(px, px), dmul(py, py)));
              t[1] = dadd(t[1], dadd(dmul(px, qx), dmul(py, qy)));
              t[2] = dadd(t[2], dsub(dmul(px, qy), dmul(py, qx)));
            }
          }
          block_sum<3>(red, t);
          if (!(t[0] > 0.0)) break;
          m.a = ddiv(t[1], t[0]);
          m.b = ddiv(t[2], t[0]);
          m.tx = dsub(mu, dsub(dmul(m.a, mx), dmul(m.b, my)));
          m.ty = dsub(mv, dadd(dmul(m.b, mx), dmul(m.a, my)));
        }
        int c = 0;
        for (int q = threadIdx.x; q < n; q += FIT_NT) c += err2(pr[q], m) <= thr2;
        double cs[1] = {static_cast<double>(c)};
        block_sum<1>(red, cs);
        ninl = static_cast<int>(cs[0]);
        if (ninl < p.min_inliers) st = LWDETR_GMC_FEW_INLIERS;
      }
    }
  }
  if (st != LWDETR_GMC_OK) m = Sim{1.0, 0.0, 0.0, 0.0};
  if (threadIdx.x == 0) {
    a.motion[row * 4 + 0] = m.a;
    a.motion[row * 4 + 1] = m.b;
    a.motion[row * 4 + 2] = m.tx;
    a.motion[row * 4 + 3] = m.ty;
    a.status[row] = st;
    a.inliers[row] = ninl;
    hp->cur = hd.cur ^ 1;
    hp->prev = hd.valid && hd.h == f.h && hd.w == f.w;
    hp->valid = 1;
    hp->h = f.h;
    hp->w = f.w;
  }
}

// lwdetr_gmc_observe: what fit_kernel does to the header, one thread per stream, with no motion estimated
__global__ void commit_kernel(const __grid_constant__ GmcArgs a, int nb) {
  pdl_sync();
  const int i = threadIdx.x;
  if (i >= nb) return;
  const GmcFrame& f = a.f[i];
  GmcHead* hp = a.t.head + f.sid;
  const GmcHead hd = *hp;
  hp->cur = hd.cur ^ 1;
  hp->prev = hd.valid && hd.h == f.h && hd.w == f.w;
  hp->valid = 1;
  hp->h = f.h;
  hp->w = f.w;
}

struct ResetArgs {
  GmcHead* head;
  int n;
  int stream[1024];
};

__global__ void reset_kernel(const __grid_constant__ ResetArgs a) {
  pdl_sync();
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
    a.head[a.stream[i]].valid = 0;
    a.head[a.stream[i]].prev = 0;
  }
}

}  // namespace

void gmc_geometry(int h, int w, const lwdetr_gmc_params& p, GmcGeo* g) {
  g->lw[0] = w / p.downscale;
  g->lh[0] = h / p.downscale;
  for (int l = 1; l <= GMC_MAX_LEVELS; ++l) {
    g->lw[l] = (g->lw[l - 1] + 1) >> 1;
    g->lh[l] = (g->lh[l - 1] + 1) >> 1;
  }
  g->nlev = 0;
  while (g->nlev < p.levels && g->lw[g->nlev + 1] > p.window && g->lh[g->nlev + 1] > p.window) ++g->nlev;
  const long long area = static_cast<long long>(g->lw[0]) * g->lh[0];
  int c = static_cast<int>(std::sqrt(static_cast<double>(area) / p.max_points));
  if (c < 1) c = 1;
  while (static_cast<long long>((g->lw[0] + c - 1) / c) * ((g->lh[0] + c - 1) / c) > p.max_points) ++c;
  g->cell = c;
  g->ncx = (g->lw[0] + c - 1) / c;
  g->ncy = (g->lh[0] + c - 1) / c;
}

int gmc_estimate_launch(const GmcTable& t, const GmcFrameHost* frames, int B, const int32_t* streams, double* motion, int32_t* status,
                        int32_t* inliers, cudaStream_t st, bool observe) {
  const int fit_smem = static_cast<int>(sizeof(double4)) * t.p.max_points;
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(fit_kernel), fit_smem)) return e;
  std::vector<GmcArgs> hold(1);          // ~12 KB of parameters: kept off the stack
  GmcArgs& a = hold[0];
  a.t = t;
  a.motion = motion;
  a.status = status;
  a.inliers = inliers;
  for (int b0 = 0; b0 < B; b0 += LAUNCH_STREAMS) {
    const int nb = B - b0 < LAUNCH_STREAMS ? B - b0 : LAUNCH_STREAMS;
    a.row0 = b0;
    long long max_px = 0;
    int max_cells = 1;
    for (int i = 0; i < nb; ++i) {
      const GmcFrameHost& h = frames[b0 + i];
      GmcGeo g;
      gmc_geometry(h.h, h.w, t.p, &g);
      a.f[i] = GmcFrame{h.data, h.pitch, h.h, h.w, streams[b0 + i], h.nv12, g.nlev, g.cell, g.ncx, g.ncy};
      const long long px = static_cast<long long>(g.lw[0]) * g.lh[0];
      if (px > max_px) max_px = px;
      if (g.ncx * g.ncy > max_cells) max_cells = g.ncx * g.ncy;
    }
    const unsigned fb = static_cast<unsigned>(std::min<long long>((max_px + 255) / 256, FLAT_BLOCKS));
    a.level = 0;
    launch_k(grey_kernel, dim3(fb, nb), dim3(256), 0, st, a);
    for (int l = 1; l <= t.p.levels; ++l) {
      a.level = l;
      const unsigned lb = fb >> (2 * l) > 0 ? fb >> (2 * l) : 1;
      launch_k(pyr_kernel, dim3(lb, nb), dim3(256), 0, st, a);
    }
    launch_k(cells_kernel, dim3(max_cells, nb), dim3(256), 0, st, a);
    launch_k(select_kernel, dim3(nb), dim3(SEL_NT), 0, st, a);
    if (observe) {
      launch_k(commit_kernel, dim3(1), dim3(LAUNCH_STREAMS), 0, st, a, nb);
    } else {
      launch_k(lk_kernel, dim3((t.p.max_points + LK_WARPS - 1) / LK_WARPS, nb), dim3(LK_WARPS * 32), 0, st, a);
      launch_k(fit_kernel, dim3(nb), dim3(FIT_NT), static_cast<size_t>(fit_smem), st, a);
    }
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

int gmc_reset_launch(const GmcTable& t, const int32_t* streams, int n, cudaStream_t st) {
  std::vector<ResetArgs> hold(1);
  ResetArgs& a = hold[0];
  a.head = t.head;
  for (int i0 = 0; i0 < n; i0 += 1024) {
    a.n = n - i0 < 1024 ? n - i0 : 1024;
    for (int i = 0; i < a.n; ++i) a.stream[i] = streams[i0 + i];
    launch_k(reset_kernel, dim3(1), dim3(256), 0, st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

}  // namespace lwb
