// The flow of lwdetr_track_flow: the Median Flow tracker (Kalal et al., 2010) for every activated tracked track of each
// stream of the call, bit for bit the contract in include/lwdetr_b200.h restated in tools/flow_spec.py.  Per call:
//   list_kernel     one CTA per stream: the activated tracked records in list order (an ordered compaction), their
//                   grid x grid seeds in level-0 pixels from the box of each record's state, the statuses reset;
//   lk_kernel       one warp per seed: forward Lucas-Kanade from the previous pyramid into the current one, then backward
//                   from the forward result (lk_point, lk.cuh: the estimator's own iteration);
//   measure_kernel  one CTA per track, one thread per seed: forward-backward error and NCC, the lower medians by an exact
//                   radix select on order-preserving keys of the float64 values (the pair scale ratios are recomputed on
//                   the fly in each pass, so no pair is stored), the selection, the box and the status.
// Everything reads the estimator's header and the tracker's records from the device, so a replayed CUDA graph follows the
// state.
#include "flow.h"

#include <algorithm>
#include <vector>

#include "launch.h"
#include "lk.cuh"

namespace lwb {
namespace {

constexpr int LAUNCH_STREAMS = 1024;
constexpr int LIST_NT = 256;
constexpr int LK_WARPS = 4;
constexpr int MEAS_NT = 256;             // >= FLOW_MAX_GRID^2: one thread per seed
constexpr double NaN = __builtin_nan("");

struct FlowArgs {
  FlowTable f;
  GmcTable g;
  TrackTable t;
  int stream[LAUNCH_STREAMS];
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// the level sizes and the levels the estimator's pyramids have for an h x w frame (gmc_geometry's rule)
__device__ int pyramid_levels(const lwdetr_gmc_params& p, int h, int w, int* lw, int* lh) {
  lw[0] = w / p.downscale;
  lh[0] = h / p.downscale;
  for (int l = 1; l <= GMC_MAX_LEVELS; ++l) {
    lw[l] = (lw[l - 1] + 1) >> 1;
    lh[l] = (lh[l - 1] + 1) >> 1;
  }
  int n = 0;
  while (n < p.levels && lw[n + 1] > p.window && lh[n + 1] > p.window) ++n;
  return n;
}

__device__ __forceinline__ long long tslot(const FlowTable& f, int sid, int j) { return static_cast<long long>(sid) * f.p.max_tracks + j; }

// ------------------------------------------------------------------------------------------------ the tracks and their seeds
__global__ void __launch_bounds__(LIST_NT) list_kernel(const __grid_constant__ FlowArgs a) {
  pdl_sync();
  __shared__ int wsum[LIST_NT / 32];
  const FlowTable& f = a.f;
  const int sid = a.stream[blockIdx.x];
  const TrackHead th = a.t.head[sid];
  const lwdetr_track_record* rec = a.t.rec + (static_cast<long long>(sid) * 2 + th.parity) * a.t.capacity;
  const int T = f.p.max_tracks, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int16_t* slot = f.slot + tslot(f, sid, 0);
  int base = 0;
  for (int i0 = 0; i0 < th.n_tracked; i0 += LIST_NT) {              // ordered compaction of the activated records
    const int i = i0 + threadIdx.x;
    const bool fl = i < th.n_tracked && rec[i].activated != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, fl);
    if (lane == 0) wsum[w] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
    for (int q = 0; q < LIST_NT / 32; ++q) {
      off += q < w ? wsum[q] : 0;
      tot += wsum[q];
    }
    const int r = base + off + __popc(bal & ((1u << lane) - 1u));
    if (fl && r < T) slot[r] = static_cast<int16_t>(i);
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) f.ntracks[sid] = base;
  const int n = min(base, T), G = f.p.grid, g2 = f.g2;
  const int prev = a.g.head[sid].prev;
  for (int j = threadIdx.x; j < n; j += LIST_NT) {
    f.status[tslot(f, sid, j)] = prev ? LWDETR_FLOW_OK : LWDETR_FLOW_NO_PREVIOUS;
    for (int q = 0; q < 8; ++q) f.meas[tslot(f, sid, j) * 8 + q] = NaN;
  }
  const double d = a.g.p.downscale;
  for (int idx = threadIdx.x; idx < n * g2; idx += LIST_NT) {
    const int j = idx / g2, q = idx - j * g2, iy = q / G, ix = q - iy * G;
    const double* m = rec[slot[j]].mean;
    // the state's box (track.cu's state_box): w = a h, x1 = cx - w / 2, y1 = cy - h / 2
    const double bw = dmul(m[2], m[3]);
    const double x1 = dsub(m[0], dmul(bw, 0.5)), y1 = dsub(m[1], dmul(m[3], 0.5));
    const double xf = dadd(x1, ddiv(dmul(ix + 0.5, bw), static_cast<double>(G)));
    const double yf = dadd(y1, ddiv(dmul(iy + 0.5, m[3]), static_cast<double>(G)));
    const long long o = tslot(f, sid, j) * g2 + q;
    f.seed[o] = make_float2(__double2float_rn(dsub(ddiv(dadd(xf, 0.5), d), 0.5)), __double2float_rn(dsub(ddiv(dadd(yf, 0.5), d), 0.5)));
    f.fb[o] = NaN;
    f.ncc[o] = NaN;
    f.valid[o] = 0;
  }
}

// ------------------------------------------------------------------------------------------------ forward and backward LK
__global__ void __launch_bounds__(LK_WARPS * 32) lk_kernel(const __grid_constant__ FlowArgs a) {
  pdl_sync();
  __shared__ LkWarp sw[LK_WARPS];
  const FlowTable& f = a.f;
  const int sid = a.stream[blockIdx.y];
  const GmcHead hd = a.g.head[sid];
  if (!hd.prev) return;
  const int n = min(f.ntracks[sid], f.p.max_tracks), total = n * f.g2;
  int lw[GMC_MAX_LEVELS + 1], lh[GMC_MAX_LEVELS + 1];
  const int nlev = pyramid_levels(a.g.p, hd.h, hd.w, lw, lh);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float eps2 = f.p.eps * f.p.eps;
  for (int wi = blockIdx.x * LK_WARPS + wid; wi < total; wi += gridDim.x * LK_WARPS) {
    const long long o = tslot(f, sid, 0) * f.g2 + wi;
    const float2 p0 = f.seed[o];
    float2 q, b;
    const bool okf = lk_point(sw[wid], a.g, sid, hd.cur ^ 1, hd.cur, lw, lh, nlev, p0, f.p.window, f.p.iterations, eps2, f.p.min_eig, &q);
    const bool okb = lk_point(sw[wid], a.g, sid, hd.cur, hd.cur ^ 1, lw, lh, nlev, q, f.p.window, f.p.iterations, eps2, f.p.min_eig, &b);
    if (lane == 0) {
      f.fwd[o] = q;
      f.bwd[o] = b;
      f.valid[o] = okf && okb;
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------ the measurement
// order-preserving keys of float64 values (no NaN among them)
__device__ __forceinline__ unsigned long long dkey(double v) {
  const unsigned long long u = static_cast<unsigned long long>(__double_as_longlong(v));
  return (u >> 63) ? ~u : u | (1ull << 63);
}
__device__ __forceinline__ double dunkey(unsigned long long k) {
  return __longlong_as_double(static_cast<long long>((k >> 63) ? k & ~(1ull << 63) : ~k));
}

struct MeasSmem {
  unsigned hist[256];
  unsigned long long prefix;
  int k, count;
  int16_t sel[FLOW_MAX_GRID * FLOW_MAX_GRID];
  double px[FLOW_MAX_GRID * FLOW_MAX_GRID], py[FLOW_MAX_GRID * FLOW_MAX_GRID];   // selected seeds, frame pixels
  double qx[FLOW_MAX_GRID * FLOW_MAX_GRID], qy[FLOW_MAX_GRID * FLOW_MAX_GRID];   // their forward points
};

// The k-th smallest (from 0) of the values val(i) of the items i in [0, n) with take(i): an exact radix select, 8 bits
// per pass, over the whole block.  The caller guarantees k < the number taken.
template <typename Take, typename Val>
__device__ double block_select(MeasSmem& S, int n, int k, Take take, Val val) {
  unsigned long long prefix = 0, mask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    S.hist[threadIdx.x] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += MEAS_NT) {
      if (!take(i)) continue;
      const unsigned long long key = dkey(val(i));
      if ((key & mask) == prefix) atomicAdd(&S.hist[(key >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned c = 0;
      int b = 0;
      for (; b < 255 && c + S.hist[b] <= static_cast<unsigned>(k); ++b) c += S.hist[b];
      S.prefix = prefix | (static_cast<unsigned long long>(b) << shift);
      S.k = k - static_cast<int>(c);
    }
    __syncthreads();
    prefix = S.prefix;
    k = S.k;
    mask |= 255ull << shift;
    __syncthreads();
  }
  return dunkey(prefix);
}

template <typename Take>
__device__ int block_count(MeasSmem& S, int n, Take take) {
  if (threadIdx.x == 0) S.count = 0;
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < n; i += MEAS_NT) c += take(i) ? 1 : 0;
  for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&S.count, c);
  __syncthreads();
  const int r = S.count;
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(MEAS_NT) measure_kernel(const __grid_constant__ FlowArgs a) {
  pdl_sync();
  __shared__ MeasSmem S;
  const FlowTable& f = a.f;
  const int sid = a.stream[blockIdx.y], j = blockIdx.x;
  const GmcHead hd = a.g.head[sid];
  if (!hd.prev || j >= min(f.ntracks[sid], f.p.max_tracks)) return;
  const int g2 = f.g2, q = threadIdx.x, tid = threadIdx.x;
  const long long o = tslot(f, sid, j) * g2;
  const double d = a.g.p.downscale;
  const int W = hd.w / a.g.p.downscale, H = hd.h / a.g.p.downscale;
  // per seed: frame-pixel points, FB error, NCC
  bool valid = false;
  double fb = NaN, ncc = NaN, px = 0, py = 0, qx = 0, qy = 0;
  if (q < g2) {
    valid = f.valid[o + q] != 0;
    const float2 s = f.seed[o + q], fw = f.fwd[o + q], bw = f.bwd[o + q];
    px = dsub(dmul(d, dadd(s.x, 0.5)), 0.5);
    py = dsub(dmul(d, dadd(s.y, 0.5)), 0.5);
    qx = dsub(dmul(d, dadd(fw.x, 0.5)), 0.5);
    qy = dsub(dmul(d, dadd(fw.y, 0.5)), 0.5);
    if (valid) {
      const double ex = dsub(dsub(dmul(d, dadd(bw.x, 0.5)), 0.5), px), ey = dsub(dsub(dmul(d, dadd(bw.y, 0.5)), 0.5), py);
      fb = __dsqrt_rn(dadd(dmul(ex, ex), dmul(ey, ey)));
      const uint8_t* I = level_ptr(a.g, sid, hd.cur ^ 1, 0);
      const uint8_t* J = level_ptr(a.g, sid, hd.cur, 0);
      const int ax = __float2int_rn(s.x), ay = __float2int_rn(s.y), bx = __float2int_rn(fw.x), by = __float2int_rn(fw.y);
      const int nw = f.p.ncc_window, hw = nw / 2;
      long long s1 = 0, s2 = 0, s11 = 0, s22 = 0, s12 = 0;
      for (int r = -hw; r <= hw; ++r) {
        const uint8_t* ir = I + static_cast<long long>(refl(ay + r, H)) * W;
        const uint8_t* jr = J + static_cast<long long>(refl(by + r, H)) * W;
        for (int c = -hw; c <= hw; ++c) {
          const long long u = ir[refl(ax + c, W)], v = jr[refl(bx + c, W)];
          s1 += u;
          s2 += v;
          s11 += u * u;
          s22 += v * v;
          s12 += u * v;
        }
      }
      const long long nn = static_cast<long long>(nw) * nw;
      const long long va = nn * s11 - s1 * s1, vb = nn * s22 - s2 * s2, cv = nn * s12 - s1 * s2;
      ncc = va > 0 && vb > 0 ? ddiv(static_cast<double>(cv), __dsqrt_rn(dmul(static_cast<double>(va), static_cast<double>(vb)))) : -1.0;
    }
    f.fb[o + q] = fb;
    f.ncc[o + q] = ncc;
    S.px[q] = px;
    S.py[q] = py;
    S.qx[q] = qx;
    S.qy[q] = qy;
  }
  __shared__ double fbv[MEAS_NT], nccv[MEAS_NT];
  __shared__ uint8_t vv[MEAS_NT];
  fbv[tid] = fb;
  nccv[tid] = ncc;
  vv[tid] = valid;
  __syncthreads();
  const long long to = tslot(f, sid, j);
  const int nv = block_count(S, g2, [&](int i) { return vv[i] != 0; });
  const lwdetr_flow_params& p = f.p;
  int st = LWDETR_FLOW_OK;
  double mfb = NaN, mncc = NaN;
  if (nv > 0) {
    mfb = block_select(S, g2, (nv - 1) / 2, [&](int i) { return vv[i] != 0; }, [&](int i) { return fbv[i]; });
    mncc = block_select(S, g2, (nv - 1) / 2, [&](int i) { return vv[i] != 0; }, [&](int i) { return nccv[i]; });
  }
  // the selection, compacted in seed order
  const auto chosen = [&](int i) { return vv[i] != 0 && fbv[i] <= mfb && nccv[i] >= mncc; };
  if (tid == 0) {
    int m = 0;
    for (int i = 0; i < g2; ++i)
      if (chosen(i)) S.sel[m++] = static_cast<int16_t>(i);
    S.count = m;
  }
  __syncthreads();
  const int m = S.count;
  __syncthreads();
  double dx = NaN, dy = NaN, s = NaN;
  if (m < p.min_points) {
    st = LWDETR_FLOW_FEW_POINTS;
  } else if (mfb > static_cast<double>(p.fb_max)) {
    st = LWDETR_FLOW_FB;
  } else {
    const auto all = [&](int) { return true; };
    dx = block_select(S, m, (m - 1) / 2, all, [&](int i) { const int k = S.sel[i]; return dsub(S.qx[k], S.px[k]); });
    dy = block_select(S, m, (m - 1) / 2, all, [&](int i) { const int k = S.sel[i]; return dsub(S.qy[k], S.py[k]); });
    // pairs i < j of the selection with a nonzero previous distance: flat index i * m + j
    const auto pd = [&](int idx) {
      const int a0 = S.sel[idx / m], b0 = S.sel[idx % m];
      const double ex = dsub(S.px[b0], S.px[a0]), ey = dsub(S.py[b0], S.py[a0]);
      return __dsqrt_rn(dadd(dmul(ex, ex), dmul(ey, ey)));
    };
    const auto pair = [&](int idx) { return idx / m < idx % m && pd(idx) > 0.0; };
    const int np = block_count(S, m * m, pair);
    if (np > 0) {
      s = block_select(S, m * m, (np - 1) / 2, pair, [&](int idx) {
        const int a0 = S.sel[idx / m], b0 = S.sel[idx % m];
        const double ex = dsub(S.qx[b0], S.qx[a0]), ey = dsub(S.qy[b0], S.qy[a0]);
        return ddiv(__dsqrt_rn(dadd(dmul(ex, ex), dmul(ey, ey))), pd(idx));
      });
    }
    if (!(isfinite(s) && s >= static_cast<double>(p.scale_min) && s <= static_cast<double>(p.scale_max))) st = LWDETR_FLOW_SCALE;
  }
  if (tid == 0) {
    double* ms = f.meas + to * 8;
    ms[0] = dx;
    ms[1] = dy;
    ms[2] = s;
    if (st == LWDETR_FLOW_OK) {
      const TrackHead th = a.t.head[sid];
      const double* mean = a.t.rec[(static_cast<long long>(sid) * 2 + th.parity) * a.t.capacity + f.slot[to]].mean;
      const double h = dmul(mean[3], s);
      ms[3] = dadd(mean[0], dx);
      ms[4] = dadd(mean[1], dy);
      ms[5] = mean[2];
      ms[6] = h;
      const double two = dmul(2.0, d);
      if (!(dmul(mean[2], h) >= two && h >= two)) st = LWDETR_FLOW_SMALL;
    }
    f.status[to] = st;
  }
}

}  // namespace

int flow_launch(const FlowTable& f, const GmcTable& g, const TrackTable& t, int B, const int32_t* streams, cudaStream_t st) {
  std::vector<FlowArgs> hold(1);         // the stream table travels in the parameters: kept off the stack
  FlowArgs& a = hold[0];
  a.f = f;
  a.g = g;
  a.t = t;
  for (int b0 = 0; b0 < B; b0 += LAUNCH_STREAMS) {
    const int nb = std::min(B - b0, LAUNCH_STREAMS);
    for (int i = 0; i < nb; ++i) a.stream[i] = streams[b0 + i];
    // LK warps per stream: every seed of max_tracks, but no more than about 4096 warps for the whole call
    const long long seeds = static_cast<long long>(f.p.max_tracks) * f.g2;
    const long long bps = std::max(1LL, std::min((seeds + LK_WARPS - 1) / LK_WARPS, std::max(8LL, 1024LL / nb)));
    launch_k(list_kernel, dim3(nb), dim3(LIST_NT), 0, st, a);
    launch_k(lk_kernel, dim3(static_cast<unsigned>(bps), nb), dim3(LK_WARPS * 32), 0, st, a);
    launch_k(measure_kernel, dim3(f.p.max_tracks, nb), dim3(MEAS_NT), 0, st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

}  // namespace lwb
