// lwdetr_speed_update: ground-plane position, velocity and speed of each track per camera stream on the device, bit for
// bit the contract stated in include/lwdetr_b200.h and restated in tools/speed_spec.py.  One CTA per stream in the call.
// The stream's records sit in fixed slots, found through the index of lifecycle.cuh (staged in shared memory); each
// record's ring of the last `window` samples (t, x, y) stays in global memory.  Per frame:
//   1. the lifecycle up to the slots of the new ids (lifecycle.cuh): keyed and sorted entries, presence, lookup, new slots;
//   2. one thread per present track projects its anchor, appends its sample to its ring (when the frame's clock is good)
//      and fits the velocity over the ring serially, oldest sample first, so the summation order is the contract's; all in
//      float64 with each operation rounded on its own (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn);
//   3. the records not seen for more than forget_after frames are dropped and the index is merged (lifecycle.cuh).
#include "speed.h"

#include <vector>

#include "launch.h"
#include "lifecycle.cuh"

namespace lwb {
namespace {

constexpr int NT = LC_NT;                // threads per CTA
constexpr int MAXE = SPEED_MAX_OUT;      // entries per frame
constexpr int LAUNCH_STREAMS = 1024;     // CTAs per launch (the stream table travels in the parameters)
static_assert(MAXE <= LC_MAXE && SPEED_CAPACITY <= LC_MAXR, "lifecycle limits");

struct SpeedArgs {
  const int32_t* ids;
  const float4* boxes;
  const int32_t* counts;
  const double* timestamps;
  float* kin;
  int32_t* samples;
  SpeedHead* head;
  const double* homography;
  RecordIndex* index;
  SpeedRec* rec;
  double* ring;
  double frame_rate;
  int max_out, capacity, window, min_samples, forget_after, anchor, row0;
  int stream[LAUNCH_STREAMS];            // stream of CTA i: batch row row0 + i
};

struct Smem {
  Lifecycle lc;
  float4 box[MAXE];                      // by entry
  double h[9];
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// (x, y) in frame pixels -> (X, Y) on the ground; false when w <= 0 or X or Y is not finite
__device__ __forceinline__ bool project(const double* h, double x, double y, double& X, double& Y) {
  const double w = dadd(dadd(dmul(h[6], x), dmul(h[7], y)), h[8]);
  X = ddiv(dadd(dadd(dmul(h[0], x), dmul(h[1], y)), h[2]), w);
  Y = ddiv(dadd(dadd(dmul(h[3], x), dmul(h[4], y)), h[5]), w);
  return w > 0.0 && isfinite(X) && isfinite(Y);
}

// The least-squares velocity over the n samples of a ring (oldest at pos) that project validly: their count, and
// (vx, vy, speed) when there is an estimate (count >= min_samples and Stt > 0), else NaN.
__device__ int fit(const double* ring, SpeedRec r, int W, int min_samples, const double* h, double& vx, double& vy, double& sp) {
  vx = vy = sp = __longlong_as_double(0x7ff8000000000000ll);
  double t0 = 0.0, X, Y;
  int i = r.n - 1;
  for (; i >= 0; --i) {                  // the newest valid sample
    const double* q = ring + ((r.pos + i) % W) * 3;
    if (project(h, q[1], q[2], X, Y)) {
      t0 = q[0];
      break;
    }
  }
  if (i < 0) return 0;
  int n = 0;
  double st = 0.0, sx = 0.0, sy = 0.0;
  for (int k = 0; k < r.n; ++k) {
    const double* q = ring + ((r.pos + k) % W) * 3;
    if (!project(h, q[1], q[2], X, Y)) continue;
    st = dadd(st, dsub(q[0], t0));
    sx = dadd(sx, X);
    sy = dadd(sy, Y);
    ++n;
  }
  const double dn = static_cast<double>(n);
  const double mt = ddiv(st, dn), mx = ddiv(sx, dn), my = ddiv(sy, dn);
  double stt = 0.0, stx = 0.0, sty = 0.0;
  for (int k = 0; k < r.n; ++k) {
    const double* q = ring + ((r.pos + k) % W) * 3;
    if (!project(h, q[1], q[2], X, Y)) continue;
    const double d = dsub(dsub(q[0], t0), mt);
    stt = dadd(stt, dmul(d, d));
    stx = dadd(stx, dmul(d, dsub(X, mx)));
    sty = dadd(sty, dmul(d, dsub(Y, my)));
  }
  if (n >= min_samples && stt > 0.0) {
    vx = ddiv(stx, stt);
    vy = ddiv(sty, stt);
    sp = __dsqrt_rn(dadd(dmul(vx, vx), dmul(vy, vy)));
  }
  return n;
}

__global__ void __launch_bounds__(NT, 1) speed_kernel(const __grid_constant__ SpeedArgs a) {
  pdl_sync();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  Lifecycle& lc = s.lc;
  const int tid = threadIdx.x;
  const int row = a.row0 + blockIdx.x, sid = a.stream[blockIdx.x];
  const SpeedHead h = a.head[sid];
  const int frame = h.frame, n_old = h.n, C = a.capacity, W = a.window;
  RecordIndex* gidx = a.index + static_cast<long long>(sid) * C;
  SpeedRec* grec = a.rec + static_cast<long long>(sid) * C;
  double* gring = a.ring + static_cast<long long>(sid) * C * W * 3;
  const int cnt = min(max(a.counts[row], 0), a.max_out);
  const long long ent0 = static_cast<long long>(row) * a.max_out;
  const double t = a.timestamps ? a.timestamps[row] : ddiv(static_cast<double>(frame), a.frame_rate);
  const bool clock_ok = isfinite(t) && t > h.last_t;

  // 1. the lifecycle up to the slots of the new ids
  if (tid < 9) s.h[tid] = a.homography[static_cast<long long>(sid) * 9 + tid];
  const int np2 = lc_stage(lc, gidx, n_old, C, cnt, [&](int j, int& id) {
    id = a.ids[ent0 + j];
    const float4 b = a.boxes[ent0 + j];
    s.box[j] = b;
    return id > 0 && isfinite(b.x) && isfinite(b.y) && isfinite(b.z) && isfinite(b.w);
  });
  lc_sort(lc, np2);
  const int P = lc_present(lc, cnt, n_old);
  const int nnew = lc_assign(lc, P, n_old, C, frame);
  const int taken = min(nnew, C - n_old);
  __syncthreads();

  // 2. per present track: this frame's ground point, the sample, the fit
  const float nanf = __int_as_float(0x7fc00000);
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int p = tid; p < P; p += NT) {
    const int j = lc.plist[p], slot = lc.jslot[j];
    double x, y, X, Y;
    box_anchor(s.box[j], a.anchor, x, y);
    const bool valid = project(s.h, x, y, X, Y);
    double vx = nan, vy = nan, sp = nan;  // no estimate
    int n = 0;
    if (slot >= 0) {
      SpeedRec r = lc.jpos[j] >= 0 ? grec[slot] : SpeedRec{0, 0};
      double* ring = gring + static_cast<long long>(slot) * W * 3;
      if (clock_ok) {
        double* q = ring + (r.n < W ? (r.pos + r.n) % W : r.pos) * 3;
        q[0] = t;
        q[1] = x;
        q[2] = y;
        if (r.n < W) ++r.n;
        else r.pos = (r.pos + 1) % W;
      }
      grec[slot] = r;
      n = fit(ring, r, W, a.min_samples, s.h, vx, vy, sp);
    }
    float* o = a.kin + (ent0 + j) * 5;
    o[0] = valid ? static_cast<float>(X) : nanf;
    o[1] = valid ? static_cast<float>(Y) : nanf;
    o[2] = static_cast<float>(vx);
    o[3] = static_cast<float>(vy);
    o[4] = static_cast<float>(sp);
    a.samples[ent0 + j] = n;
  }
  for (int j = tid; j < a.max_out; j += NT) {    // absent entries
    if (j < cnt && lc_is_present(lc, j, cnt, P)) continue;
    float* o = a.kin + (ent0 + j) * 5;
    for (int c = 0; c < 5; ++c) o[c] = nanf;
    a.samples[ent0 + j] = 0;
  }

  // 3. forget, and the new index
  const int n_new = lc_merge(lc, gidx, n_old, cnt, P, frame, a.forget_after);
  if (tid == 0)
    a.head[sid] = SpeedHead{frame + 1, n_new, h.overflow + nnew - taken, h.clock_errors + (clock_ok ? 0 : 1), clock_ok ? t : h.last_t};
}

struct SpeedResetArgs {
  SpeedHead* head;
  int n;
  int stream[LAUNCH_STREAMS];
};

__global__ void speed_reset_kernel(const __grid_constant__ SpeedResetArgs a) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.n) a.head[a.stream[i]] = SpeedHead{1, 0, 0, 0, -__longlong_as_double(0x7ff0000000000000ll)};
}

}  // namespace

int speed_launch(const SpeedTable& t, const int32_t* ids, const float* boxes, const int32_t* counts, int B, int max_out,
                 const int32_t* streams, const double* timestamps, float* kin, int32_t* samples, cudaStream_t st) {
  constexpr int smem = static_cast<int>(sizeof(Smem));
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(speed_kernel), smem)) return e;
  std::vector<SpeedArgs> hold(1);        // ~4 KB of parameters: kept off the stack
  SpeedArgs& a = hold[0];
  a.ids = ids;
  a.boxes = reinterpret_cast<const float4*>(boxes);
  a.counts = counts;
  a.timestamps = timestamps;
  a.kin = kin;
  a.samples = samples;
  a.head = t.head;
  a.homography = t.homography;
  a.index = t.index;
  a.rec = t.rec;
  a.ring = t.ring;
  a.frame_rate = t.frame_rate;
  a.max_out = max_out;
  a.capacity = t.capacity;
  a.window = t.window;
  a.min_samples = t.min_samples;
  a.forget_after = t.forget_after;
  a.anchor = t.anchor;
  for (int b0 = 0; b0 < B; b0 += LAUNCH_STREAMS) {
    const int nb = B - b0 < LAUNCH_STREAMS ? B - b0 : LAUNCH_STREAMS;
    a.row0 = b0;
    for (int i = 0; i < nb; ++i) a.stream[i] = streams[b0 + i];
    launch_k(speed_kernel, dim3(nb), dim3(NT), static_cast<size_t>(smem), st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

int speed_reset_launch(const SpeedTable& t, const int32_t* streams, int n, cudaStream_t st) {
  std::vector<SpeedResetArgs> hold(1);
  SpeedResetArgs& a = hold[0];
  a.head = t.head;
  for (int i0 = 0; i0 < n; i0 += LAUNCH_STREAMS) {
    a.n = n - i0 < LAUNCH_STREAMS ? n - i0 : LAUNCH_STREAMS;
    for (int i = 0; i < a.n; ++i) a.stream[i] = streams[i0 + i];
    launch_k(speed_reset_kernel, dim3((a.n + 255) / 256), dim3(256), 0, st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

}  // namespace lwb
