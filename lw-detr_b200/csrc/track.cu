// lwdetr_track: ByteTrack (BYTETracker.update) per camera stream on the device, bit for bit the contract stated in
// include/lwdetr_b200.h and restated in tools/track_spec.py.  One CTA per stream in the call; the stream's lists live in
// a device table (two record buffers per stream, the frame's result written to the other one), so a call allocates and
// copies nothing and replays correctly from a CUDA graph.  Per frame:
//   1. the frame's entries and the stream's records are loaded; the pool (confirmed tracks, then lost ones) is predicted,
//      one thread per track, in float64 with every operation rounded on its own (__dadd_rn / __dmul_rn / __ddiv_rn);
//      with a camera motion (lwdetr_track_ex) every record is then warped by the frame's similarity;
//   2. each association lists its admissible (track, detection) pairs, finds the connected components by label
//      propagation in shared memory, sorts the nodes by (component, index) and gives each component to one warp, which
//      runs the shortest-augmenting-path Hungarian method on it: lanes scan the component's columns (costs recomputed on
//      the fly, nothing n x m is stored) and a shuffle argmin takes the smallest slack, lowest column on ties.  A row's
//      search never leaves its component, so this gives the bits of the whole-matrix solve;
//   3. the lifecycle (updates, lost, removed, births under the capacity, ageing, duplicates) and a compaction into the
//      other buffer in ByteTrack's list order; the activated tracked tracks are the output.
// lwdetr_track_reid is a second instantiation of the same kernel (ReidArgs / SmemReid; the ByteTrack one compiles as
// before).  After the entry lists it computes each high entry's norm (one warp each), lists the (track, high entry) pairs
// that pass the proximity test, both with appearance, sorted by (track, entry) into a per-stream global table of
// TRACK_PAIRS, and gives each its emb' (one warp per pair).  The Hungarian lanes look a pair up by binary search within its
// track's row (row offsets in shared memory).  Beyond TRACK_PAIRS pairs a lane computes emb' itself, in the same summation
// order, so the bits do not depend on the table.  Track embeddings live in stable per-stream slots: a record carries its
// slot through the compaction (a parallel slot array, double-buffered like the records) and a birth takes the lowest free
// slot, so a frame moves no embedding; only updates and births write D floats.
#include "track.h"
#include "flow.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <climits>
#include <type_traits>
#include <vector>

#include "launch.h"
#include "postproc.cuh"

namespace lwb {
namespace {

constexpr int NT = 512;                  // threads per CTA
constexpr int NW = NT / 32;
constexpr int MAXN = TRACK_MAX;
constexpr int EMAX = 8192;               // admissible pairs kept for the component search; beyond: one component
constexpr int LAUNCH_STREAMS = 1024;     // CTAs per launch (the stream table travels in the parameters)
constexpr double INF = __builtin_huge_val();

enum : uint8_t { TF_ACT = 1, TF_LOSTLIST = 2, TF_MATCHED = 4, TF_REFOUND = 8, TF_NEWLOST = 16, TF_REMOVED = 32, TF_DROP = 64 };

struct TrackArgs {
  const float* scores;
  const int32_t* labels;
  const float4* boxes;
  int32_t* out_ids;
  float* out_scores;
  int32_t* out_labels;
  float4* out_boxes;
  int32_t* out_index;
  int32_t* counts;
  TrackHead* head;
  lwdetr_track_record* rec;
  const double* motion;                  // [rows][4] (a, b, tx, ty) or null
  float track_thresh, low_thresh, new_thresh, match_thresh, second_thresh, unconf_thresh, dup_thresh;
  int k, max_out, capacity, max_time_lost, fuse, class_aware, row0;
  int stream[LAUNCH_STREAMS];            // stream of CTA i: batch row row0 + i
};

struct ReidArgs : TrackArgs {
  const void* emb;                       // entry embeddings [rows][k] rows of ld_emb elements, or null (no appearance)
  long long ld_emb;
  int dtype, dim;                        // LWDETR_ET_*, D
  float prox, app, alpha;
  int16_t* slot;                         // [streams][2][capacity], parallel to rec
  uint8_t* has;                          // [streams][capacity] by slot
  float* temb;                           // [streams][capacity][dim] by slot
  uint32_t* pkey;                        // [streams][TRACK_PAIRS]: (record << 16) | entry, ascending
  double* pval;                          // [streams][TRACK_PAIRS]: emb' of the pair
};

struct Smem {
  double4 tbox[MAXN];                    // track slot boxes (after predict / update)
  double u[2 * MAXN], v[2 * MAXN], minv[2 * MAXN];
  float4 ebox[MAXN];
  float escore[MAXN];
  int elab[MAXN], tlab[MAXN], tdiff[MAXN];
  uint32_t key[2 * MAXN];
  int lab[2 * MAXN];
  uint32_t edge[EMAX];
  int16_t p[2 * MAXN], way[2 * MAXN], seg[2 * MAXN + 1];
  int16_t high[MAXN], low[MAXN], pool[MAXN], unconf[MAXN], rows[MAXN], rest[MAXN], births[MAXN], match[MAXN], tdet[MAXN];
  int16_t tlist[MAXN], llist[MAXN];
  uint8_t used[2 * MAXN], tf[MAXN], eused[MAXN], bdrop[MAXN];
  int wsum[NW];
  int n_edges, changed, n_removed;
};

struct SmemReid : Smem {
  double enorm[MAXN];                    // entry norm ne, 0 without appearance (high entries only)
  int16_t tslot[MAXN], bslot[MAXN], poff[MAXN + 1];
  uint8_t thas[MAXN], sused[MAXN];
  const uint32_t* pkey;                  // this stream's pair table
  const double* pval;
  const float* temb;                     // this stream's track embeddings
  const char* erow;                      // entry 0 of this frame's embeddings, or null
  long long ld_bytes;
  double prox, app;
  int dtype, dim, overflow, app_on;
};

template <class SM>
constexpr bool kReid = std::is_same<SM, SmemReid>::value;

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dsqrt(double a) { return __dsqrt_rn(a); }

struct KState {
  double p[4], v[4], P[4], C[4], V[4];
};

__device__ __forceinline__ void load_state(const lwdetr_track_record& r, KState& s) {
  for (int q = 0; q < 4; ++q) {
    s.p[q] = r.mean[q];
    s.v[q] = r.mean[4 + q];
    s.P[q] = r.cov[q];
    s.C[q] = r.cov[4 + q];
    s.V[q] = r.cov[8 + q];
  }
}

__device__ __forceinline__ void store_state(lwdetr_track_record& r, const KState& s) {
  for (int q = 0; q < 4; ++q) {
    r.mean[q] = s.p[q];
    r.mean[4 + q] = s.v[q];
    r.cov[q] = s.P[q];
    r.cov[4 + q] = s.C[q];
    r.cov[8 + q] = s.V[q];
  }
}

// (w * h, w * h, fixed, w * h)[q]
__device__ __forceinline__ double std_of(int q, double h, double w, double fixed) { return q == 2 ? fixed : dmul(w, h); }

__device__ __forceinline__ double4 state_box(const double* p) {
  const double w = dmul(p[2], p[3]);
  const double x1 = dsub(p[0], dmul(w, 0.5));
  const double y1 = dsub(p[1], dmul(p[3], 0.5));
  return make_double4(x1, y1, dadd(x1, w), dadd(y1, p[3]));
}

__device__ __forceinline__ void measurement(float4 b, double* z) {
  const double x1 = b.x, y1 = b.y, w = dsub(static_cast<double>(b.z), x1), h = dsub(static_cast<double>(b.w), y1);
  z[0] = dadd(x1, dmul(w, 0.5));
  z[1] = dadd(y1, dmul(h, 0.5));
  z[2] = ddiv(w, h);
  z[3] = h;
}

__device__ void initiate(KState& s, const double* z) {
  const double h = z[3];
  for (int q = 0; q < 4; ++q) {
    const double sp = std_of(q, h, 2 * (1.0 / 20), 1e-2), sv = std_of(q, h, 10 * (1.0 / 160), 1e-5);
    s.p[q] = z[q];
    s.v[q] = 0.0;
    s.P[q] = dmul(sp, sp);
    s.C[q] = 0.0;
    s.V[q] = dmul(sv, sv);
  }
}

__device__ void predict(KState& s, bool tracked) {
  if (!tracked) s.v[3] = 0.0;
  const double h = s.p[3];
  for (int q = 0; q < 4; ++q) {
    const double sp = std_of(q, h, 1.0 / 20, 1e-2), sv = std_of(q, h, 1.0 / 160, 1e-5);
    s.p[q] = dadd(s.p[q], s.v[q]);
    s.P[q] = dadd(dadd(dadd(s.P[q], dadd(s.C[q], s.C[q])), s.V[q]), dmul(sp, sp));
    s.C[q] = dadd(s.C[q], s.V[q]);
    s.V[q] = dadd(s.V[q], dmul(sv, sv));
  }
}

// camera motion x' = a x - b y + tx, y' = b x + a y + ty applied to the state.  s = sqrt(a^2 + b^2); x, y and h scale by s,
// so their (P, C, V) scale by s^2 (the x and y blocks are equal, so the rotation leaves them diagonal); the aspect keeps its own.
__device__ void warp_state(KState& s, const double* m) {
  const double a = m[0], b = m[1];
  const double s2 = dadd(dmul(a, a), dmul(b, b)), sc = dsqrt(s2);
  const double cx = s.p[0], cy = s.p[1], vx = s.v[0], vy = s.v[1];
  s.p[0] = dadd(dsub(dmul(a, cx), dmul(b, cy)), m[2]);
  s.p[1] = dadd(dadd(dmul(b, cx), dmul(a, cy)), m[3]);
  s.v[0] = dsub(dmul(a, vx), dmul(b, vy));
  s.v[1] = dadd(dmul(b, vx), dmul(a, vy));
  s.p[3] = dmul(sc, s.p[3]);
  s.v[3] = dmul(sc, s.v[3]);
  const int scaled[3] = {0, 1, 3};
  for (int q : scaled) {
    s.P[q] = dmul(s2, s.P[q]);
    s.C[q] = dmul(s2, s.C[q]);
    s.V[q] = dmul(s2, s.V[q]);
  }
}

__device__ void kalman_update(KState& s, const double* z) {
  const double h = s.p[3];
  for (int q = 0; q < 4; ++q) {
    const double sr = std_of(q, h, 1.0 / 20, 1e-1);
    const double S = dadd(s.P[q], dmul(sr, sr));
    const double Kp = ddiv(s.P[q], S), Kv = ddiv(s.C[q], S);
    const double y = dsub(z[q], s.p[q]);
    s.p[q] = dadd(s.p[q], dmul(Kp, y));
    s.v[q] = dadd(s.v[q], dmul(Kv, y));
    s.P[q] = dsub(s.P[q], dmul(dmul(Kp, Kp), S));
    s.C[q] = dsub(s.C[q], dmul(dmul(Kp, Kv), S));
    s.V[q] = dsub(s.V[q], dmul(dmul(Kv, Kv), S));
  }
}

__device__ __forceinline__ double iou_d(double4 a, double4 b) {
  const double ix = fmax(0.0, dsub(fmin(a.z, b.z), fmax(a.x, b.x)));
  const double iy = fmax(0.0, dsub(fmin(a.w, b.w), fmax(a.y, b.y)));
  const double inter = dmul(ix, iy);
  const double aa = dmul(fmax(0.0, dsub(a.z, a.x)), fmax(0.0, dsub(a.w, a.y)));
  const double ab = dmul(fmax(0.0, dsub(b.z, b.x)), fmax(0.0, dsub(b.w, b.y)));
  const double uni = dsub(dadd(aa, ab), inter);
  if (!(aa > 0.0) || !(ab > 0.0) || !(uni > 0.0)) return 0.0;
  return ddiv(inter, uni);
}

__device__ __forceinline__ double4 widen(float4 b) { return make_double4(b.x, b.y, b.z, b.w); }

struct Assoc {
  double L;
  bool fuse, class_aware;
};

__device__ __forceinline__ double emb_at(const char* row, int dtype, int i) {
  if (dtype == LWDETR_ET_F32) return reinterpret_cast<const float*>(row)[i];
  if (dtype == LWDETR_ET_F16) return __half2float(reinterpret_cast<const __half*>(row)[i]);
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(row)[i]);
}

// the header's fixed order, one lane: partial J of dot(t, e) (terms J, J + 32, ... from 0), combined as the xor butterfly
// 16, 8, 4, 2, 1 combines them for lane 0
template <int J, int O>
__device__ double tree_dot(const float* t, const char* e, int dtype, int D) {
  if constexpr (O == 32) {
    double p = 0.0;
    for (int i = J; i < D; i += 32) p = dadd(p, dmul(t[i], emb_at(e, dtype, i)));
    return p;
  } else {
    return dadd(tree_dot<J, 2 * O>(t, e, dtype, D), tree_dot<J + O, 2 * O>(t, e, dtype, D));
  }
}

// the same order over a warp: every lane holds its partial, every lane ends with the sum
__device__ __forceinline__ double warp_tree(double p) {
  for (int o = 16; o > 0; o >>= 1) p = dadd(p, __shfl_xor_sync(0xffffffffu, p, o));
  return p;
}

// emb' = max(0, 1 - dot / ne) / 2, or 1 above appearance_thresh
__device__ __forceinline__ double emb_cost(double dot, double ne, double app) {
  const double m = ddiv(fmax(0.0, dsub(1.0, ddiv(dot, ne))), 2.0);
  return m <= app ? m : 1.0;
}

// emb' of (record sl, entry e) whose IoU is io: from the pair table, or computed here when the table overflowed
__device__ double appearance(const SmemReid& S, int sl, int e, double io) {
  if (!(dsub(1.0, io) <= S.prox)) return 1.0;
  if (S.overflow) {
    if (!S.thas[sl] || !(S.enorm[e] > 0.0)) return 1.0;
    const char* er = S.erow + e * S.ld_bytes;
    return emb_cost(tree_dot<0, 1>(S.temb + static_cast<long long>(S.tslot[sl]) * S.dim, er, S.dtype, S.dim), S.enorm[e], S.app);
  }
  const uint32_t key = (static_cast<uint32_t>(sl) << 16) | static_cast<uint32_t>(e);
  int lo = S.poff[sl];
  const int end = S.poff[sl + 1];
  for (int hi = end; lo < hi;) {
    const int mid = (lo + hi) >> 1;
    if (S.pkey[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo < end && S.pkey[lo] == key ? S.pval[lo] : 1.0;
}

// cost of (record sl: track box tb with label tl, entry e), +inf when not admissible.  L <= 1 (checked by the C ABI), so
// a pair without overlap (cost 1) is never admissible; with appearance the cost is min(cost, emb'), and emb' < 1 needs
// 1 - iou <= proximity_thresh < 1, so that still holds.
template <class SM>
__device__ __forceinline__ double pair_cost(const SM& S, double4 tb, int tl, int e, const Assoc& A, int sl) {
  if (A.class_aware && tl != S.elab[e]) return INF;
  const double io = iou_d(tb, widen(S.ebox[e]));
  double c = A.fuse ? dsub(1.0, dmul(io, static_cast<double>(S.escore[e]))) : dsub(1.0, io);
  if constexpr (kReid<SM>) {
    if (S.app_on) {
      const double m = appearance(S, sl, e, io);
      if (m < c) c = m;
    }
  }
  return c < A.L ? c : INF;
}

// Ordered compaction over i in [0, n): emit(i, rank) for every i with pred(i), rank counting those before it.  Returns
// the count.  Every thread of the block calls it.
template <typename Pred, typename Emit>
__device__ int ordered_scan(Smem& S, int n, Pred pred, Emit emit) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int base = 0;
  for (int i0 = 0; i0 < n; i0 += NT) {
    const int i = i0 + threadIdx.x;
    const bool f = i < n && pred(i);
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) S.wsum[w] = __popc(bal);
    __syncthreads();
    int off = 0, tot = 0;
    for (int q = 0; q < NW; ++q) {
      const int c = S.wsum[q];
      off += q < w ? c : 0;
      tot += c;
    }
    if (f) emit(i, base + off + __popc(bal & ((1u << lane) - 1u)));
    base += tot;
    __syncthreads();
  }
  return base;
}

__device__ void bitonic_sort_asc(uint32_t* key, int np2) {
  for (int size = 2; size <= np2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < np2 / 2; i += NT) {
        const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
        const bool asc = (lo & size) == 0;
        const uint32_t a = key[lo], b = key[hi];
        if ((a > b) == asc && a != b) {
          key[lo] = b;
          key[hi] = a;
        }
      }
      __syncthreads();
    }
  }
}

// One warp: the Hungarian method on one component, nodes key[q0, q1) sorted rows first (R of them), then C columns.
// Local column t < C is the t-th real column, t = C + i the own "unmatched" column of local row i (cost L).
template <class SM>
__device__ void solve_component(SM& S, int q0, int R, int C, int nr, const int16_t* rows, const int16_t* cols, const Assoc& A) {
  const int lane = threadIdx.x & 31;
  const int T = R + C;
  double* u = S.u + q0;
  double* v = S.v + q0;
  double* minv = S.minv + q0;
  int16_t* p = S.p + q0;
  int16_t* way = S.way + q0;
  uint8_t* used = S.used + q0;
  const uint32_t* key = S.key + q0;
  for (int t = lane; t < T; t += 32) {
    v[t] = 0.0;
    p[t] = -1;
  }
  for (int t = lane; t < R; t += 32) u[t] = 0.0;
  __syncwarp();
  for (int ri = 0; ri < R; ++ri) {
    for (int t = lane; t < T; t += 32) {
      minv[t] = INF;
      used[t] = 0;
    }
    __syncwarp();
    int j0 = -1;                                     // the virtual column holding row ri
    for (;;) {
      int i0 = ri;
      if (j0 >= 0) {
        i0 = p[j0];
        if (lane == 0) used[j0] = 1;
      }
      __syncwarp();
      const int slot = rows[key[i0] & 2047];
      const double4 tb = S.tbox[slot];
      const int tl = S.tlab[slot];
      const double ui0 = u[i0];
      double best = INF;
      int bt = INT_MAX;
      for (int t = lane; t < T; t += 32) {
        if (used[t]) continue;
        const double c = t < C ? pair_cost(S, tb, tl, cols[(key[R + t] & 2047) - nr], A, slot) : (t - C == i0 ? A.L : INF);
        const double cur = dsub(dsub(c, ui0), v[t]);
        double mv = minv[t];
        if (cur < mv) {
          mv = cur;
          minv[t] = cur;
          way[t] = static_cast<int16_t>(j0);
        }
        if (mv < best) {
          best = mv;
          bt = t;
        }
      }
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
        if (ob < best || (ob == best && ot < bt)) {
          best = ob;
          bt = ot;
        }
      }
      const double delta = best;
      for (int t = lane; t < T; t += 32) {
        if (used[t]) {
          u[p[t]] = dadd(u[p[t]], delta);
          v[t] = dsub(v[t], delta);
        } else {
          minv[t] = dsub(minv[t], delta);
        }
      }
      if (lane == 0) u[ri] = dadd(u[ri], delta);
      __syncwarp();
      j0 = bt;
      if (p[j0] < 0) break;
    }
    if (lane == 0) {
      for (int j = j0; j >= 0;) {
        const int jp = way[j];
        p[j] = static_cast<int16_t>(jp < 0 ? ri : p[jp]);
        j = jp;
      }
    }
    __syncwarp();
  }
  for (int t = lane; t < C; t += 32)
    if (p[t] >= 0) S.match[key[p[t]] & 2047] = static_cast<int16_t>((key[R + t] & 2047) - nr);
  __syncwarp();
}

// rows: nr track slots, cols: nc entry indices -> S.match[r]: the column position matched to row r, or -1.
template <class SM>
__device__ void associate(SM& S, const int16_t* rows, int nr, const int16_t* cols, int nc, const Assoc& A) {
  const int tid = threadIdx.x;
  for (int r = tid; r < nr; r += NT) S.match[r] = -1;
  if (tid == 0) S.n_edges = 0;
  __syncthreads();
  if (nr == 0 || nc == 0) return;
  const int n = nr + nc;
  for (int idx = tid; idx < nr * nc; idx += NT) {
    const int r = idx / nc, c = idx - r * nc;
    const int slot = rows[r];
    if (pair_cost(S, S.tbox[slot], S.tlab[slot], cols[c], A, slot) < INF) {
      const int e = atomicAdd(&S.n_edges, 1);
      if (e < EMAX) S.edge[e] = (static_cast<uint32_t>(r) << 16) | static_cast<uint32_t>(c);
    }
  }
  __syncthreads();
  const int ne = S.n_edges;
  if (ne == 0) return;
  const bool one = ne > EMAX;                          // too many pairs to keep: solve everything as one component
  for (int x = tid; x < n; x += NT) S.lab[x] = one ? 0 : x;
  __syncthreads();
  while (!one) {
    if (tid == 0) S.changed = 0;
    __syncthreads();
    for (int i = tid; i < ne; i += NT) {
      const uint32_t e = S.edge[i];
      const int la = S.lab[e >> 16], lb = S.lab[nr + (e & 0xffff)];
      if (la != lb) {
        const int lo = min(la, lb);
        if (atomicMin(&S.lab[max(la, lb)], lo) > lo) S.changed = 1;
      }
    }
    __syncthreads();
    for (int x = tid; x < n; x += NT) {
      const int l = S.lab[x], ll = S.lab[l];
      if (ll != l) {
        S.lab[x] = ll;
        S.changed = 1;
      }
    }
    __syncthreads();
    const int ch = S.changed;
    __syncthreads();
    if (!ch) break;
  }
  int np2 = 2;
  while (np2 < n) np2 <<= 1;
  for (int x = tid; x < np2; x += NT) S.key[x] = x < n ? (static_cast<uint32_t>(S.lab[x]) << 11) | static_cast<uint32_t>(x) : 0xffffffffu;
  __syncthreads();
  bitonic_sort_asc(S.key, np2);
  const int nseg = ordered_scan(S, n, [&](int q) { return q == 0 || (S.key[q] >> 11) != (S.key[q - 1] >> 11); },
                                [&](int q, int rank) { S.seg[rank] = static_cast<int16_t>(q); });
  if (tid == 0) S.seg[nseg] = static_cast<int16_t>(n);
  __syncthreads();
  const int lane = tid & 31;
  for (int g = tid >> 5; g < nseg; g += NW) {
    const int q0 = S.seg[g], q1 = S.seg[g + 1];
    int R = 0;                                       // rows sort first within a segment
    for (int base = q0; base < q1; base += 32) {
      const int q = base + lane;
      R += __popc(__ballot_sync(0xffffffffu, q < q1 && (S.key[q] & 2047) < static_cast<uint32_t>(nr)));
    }
    const int C = q1 - q0 - R;
    if (R > 0 && C > 0) solve_component(S, q0, R, C, nr, rows, cols, A);
  }
  __syncthreads();
}

__device__ void write_output(const TrackArgs& a, long long o, int id, float score, int label, float4 box, int index) {
  a.out_ids[o] = id;
  a.out_scores[o] = score;
  a.out_labels[o] = label;
  a.out_boxes[o] = box;
  a.out_index[o] = index;
}

__device__ __forceinline__ float4 narrow(double4 b) {
  return make_float4(__double2float_rn(b.x), __double2float_rn(b.y), __double2float_rn(b.z), __double2float_rn(b.w));
}

// An update of a track's embedding t (slot es) by an entry with appearance (row er, norm ne), one warp: t = e / ne for a
// track without one, else s = alpha t + (1 - alpha) e / ne and t = s / |s| (t unchanged when |s| is not finite or not > 0).
// Each lane recomputes its s_i in the second pass, so nothing of length D is kept.
__device__ void ema_update(const ReidArgs& a, float* t, uint8_t* has, const char* er, double ne) {
  const int lane = threadIdx.x & 31, D = a.dim;
  if (!*has) {
    for (int i = lane; i < D; i += 32) t[i] = __double2float_rn(ddiv(emb_at(er, a.dtype, i), ne));
    __syncwarp();
    if (lane == 0) *has = 1;
    return;
  }
  const double al = a.alpha, om = dsub(1.0, al);
  double p = 0.0;
  for (int i = lane; i < D; i += 32) {
    const double si = dadd(dmul(al, static_cast<double>(t[i])), dmul(om, ddiv(emb_at(er, a.dtype, i), ne)));
    p = dadd(p, dmul(si, si));
  }
  const double n = dsqrt(warp_tree(p));
  if (!(isfinite(n) && n > 0.0)) return;
  for (int i = lane; i < D; i += 32) {
    const double si = dadd(dmul(al, static_cast<double>(t[i])), dmul(om, ddiv(emb_at(er, a.dtype, i), ne)));
    t[i] = __double2float_rn(ddiv(si, n));
  }
}

template <class Args>
__global__ void __launch_bounds__(NT, 1) track_kernel(const __grid_constant__ Args a) {
  constexpr bool REID = std::is_same<Args, ReidArgs>::value;
  using SM = std::conditional_t<REID, SmemReid, Smem>;
  pdl_sync();   // programmatic dependent launch: release the successor, wait for the predecessor (launch.h)
  extern __shared__ __align__(16) uint8_t sm_track[];
  SM& S = *reinterpret_cast<SM*>(sm_track);
  const int tid = threadIdx.x;
  const int sid = a.stream[blockIdx.x];
  const long long row = a.row0 + blockIdx.x;
  TrackHead* hp = a.head + sid;
  const int frame = hp->frame, next_id = hp->next_id, nT = hp->n_tracked, nL = hp->n_lost, parity = hp->parity;
  const int nS = nT + nL, k = a.k, cap = a.capacity;
  lwdetr_track_record* cur = a.rec + (static_cast<long long>(sid) * 2 + parity) * cap;
  lwdetr_track_record* nxt = a.rec + (static_cast<long long>(sid) * 2 + (parity ^ 1)) * cap;
  const float* sc = a.scores + row * k;
  const int32_t* lb = a.labels + row * k;
  const float4* bx = a.boxes + row * k;

  if (tid == 0) S.n_removed = 0;
  [[maybe_unused]] const int lane = tid & 31, warp = tid >> 5;
  [[maybe_unused]] int16_t *slot_cur = nullptr, *slot_nxt = nullptr;
  [[maybe_unused]] uint8_t* has = nullptr;
  [[maybe_unused]] float* temb = nullptr;
  if constexpr (REID) {
    slot_cur = a.slot + (static_cast<long long>(sid) * 2 + parity) * cap;
    slot_nxt = a.slot + (static_cast<long long>(sid) * 2 + (parity ^ 1)) * cap;
    has = a.has + static_cast<long long>(sid) * cap;
    temb = a.temb + static_cast<long long>(sid) * cap * a.dim;
    if (tid == 0) {
      const int esz = a.dtype == LWDETR_ET_F32 ? 4 : 2;
      S.pkey = a.pkey + static_cast<long long>(sid) * TRACK_PAIRS;
      S.pval = a.pval + static_cast<long long>(sid) * TRACK_PAIRS;
      S.temb = temb;
      S.ld_bytes = a.ld_emb * esz;
      S.erow = a.emb ? static_cast<const char*>(a.emb) + row * k * S.ld_bytes : nullptr;
      S.prox = a.prox;
      S.app = a.app;
      S.dtype = a.dtype;
      S.dim = a.dim;
      S.app_on = 0;
    }
  }
  for (int i = tid; i < k; i += NT) {
    S.ebox[i] = bx[i];
    S.escore[i] = sc[i];
    S.elab[i] = lb[i];
    S.eused[i] = 0;
  }
  for (int sl = tid; sl < nS; sl += NT) {
    lwdetr_track_record& r = cur[sl];
    const bool lost = sl >= nT, act = r.activated != 0;
    KState ks;
    load_state(r, ks);
    if (lost || act) predict(ks, !lost);
    if (a.motion) warp_state(ks, a.motion + row * 4);
    if (lost || act || a.motion) store_state(r, ks);
    S.tbox[sl] = state_box(ks.p);
    S.tlab[sl] = r.label;
    S.tdiff[sl] = r.end_frame - r.start_frame;
    S.tdet[sl] = -1;
    S.tf[sl] = static_cast<uint8_t>((act ? TF_ACT : 0) | (lost ? TF_LOSTLIST : 0));
    if constexpr (REID) {
      S.tslot[sl] = slot_cur[sl];
      S.thas[sl] = has[slot_cur[sl]];
    }
  }
  __syncthreads();
  const auto valid = [&](int i) {
    const double x1 = S.ebox[i].x, y1 = S.ebox[i].y, x2 = S.ebox[i].z, y2 = S.ebox[i].w;
    return isfinite(x1) && isfinite(y1) && isfinite(x2) && isfinite(y2) && dsub(x2, x1) > 0.0 && dsub(y2, y1) > 0.0;
  };
  const int nh = ordered_scan(S, k, [&](int i) { return S.escore[i] > a.track_thresh && valid(i); },
                              [&](int i, int r) { S.high[r] = static_cast<int16_t>(i); });
  const int nl = ordered_scan(S, k, [&](int i) { return S.escore[i] > a.low_thresh && S.escore[i] < a.track_thresh && valid(i); },
                              [&](int i, int r) { S.low[r] = static_cast<int16_t>(i); });
  const int np = ordered_scan(S, nS, [&](int sl) { return (S.tf[sl] & (TF_ACT | TF_LOSTLIST)) != 0; },
                              [&](int sl, int r) { S.pool[r] = static_cast<int16_t>(sl); });
  const int nu = ordered_scan(S, nT, [&](int sl) { return !(S.tf[sl] & TF_ACT); },
                              [&](int sl, int r) { S.unconf[r] = static_cast<int16_t>(sl); });
  [[maybe_unused]] const auto update_embedding = [&](int sl, int e) {
    if constexpr (REID) {
      if (S.enorm[e] > 0.0) {
        const int es = S.tslot[sl];
        ema_update(a, temb + static_cast<long long>(es) * a.dim, has + es, S.erow + e * S.ld_bytes, S.enorm[e]);
      }
    }
  };
  if constexpr (REID) {
    // entry norms of the high entries, one warp each, in the fixed order
    for (int c = warp; c < nh; c += NW) {
      const int e = S.high[c];
      double p = 0.0;
      if (S.erow) {
        const char* er = S.erow + e * S.ld_bytes;
        for (int i = lane; i < a.dim; i += 32) {
          const double x = emb_at(er, a.dtype, i);
          p = dadd(p, dmul(x, x));
        }
      }
      const double ne = dsqrt(warp_tree(p));
      if (lane == 0) S.enorm[e] = isfinite(ne) && ne > 0.0 ? ne : 0.0;
    }
    __syncthreads();
    // the (record, high entry) pairs within proximity, both with appearance, in (record, entry) order
    uint32_t* pkey = a.pkey + static_cast<long long>(sid) * TRACK_PAIRS;
    double* pval = a.pval + static_cast<long long>(sid) * TRACK_PAIRS;
    const int npairs = ordered_scan(S, nS * nh, [&](int idx) {
      const int sl = idx / nh, e = S.high[idx - sl * nh];
      return S.thas[sl] && S.enorm[e] > 0.0 && dsub(1.0, iou_d(S.tbox[sl], widen(S.ebox[e]))) <= S.prox;
    }, [&](int idx, int r) {
      const int sl = idx / nh, e = S.high[idx - sl * nh];
      if (r < TRACK_PAIRS) pkey[r] = (static_cast<uint32_t>(sl) << 16) | static_cast<uint32_t>(e);
    });
    const bool overflow = npairs > TRACK_PAIRS;
    if (tid == 0) S.overflow = overflow;
    if (!overflow) {
      __syncthreads();                   // the keys written by other threads
      for (int i = warp; i < npairs; i += NW) {
        const uint32_t key = pkey[i];
        const int sl = key >> 16, e = key & 0xffff;
        const float* t = temb + static_cast<long long>(S.tslot[sl]) * a.dim;
        const char* er = S.erow + e * S.ld_bytes;
        double p = 0.0;
        for (int j = lane; j < a.dim; j += 32) p = dadd(p, dmul(static_cast<double>(t[j]), emb_at(er, a.dtype, j)));
        const double dot = warp_tree(p);
        if (lane == 0) pval[i] = emb_cost(dot, S.enorm[e], S.app);
      }
      for (int sl = tid; sl <= nS; sl += NT) {
        const uint32_t key = static_cast<uint32_t>(sl) << 16;
        int lo = 0;
        for (int hi = npairs; lo < hi;) {
          const int mid = (lo + hi) >> 1;
          if (pkey[mid] < key) lo = mid + 1;
          else hi = mid;
        }
        S.poff[sl] = static_cast<int16_t>(lo);
      }
    }
    if (tid == 0) S.app_on = 1;
    __syncthreads();
  }

  // a matched track takes the entry's measurement, score, label and this frame
  const auto take = [&](int sl, int e) {
    lwdetr_track_record& r = cur[sl];
    KState ks;
    load_state(r, ks);
    double z[4];
    measurement(S.ebox[e], z);
    kalman_update(ks, z);
    store_state(r, ks);
    r.state = LWDETR_TRACK_TRACKED;
    r.activated = 1;
    r.end_frame = frame;
    r.score = S.escore[e];
    r.label = S.elab[e];
    r.index = e;
    S.tbox[sl] = state_box(ks.p);
    S.tlab[sl] = S.elab[e];
    S.tdiff[sl] = frame - r.start_frame;
    S.tdet[sl] = static_cast<int16_t>(e);
    S.eused[e] = 1;
  };

  // 1. pool x high detections
  associate(S, S.pool, np, S.high, nh, Assoc{static_cast<double>(a.match_thresh), a.fuse != 0, a.class_aware != 0});
  for (int r = tid; r < np; r += NT) {
    const int sl = S.pool[r], c = S.match[r];
    if (c >= 0) {
      take(sl, S.high[c]);
      S.tf[sl] |= TF_MATCHED | ((S.tf[sl] & TF_LOSTLIST) ? TF_REFOUND : 0);
    }
  }
  __syncthreads();
  if constexpr (REID) {
    for (int r = warp; r < np; r += NW)
      if (S.match[r] >= 0) update_embedding(S.pool[r], S.high[S.match[r]]);
    if (tid == 0) S.app_on = 0;          // association 2 (low entries) is IoU only
  }
  const int nrest = ordered_scan(S, nh, [&](int c) { return !S.eused[S.high[c]]; },
                                 [&](int c, int r) { S.rest[r] = S.high[c]; });
  const int nrt = ordered_scan(S, np, [&](int r) { return S.match[r] < 0 && !(S.tf[S.pool[r]] & TF_LOSTLIST); },
                               [&](int r, int q) { S.rows[q] = S.pool[r]; });
  // 2. the pool's unmatched Tracked tracks x low detections, no score fusion
  associate(S, S.rows, nrt, S.low, nl, Assoc{static_cast<double>(a.second_thresh), false, a.class_aware != 0});
  for (int r = tid; r < nrt; r += NT) {
    const int sl = S.rows[r], c = S.match[r];
    if (c >= 0) {
      take(sl, S.low[c]);
      S.tf[sl] |= TF_MATCHED;
    } else {
      cur[sl].state = LWDETR_TRACK_LOST;
      S.tf[sl] |= TF_NEWLOST;
    }
  }
  __syncthreads();
  // 3. unconfirmed tracks x the high detections left
  if constexpr (REID) {
    if (tid == 0) S.app_on = 1;
  }
  associate(S, S.unconf, nu, S.rest, nrest, Assoc{static_cast<double>(a.unconf_thresh), a.fuse != 0, a.class_aware != 0});
  for (int r = tid; r < nu; r += NT) {
    const int sl = S.unconf[r], c = S.match[r];
    if (c >= 0) {
      take(sl, S.rest[c]);
      S.tf[sl] |= TF_MATCHED;
    } else {
      S.tf[sl] |= TF_REMOVED;
      atomicAdd(&S.n_removed, 1);
    }
  }
  // ageing of the lost list as it was (a refound track has end_frame == frame)
  for (int sl = nT + tid; sl < nS; sl += NT) {
    if (!(S.tf[sl] & TF_REFOUND) && frame - cur[sl].end_frame > a.max_time_lost) {
      S.tf[sl] |= TF_REMOVED;
      atomicAdd(&S.n_removed, 1);
    }
  }
  __syncthreads();
  // births, refused beyond the capacity
  const int live = nS - S.n_removed;
  const int ncand = ordered_scan(S, nrest, [&](int c) { return !S.eused[S.rest[c]] && S.escore[S.rest[c]] >= a.new_thresh; },
                                 [&](int c, int r) { S.births[r] = S.rest[c]; });
  const int nb = min(ncand, cap - live);
  for (int b = tid; b < nb; b += NT) S.bdrop[b] = 0;
  if constexpr (REID) {
    for (int r = warp; r < nu; r += NW)
      if (S.match[r] >= 0) update_embedding(S.unconf[r], S.rest[S.match[r]]);
    // births take the lowest slots no live record holds (there are cap - live >= nb of them)
    for (int es = tid; es < cap; es += NT) S.sused[es] = 0;
    __syncthreads();
    for (int sl = tid; sl < nS; sl += NT)
      if (!(S.tf[sl] & TF_REMOVED)) S.sused[S.tslot[sl]] = 1;
    __syncthreads();
    ordered_scan(S, cap, [&](int es) { return !S.sused[es]; },
                 [&](int es, int r) { if (r < nb) S.bslot[r] = static_cast<int16_t>(es); });
    for (int b = warp; b < nb; b += NW) {
      const int e = S.births[b], es = S.bslot[b];
      if (S.enorm[e] > 0.0) {
        float* t = temb + static_cast<long long>(es) * a.dim;
        const char* er = S.erow + e * S.ld_bytes;
        for (int i = lane; i < a.dim; i += 32) t[i] = __double2float_rn(ddiv(emb_at(er, a.dtype, i), S.enorm[e]));
      }
      if (lane == 0) has[es] = S.enorm[e] > 0.0;
    }
  }
  // new lists: tracked = still-tracked previous tracked, births, refound; lost = remaining previous lost, new lost
  const int nA = ordered_scan(S, nT, [&](int sl) { return (S.tf[sl] & TF_MATCHED) != 0; },
                              [&](int sl, int r) { S.tlist[r] = static_cast<int16_t>(sl); });
  for (int b = tid; b < nb; b += NT) S.tlist[nA + b] = static_cast<int16_t>(MAXN + b);
  const int nC = ordered_scan(S, nL, [&](int q) { return (S.tf[nT + q] & TF_REFOUND) != 0; },
                              [&](int q, int r) { S.tlist[nA + nb + r] = static_cast<int16_t>(nT + q); });
  const int nD = ordered_scan(S, nL, [&](int q) { return !(S.tf[nT + q] & (TF_REFOUND | TF_REMOVED)); },
                              [&](int q, int r) { S.llist[r] = static_cast<int16_t>(nT + q); });
  const int nE = ordered_scan(S, nT, [&](int sl) { return (S.tf[sl] & TF_NEWLOST) != 0; },
                              [&](int sl, int r) { S.llist[nD + r] = static_cast<int16_t>(sl); });
  const int ntr = nA + nb + nC, nlo = nD + nE;
  // a birth's box and state come from its entry
  const auto birth_state = [&](int b, KState& ks) {
    double z[4];
    measurement(S.ebox[S.births[b]], z);
    initiate(ks, z);
  };
  const auto tracked_box = [&](int x) {
    if (x < MAXN) return S.tbox[x];
    KState ks;
    birth_state(x - MAXN, ks);
    return state_box(ks.p);
  };
  // duplicates: a (tracked, lost) pair closer than duplicate_thresh in IoU distance drops the younger track (the tracked
  // one on a tie)
  const double dup = a.dup_thresh;
  for (int idx = tid; idx < ntr * nlo; idx += NT) {
    const int i = idx / nlo, j = idx - i * nlo;
    const int x = S.tlist[i], y = S.llist[j];
    const int lx = x < MAXN ? S.tlab[x] : S.elab[S.births[x - MAXN]];
    if (a.class_aware && lx != S.tlab[y]) continue;
    if (dsub(1.0, iou_d(tracked_box(x), S.tbox[y])) < dup) {
      const int dx = x < MAXN ? S.tdiff[x] : 0;
      if (dx > S.tdiff[y]) S.tf[y] |= TF_DROP;
      else if (x < MAXN) S.tf[x] |= TF_DROP;
      else S.bdrop[x - MAXN] = 1;
    }
  }
  __syncthreads();
  const auto dropped = [&](int x) { return x < MAXN ? (S.tf[x] & TF_DROP) != 0 : S.bdrop[x - MAXN] != 0; };
  // compaction into the other buffer, and the output (activated tracked tracks; births only on frame 1)
  const int newT = ordered_scan(S, ntr, [&](int i) { return !dropped(S.tlist[i]); }, [&](int i, int r) {
    const int x = S.tlist[i];
    lwdetr_track_record& o = nxt[r];
    if constexpr (REID) slot_nxt[r] = x < MAXN ? S.tslot[x] : S.bslot[x - MAXN];
    if (x < MAXN) {
      o = cur[x];
    } else {
      const int b = x - MAXN, e = S.births[b];
      KState ks;
      birth_state(b, ks);
      store_state(o, ks);
      o.id = next_id + b;
      o.state = LWDETR_TRACK_TRACKED;
      o.activated = frame == 1;
      o.start_frame = frame;
      o.end_frame = frame;
      o.label = S.elab[e];
      o.score = S.escore[e];
      o.index = e;
    }
  });
  const int newL = ordered_scan(S, nlo, [&](int j) { return !dropped(S.llist[j]); }, [&](int j, int r) {
    nxt[newT + r] = cur[S.llist[j]];
    if constexpr (REID) slot_nxt[newT + r] = S.tslot[S.llist[j]];
  });
  const long long ob = row * a.max_out;
  const int nout = ordered_scan(S, ntr, [&](int i) {
    const int x = S.tlist[i];
    return !dropped(x) && (x < MAXN || frame == 1);
  }, [&](int i, int r) {
    if (r >= a.max_out) return;
    const int x = S.tlist[i];
    if (x < MAXN) {
      const int e = S.tdet[x];
      write_output(a, ob + r, cur[x].id, S.escore[e], S.elab[e], narrow(S.tbox[x]), e);
    } else {
      const int b = x - MAXN, e = S.births[b];
      write_output(a, ob + r, next_id + b, S.escore[e], S.elab[e], narrow(tracked_box(x)), e);
    }
  });
  const int cnt = min(nout, a.max_out);
  for (int r = cnt + tid; r < a.max_out; r += NT) write_output(a, ob + r, 0, 0.f, -1, make_float4(0.f, 0.f, 0.f, 0.f), -1);
  if (tid == 0) {
    a.counts[row] = cnt;
    hp->frame = frame + 1;
    hp->next_id = next_id + nb;
    hp->overflow += ncand - nb;
    hp->n_tracked = newT;
    hp->n_lost = newL;
    hp->parity = parity ^ 1;
  }
}

// lwdetr_track_flow: a frame without detections.  Confirmed Tracked tracks take the flow's measurement or go Lost; the rest
// of the frame (predict, warp, ageing, lists, duplicates, output) is track_kernel's, without associations and births.
struct FlowTrackArgs {
  TrackArgs t;
  const int32_t* fstatus;                // [streams][max_tracks]
  const double* fmeas;                   // [streams][max_tracks][8]: z at 3..6
  int max_tracks;
  int16_t* slot;                         // the appearance slots, or null
};

__global__ void __launch_bounds__(NT, 1) track_flow_kernel(const __grid_constant__ FlowTrackArgs fa) {
  pdl_sync();
  extern __shared__ __align__(16) uint8_t sm_track[];
  Smem& S = *reinterpret_cast<Smem*>(sm_track);
  const TrackArgs& a = fa.t;
  const int tid = threadIdx.x;
  const int sid = a.stream[blockIdx.x];
  const long long row = a.row0 + blockIdx.x;
  TrackHead* hp = a.head + sid;
  const int frame = hp->frame, nT = hp->n_tracked, nL = hp->n_lost, parity = hp->parity;
  const int nS = nT + nL, cap = a.capacity;
  lwdetr_track_record* cur = a.rec + (static_cast<long long>(sid) * 2 + parity) * cap;
  lwdetr_track_record* nxt = a.rec + (static_cast<long long>(sid) * 2 + (parity ^ 1)) * cap;
  if (tid == 0) S.n_removed = 0;
  for (int sl = tid; sl < nS; sl += NT) {
    lwdetr_track_record& r = cur[sl];
    const bool lost = sl >= nT, act = r.activated != 0;
    KState ks;
    load_state(r, ks);
    if (lost || act) predict(ks, !lost);
    if (a.motion) warp_state(ks, a.motion + row * 4);
    if (lost || act || a.motion) store_state(r, ks);
    S.tbox[sl] = state_box(ks.p);
    S.tlab[sl] = r.label;
    S.tdiff[sl] = r.end_frame - r.start_frame;
    S.tf[sl] = static_cast<uint8_t>((act ? TF_ACT : 0) | (lost ? TF_LOSTLIST : 0));
  }
  __syncthreads();
  // the flow's track j is the j-th activated record of the tracked list
  ordered_scan(S, nT, [&](int sl) { return (S.tf[sl] & TF_ACT) != 0; }, [&](int sl, int j) { S.tdet[sl] = static_cast<int16_t>(j); });
  const long long fo = static_cast<long long>(sid) * fa.max_tracks;
  for (int sl = tid; sl < nT; sl += NT) {
    if (!(S.tf[sl] & TF_ACT)) {
      S.tf[sl] |= TF_MATCHED;            // unconfirmed: carried
      continue;
    }
    const int j = S.tdet[sl];
    lwdetr_track_record& r = cur[sl];
    if (j < fa.max_tracks && fa.fstatus[fo + j] == LWDETR_FLOW_OK) {
      KState ks;
      load_state(r, ks);
      double z[4];
      for (int q = 0; q < 4; ++q) z[q] = fa.fmeas[(fo + j) * 8 + 3 + q];
      kalman_update(ks, z);
      store_state(r, ks);
      r.end_frame = frame;
      r.index = -1;
      S.tbox[sl] = state_box(ks.p);
      S.tdiff[sl] = frame - r.start_frame;
      S.tf[sl] |= TF_MATCHED;
    } else {
      r.state = LWDETR_TRACK_LOST;
      S.tf[sl] |= TF_NEWLOST;
    }
  }
  for (int sl = nT + tid; sl < nS; sl += NT)
    if (frame - cur[sl].end_frame > a.max_time_lost) S.tf[sl] |= TF_REMOVED;
  __syncthreads();
  const int ntr = ordered_scan(S, nT, [&](int sl) { return (S.tf[sl] & TF_MATCHED) != 0; },
                               [&](int sl, int r) { S.tlist[r] = static_cast<int16_t>(sl); });
  const int nD = ordered_scan(S, nL, [&](int q) { return !(S.tf[nT + q] & TF_REMOVED); },
                              [&](int q, int r) { S.llist[r] = static_cast<int16_t>(nT + q); });
  const int nE = ordered_scan(S, nT, [&](int sl) { return (S.tf[sl] & TF_NEWLOST) != 0; },
                              [&](int sl, int r) { S.llist[nD + r] = static_cast<int16_t>(sl); });
  const int nlo = nD + nE;
  const double dup = a.dup_thresh;
  for (int idx = tid; idx < ntr * nlo; idx += NT) {
    const int i = idx / nlo, j = idx - i * nlo;
    const int x = S.tlist[i], y = S.llist[j];
    if (a.class_aware && S.tlab[x] != S.tlab[y]) continue;
    if (dsub(1.0, iou_d(S.tbox[x], S.tbox[y])) < dup) {
      if (S.tdiff[x] > S.tdiff[y]) S.tf[y] |= TF_DROP;
      else S.tf[x] |= TF_DROP;
    }
  }
  __syncthreads();
  int16_t* slot_cur = fa.slot ? fa.slot + (static_cast<long long>(sid) * 2 + parity) * cap : nullptr;
  int16_t* slot_nxt = fa.slot ? fa.slot + (static_cast<long long>(sid) * 2 + (parity ^ 1)) * cap : nullptr;
  const int newT = ordered_scan(S, ntr, [&](int i) { return !(S.tf[S.tlist[i]] & TF_DROP); }, [&](int i, int r) {
    nxt[r] = cur[S.tlist[i]];
    if (slot_nxt) slot_nxt[r] = slot_cur[S.tlist[i]];
  });
  const int newL = ordered_scan(S, nlo, [&](int j) { return !(S.tf[S.llist[j]] & TF_DROP); }, [&](int j, int r) {
    nxt[newT + r] = cur[S.llist[j]];
    if (slot_nxt) slot_nxt[newT + r] = slot_cur[S.llist[j]];
  });
  const long long ob = row * a.max_out;
  const int nout = ordered_scan(S, ntr, [&](int i) {
    const int x = S.tlist[i];
    return !(S.tf[x] & TF_DROP) && (S.tf[x] & TF_ACT);
  }, [&](int i, int r) {
    if (r >= a.max_out) return;
    const lwdetr_track_record& t = cur[S.tlist[i]];
    write_output(a, ob + r, t.id, t.score, t.label, narrow(S.tbox[S.tlist[i]]), -1);
  });
  const int cnt = min(nout, a.max_out);
  for (int r = cnt + tid; r < a.max_out; r += NT) write_output(a, ob + r, 0, 0.f, -1, make_float4(0.f, 0.f, 0.f, 0.f), -1);
  if (tid == 0) {
    a.counts[row] = cnt;
    hp->frame = frame + 1;
    hp->n_tracked = newT;
    hp->n_lost = newL;
    hp->parity = parity ^ 1;
  }
}

struct ResetArgs {
  TrackHead* head;
  int n;
  int stream[LAUNCH_STREAMS];
};

__global__ void track_reset_kernel(const __grid_constant__ ResetArgs a) {
  pdl_sync();
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
    TrackHead h = {};
    h.frame = 1;
    h.next_id = 1;
    a.head[a.stream[i]] = h;
  }
}

// lwdetr_query_best: one thread per query, the classes scanned in order (ties to the lower class)
__global__ void query_best_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const float* __restrict__ target_sizes,
                                  int B, int nq, int ncls, float* __restrict__ scores, int32_t* __restrict__ labels,
                                  float* __restrict__ out_boxes) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(B) * nq) return;
  const int b = static_cast<int>(i / nq);
  const float* lg = logits + i * ncls;
  float best = sigmoid_f32(lg[0]);
  int lab = 0;
  for (int c = 1; c < ncls; ++c) {
    const float s = sigmoid_f32(lg[c]);
    if (s > best) {
      best = s;
      lab = c;
    }
  }
  const float4 bx = *reinterpret_cast<const float4*>(boxes + i * 4);
  scores[i] = best;
  labels[i] = lab;
  *reinterpret_cast<float4*>(out_boxes + i * 4) = box_cxcywh_to_xyxy(bx, target_sizes[2 * b], target_sizes[2 * b + 1]);
}

}  // namespace

int track_launch(const TrackTable& t, const lwdetr_track_params& p, const float* scores, const int32_t* labels, const float* boxes,
                 const double* motion, int B, int k, const int32_t* streams, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels,
                 float* out_boxes, int32_t* out_index, int32_t* counts, cudaStream_t st, const ReidInput* reid) {
  if (B < 1 || k < 1 || k > TRACK_MAX || max_out < 1) return -2;
  const int smem = static_cast<int>(reid ? sizeof(SmemReid) : sizeof(Smem));
  const void* kern = reid ? reinterpret_cast<const void*>(track_kernel<ReidArgs>) : reinterpret_cast<const void*>(track_kernel<TrackArgs>);
  if (int e = ensure_max_dyn_smem(kern, smem)) return e;
  std::vector<ReidArgs> hold(1);         // ~4 KB of parameters: kept off the stack
  TrackArgs& a = hold[0];
  a.scores = scores;
  a.labels = labels;
  a.boxes = reinterpret_cast<const float4*>(boxes);
  a.out_ids = out_ids;
  a.out_scores = out_scores;
  a.out_labels = out_labels;
  a.out_boxes = reinterpret_cast<float4*>(out_boxes);
  a.out_index = out_index;
  a.counts = counts;
  a.head = t.head;
  a.rec = t.rec;
  a.motion = motion;
  a.track_thresh = p.track_thresh;
  a.low_thresh = p.low_thresh;
  a.new_thresh = p.new_track_thresh;
  a.match_thresh = p.match_thresh;
  a.second_thresh = p.second_thresh;
  a.unconf_thresh = p.unconfirmed_thresh;
  a.dup_thresh = p.duplicate_thresh;
  a.k = k;
  a.max_out = max_out;
  a.capacity = t.capacity;
  a.max_time_lost = static_cast<int>(p.frame_rate / 30.0 * p.track_buffer);
  a.fuse = p.fuse_score;
  a.class_aware = p.class_aware;
  ReidArgs& r = hold[0];
  if (reid) {
    const ReidTable& rt = *reid->table;
    r.emb = reid->emb;
    r.ld_emb = reid->ld;
    r.dtype = reid->dtype;
    r.dim = rt.params.embedding_dim;
    r.prox = rt.params.proximity_thresh;
    r.app = rt.params.appearance_thresh;
    r.alpha = rt.params.ema_alpha;
    r.slot = rt.slot;
    r.has = rt.has;
    r.temb = rt.emb;
    r.pkey = rt.pkey;
    r.pval = rt.pval;
  }
  for (int b0 = 0; b0 < B; b0 += LAUNCH_STREAMS) {
    const int nb = B - b0 < LAUNCH_STREAMS ? B - b0 : LAUNCH_STREAMS;
    a.row0 = b0;
    for (int i = 0; i < nb; ++i) a.stream[i] = streams[b0 + i];
    if (reid) launch_k(track_kernel<ReidArgs>, dim3(nb), dim3(NT), static_cast<size_t>(smem), st, r);
    else launch_k(track_kernel<TrackArgs>, dim3(nb), dim3(NT), static_cast<size_t>(smem), st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

int track_flow_launch(const TrackTable& t, const lwdetr_track_params& p, const FlowTable& f, const double* motion, int16_t* slot, int B,
                      const int32_t* streams, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes,
                      int32_t* out_index, int32_t* counts, cudaStream_t st) {
  const int smem = static_cast<int>(sizeof(Smem));
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(track_flow_kernel), smem)) return e;
  std::vector<FlowTrackArgs> hold(1);
  FlowTrackArgs& fa = hold[0];
  TrackArgs& a = fa.t;
  a.out_ids = out_ids;
  a.out_scores = out_scores;
  a.out_labels = out_labels;
  a.out_boxes = reinterpret_cast<float4*>(out_boxes);
  a.out_index = out_index;
  a.counts = counts;
  a.head = t.head;
  a.rec = t.rec;
  a.motion = motion;
  a.dup_thresh = p.duplicate_thresh;
  a.max_out = max_out;
  a.capacity = t.capacity;
  a.max_time_lost = static_cast<int>(p.frame_rate / 30.0 * p.track_buffer);
  a.class_aware = p.class_aware;
  fa.fstatus = f.status;
  fa.fmeas = f.meas;
  fa.max_tracks = f.p.max_tracks;
  fa.slot = slot;
  for (int b0 = 0; b0 < B; b0 += LAUNCH_STREAMS) {
    const int nb = B - b0 < LAUNCH_STREAMS ? B - b0 : LAUNCH_STREAMS;
    a.row0 = b0;
    for (int i = 0; i < nb; ++i) a.stream[i] = streams[b0 + i];
    launch_k(track_flow_kernel, dim3(nb), dim3(NT), static_cast<size_t>(smem), st, fa);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

int track_reset_launch(const TrackTable& t, const int32_t* streams, int n, cudaStream_t st) {
  std::vector<ResetArgs> hold(1);
  ResetArgs& a = hold[0];
  a.head = t.head;
  for (int i0 = 0; i0 < n; i0 += LAUNCH_STREAMS) {
    a.n = n - i0 < LAUNCH_STREAMS ? n - i0 : LAUNCH_STREAMS;
    for (int i = 0; i < a.n; ++i) a.stream[i] = streams[i0 + i];
    launch_k(track_reset_kernel, dim3(1), dim3(256), 0, st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

int query_best_launch(const float* logits, const float* boxes, const float* target_sizes, int B, int nq, int ncls, float* scores,
                      int32_t* labels, float* out_boxes, cudaStream_t st) {
  const long long n = static_cast<long long>(B) * nq;
  launch_k(query_best_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st, logits, boxes, target_sizes, B, nq, ncls,
           scores, labels, out_boxes);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace lwb
