// lwdetr_zones_update: line crossings and zone occupancy per camera stream on the device, bit for bit the contract stated in
// include/lwdetr_b200.h and restated in tools/zone_spec.py.  One CTA per stream in the call.  A stream's records sit in
// fixed slots; an index of (id, slot, last_seen) sorted by id is staged in shared memory with the stream's geometry, so
// the lookup of a present id is a binary search there.  Per frame:
//   1. the frame's entries are keyed (id, entry) and bitonic-sorted: the first entry of each id is present, a repeat is
//      ignored; present ids are looked up in the index, and new ones take free slots (lowest first) in input order;
//   2. the side and point-in-polygon tests run over all (present track, line or polygon) pairs in parallel, in float64
//      with each operation rounded on its own (__dadd_rn / __dmul_rn / __ddiv_rn);
//   3. each present track counts its events, a block-wide scan gives each its offset in the frame's fixed event order,
//      and each writes its events and its record; the forgotten records follow in ascending id, through a second scan;
//   4. the index is rebuilt by a merge of the surviving records and the new ones (both sorted by id), written in place.
#include "zones.h"

#include <vector>

#include "launch.h"
#include "lwdetr_b200.h"

namespace lwb {
namespace {

constexpr int NT = 512;                  // threads per CTA
constexpr int NW = NT / 32;
constexpr int MAXE = ZONE_MAX_OUT;       // entries per frame
constexpr int MAXR = ZONE_CAPACITY;      // records per stream
constexpr int LAUNCH_STREAMS = 1024;     // CTAs per launch (the stream table travels in the parameters)
constexpr unsigned long long NOKEY = ~0ull;

struct ZoneArgs {
  const int32_t* ids;
  const int32_t* labels;
  const float4* boxes;
  const int32_t* counts;
  uint32_t* inside;
  int32_t* occupancy;
  int32_t* events;
  int32_t* event_counts;
  ZoneHead* head;
  const ZoneGeom* geom;
  const double2* verts;
  ZoneIndex* index;
  ZoneRec* rec;
  int32_t* line_counts;
  int32_t* entries;
  int max_out, max_events, capacity, num_classes, forget_after, zone_anchor, line_anchors, row0;
  int stream[LAUNCH_STREAMS];            // stream of CTA i: batch row row0 + i
};

struct Smem {
  double line[ZONE_LINES][4];
  double2 vert[ZONE_VERTS];
  ZoneIndex idx[MAXR];                   // the stream's index; last_seen of present records set to the frame
  int rscan[MAXR];                       // per record: forget events, then survivors (exclusive scans)
  unsigned long long key[MAXE];          // (id << 32) | entry, sorted
  float4 box[MAXE];                      // by entry
  int eid[MAXE], elab[MAXE];
  int jscan[MAXE];                       // by entry: position among the present entries (exclusive scan)
  int jpos[MAXE], jslot[MAXE];           // by entry: index position (-1: no record before this frame), slot (-1: none)
  int plist[MAXE];                       // present entries in input order
  int pnew[MAXE];                        // by present position: rank among the new ids
  int pscan[MAXE];                       // by present position: event offset
  uint32_t dset[MAXE], dpos[MAXE], pmask[MAXE];   // by present position: decided lines, +1 lines, zones inside
  int sscan[MAXE];                       // by sorted position: rank among the new records
  int newj[MAXE];                        // new records by ascending id: their entry
  uint32_t used[MAXR / 32];              // slot bitmap
  int freepref[MAXR / 32 + 1];
  int start[ZONE_POLYS + 1];
  int occ[ZONE_POLYS];
  int wsum[NW];
  int total;
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// exclusive prefix sums of a[0, n) in place; every thread gets the total
__device__ int block_scan(int* a, int n, Smem& s) {
  __syncthreads();
  const int per = (n + NT - 1) / NT;
  const int lo = min(n, static_cast<int>(threadIdx.x) * per), hi = min(n, lo + per);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += a[i];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int inc = sum;
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(~0u, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) s.wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    const int v = lane < NW ? s.wsum[lane] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(~0u, x, o);
      if (lane >= o) x += u;
    }
    if (lane < NW) s.wsum[lane] = x - v;
    if (lane == 31) s.total = x;
  }
  __syncthreads();
  int run = s.wsum[w] + inc - sum;
  for (int i = lo; i < hi; ++i) {
    const int v = a[i];
    a[i] = run;
    run += v;
  }
  const int total = s.total;
  __syncthreads();
  return total;
}

// anchor 3 * row + column of an fp32 xyxy box, widened
__device__ __forceinline__ void anchor(const float4 b, int which, double& x, double& y) {
  const int row = which / 3, col = which % 3;
  x = col == 0 ? static_cast<double>(b.x) : col == 1 ? dmul(dadd(b.x, b.z), 0.5) : static_cast<double>(b.z);
  y = row == 0 ? static_cast<double>(b.y) : row == 1 ? dmul(dadd(b.y, b.w), 0.5) : static_cast<double>(b.w);
}

__device__ int line_side(const double* ln, const float4 b, int mask) {
  const double ax = ln[0], ay = ln[1], dx = dsub(ln[2], ax), dy = dsub(ln[3], ay);
  const double L2 = dadd(dmul(dx, dx), dmul(dy, dy));
  bool pos = true, neg = true;
  for (int w = 0; w < 9; ++w) {
    if (!(mask >> w & 1)) continue;
    double px, py;
    anchor(b, w, px, py);
    const double ux = dsub(px, ax), uy = dsub(py, ay);
    const double t = dadd(dmul(ux, dx), dmul(uy, dy));
    const double c = dsub(dmul(dx, uy), dmul(dy, ux));
    const bool within = t >= 0.0 && t <= L2;
    pos = pos && within && c > 0.0;
    neg = neg && within && c < 0.0;
  }
  return pos ? 1 : neg ? -1 : 0;
}

__device__ bool in_polygon(const double2* v, int n, double px, double py) {
  bool in = false;
  for (int i = 0; i < n; ++i) {
    const double2 p = v[i], q = v[i == 0 ? n - 1 : i - 1];
    if ((p.y > py) != (q.y > py) && px < dadd(ddiv(dmul(dsub(q.x, p.x), dsub(py, p.y)), dsub(q.y, p.y)), p.x)) in = !in;
  }
  return in;
}

__device__ __forceinline__ int index_lower_bound(const ZoneIndex* idx, int n, int id) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (idx[m].id < id) lo = m + 1;
    else hi = m;
  }
  return lo;
}

__device__ __forceinline__ void put_event(const ZoneArgs& a, int row, int e, int id, int kind, int index, int label, int dwell) {
  if (e >= a.max_events) return;
  int32_t* o = a.events + (static_cast<long long>(row) * a.max_events + e) * 5;
  o[0] = id;
  o[1] = kind;
  o[2] = index;
  o[3] = label;
  o[4] = dwell;
}

__global__ void __launch_bounds__(NT, 1) zones_kernel(const __grid_constant__ ZoneArgs a) {
  pdl_sync();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x;
  const int row = a.row0 + blockIdx.x, sid = a.stream[blockIdx.x];
  const ZoneHead h = a.head[sid];
  const ZoneGeom* g = a.geom + sid;
  const int nl = g->n_lines, nz = g->n_polys, frame = h.frame, n_old = h.n, C = a.capacity, ncls = a.num_classes;
  ZoneIndex* gidx = a.index + static_cast<long long>(sid) * C;
  ZoneRec* grec = a.rec + static_cast<long long>(sid) * C;
  const int cnt = min(max(a.counts[row], 0), a.max_out);
  const long long ent0 = static_cast<long long>(row) * a.max_out;

  // 1. stage the geometry, the index and the entries
  for (int i = tid; i < nl * 4; i += NT) s.line[i >> 2][i & 3] = g->line[i >> 2][i & 3];
  if (tid <= nz) s.start[tid] = g->start[tid];
  if (tid < ZONE_POLYS) s.occ[tid] = 0;
  const int nv = g->start[nz];
  for (int i = tid; i < nv; i += NT) s.vert[i] = a.verts[static_cast<long long>(sid) * ZONE_VERTS + i];
  for (int i = tid; i < n_old; i += NT) s.idx[i] = gidx[i];
  const int words = (C + 31) / 32;
  for (int w = tid; w < words; w += NT) s.used[w] = C - w * 32 >= 32 ? 0u : ~0u << (C - w * 32);
  int np2 = 1;
  while (np2 < cnt) np2 <<= 1;
  for (int j = tid; j < np2; j += NT) {
    unsigned long long k = NOKEY;
    if (j < cnt) {
      const int id = a.ids[ent0 + j];
      const float4 b = a.boxes[ent0 + j];
      s.eid[j] = id;
      s.elab[j] = a.labels[ent0 + j];
      s.box[j] = b;
      s.jscan[j] = 0;
      if (id > 0 && isfinite(b.x) && isfinite(b.y) && isfinite(b.z) && isfinite(b.w))
        k = static_cast<unsigned long long>(static_cast<uint32_t>(id)) << 32 | static_cast<uint32_t>(j);
    }
    s.key[j] = k;
  }
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < np2; i += NT) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long x = s.key[i], y = s.key[l];
          if ((x > y) == ((i & k) == 0)) {
            s.key[i] = y;
            s.key[l] = x;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int p = tid; p < cnt; p += NT) {       // the first entry of each id is present
    const unsigned long long k = s.key[p];
    if (k != NOKEY && (p == 0 || s.key[p - 1] >> 32 != k >> 32)) s.jscan[static_cast<uint32_t>(k)] = 1;
  }
  const int P = block_scan(s.jscan, cnt, s);
  auto present = [&](int j) { return (j + 1 < cnt ? s.jscan[j + 1] : P) != s.jscan[j]; };
  for (int j = tid; j < cnt; j += NT)
    if (present(j)) s.plist[s.jscan[j]] = j;
  for (int i = tid; i < n_old; i += NT) atomicOr(&s.used[s.idx[i].slot >> 5], 1u << (s.idx[i].slot & 31));
  __syncthreads();
  for (int p = tid; p < P; p += NT) {
    const int j = s.plist[p], id = s.eid[j];
    const int lb = index_lower_bound(s.idx, n_old, id);
    const bool found = lb < n_old && s.idx[lb].id == id;
    s.jpos[j] = found ? lb : -1;
    s.jslot[j] = found ? s.idx[lb].slot : -1;
    if (found) s.idx[lb].last_seen = frame;
    s.pnew[p] = found ? 0 : 1;
    s.dset[p] = s.dpos[p] = s.pmask[p] = 0;
  }
  if (tid == 0) {
    int acc = 0;
    for (int w = 0; w < words; ++w) {
      s.freepref[w] = acc;
      acc += __popc(~s.used[w]);
    }
    s.freepref[words] = acc;
  }
  const int nnew = block_scan(s.pnew, P, s);
  const int nfree = C - n_old, taken = min(nnew, nfree);
  for (int p = tid; p < P; p += NT) {          // the r-th new id takes the r-th free slot, while there is one
    const int j = s.plist[p], r = s.pnew[p];
    if (s.jpos[j] >= 0 || r >= nfree) continue;
    int lo = 0, hi = words - 1;                 // the last word w with freepref[w] <= r
    while (lo < hi) {
      const int m = (lo + hi + 1) >> 1;
      if (s.freepref[m] <= r) lo = m;
      else hi = m - 1;
    }
    s.jslot[j] = lo * 32 + static_cast<int>(__fns(~s.used[lo], 0, r - s.freepref[lo] + 1));
  }

  // 2. side and point-in-polygon tests over (present track, line or polygon) pairs
  const int K = nl + nz;
  for (int q = tid; q < P * K; q += NT) {
    const int p = q / K, k = q - p * K;
    const float4 b = s.box[s.plist[p]];
    if (k < nl) {
      const int d = line_side(s.line[k], b, a.line_anchors);
      if (d != 0) atomicOr(&s.dset[p], 1u << k);
      if (d > 0) atomicOr(&s.dpos[p], 1u << k);
    } else {
      const int z = k - nl;
      double px, py;
      anchor(b, a.zone_anchor, px, py);
      if (in_polygon(s.vert + s.start[z], s.start[z + 1] - s.start[z], px, py)) atomicOr(&s.pmask[p], 1u << z);
    }
  }
  __syncthreads();

  // 3. events: counts, offsets, then the events and the records
  for (int p = tid; p < P; p += NT) {
    const int j = s.plist[p], slot = s.jslot[j];
    const uint32_t m = s.pmask[p];
    for (uint32_t x = m; x; x &= x - 1) atomicAdd(&s.occ[__ffs(x) - 1], 1);
    int ev = 0;
    if (slot >= 0) {
      uint32_t ins = 0, ss = 0, sp = 0;
      if (s.jpos[j] >= 0) {
        ins = grec[slot].inside;
        ss = grec[slot].side_set;
        sp = grec[slot].side_pos;
      }
      ev = __popc(s.dset[p] & ss & (s.dpos[p] ^ sp)) + __popc(m ^ ins);
    }
    s.pscan[p] = ev;
  }
  for (int i = tid; i < n_old; i += NT) {
    const ZoneIndex e = s.idx[i];
    s.rscan[i] = frame - e.last_seen > a.forget_after ? __popc(grec[e.slot].inside) : 0;
  }
  const int E1 = block_scan(s.pscan, P, s);
  const int E2 = block_scan(s.rscan, n_old, s);
  const int ncol = ncls + 1;
  for (int p = tid; p < P; p += NT) {
    const int j = s.plist[p], slot = s.jslot[j];
    if (slot < 0) continue;
    const int id = s.eid[j], lab = s.elab[j], col = lab >= 0 && lab < ncls ? lab : ncls;
    ZoneRec* r = grec + slot;
    uint32_t ins = 0, ss = 0, sp = 0;
    if (s.jpos[j] >= 0) {
      ins = r->inside;
      ss = r->side_set;
      sp = r->side_pos;
    } else {
      for (int z = 0; z < ZONE_POLYS; ++z) r->entry[z] = 0;
    }
    int e = s.pscan[p];
    const uint32_t ds = s.dset[p], dp = s.dpos[p], m = s.pmask[p];
    for (uint32_t x = ds & ss & (dp ^ sp); x; x &= x - 1) {
      const int l = __ffs(x) - 1;
      const bool in = dp >> l & 1;
      put_event(a, row, e++, id, in ? LWDETR_ZONE_LINE_IN : LWDETR_ZONE_LINE_OUT, l, lab, 0);
      atomicAdd(a.line_counts + ((static_cast<long long>(sid) * ZONE_LINES + l) * ncol + col) * 2 + (in ? 0 : 1), 1);
    }
    for (uint32_t x = m ^ ins; x; x &= x - 1) {
      const int z = __ffs(x) - 1;
      if (m >> z & 1) {
        r->entry[z] = frame;
        put_event(a, row, e++, id, LWDETR_ZONE_ENTER, z, lab, 0);
        atomicAdd(a.entries + (static_cast<long long>(sid) * ZONE_POLYS + z) * ncol + col, 1);
      } else {
        put_event(a, row, e++, id, LWDETR_ZONE_EXIT, z, lab, frame - r->entry[z]);
        r->entry[z] = 0;
      }
    }
    r->inside = m;
    r->side_set = ss | ds;
    r->side_pos = (sp & ~ds) | (dp & ds);
    r->label = lab;
  }
  for (int i = tid; i < n_old; i += NT) {       // forgotten records: none of them is present
    const ZoneIndex x = s.idx[i];
    if (frame - x.last_seen <= a.forget_after) continue;
    const ZoneRec* r = grec + x.slot;
    const int lab = r->label;
    int e = E1 + s.rscan[i];
    for (uint32_t y = r->inside; y; y &= y - 1) {
      const int z = __ffs(y) - 1;
      put_event(a, row, e++, x.id, LWDETR_ZONE_FORGET, z, lab, x.last_seen - r->entry[z]);
    }
  }

  // 4. the new index: the survivors and the new records merged by id
  __syncthreads();
  for (int i = tid; i < n_old; i += NT) s.rscan[i] = frame - s.idx[i].last_seen <= a.forget_after ? 1 : 0;
  for (int p = tid; p < cnt; p += NT) {
    const unsigned long long k = s.key[p];
    const int j = static_cast<int>(static_cast<uint32_t>(k));
    s.sscan[p] = k != NOKEY && present(j) && s.jpos[j] < 0 && s.jslot[j] >= 0 ? 1 : 0;
  }
  const int S = block_scan(s.rscan, n_old, s);
  const int A = block_scan(s.sscan, cnt, s);
  for (int p = tid; p < cnt; p += NT) {
    const unsigned long long k = s.key[p];
    const int j = static_cast<int>(static_cast<uint32_t>(k));
    if (k != NOKEY && present(j) && s.jpos[j] < 0 && s.jslot[j] >= 0) s.newj[s.sscan[p]] = j;
  }
  __syncthreads();
  for (int i = tid; i < n_old; i += NT) {
    const ZoneIndex x = s.idx[i];
    if (frame - x.last_seen > a.forget_after) continue;
    int lo = 0, hi = A;                         // new ids below x.id
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (s.eid[s.newj[m]] < x.id) lo = m + 1;
      else hi = m;
    }
    gidx[s.rscan[i] + lo] = x;
  }
  for (int r = tid; r < A; r += NT) {
    const int j = s.newj[r], id = s.eid[j];
    const int lb = index_lower_bound(s.idx, n_old, id);
    gidx[r + (lb < n_old ? s.rscan[lb] : S)] = ZoneIndex{id, s.jslot[j], frame};
  }

  // outputs
  uint32_t* ins_out = a.inside + ent0;
  for (int j = tid; j < a.max_out; j += NT) ins_out[j] = j < cnt && present(j) ? s.pmask[s.jscan[j]] : 0u;
  if (tid < ZONE_POLYS) a.occupancy[row * ZONE_POLYS + tid] = s.occ[tid];
  for (long long e = E1 + E2 + tid; e < a.max_events; e += NT)
    for (int c = 0; c < 5; ++c) a.events[(static_cast<long long>(row) * a.max_events + e) * 5 + c] = 0;
  if (tid == 0) {
    a.event_counts[row] = E1 + E2;
    a.head[sid] = ZoneHead{frame + 1, S + A, h.overflow + nnew - taken, 0};
  }
}

struct ZoneResetArgs {
  ZoneHead* head;
  int32_t* line_counts;
  int32_t* entries;
  int ncol, n;
  int stream[LAUNCH_STREAMS];
};

__global__ void zones_reset_kernel(const __grid_constant__ ZoneResetArgs a) {
  pdl_sync();
  const long long sid = a.stream[blockIdx.x];
  const int nlc = ZONE_LINES * a.ncol * 2, nen = ZONE_POLYS * a.ncol;
  for (int i = threadIdx.x; i < nlc; i += blockDim.x) a.line_counts[sid * nlc + i] = 0;
  for (int i = threadIdx.x; i < nen; i += blockDim.x) a.entries[sid * nen + i] = 0;
  if (threadIdx.x == 0) a.head[sid] = ZoneHead{1, 0, 0, 0};
}

}  // namespace

int zones_launch(const ZoneTable& t, const int32_t* ids, const int32_t* labels, const float* boxes, const int32_t* counts, int B, int max_out,
                 const int32_t* streams, uint32_t* inside, int32_t* occupancy, int32_t* events, int max_events, int32_t* event_counts,
                 cudaStream_t st) {
  constexpr int smem = static_cast<int>(sizeof(Smem));
  if (int e = ensure_max_dyn_smem(reinterpret_cast<const void*>(zones_kernel), smem)) return e;
  std::vector<ZoneArgs> hold(1);         // ~4 KB of parameters: kept off the stack
  ZoneArgs& a = hold[0];
  a.ids = ids;
  a.labels = labels;
  a.boxes = reinterpret_cast<const float4*>(boxes);
  a.counts = counts;
  a.inside = inside;
  a.occupancy = occupancy;
  a.events = events;
  a.event_counts = event_counts;
  a.head = t.head;
  a.geom = t.geom;
  a.verts = t.verts;
  a.index = t.index;
  a.rec = t.rec;
  a.line_counts = t.line_counts;
  a.entries = t.entries;
  a.max_out = max_out;
  a.max_events = max_events;
  a.capacity = t.capacity;
  a.num_classes = t.num_classes;
  a.forget_after = t.forget_after;
  a.zone_anchor = t.zone_anchor;
  a.line_anchors = t.line_anchors;
  for (int b0 = 0; b0 < B; b0 += LAUNCH_STREAMS) {
    const int nb = B - b0 < LAUNCH_STREAMS ? B - b0 : LAUNCH_STREAMS;
    a.row0 = b0;
    for (int i = 0; i < nb; ++i) a.stream[i] = streams[b0 + i];
    launch_k(zones_kernel, dim3(nb), dim3(NT), static_cast<size_t>(smem), st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

int zones_reset_launch(const ZoneTable& t, const int32_t* streams, int n, cudaStream_t st) {
  std::vector<ZoneResetArgs> hold(1);
  ZoneResetArgs& a = hold[0];
  a.head = t.head;
  a.line_counts = t.line_counts;
  a.entries = t.entries;
  a.ncol = t.num_classes + 1;
  for (int i0 = 0; i0 < n; i0 += LAUNCH_STREAMS) {
    a.n = n - i0 < LAUNCH_STREAMS ? n - i0 : LAUNCH_STREAMS;
    for (int i = 0; i < a.n; ++i) a.stream[i] = streams[i0 + i];
    launch_k(zones_reset_kernel, dim3(a.n), dim3(256), 0, st, a);
    if (cudaError_t e = cudaGetLastError()) return static_cast<int>(e);
  }
  return 0;
}

}  // namespace lwb
