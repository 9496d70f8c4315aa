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
// Steps 1 and 4 are the record lifecycle of lifecycle.cuh, which lwdetr_speed_update shares.
#include "zones.h"

#include <vector>

#include "launch.h"
#include "lifecycle.cuh"
#include "lwdetr_b200.h"

namespace lwb {
namespace {

constexpr int NT = LC_NT;                // threads per CTA
constexpr int MAXE = ZONE_MAX_OUT;       // entries per frame
constexpr int LAUNCH_STREAMS = 1024;     // CTAs per launch (the stream table travels in the parameters)
static_assert(MAXE <= LC_MAXE && ZONE_CAPACITY <= LC_MAXR, "lifecycle limits");

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
  Lifecycle lc;                          // index, keys, presence, slots (lifecycle.cuh); lc.rscan: forget events first
  double line[ZONE_LINES][4];
  double2 vert[ZONE_VERTS];
  float4 box[MAXE];                      // by entry
  int elab[MAXE];
  int pscan[MAXE];                       // by present position: event offset
  uint32_t dset[MAXE], dpos[MAXE], pmask[MAXE];   // by present position: decided lines, +1 lines, zones inside
  int start[ZONE_POLYS + 1];
  int occ[ZONE_POLYS];
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

__device__ int line_side(const double* ln, const float4 b, int mask) {
  const double ax = ln[0], ay = ln[1], dx = dsub(ln[2], ax), dy = dsub(ln[3], ay);
  const double L2 = dadd(dmul(dx, dx), dmul(dy, dy));
  bool pos = true, neg = true;
  for (int w = 0; w < 9; ++w) {
    if (!(mask >> w & 1)) continue;
    double px, py;
    box_anchor(b, w, px, py);
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
  Lifecycle& lc = s.lc;
  const int tid = threadIdx.x;
  const int row = a.row0 + blockIdx.x, sid = a.stream[blockIdx.x];
  const ZoneHead h = a.head[sid];
  const ZoneGeom* g = a.geom + sid;
  const int nl = g->n_lines, nz = g->n_polys, frame = h.frame, n_old = h.n, C = a.capacity, ncls = a.num_classes;
  ZoneIndex* gidx = a.index + static_cast<long long>(sid) * C;
  ZoneRec* grec = a.rec + static_cast<long long>(sid) * C;
  const int cnt = min(max(a.counts[row], 0), a.max_out);
  const long long ent0 = static_cast<long long>(row) * a.max_out;

  // 1. stage the geometry, the index and the entries; the lifecycle up to the slots of the new ids
  for (int i = tid; i < nl * 4; i += NT) s.line[i >> 2][i & 3] = g->line[i >> 2][i & 3];
  if (tid <= nz) s.start[tid] = g->start[tid];
  if (tid < ZONE_POLYS) s.occ[tid] = 0;
  const int nv = g->start[nz];
  for (int i = tid; i < nv; i += NT) s.vert[i] = a.verts[static_cast<long long>(sid) * ZONE_VERTS + i];
  const int np2 = lc_stage(lc, gidx, n_old, C, cnt, [&](int j, int& id) {
    id = a.ids[ent0 + j];
    const float4 b = a.boxes[ent0 + j];
    s.elab[j] = a.labels[ent0 + j];
    s.box[j] = b;
    return id > 0 && isfinite(b.x) && isfinite(b.y) && isfinite(b.z) && isfinite(b.w);
  });
  lc_sort(lc, np2);
  const int P = lc_present(lc, cnt, n_old);
  for (int p = tid; p < P; p += NT) s.dset[p] = s.dpos[p] = s.pmask[p] = 0;
  const int nnew = lc_assign(lc, P, n_old, C, frame);
  const int taken = min(nnew, C - n_old);

  // 2. side and point-in-polygon tests over (present track, line or polygon) pairs
  const int K = nl + nz;
  for (int q = tid; q < P * K; q += NT) {
    const int p = q / K, k = q - p * K;
    const float4 b = s.box[lc.plist[p]];
    if (k < nl) {
      const int d = line_side(s.line[k], b, a.line_anchors);
      if (d != 0) atomicOr(&s.dset[p], 1u << k);
      if (d > 0) atomicOr(&s.dpos[p], 1u << k);
    } else {
      const int z = k - nl;
      double px, py;
      box_anchor(b, a.zone_anchor, px, py);
      if (in_polygon(s.vert + s.start[z], s.start[z + 1] - s.start[z], px, py)) atomicOr(&s.pmask[p], 1u << z);
    }
  }
  __syncthreads();

  // 3. events: counts, offsets, then the events and the records
  for (int p = tid; p < P; p += NT) {
    const int j = lc.plist[p], slot = lc.jslot[j];
    const uint32_t m = s.pmask[p];
    for (uint32_t x = m; x; x &= x - 1) atomicAdd(&s.occ[__ffs(x) - 1], 1);
    int ev = 0;
    if (slot >= 0) {
      uint32_t ins = 0, ss = 0, sp = 0;
      if (lc.jpos[j] >= 0) {
        ins = grec[slot].inside;
        ss = grec[slot].side_set;
        sp = grec[slot].side_pos;
      }
      ev = __popc(s.dset[p] & ss & (s.dpos[p] ^ sp)) + __popc(m ^ ins);
    }
    s.pscan[p] = ev;
  }
  for (int i = tid; i < n_old; i += NT) {
    const ZoneIndex e = lc.idx[i];
    lc.rscan[i] = frame - e.last_seen > a.forget_after ? __popc(grec[e.slot].inside) : 0;
  }
  const int E1 = block_scan(s.pscan, P, lc);
  const int E2 = block_scan(lc.rscan, n_old, lc);
  const int ncol = ncls + 1;
  for (int p = tid; p < P; p += NT) {
    const int j = lc.plist[p], slot = lc.jslot[j];
    if (slot < 0) continue;
    const int id = lc.eid[j], lab = s.elab[j], col = lab >= 0 && lab < ncls ? lab : ncls;
    ZoneRec* r = grec + slot;
    uint32_t ins = 0, ss = 0, sp = 0;
    if (lc.jpos[j] >= 0) {
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
    const ZoneIndex x = lc.idx[i];
    if (frame - x.last_seen <= a.forget_after) continue;
    const ZoneRec* r = grec + x.slot;
    const int lab = r->label;
    int e = E1 + lc.rscan[i];
    for (uint32_t y = r->inside; y; y &= y - 1) {
      const int z = __ffs(y) - 1;
      put_event(a, row, e++, x.id, LWDETR_ZONE_FORGET, z, lab, x.last_seen - r->entry[z]);
    }
  }

  // 4. the new index: the survivors and the new records merged by id
  const int n_new = lc_merge(lc, gidx, n_old, cnt, P, frame, a.forget_after);

  // outputs
  uint32_t* ins_out = a.inside + ent0;
  for (int j = tid; j < a.max_out; j += NT) ins_out[j] = j < cnt && lc_is_present(lc, j, cnt, P) ? s.pmask[lc.jscan[j]] : 0u;
  if (tid < ZONE_POLYS) a.occupancy[row * ZONE_POLYS + tid] = s.occ[tid];
  for (long long e = E1 + E2 + tid; e < a.max_events; e += NT)
    for (int c = 0; c < 5; ++c) a.events[(static_cast<long long>(row) * a.max_events + e) * 5 + c] = 0;
  if (tid == 0) {
    a.event_counts[row] = E1 + E2;
    a.head[sid] = ZoneHead{frame + 1, n_new, h.overflow + nnew - taken, 0};
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
