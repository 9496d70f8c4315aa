// Drawing into the frames in place (lwdetr_annotate / _nv12; the contract is in include/lwdetr_b200.h, tools/annotate_spec.py
// restates it).  Frames go in groups of ANN_GROUP (their descriptors travel as kernel parameters); per group two kernels:
//   1. setup, one CTA of 1024 threads per frame (thread j = entry j): each entry's rectangle, colour and label text, the
//      zone geometry's bounding boxes and the zone texts, written as the frame's primitive list in painter's order into the
//      object's scratch.  The order comes from one block-wide scan: privacy rectangles first, then zone fills, edges,
//      lines, box fills, outlines, labels and zone texts at fixed offsets of the counts.
//   2. draw, one CTA of 256 threads per 64 x 64 tile of a frame (aligned to the frame's origin, so no privacy block, at most
//      64 pixels, crosses a tile).  The CTA culls the frame's list against its tile into shared memory (an ordered
//      compaction, in rounds of at most CULL_CAP primitives) and exits at once when nothing overlaps.  Otherwise each thread
//      owns four 2x2 pixel blocks (and their chroma samples) of the tile: it stages them in shared memory, pixelates,
//      composites every primitive in order and stores only the bytes a primitive covered.  No two threads touch one byte;
//      the privacy sums are shared-memory integer atomics, whose result does not depend on their order.
#include "annotate.h"
#include "font5x7.cuh"
#include "frame.cuh"
#include "launch.h"

#include <algorithm>
#include <type_traits>

namespace lwb {

namespace {
constexpr int TILE = 64, NT = 256, SETUP_NT = 1024, CULL_CAP = 512, POLY_EDGES = 32;
constexpr int MAX_COORD = 1 << 20;              // zone text origins are clamped to [-MAX_COORD, MAX_COORD]

template <typename F>
struct AnnFrames {
  F f[ANN_GROUP];
  int32_t stream[ANN_GROUP];
};
struct AnnArgs {
  int f0, nb;                                   // first frame of the group in the call, frames in the group
  AnnOptions o;
  const int32_t* ids;
  const float* scores;
  const int32_t* labels;
  const float* boxes;
  const int32_t* counts;
  int k;
  float threshold;
  const ZoneGeom* geom;                         // NULL without zones
  const double2* verts;
  const int32_t* line_counts;
  int zone_ncol;                                // num_classes + 1 of the zones object
  const int32_t* occupancy;
};
static_assert(sizeof(AnnFrames<lwdetr_frame_nv12>) + sizeof(AnnArgs) + sizeof(AnnTable) + 64 <= 4096, "annotate launch exceeds 4 KB of parameters");

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }

__device__ __forceinline__ int clamp_coord(double v, int lo, int hi) { return static_cast<int>(fmin(fmax(v, static_cast<double>(lo)), static_cast<double>(hi))); }

// decimal of v into s, returns the characters written
__device__ int put_int(char* s, long long v) {
  char tmp[24];
  int n = 0;
  const bool neg = v < 0;
  unsigned long long u = neg ? 0ull - static_cast<unsigned long long>(v) : static_cast<unsigned long long>(v);
  do { tmp[n++] = static_cast<char>('0' + u % 10); u /= 10; } while (u);
  int m = 0;
  if (neg) s[m++] = '-';
  while (n) s[m++] = tmp[--n];
  return m;
}

__device__ __forceinline__ uint32_t palette_rgb(const AnnTable& t, long long i) {
  const long long n = __ldg(t.palette_n);
  const long long p = ((i % n) + n) % n;
  return t.palette[3 * p] | static_cast<uint32_t>(t.palette[3 * p + 1]) << 8 | static_cast<uint32_t>(t.palette[3 * p + 2]) << 16;
}
// black text on a light colour, white on a dark one (the grey of the motion estimator)
__device__ __forceinline__ uint32_t text_rgb(uint32_t c) {
  const int g = (9798 * static_cast<int>(c & 255) + 19235 * static_cast<int>(c >> 8 & 255) + 3735 * static_cast<int>(c >> 16 & 255) + 16384) >> 15;
  return g >= 128 ? 0u : 0xFFFFFFu;
}

__device__ __forceinline__ void put_rect(AnnPrim* p, int kind, int alpha, uint32_t rgb, int x0, int y0, int x1, int y1) {
  p->x0 = x0; p->y0 = y0; p->x1 = x1; p->y1 = y1; p->kind = kind; p->alpha = alpha; p->rgb = rgb; p->p0 = p->p1 = p->p2 = 0;
}
// background and glyphs of a text of n characters at (ox, oy), clipped to the frame
__device__ void put_text(AnnPrim* p, uint32_t rgb, int ox, int oy, int n, int slot, int s, int h, int w) {
  const int x0 = max(ox, 0), y0 = max(oy, 0), x1 = min(ox + 6 * s * n, w), y1 = min(oy + 8 * s, h);
  put_rect(p, ANN_FILL, 256, rgb, x0, y0, x1, y1);
  put_rect(p + 1, ANN_TEXT_GLYPHS, 256, text_rgb(rgb), x0, y0, x1, y1);
  p[1].p0 = ox; p[1].p1 = oy; p[1].p2 = slot;
}

// a segment's conservative pixel bounding box (a covered pixel's centre is within r of the segment)
__device__ void put_seg(AnnPrim* p, uint32_t rgb, double ax, double ay, double bx, double by, double r, int h, int w) {
  const int x0 = clamp_coord(floor(fmin(ax, bx) - r) - 1.0, 0, w), x1 = clamp_coord(ceil(fmax(ax, bx) + r) + 1.0, 0, w);
  const int y0 = clamp_coord(floor(fmin(ay, by) - r) - 1.0, 0, h), y1 = clamp_coord(ceil(fmax(ay, by) + r) + 1.0, 0, h);
  put_rect(p, ANN_SEG, 256, rgb, x0, y0, x1, y1);
}

// exclusive block scan of v over the SETUP_NT threads; *total = the sum
__device__ int block_scan(int v, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += u;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int y = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, y, o);
      if (lane >= o) y += u;
    }
    warp_sums[lane] = y;
  }
  __syncthreads();
  const int r = x - v + (wid ? warp_sums[wid - 1] : 0);
  *total = warp_sums[31];
  __syncthreads();
  return r;
}

template <typename F>
__global__ void __launch_bounds__(SETUP_NT) ann_setup_kernel(const __grid_constant__ AnnFrames<F> g, const __grid_constant__ AnnArgs a,
                                                             const __grid_constant__ AnnTable t) {
  pdl_sync();
  __shared__ int warp_sums[32];
  const int z = blockIdx.x, b = a.f0 + z, j = threadIdx.x;
  const F& f = g.f[z];
  const int h = f.height, w = f.width, s = a.o.text_scale;
  AnnPrim* P = t.prims + static_cast<long long>(z) * ANN_PRIMS;
  char* T = t.texts + static_cast<long long>(z) * ANN_TEXTS * ANN_TEXT;

  // the entry of this thread
  bool drawn = false, priv = false;
  int r[4] = {0, 0, 0, 0}, nch = 0;
  uint32_t rgb = 0;
  if (j < a.k && j < (a.counts ? __ldg(a.counts + b) : a.k)) {
    const long long e = static_cast<long long>(b) * a.k + j;
    const float sc = __ldg(a.scores + e);
    const int lab = __ldg(a.labels + e);
    const float* bx = a.boxes + 4 * e;
    const float x1 = __ldg(bx), y1 = __ldg(bx + 1), x2 = __ldg(bx + 2), y2 = __ldg(bx + 3);
    if (sc >= a.threshold && isfinite(x1) && isfinite(y1) && isfinite(x2) && isfinite(y2)) {
      r[0] = static_cast<int>(fminf(fmaxf(floorf(x1), 0.f), static_cast<float>(w)));
      r[1] = static_cast<int>(fminf(fmaxf(floorf(y1), 0.f), static_cast<float>(h)));
      r[2] = static_cast<int>(fminf(fmaxf(floorf(x2), 0.f), static_cast<float>(w)));
      r[3] = static_cast<int>(fminf(fmaxf(floorf(y2), 0.f), static_cast<float>(h)));
      drawn = r[2] > r[0] && r[3] > r[1];
    }
    if (drawn) {
      const bool known = lab >= 0 && lab < t.num_classes;
      priv = known && t.privacy[lab];
      const int id = a.ids ? __ldg(a.ids + e) : 0;
      rgb = palette_rgb(t, a.ids ? static_cast<long long>(id) : static_cast<long long>(lab));
      if (!priv && a.o.label) {                                     // "name #id 0.xx"
        char* out = T + static_cast<long long>(j) * ANN_TEXT;
        if (a.o.label & LWDETR_LABEL_NAME) {
          const char* nm = known ? t.names + static_cast<long long>(lab) * ANN_NAME : nullptr;
          if (nm && nm[0])
            for (int c = 0; c < ANN_NAME - 1 && nm[c]; ++c) out[nch++] = nm[c];
          else
            nch += put_int(out + nch, lab);
        }
        if ((a.o.label & LWDETR_LABEL_ID) && a.ids) {
          if (nch) out[nch++] = ' ';
          out[nch++] = '#';
          nch += put_int(out + nch, id);
        }
        if (a.o.label & LWDETR_LABEL_SCORE) {
          const int pc = static_cast<int>(fminf(fmaxf(floorf(__fadd_rn(__fmul_rn(sc, 100.f), 0.5f)), 0.f), 100.f));
          if (nch) out[nch++] = ' ';
          out[nch++] = pc == 100 ? '1' : '0';
          out[nch++] = '.';
          out[nch++] = static_cast<char>('0' + pc % 100 / 10);
          out[nch++] = static_cast<char>('0' + pc % 10);
        }
        out[nch] = 0;
      }
    }
  }

  // zone geometry of the frame's stream
  const ZoneGeom* zg = a.geom ? a.geom + g.stream[z] : nullptr;
  const int L = zg ? zg->n_lines : 0, Z = zg ? zg->n_polys : 0, V = zg ? zg->start[Z] : 0;
  const double2* vt = zg ? a.verts + static_cast<long long>(g.stream[z]) * ZONE_VERTS : nullptr;

  // painter's order: counts -> offsets
  int total;
  const int ex = block_scan((drawn && priv ? 1 : 0) | (drawn && !priv ? 1 << 16 : 0), warp_sums, &total);
  const int npriv = total & 0xFFFF, nbox = total >> 16;
  const bool labelled = nch > 0;
  int nlab;
  const int exl = block_scan(labelled ? 1 : 0, warp_sums, &nlab);
  const int o_poly = npriv, o_edge = o_poly + (a.o.zone_fill_alpha > 0 ? Z : 0), o_line = o_edge + V, o_fill = o_line + L;
  const int o_outline = o_fill + (a.o.box_fill_alpha > 0 ? nbox : 0), o_label = o_outline + nbox, o_ltext = o_label + 2 * nlab;
  const int o_ptext = o_ltext + 2 * L, n = o_ptext + (a.occupancy ? 2 * Z : 0);

  if (drawn && priv) put_rect(P + (ex & 0xFFFF), ANN_PRIV, 256, 0, r[0], r[1], r[2], r[3]);
  if (drawn && !priv) {
    const int q = ex >> 16;
    if (a.o.box_fill_alpha > 0) put_rect(P + o_fill + q, ANN_FILL, a.o.box_fill_alpha, rgb, r[0], r[1], r[2], r[3]);
    put_rect(P + o_outline + q, ANN_OUTLINE, 256, rgb, r[0], r[1], r[2], r[3]);
  }
  if (labelled) {
    const int oy = r[1] - 8 * s >= 0 ? r[1] - 8 * s : r[1];
    put_text(P + o_label + 2 * exl, rgb, r[0], oy, nch, j, s, h, w);
  }
  if (zg) {
    const double rad = dmul(static_cast<double>(a.o.zone_thickness), 0.5);
    for (int v = j; v < V; v += SETUP_NT) {                          // polygon edges v -> next vertex of its polygon
      int p = 0;
      while (zg->start[p + 1] <= v) ++p;
      const int nx = v + 1 == zg->start[p + 1] ? zg->start[p] : v + 1;
      const double2 A = vt[v], Bv = vt[nx];
      put_seg(P + o_edge + v, palette_rgb(t, p), A.x, A.y, Bv.x, Bv.y, rad, h, w);
      P[o_edge + v].p0 = -1; P[o_edge + v].p1 = v; P[o_edge + v].p2 = nx;
    }
    if (j < Z && a.o.zone_fill_alpha > 0) {                          // polygon fills
      const int v0 = zg->start[j], nv = zg->start[j + 1] - v0;
      double mnx = vt[v0].x, mxx = mnx, mny = vt[v0].y, mxy = mny;
      for (int v = 1; v < nv; ++v) {
        const double2 q = vt[v0 + v];
        mnx = fmin(mnx, q.x); mxx = fmax(mxx, q.x); mny = fmin(mny, q.y); mxy = fmax(mxy, q.y);
      }
      AnnPrim* p = P + o_poly + j;
      put_rect(p, ANN_POLY, a.o.zone_fill_alpha, palette_rgb(t, j), clamp_coord(floor(mnx) - 1.0, 0, w), clamp_coord(floor(mny) - 1.0, 0, h),
               clamp_coord(ceil(mxx) + 1.0, 0, w), clamp_coord(ceil(mxy) + 1.0, 0, h));
      p->p0 = v0; p->p1 = nv;
    }
    if (j < L) {
      const double* ln = zg->line[j];
      put_seg(P + o_line + j, palette_rgb(t, j), ln[0], ln[1], ln[2], ln[3], rad, h, w);
      P[o_line + j].p0 = j;
    }
    const int lane = j & 31, wid = j >> 5;
    if (wid < L) {                                                   // "in N out M" of line wid
      const int32_t* lc = a.line_counts + (static_cast<long long>(g.stream[z]) * ZONE_LINES + wid) * a.zone_ncol * 2;
      long long cin = 0, cout = 0;
      for (int c = lane; c < a.zone_ncol; c += 32) { cin += lc[2 * c]; cout += lc[2 * c + 1]; }
#pragma unroll
      for (int o = 16; o; o >>= 1) { cin += __shfl_xor_sync(0xffffffffu, cin, o); cout += __shfl_xor_sync(0xffffffffu, cout, o); }
      if (lane == 0) {
        const int slot = ANN_K + wid;
        char* out = T + static_cast<long long>(slot) * ANN_TEXT;
        int m = 0;
        out[m++] = 'i'; out[m++] = 'n'; out[m++] = ' ';
        m += put_int(out + m, cin);
        out[m++] = ' '; out[m++] = 'o'; out[m++] = 'u'; out[m++] = 't'; out[m++] = ' ';
        m += put_int(out + m, cout);
        out[m] = 0;
        const double* ln = zg->line[wid];
        const int ox = clamp_coord(floor(dmul(dadd(ln[0], ln[2]), 0.5)), -MAX_COORD, MAX_COORD);
        const int oy = clamp_coord(floor(dmul(dadd(ln[1], ln[3]), 0.5)), -MAX_COORD, MAX_COORD);
        put_text(P + o_ltext + 2 * wid, palette_rgb(t, wid), ox, oy, m, slot, s, h, w);
      }
    }
    if (a.occupancy && j < Z) {                                      // occupancy of polygon j at its first vertex
      const int slot = ANN_K + ZONE_LINES + j;
      char* out = T + static_cast<long long>(slot) * ANN_TEXT;
      const int m = put_int(out, __ldg(a.occupancy + static_cast<long long>(b) * ZONE_POLYS + j));
      out[m] = 0;
      const double2 q = vt[zg->start[j]];
      put_text(P + o_ptext + 2 * j, palette_rgb(t, j), clamp_coord(floor(q.x), -MAX_COORD, MAX_COORD), clamp_coord(floor(q.y), -MAX_COORD, MAX_COORD),
               m, slot, s, h, w);
    }
  }
  if (j == 0) {
    t.nprims[2 * z] = n;
    t.nprims[2 * z + 1] = npriv;
  }
}

// ---------------------------------------------------------------------------------------------------------------- draw

// palette colour -> Y, Cb, Cr of a colorspace (the header's table)
__constant__ int kRgb2Yuv[4][9] = {{16840, 33058, 6405, -9713, -19068, 28781, 28781, -24110, -4671},
                                   {11966, 40254, 4064, -6596, -22189, 28784, 28784, -26145, -2639},
                                   {19595, 38470, 7471, -11058, -21710, 32768, 32768, -27439, -5329},
                                   {13933, 46871, 4732, -7509, -25259, 32768, 32768, -29763, -3005}};
__device__ __forceinline__ uint32_t rgb_to_yuv(uint32_t c, int cs) {
  const int R = c & 255, G = c >> 8 & 255, B = c >> 16 & 255;
  const int* k = kRgb2Yuv[cs];
  const int Y = min(max(((k[0] * R + k[1] * G + k[2] * B + (1 << 15)) >> 16) + (cs < LWDETR_CSC_BT601_FULL ? 16 : 0), 0), 255);
  const int U = min(max(((k[3] * R + k[4] * G + k[5] * B + (1 << 15)) >> 16) + 128, 0), 255);
  const int V = min(max(((k[6] * R + k[7] * G + k[8] * B + (1 << 15)) >> 16) + 128, 0), 255);
  return Y | U << 8 | V << 16;
}
__device__ __forceinline__ int colorspace_of(const lwdetr_frame&) { return 0; }
__device__ __forceinline__ int colorspace_of(const lwdetr_frame_nv12& f) { return f.colorspace; }
__device__ __forceinline__ uint8_t blend(int src, int c, int a) { return static_cast<uint8_t>((src * (256 - a) + c * a + 128) >> 8); }

// is pixel (x, y) (inside the primitive's box and the frame) covered by p; polygons are tested in ann_draw_kernel, by rows
__device__ __forceinline__ bool covers(const AnnPrim& p, int x, int y, const AnnArgs& a, const ZoneGeom* zg, const double2* vt,
                                       const char* texts) {
  if (x < p.x0 || x >= p.x1 || y < p.y0 || y >= p.y1) return false;
  switch (p.kind) {
    case ANN_PRIV:
    case ANN_FILL: return true;
    case ANN_OUTLINE: {
      const int th = a.o.thickness;
      return x < p.x0 + th || x >= p.x1 - th || y < p.y0 + th || y >= p.y1 - th;
    }
    case ANN_SEG: {
      double ax, ay, bx, by;
      if (p.p0 >= 0) {
        ax = zg->line[p.p0][0]; ay = zg->line[p.p0][1]; bx = zg->line[p.p0][2]; by = zg->line[p.p0][3];
      } else {
        ax = vt[p.p1].x; ay = vt[p.p1].y; bx = vt[p.p2].x; by = vt[p.p2].y;
      }
      const double cx = static_cast<double>(x) + 0.5, cy = static_cast<double>(y) + 0.5;
      const double dx = dsub(bx, ax), dy = dsub(by, ay), L2 = dadd(dmul(dx, dx), dmul(dy, dy));
      const double qx = dsub(cx, ax), qy = dsub(cy, ay), u = dadd(dmul(qx, dx), dmul(qy, dy));
      double d2;
      if (u <= 0.0) {
        d2 = dadd(dmul(qx, qx), dmul(qy, qy));
      } else if (u >= L2) {
        const double ex = dsub(cx, bx), ey = dsub(cy, by);
        d2 = dadd(dmul(ex, ex), dmul(ey, ey));
      } else {
        const double c = dsub(dmul(dx, qy), dmul(dy, qx));
        d2 = __ddiv_rn(dmul(c, c), L2);
      }
      const double r = dmul(static_cast<double>(a.o.zone_thickness), 0.5);
      return d2 <= dmul(r, r);
    }
    default: {                                                      // ANN_TEXT_GLYPHS
      const int s = a.o.text_scale;
      const int cx = (x - p.p0) / s, gy = (y - p.p1) / s, ci = cx / kCellW, gx = cx - kCellW * ci;
      if (gx >= kFontCols || gy >= kFontRows) return false;
      int ch = static_cast<unsigned char>(texts[static_cast<long long>(p.p2) * ANN_TEXT + ci]);
      if (ch < kFontFirst || ch >= kFontFirst + kFontGlyphs) ch = '?';
      return kFont5x7[ch - kFontFirst][gy] >> (kFontCols - 1 - gx) & 1;
    }
  }
}

template <typename F>
__global__ void __launch_bounds__(NT) ann_draw_kernel(const __grid_constant__ AnnFrames<F> g, const __grid_constant__ AnnArgs a,
                                                      const __grid_constant__ AnnTable t) {
  constexpr bool kNV12 = std::is_same<F, lwdetr_frame_nv12>::value;
  constexpr int CH = kNV12 ? 1 : 3;                                 // bytes of one staged pixel (NV12: luma; chroma apart)
  pdl_sync();
  __shared__ int list[CULL_CAP];
  __shared__ int warp_n[NT / 32];
  __shared__ int s_count, s_next;
  __shared__ uint8_t px[TILE * TILE * CH];
  __shared__ uint8_t cpx[kNV12 ? (TILE / 2) * (TILE / 2) * 2 : 2];
  __shared__ int acc[(TILE / 2) * (TILE / 2)][kNV12 ? 5 : 4];       // privacy sums per block: RGB r, g, b, n; NV12 y, n, u, v, n
  __shared__ double xcross[TILE][POLY_EDGES];                       // polygon fill: each (tile row, edge)'s crossing abscissa

  const int z = blockIdx.z;
  const F& f = g.f[z];
  const int h = f.height, w = f.width;
  const int tx0 = blockIdx.x * TILE, ty0 = blockIdx.y * TILE;
  if (tx0 >= w || ty0 >= h) return;
  const int tx1 = min(tx0 + TILE, w), ty1 = min(ty0 + TILE, h);
  const int n = t.nprims[2 * z], npriv = t.nprims[2 * z + 1];
  const AnnPrim* P = t.prims + static_cast<long long>(z) * ANN_PRIMS;
  const char* texts = t.texts + static_cast<long long>(z) * ANN_TEXTS * ANN_TEXT;
  const ZoneGeom* zg = a.geom ? a.geom + g.stream[z] : nullptr;
  const double2* vt = a.geom ? a.verts + static_cast<long long>(g.stream[z]) * ZONE_VERTS : nullptr;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;

  // one cull round: the primitives from `pos` on whose box meets the tile, in order, while the list has room for a chunk
  auto cull = [&](int pos) {
    __syncthreads();                                                // every thread is done with the previous list
    int cnt = 0;
    while (pos < n && cnt + NT <= CULL_CAP) {
      const int i = pos + tid;
      bool hit = false;
      if (i < n) {
        const AnnPrim& p = P[i];
        hit = p.x0 < tx1 && p.x1 > tx0 && p.y0 < ty1 && p.y1 > ty0 && p.x1 > p.x0 && p.y1 > p.y0;
      }
      const unsigned m = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) warp_n[wid] = __popc(m);
      __syncthreads();
      int before = 0, all = 0;
#pragma unroll
      for (int q = 0; q < NT / 32; ++q) { before += q < wid ? warp_n[q] : 0; all += warp_n[q]; }
      if (hit) list[cnt + before + __popc(m & ((1u << lane) - 1u))] = i;
      cnt += all;
      pos += NT;
      __syncthreads();
    }
    if (tid == 0) { s_count = cnt; s_next = min(pos, n); }
    __syncthreads();
  };

  cull(0);
  if (s_count == 0 && s_next >= n) return;                          // nothing meets this tile: the common case

  // stage the thread's four 2x2 blocks; bit 4 q + 2 dy + dx of `mine` = pixel in the frame, of `wr` = written
  uint32_t mine = 0, wr = 0, pm = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int ly = 2 * by + (d >> 1), lx = 2 * bx + (d & 1), y = ty0 + ly, x = tx0 + lx;
      if (y < ty1 && x < tx1) {
        mine |= 1u << (4 * q + d);
        if constexpr (kNV12) {
          px[ly * TILE + lx] = f.luma[static_cast<long long>(y) * f.luma_pitch + x];
        } else {
          const uint8_t* s = f.data + static_cast<long long>(y) * f.pitch_bytes + 3LL * x;
          for (int c = 0; c < 3; ++c) px[(ly * TILE + lx) * 3 + c] = s[c];
        }
      }
    }
    if constexpr (kNV12) {
      if (mine >> (4 * q) & 1) {                                    // the chroma sample of an in-frame top-left pixel
        const uint8_t* s = f.chroma + static_cast<long long>((ty0 >> 1) + by) * f.chroma_pitch + 2LL * ((tx0 >> 1) + bx);
        cpx[2 * blk] = s[0];
        cpx[2 * blk + 1] = s[1];
      }
    }
  }

  const int PB = a.o.privacy_block, nbx = TILE / PB;
  bool pixelated = false;
  auto pixelate = [&]() {
    pixelated = true;
    if (!__syncthreads_or(pm)) return;
    for (int i = tid; i < nbx * nbx; i += NT)
      for (int c = 0; c < (kNV12 ? 5 : 4); ++c) acc[i][c] = 0;
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        if (!(pm >> (4 * q + d) & 1)) continue;
        const int ly = 2 * by + (d >> 1), lx = 2 * bx + (d & 1), pb = (ly / PB) * nbx + lx / PB;
        if constexpr (kNV12) {
          atomicAdd(&acc[pb][0], px[ly * TILE + lx]);
          atomicAdd(&acc[pb][1], 1);
        } else {
          for (int c = 0; c < 3; ++c) atomicAdd(&acc[pb][c], px[(ly * TILE + lx) * 3 + c]);
          atomicAdd(&acc[pb][3], 1);
        }
      }
      if constexpr (kNV12) {
        if (pm >> (4 * q) & 1) {                                    // chroma blocks of PB / 2 samples: the same block index
          const int pb = (by / (PB / 2)) * nbx + bx / (PB / 2);
          atomicAdd(&acc[pb][2], cpx[2 * blk]);
          atomicAdd(&acc[pb][3], cpx[2 * blk + 1]);
          atomicAdd(&acc[pb][4], 1);
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        if (!(pm >> (4 * q + d) & 1)) continue;
        const int ly = 2 * by + (d >> 1), lx = 2 * bx + (d & 1), pb = (ly / PB) * nbx + lx / PB;
        if constexpr (kNV12) {
          const int cn = acc[pb][1];
          px[ly * TILE + lx] = static_cast<uint8_t>((acc[pb][0] + cn / 2) / cn);
        } else {
          const int cn = acc[pb][3];
          for (int c = 0; c < 3; ++c) px[(ly * TILE + lx) * 3 + c] = static_cast<uint8_t>((acc[pb][c] + cn / 2) / cn);
        }
      }
      if constexpr (kNV12) {
        if (pm >> (4 * q) & 1) {
          const int pb = (by / (PB / 2)) * nbx + bx / (PB / 2), cn = acc[pb][4];
          cpx[2 * blk] = static_cast<uint8_t>((acc[pb][2] + cn / 2) / cn);
          cpx[2 * blk + 1] = static_cast<uint8_t>((acc[pb][3] + cn / 2) / cn);
          wr |= 1u << (16 + q);
        }
      }
    }
    wr |= pm;
  };

  for (;;) {
    const int cnt = s_count;
    for (int li = 0; li < cnt; ++li) {
      const int i = list[li];
      if (i >= npriv && !pixelated) pixelate();
      const AnnPrim p = P[i];
      if (p.kind == ANN_PRIV) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
#pragma unroll
          for (int d = 0; d < 4; ++d)
            if ((mine >> (4 * q + d) & 1) && covers(p, tx0 + 2 * bx + (d & 1), ty0 + 2 * by + (d >> 1), a, zg, vt, texts)) pm |= 1u << (4 * q + d);
        }
        continue;
      }
      const uint32_t col = kNV12 ? rgb_to_yuv(p.rgb, colorspace_of(f)) : p.rgb;
      // polygon fill: lwdetr_zones' even-odd rule at the pixel centres.  Whether edge (i, j) straddles a row and where it
      // crosses it depend on the row only, so they are computed once per (tile row, edge), in chunks of POLY_EDGES edges,
      // with the same operations as the rule: x = (xj - xi) * (py - yi) / (yj - yi) + xi, -inf (no flip) off the row
      // polygon fill: lwdetr_zones' even-odd rule at the pixel centres.  Whether edge (i, j) straddles a row and where it
      // crosses it depend on the row only, so they are computed once per (tile row, edge), in chunks of POLY_EDGES edges,
      // with the rule's operations: x = (xj - xi) * (py - yi) / (yj - yi) + xi, and -inf (no flip) off the row
      uint32_t pin = 0;
      if (p.kind == ANN_POLY) {
        const int v0 = p.p0, nv = p.p1;
        for (int e0 = 0; e0 < nv; e0 += POLY_EDGES) {
          __syncthreads();                                          // the previous chunk is read
          for (int u = tid; u < TILE * POLY_EDGES; u += NT) {
            const int row = u / POLY_EDGES, e = u % POLY_EDGES, i = e0 + e;
            double x = -INFINITY;
            if (i < nv) {
              const double py = static_cast<double>(ty0 + row) + 0.5;
              const double2 vi = vt[v0 + i], vj = vt[v0 + (i + nv - 1) % nv];
              if ((vi.y > py) != (vj.y > py)) x = dadd(__ddiv_rn(dmul(dsub(vj.x, vi.x), dsub(py, vi.y)), dsub(vj.y, vi.y)), vi.x);
            }
            xcross[row][e] = x;
          }
          __syncthreads();
          const int ne = min(POLY_EDGES, nv - e0);
#pragma unroll 1
          for (int q = 0; q < 4; ++q) {
            const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
#pragma unroll 1
            for (int d = 0; d < 4; ++d) {
              const double pxc = static_cast<double>(tx0 + 2 * bx + (d & 1)) + 0.5;
              const double* xr = xcross[2 * by + (d >> 1)];
              uint32_t flips = 0;
              for (int e = 0; e < ne; ++e) flips ^= pxc < xr[e] ? 1u : 0u;
              pin ^= flips << (4 * q + d);
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
        uint32_t cov = 0;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          if (!(mine >> (4 * q + d) & 1)) continue;
          const int x = tx0 + 2 * bx + (d & 1), y = ty0 + 2 * by + (d >> 1);
          const bool c = p.kind == ANN_POLY ? (x >= p.x0 && x < p.x1 && y >= p.y0 && y < p.y1 && (pin >> (4 * q + d) & 1))
                                            : covers(p, x, y, a, zg, vt, texts);
          if (c) cov |= 1u << d;
        }
        if (!cov) continue;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          if (!(cov >> d & 1)) continue;
          const int o = (2 * by + (d >> 1)) * TILE + 2 * bx + (d & 1);
          for (int c = 0; c < CH; ++c) px[o * CH + c] = blend(px[o * CH + c], col >> (8 * c) & 255, p.alpha);
        }
        wr |= cov << (4 * q);
        if constexpr (kNV12) {
          const int ac = (p.alpha * __popc(cov) + 2) >> 2;
          cpx[2 * blk] = blend(cpx[2 * blk], col >> 8 & 255, ac);
          cpx[2 * blk + 1] = blend(cpx[2 * blk + 1], col >> 16 & 255, ac);
          wr |= 1u << (16 + q);
        }
      }
    }
    if (s_next >= n) break;
    cull(s_next);
  }
  if (!pixelated) pixelate();

  // store the written bytes only
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int blk = tid + q * NT, by = blk >> 5, bx = blk & 31;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      if (!(wr >> (4 * q + d) & 1)) continue;
      const int ly = 2 * by + (d >> 1), lx = 2 * bx + (d & 1), y = ty0 + ly, x = tx0 + lx;
      if constexpr (kNV12) {
        const_cast<uint8_t*>(f.luma)[static_cast<long long>(y) * f.luma_pitch + x] = px[ly * TILE + lx];
      } else {
        uint8_t* d8 = const_cast<uint8_t*>(f.data) + static_cast<long long>(y) * f.pitch_bytes + 3LL * x;
        for (int c = 0; c < 3; ++c) d8[c] = px[(ly * TILE + lx) * 3 + c];
      }
    }
    if constexpr (kNV12) {
      if (wr >> (16 + q) & 1) {
        uint8_t* d8 = const_cast<uint8_t*>(f.chroma) + static_cast<long long>((ty0 >> 1) + by) * f.chroma_pitch + 2LL * ((tx0 >> 1) + bx);
        d8[0] = cpx[2 * blk];
        d8[1] = cpx[2 * blk + 1];
      }
    }
  }
}

template <typename F>
int annotate_impl(const AnnTable& t, const AnnOptions& o, const F* frames, int B, const AnnCall& c, cudaStream_t st) {
  AnnArgs a = {};
  a.o = o;
  a.ids = c.ids; a.scores = c.scores; a.labels = c.labels; a.boxes = c.boxes; a.counts = c.counts; a.k = c.k; a.threshold = c.threshold;
  if (c.zones) {
    a.geom = c.zones->geom; a.verts = c.zones->verts; a.line_counts = c.zones->line_counts; a.zone_ncol = c.zones->num_classes + 1;
    a.occupancy = c.occupancy;
  }
  for (int f0 = 0; f0 < B; f0 += ANN_GROUP) {
    AnnFrames<F> g = {};
    a.f0 = f0;
    a.nb = std::min(ANN_GROUP, B - f0);
    int hmax = 1, wmax = 1;
    for (int j = 0; j < a.nb; ++j) {
      g.f[j] = frames[f0 + j];
      g.stream[j] = c.zones ? c.streams[f0 + j] : 0;
      hmax = std::max(hmax, frames[f0 + j].height);
      wmax = std::max(wmax, frames[f0 + j].width);
    }
    cudaError_t e = launch_k(ann_setup_kernel<F>, dim3(a.nb), dim3(SETUP_NT), 0, st, g, a, t);
    if (e == cudaSuccess)
      e = launch_k(ann_draw_kernel<F>, dim3((wmax + TILE - 1) / TILE, (hmax + TILE - 1) / TILE, a.nb), dim3(NT), 0, st, g, a, t);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  return 0;
}
}  // namespace

int annotate_launch(const AnnTable& t, const AnnOptions& o, const lwdetr_frame* frames, int B, const AnnCall& c, cudaStream_t st) {
  return annotate_impl(t, o, frames, B, c, st);
}
int annotate_launch(const AnnTable& t, const AnnOptions& o, const lwdetr_frame_nv12* frames, int B, const AnnCall& c, cudaStream_t st) {
  return annotate_impl(t, o, frames, B, c, st);
}

}  // namespace lwb
