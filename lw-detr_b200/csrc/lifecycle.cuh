// The id -> record lifecycle that lwdetr_zones_update and lwdetr_speed_update share: one CTA of LC_NT threads per stream,
// the stream's records in fixed slots and an index of (id, slot, last_seen) sorted by id, staged in shared memory.  Per
// frame, on the entries of one lwdetr_track output row:
//   lc_stage    the index and the slot bitmap are staged; each entry is keyed (id, entry) when valid, NOKEY otherwise;
//   lc_sort     the keys are bitonic-sorted;
//   lc_present  the first entry of each id is present (a repeat is ignored); P present entries in input order;
//   lc_assign   present ids are looked up in the index (last_seen of a found record becomes the frame), and new ones take
//               free slots (lowest first) in input order while there is one;
//   lc_merge    records with frame - last_seen > forget_after are dropped, and the index is rebuilt by a merge of the
//               survivors and the new records (both sorted by id), written in place.
// Between the phases the caller runs its own per-track work on Lifecycle's arrays (jslot, jpos, plist, ...).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "records.h"

namespace lwb {

constexpr int LC_NT = 512;                    // threads per CTA
constexpr int LC_NW = LC_NT / 32;
constexpr int LC_MAXE = 1024;                 // entries per frame
constexpr int LC_MAXR = 4096;                 // records per stream
constexpr unsigned long long LC_NOKEY = ~0ull;

struct Lifecycle {
  RecordIndex idx[LC_MAXR];                   // the stream's index; last_seen of present records set to the frame
  int rscan[LC_MAXR];                         // per record: scratch for the caller, then survivors (exclusive scan)
  unsigned long long key[LC_MAXE];            // (id << 32) | entry, sorted
  int eid[LC_MAXE];                           // by entry: id
  int jscan[LC_MAXE];                         // by entry: position among the present entries (exclusive scan)
  int jpos[LC_MAXE], jslot[LC_MAXE];          // by entry: index position (-1: no record before this frame), slot (-1: none)
  int plist[LC_MAXE];                         // present entries in input order
  int pnew[LC_MAXE];                          // by present position: rank among the new ids
  int sscan[LC_MAXE];                         // by sorted position: rank among the new records
  int newj[LC_MAXE];                          // new records by ascending id: their entry
  uint32_t used[LC_MAXR / 32];                // slot bitmap
  int freepref[LC_MAXR / 32 + 1];
  int wsum[LC_NW];
  int total;
};

// exclusive prefix sums of a[0, n) in place; every thread gets the total
__device__ inline int block_scan(int* a, int n, Lifecycle& s) {
  __syncthreads();
  const int per = (n + LC_NT - 1) / LC_NT;
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
    const int v = lane < LC_NW ? s.wsum[lane] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(~0u, x, o);
      if (lane >= o) x += u;
    }
    if (lane < LC_NW) s.wsum[lane] = x - v;
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

// the tracks' anchor rule (LWDETR_ANCHOR_*): anchor 3 * row + column of an fp32 xyxy box, widened to float64, rows y1,
// (y1 + y2) * 0.5, y2 and columns x1, (x1 + x2) * 0.5, x2
__device__ __forceinline__ void box_anchor(const float4 b, int which, double& x, double& y) {
  const int row = which / 3, col = which % 3;
  x = col == 0 ? static_cast<double>(b.x) : col == 1 ? __dmul_rn(__dadd_rn(b.x, b.z), 0.5) : static_cast<double>(b.z);
  y = row == 0 ? static_cast<double>(b.y) : row == 1 ? __dmul_rn(__dadd_rn(b.y, b.w), 0.5) : static_cast<double>(b.w);
}

__device__ __forceinline__ int index_lower_bound(const RecordIndex* idx, int n, int id) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (idx[m].id < id) lo = m + 1;
    else hi = m;
  }
  return lo;
}

// Stages the n_old records of gidx and the slot bitmap of C slots, and keys the cnt entries: load(j, id) reads entry j
// (and whatever the caller keeps of it), sets its id and returns whether it is valid.  Returns np2, the sort's length.
// Ends without a barrier: lc_sort begins with one.
template <class Load>
__device__ int lc_stage(Lifecycle& s, const RecordIndex* gidx, int n_old, int C, int cnt, Load load) {
  const int tid = threadIdx.x;
  for (int i = tid; i < n_old; i += LC_NT) s.idx[i] = gidx[i];
  const int words = (C + 31) / 32;
  for (int w = tid; w < words; w += LC_NT) s.used[w] = C - w * 32 >= 32 ? 0u : ~0u << (C - w * 32);
  int np2 = 1;
  while (np2 < cnt) np2 <<= 1;
  for (int j = tid; j < np2; j += LC_NT) {
    unsigned long long k = LC_NOKEY;
    if (j < cnt) {
      int id = 0;
      const bool ok = load(j, id);
      s.eid[j] = id;
      s.jscan[j] = 0;
      if (ok) k = static_cast<unsigned long long>(static_cast<uint32_t>(id)) << 32 | static_cast<uint32_t>(j);
    }
    s.key[j] = k;
  }
  return np2;
}

__device__ inline void lc_sort(Lifecycle& s, int np2) {
  const int tid = threadIdx.x;
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < np2; i += LC_NT) {
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
}

// The present entries: P of them, in plist[0, P) in input order; marks the old records' slots used.  Ends on a barrier.
__device__ inline int lc_present(Lifecycle& s, int cnt, int n_old) {
  const int tid = threadIdx.x;
  for (int p = tid; p < cnt; p += LC_NT) {       // the first entry of each id is present
    const unsigned long long k = s.key[p];
    if (k != LC_NOKEY && (p == 0 || s.key[p - 1] >> 32 != k >> 32)) s.jscan[static_cast<uint32_t>(k)] = 1;
  }
  const int P = block_scan(s.jscan, cnt, s);
  for (int j = tid; j < cnt; j += LC_NT)
    if ((j + 1 < cnt ? s.jscan[j + 1] : P) != s.jscan[j]) s.plist[s.jscan[j]] = j;
  for (int i = tid; i < n_old; i += LC_NT) atomicOr(&s.used[s.idx[i].slot >> 5], 1u << (s.idx[i].slot & 31));
  __syncthreads();
  return P;
}

// whether entry j (< cnt) is present, once lc_present has run
__device__ __forceinline__ bool lc_is_present(const Lifecycle& s, int j, int cnt, int P) {
  return (j + 1 < cnt ? s.jscan[j + 1] : P) != s.jscan[j];
}

// Looks the P present ids up and gives the new ones the lowest free slots of C, in input order: jpos and jslot of each
// present entry (jslot -1: not recorded).  Returns the number of new ids; min(new, C - n_old) of them are recorded.  Ends
// without a barrier: jslot of new ids is written last.
__device__ inline int lc_assign(Lifecycle& s, int P, int n_old, int C, int frame) {
  const int tid = threadIdx.x, words = (C + 31) / 32;
  for (int p = tid; p < P; p += LC_NT) {
    const int j = s.plist[p], id = s.eid[j];
    const int lb = index_lower_bound(s.idx, n_old, id);
    const bool found = lb < n_old && s.idx[lb].id == id;
    s.jpos[j] = found ? lb : -1;
    s.jslot[j] = found ? s.idx[lb].slot : -1;
    if (found) s.idx[lb].last_seen = frame;
    s.pnew[p] = found ? 0 : 1;
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
  const int nfree = C - n_old;
  for (int p = tid; p < P; p += LC_NT) {          // the r-th new id takes the r-th free slot, while there is one
    const int j = s.plist[p], r = s.pnew[p];
    if (s.jpos[j] >= 0 || r >= nfree) continue;
    int lo = 0, hi = words - 1;                    // the last word w with freepref[w] <= r
    while (lo < hi) {
      const int m = (lo + hi + 1) >> 1;
      if (s.freepref[m] <= r) lo = m;
      else hi = m - 1;
    }
    s.jslot[j] = lo * 32 + static_cast<int>(__fns(~s.used[lo], 0, r - s.freepref[lo] + 1));
  }
  return nnew;
}

// Drops the records with frame - last_seen > forget_after and writes the new index to gidx: the survivors and the new
// records merged by id.  Returns the number of records.  Begins with a barrier; rscan is overwritten.
__device__ inline int lc_merge(Lifecycle& s, RecordIndex* gidx, int n_old, int cnt, int P, int frame, int forget_after) {
  const int tid = threadIdx.x;
  __syncthreads();
  for (int i = tid; i < n_old; i += LC_NT) s.rscan[i] = frame - s.idx[i].last_seen <= forget_after ? 1 : 0;
  for (int p = tid; p < cnt; p += LC_NT) {
    const unsigned long long k = s.key[p];
    const int j = static_cast<int>(static_cast<uint32_t>(k));
    s.sscan[p] = k != LC_NOKEY && lc_is_present(s, j, cnt, P) && s.jpos[j] < 0 && s.jslot[j] >= 0 ? 1 : 0;
  }
  const int S = block_scan(s.rscan, n_old, s);
  const int A = block_scan(s.sscan, cnt, s);
  for (int p = tid; p < cnt; p += LC_NT) {
    const unsigned long long k = s.key[p];
    const int j = static_cast<int>(static_cast<uint32_t>(k));
    if (k != LC_NOKEY && lc_is_present(s, j, cnt, P) && s.jpos[j] < 0 && s.jslot[j] >= 0) s.newj[s.sscan[p]] = j;
  }
  __syncthreads();
  for (int i = tid; i < n_old; i += LC_NT) {
    const RecordIndex x = s.idx[i];
    if (frame - x.last_seen > forget_after) continue;
    int lo = 0, hi = A;                            // new ids below x.id
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (s.eid[s.newj[m]] < x.id) lo = m + 1;
      else hi = m;
    }
    gidx[s.rscan[i] + lo] = x;
  }
  for (int r = tid; r < A; r += LC_NT) {
    const int j = s.newj[r], id = s.eid[j];
    const int lb = index_lower_bound(s.idx, n_old, id);
    gidx[r + (lb < n_old ? s.rscan[lb] : S)] = RecordIndex{id, s.jslot[j], frame};
  }
  return S + A;
}

}  // namespace lwb
