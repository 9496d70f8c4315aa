// calcOpticalFlowPyrLK's iteration for one point by one warp, shared by the camera-motion estimator (gmc.cu, lk_kernel)
// and the per-object flow (flow.cu): the pyramids are the estimator's (GmcTable), window sums in exact int64.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gmc.h"

namespace lwb {
namespace {

// BORDER_REFLECT_101 (cv::borderInterpolate)
__device__ __forceinline__ int refl(int p, int n) {
  if (n == 1) return 0;
  while (static_cast<unsigned>(p) >= static_cast<unsigned>(n)) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

__device__ __forceinline__ uint8_t* level_ptr(const GmcTable& t, int sid, int buf, int l) {
  return t.pyr + (static_cast<long long>(sid) * 2 + buf) * t.slot_bytes + t.off[l];
}

constexpr int WB = 14;                   // OpenCV's W_BITS
constexpr int PP = GMC_MAX_WINDOW + 3;   // previous-image patch side (window + 1 for interpolation + 1 each side)
constexpr int DP = GMC_MAX_WINDOW + 1;   // derivative patch side

struct LkWarp {
  uint8_t patch[PP * PP];
  short2 deriv[DP * DP];
  short iw[GMC_MAX_WINDOW * GMC_MAX_WINDOW];
  short2 diw[GMC_MAX_WINDOW * GMC_MAX_WINDOW];
};

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

__device__ __forceinline__ long long warp_sum(long long v) {
  for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}

// The whole warp: the point p0 (level-0 pixels) of the pyramid in buffer bi of stream sid, tracked into buffer bj from level
// nlev down to 0 (level sizes lw / lh), no initial guess.  Returns the status (false: lost at level 0) and the point in *out.
__device__ __forceinline__ bool lk_point(LkWarp& S, const GmcTable& t, int sid, int bi, int bj, const int* lw, const int* lh, int nlev,
                                         float2 p0, int win, int iterations, float eps2, float min_eig_thr, float2* out) {
  const int lane = threadIdx.x & 31;
  const int half = (win - 1) / 2, area = win * win;
  float2 nxt = p0;
  bool ok = true;
  for (int l = nlev; l >= 0; --l) {
    const int W = lw[l], H = lh[l];
    const uint8_t* I = level_ptr(t, sid, bi, l);
    const uint8_t* J = level_ptr(t, sid, bj, l);
    const float sc = 1.f / static_cast<float>(1 << l);
    float2 prev = make_float2(p0.x * sc - half, p0.y * sc - half);
    nxt = l == nlev ? make_float2(p0.x * sc, p0.y * sc) : make_float2(nxt.x * 2.f, nxt.y * 2.f);
    const int ipx = static_cast<int>(floorf(prev.x)), ipy = static_cast<int>(floorf(prev.y));
    if (ipx < -win || ipx >= W || ipy < -win || ipy >= H) {
      if (l == 0) ok = false;
      continue;
    }
    float ax = prev.x - ipx, ay = prev.y - ipy;
    int w00 = __float2int_rn((1.f - ax) * (1.f - ay) * (1 << WB));
    int w01 = __float2int_rn(ax * (1.f - ay) * (1 << WB));
    int w10 = __float2int_rn((1.f - ax) * ay * (1 << WB));
    int w11 = (1 << WB) - w00 - w01 - w10;
    // previous image around the window (reflected), its Scharr derivatives (0 outside the image), the window interpolated
    for (int q = lane; q < (win + 3) * (win + 3); q += 32) {
      const int qy = q / (win + 3), qx = q - qy * (win + 3);
      S.patch[qy * PP + qx] = I[static_cast<long long>(refl(ipy - 1 + qy, H)) * W + refl(ipx - 1 + qx, W)];
    }
    __syncwarp();
    for (int q = lane; q < (win + 1) * (win + 1); q += 32) {
      const int qy = q / (win + 1), qx = q - qy * (win + 1);
      const int y = ipy + qy, x = ipx + qx;
      short2 dv = make_short2(0, 0);
      if (y >= 0 && y < H && x >= 0 && x < W) {
        const uint8_t* c = S.patch + (qy + 1) * PP + (qx + 1);
        // the patch holds reflected pixels, which is calcSharrDeriv's border.  t0 = 3 (up + down) + 10 mid, t1 = down - up; dx = t0[x+1] - t0[x-1], dy = 3 (t1[x+1] + t1[x-1]) + 10 t1[x]
        const auto t0 = [&](int o) { return 3 * (c[o - PP] + c[o + PP]) + 10 * c[o]; };
        const auto t1 = [&](int o) { return c[o + PP] - c[o - PP]; };
        dv = make_short2(static_cast<short>(t0(1) - t0(-1)), static_cast<short>(3 * (t1(1) + t1(-1)) + 10 * t1(0)));
      }
      S.deriv[qy * DP + qx] = dv;
    }
    __syncwarp();
    long long a11 = 0, a12 = 0, a22 = 0;
    for (int q = lane; q < area; q += 32) {
      const int qy = q / win, qx = q - qy * win;
      const uint8_t* s = S.patch + (qy + 1) * PP + (qx + 1);
      const int ival = descale(s[0] * w00 + s[1] * w01 + s[PP] * w10 + s[PP + 1] * w11, WB - 5);
      const short2* ds = S.deriv + qy * DP + qx;
      const int ixv = descale(ds[0].x * w00 + ds[1].x * w01 + ds[DP].x * w10 + ds[DP + 1].x * w11, WB);
      const int iyv = descale(ds[0].y * w00 + ds[1].y * w01 + ds[DP].y * w10 + ds[DP + 1].y * w11, WB);
      S.iw[q] = static_cast<short>(ival);
      S.diw[q] = make_short2(static_cast<short>(ixv), static_cast<short>(iyv));
      a11 += static_cast<long long>(ixv) * ixv;
      a12 += static_cast<long long>(ixv) * iyv;
      a22 += static_cast<long long>(iyv) * iyv;
    }
    const float fs = 1.f / static_cast<float>(1 << 20);
    const float A11 = static_cast<float>(warp_sum(a11)) * fs, A12 = static_cast<float>(warp_sum(a12)) * fs,
                A22 = static_cast<float>(warp_sum(a22)) * fs;
    __syncwarp();
    float D = A11 * A22 - A12 * A12;
    const float min_eig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / static_cast<float>(2 * area);
    if (min_eig < min_eig_thr || D < 1.1920929e-7f) {
      if (l == 0) ok = false;
      continue;
    }
    D = 1.f / D;
    float2 np_ = make_float2(nxt.x - half, nxt.y - half);
    float2 pd = make_float2(0.f, 0.f);
    for (int it = 0; it < iterations; ++it) {
      const int inx = static_cast<int>(floorf(np_.x)), iny = static_cast<int>(floorf(np_.y));
      if (inx < -win || inx >= W || iny < -win || iny >= H) {
        if (l == 0) ok = false;
        break;
      }
      ax = np_.x - inx;
      ay = np_.y - iny;
      w00 = __float2int_rn((1.f - ax) * (1.f - ay) * (1 << WB));
      w01 = __float2int_rn(ax * (1.f - ay) * (1 << WB));
      w10 = __float2int_rn((1.f - ax) * ay * (1 << WB));
      w11 = (1 << WB) - w00 - w01 - w10;
      long long b1 = 0, b2 = 0;
      for (int q = lane; q < area; q += 32) {
        const int qy = q / win, qx = q - qy * win;
        const long long r0 = static_cast<long long>(refl(iny + qy, H)) * W, r1 = static_cast<long long>(refl(iny + qy + 1, H)) * W;
        const int c0 = refl(inx + qx, W), c1 = refl(inx + qx + 1, W);
        const int diff = descale(J[r0 + c0] * w00 + J[r0 + c1] * w01 + J[r1 + c0] * w10 + J[r1 + c1] * w11, WB - 5) - S.iw[q];
        b1 += static_cast<long long>(diff) * S.diw[q].x;
        b2 += static_cast<long long>(diff) * S.diw[q].y;
      }
      const float B1 = static_cast<float>(warp_sum(b1)) * fs, B2 = static_cast<float>(warp_sum(b2)) * fs;
      const float2 delta = make_float2((A12 * B2 - A22 * B1) * D, (A12 * B1 - A11 * B2) * D);
      np_.x += delta.x;
      np_.y += delta.y;
      nxt = make_float2(np_.x + half, np_.y + half);
      if (delta.x * delta.x + delta.y * delta.y <= eps2) break;
      if (it > 0 && fabsf(delta.x + pd.x) < 0.01f && fabsf(delta.y + pd.y) < 0.01f) {
        nxt.x -= delta.x * 0.5f;
        nxt.y -= delta.y * 0.5f;
        break;
      }
      pd = delta;
    }
  }
  *out = nxt;
  return ok;
}

}  // namespace
}  // namespace lwb
