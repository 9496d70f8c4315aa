// Camera-motion estimation per video stream on the device (lwdetr_gmc_*, include/lwdetr_b200.h): grey + downscale,
// pyrDown pyramid, grid Shi-Tomasi corners, pyramidal Lucas-Kanade and a deterministic RANSAC + float64 refit of a
// similarity.  State (two pyramids and two corner lists per stream) lives in a device table allocated once.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lwdetr_b200.h"

namespace lwb {

constexpr int GMC_MAX_LEVELS = 5;        // pyramid levels above level 0
constexpr int GMC_MAX_POINTS = 4096;
constexpr int GMC_MAX_WINDOW = 31;
constexpr int GMC_MAX_HYPOTHESES = 4096;
constexpr int GMC_MIN_SIDE = 16;         // level-0 sides
constexpr int GMC_REFITS = 3;            // least-squares rounds after RANSAC

struct GmcHead {                         // per stream, on the device
  int32_t cur;                           // buffer holding the stream's last frame
  int32_t valid;                         // a last frame exists
  int32_t h, w;                          // its size
  int32_t npts[2];                       // corner count of each buffer
  int32_t prev;                          // the other buffer holds the frame before the last one, of the same size
  int32_t pad1;
};

struct GmcTable {
  int num_streams;
  lwdetr_gmc_params p;
  GmcHead* head;                         // [num_streams]
  uint8_t* pyr;                          // [num_streams][2][slot_bytes]: levels 0..levels at off[l], rows pitch = level width
  long long slot_bytes;
  long long off[GMC_MAX_LEVELS + 1];
  float2* pts;                           // [num_streams][2][max_points]: corners of each buffer, level-0 pixels
  double* cell_r;                        // [num_streams][max_points]: best response of each grid cell
  int32_t* cell_i;                       // its pixel index (y * width + x), -1: none
  float4* flow;                          // [num_streams][max_points]: (from, to) of each tracked corner, level-0 pixels
  int8_t* found;                         // [num_streams][max_points]
};

// Geometry of one frame size: level sizes, levels used (OpenCV's buildOpticalFlowPyramid rule), corner grid.
struct GmcGeo {
  int lw[GMC_MAX_LEVELS + 1], lh[GMC_MAX_LEVELS + 1];
  int nlev, cell, ncx, ncy;
};
void gmc_geometry(int h, int w, const lwdetr_gmc_params& p, GmcGeo* g);

// One frame of one stream: an RGB frame (nv12 = 0, data / pitch of the pixels) or the luma plane of an NV12 frame.
struct GmcFrameHost {
  const uint8_t* data;
  long long pitch;
  int h, w, nv12;
};

// streams: HOST, B distinct ids in [0, num_streams) (checked by the caller); frames validated by the caller.  observe:
// lwdetr_gmc_observe (grey, pyramid and corners only; motion, status and inliers unused).
int gmc_estimate_launch(const GmcTable& t, const GmcFrameHost* frames, int B, const int32_t* streams, double* motion, int32_t* status,
                        int32_t* inliers, cudaStream_t st, bool observe = false);
int gmc_reset_launch(const GmcTable& t, const int32_t* streams, int n, cudaStream_t st);

}  // namespace lwb
