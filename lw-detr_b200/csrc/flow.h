// Per-object flow between two frames of a stream (lwdetr_flow_*, lwdetr_track_flow, include/lwdetr_b200.h): the Median
// Flow tracker for every activated tracked track of the device tracker, read from the camera-motion estimator's two
// pyramids of the stream.  Scratch (one slot of max_tracks x grid^2 points per stream) is allocated once at create.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "gmc.h"
#include "lwdetr_b200.h"
#include "track.h"

namespace lwb {

constexpr int FLOW_MAX_GRID = 16;

struct FlowTable {
  lwdetr_flow_params p;
  int num_streams, g2;
  int32_t* ntracks;                      // [num_streams]: activated tracked tracks of the stream at the last call
  int16_t* slot;                         // [num_streams][max_tracks]: their records, in list order
  float2* seed;                          // [num_streams][max_tracks][g2]: level-0 pixels
  float2* fwd;                           // forward Lucas-Kanade, previous -> current
  float2* bwd;                           // backward, current -> previous, from fwd
  int8_t* valid;                         // both directions found
  double* fb;                            // forward-backward error, frame pixels (NaN where not valid)
  double* ncc;                           // NCC of the two patches (NaN where not valid)
  int32_t* status;                       // [num_streams][max_tracks]: LWDETR_FLOW_*
  double* meas;                          // [num_streams][max_tracks][8]: dx, dy, s, then the measurement (cx, cy, a, h)
};

// The flow of the B HOST streams (distinct, checked by the caller) of one call: reads the tracker's records as they are
// and the estimator's current and previous pyramids.  0 or a cudaError_t.
int flow_launch(const FlowTable& f, const GmcTable& g, const TrackTable& t, int B, const int32_t* streams, cudaStream_t st);

// lwdetr_track_flow's tracker step from the flow's measurements (track.cu).  motion: DEVICE [B][4] or null.  slot: the
// tracker's embedding slots (ReidTable::slot) or null.
int track_flow_launch(const TrackTable& t, const lwdetr_track_params& p, const FlowTable& f, const double* motion, int16_t* slot, int B,
                      const int32_t* streams, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels, float* out_boxes,
                      int32_t* out_index, int32_t* counts, cudaStream_t st);

}  // namespace lwb
