// Multi-object tracking on the device (lwdetr_track, include/lwdetr_b200.h): ByteTrack's association per camera stream,
// one CTA per stream, state in a device table allocated once per tracker.  lwdetr_query_best: one detection per query.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lwdetr_b200.h"

namespace lwb {

constexpr int TRACK_MAX = 1024;          // entries per frame, and tracks per stream (capacity)

struct TrackHead {                       // per stream, on the device
  int32_t frame, next_id, overflow, n_tracked, n_lost, parity, pad0, pad1;
};

struct TrackTable {
  int num_streams, capacity;
  TrackHead* head;                       // [num_streams]
  lwdetr_track_record* rec;              // [num_streams][2][capacity]: two buffers per stream, head.parity the current one
};

// -2: a limit is exceeded (k, streams); otherwise a cudaError_t.  streams: HOST, B distinct ids in [0, num_streams).
// motion: DEVICE [B][4] camera motion of each frame (lwdetr_track_ex), or null.
int track_launch(const TrackTable& t, const lwdetr_track_params& p, const float* scores, const int32_t* labels, const float* boxes,
                 const double* motion, int B, int k, const int32_t* streams, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels,
                 float* out_boxes, int32_t* out_index, int32_t* counts, cudaStream_t st);
// frame and next id back to 1, lists emptied, overflow count 0, for n HOST stream ids
int track_reset_launch(const TrackTable& t, const int32_t* streams, int n, cudaStream_t st);
int query_best_launch(const float* logits, const float* boxes, const float* target_sizes, int B, int nq, int ncls, float* scores,
                      int32_t* labels, float* out_boxes, cudaStream_t st);

}  // namespace lwb
