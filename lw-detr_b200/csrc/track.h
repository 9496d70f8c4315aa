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

constexpr int TRACK_PAIRS = 8192;        // proximity pairs per stream and frame kept with their appearance cost

// the appearance state of a tracker made by lwdetr_tracker_create_reid (track.cu: stable embedding slots)
struct ReidTable {
  lwdetr_reid_params params;
  int16_t* slot;                         // [num_streams][2][capacity]: embedding slot of each record, parallel to rec
  uint8_t* has;                          // [num_streams][capacity] by slot: the slot holds an embedding
  float* emb;                            // [num_streams][capacity][embedding_dim] by slot
  uint32_t* pkey;                        // [num_streams][TRACK_PAIRS] scratch of one frame
  double* pval;                          // [num_streams][TRACK_PAIRS]
};

// the embeddings of one lwdetr_track_reid call: DEVICE [B][k] rows of ld elements of type dtype (LWDETR_ET_*), or null
struct ReidInput {
  const ReidTable* table;
  const void* emb;
  int dtype;
  long long ld;
};

// -2: a limit is exceeded (k, streams); otherwise a cudaError_t.  streams: HOST, B distinct ids in [0, num_streams).
// motion: DEVICE [B][4] camera motion of each frame (lwdetr_track_ex), or null.  reid: null for ByteTrack, else the
// appearance instantiation runs (lwdetr_track_reid).
int track_launch(const TrackTable& t, const lwdetr_track_params& p, const float* scores, const int32_t* labels, const float* boxes,
                 const double* motion, int B, int k, const int32_t* streams, int max_out, int32_t* out_ids, float* out_scores, int32_t* out_labels,
                 float* out_boxes, int32_t* out_index, int32_t* counts, cudaStream_t st, const ReidInput* reid = nullptr);
// frame and next id back to 1, lists emptied, overflow count 0, for n HOST stream ids
int track_reset_launch(const TrackTable& t, const int32_t* streams, int n, cudaStream_t st);
int query_best_launch(const float* logits, const float* boxes, const float* target_sizes, int B, int nq, int ncls, float* scores,
                      int32_t* labels, float* out_boxes, cudaStream_t st);

}  // namespace lwb
