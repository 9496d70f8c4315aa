// Ground-plane position, velocity and speed of each track per camera stream (lwdetr_speed_*, include/lwdetr_b200.h): one
// CTA per stream in the call, state in a device table allocated once per object.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "records.h"

namespace lwb {

constexpr int SPEED_CAPACITY = 4096, SPEED_WINDOW = 64, SPEED_MAX_OUT = 1024;

struct SpeedHead {                       // per stream
  int32_t frame, n, overflow, clock_errors;   // n records, in index[0, n) by ascending id
  double last_t;                         // the last timestamp that added samples (-inf: none)
};

struct SpeedRec {                        // per slot: the ring holds n samples, the oldest at pos
  int32_t n, pos;
};

struct SpeedTable {
  int num_streams, capacity, window, min_samples, forget_after, anchor;
  double frame_rate;
  SpeedHead* head;                       // [num_streams]
  double* homography;                    // [num_streams][9], row-major, frame pixels -> ground units
  RecordIndex* index;                    // [num_streams][capacity]
  SpeedRec* rec;                         // [num_streams][capacity]
  double* ring;                          // [num_streams][capacity][window][3]: (t, x, y), x and y the anchor in pixels
};

// streams HOST, B distinct ids in [0, num_streams); timestamps DEVICE float64 [B] or null; everything else DEVICE.  A
// cudaError_t.
int speed_launch(const SpeedTable& t, const int32_t* ids, const float* boxes, const int32_t* counts, int B, int max_out,
                 const int32_t* streams, const double* timestamps, float* kin, int32_t* samples, cudaStream_t st);
// frame back to 1, no records, counters 0, last timestamp -inf, for n HOST stream ids; the homography is kept
int speed_reset_launch(const SpeedTable& t, const int32_t* streams, int n, cudaStream_t st);

}  // namespace lwb
