// Cross-view merge of tiled detection (lwdetr_tile_merge, include/lwdetr_b200.h): per frame, the per-view top-k of
// lwdetr_postprocess moved into frame pixels, sorted by score and thinned by a greedy class-aware NMS.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lwb {

constexpr int TILE_MAX_CAND = 16384;     // candidates (views * k) of one frame: the shared-memory sort
constexpr int TILE_MAX_DET = 1024;       // kept boxes per frame
constexpr int TILE_MAX_VIEWS = 2048;     // views of one frame: the view table travels in the kernel's parameters
enum { TILE_IOU = 0, TILE_IOS = 1 };

struct TileViewHost {
  int32_t frame, x0, y0;
};

// -2: a limit above is exceeded; otherwise a cudaError_t.  views: HOST, validated by the caller (frames non-decreasing in
// [0, num_frames)).
int tile_merge_launch(const float* scores, const int32_t* labels, const float* boxes, int V, int k, const TileViewHost* views,
                      int num_frames, float score_threshold, float iou_threshold, int metric, int max_det, float* out_scores,
                      int32_t* out_labels, float* out_boxes, int32_t* counts, cudaStream_t st);

}  // namespace lwb
