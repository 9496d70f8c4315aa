// Detection crops out of raw frames for second-stage networks (lwdetr_crops, lwdetr_crop_select, lwdetr_scatter_rows; see crops.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "lwdetr_b200.h"

namespace lwb {

constexpr int kCropMinSide = 8, kCropMaxSide = 1024;   // output sides
constexpr int kCropMaxCount = 65536, kCropMaxFrames = 1024;

struct CropDesc {
  int out_h, out_w, filter, normalize, etype;          // etype: LWDETR_ET_*
  float mean[3], stdv[3];
};

// 0 when every frame is one the crop kernel reads (pointers, sides in [kFrameMinSide, kFrameMaxSide], pitches, colour space),
// else -1 with the broken limit named in *err.  Host only.
int crop_frames_check(const lwdetr_frame* frames, int B, std::string* err);
int crop_frames_check(const lwdetr_frame_nv12* frames, int B, std::string* err);
// frames: HOST array of B validated descriptors (dst sides unused); boxes fp32 [N, 4], frame_index int32 [N], count int32 [1] or
// NULL, out [N, 3, out_h, out_w] of etype, valid int8 [N]: DEVICE.  A cudaError_t, or -2 when a group's shared memory exceeds
// what a CTA can have.
int crops_launch(const lwdetr_frame* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                 const CropDesc& d, void* out, int8_t* valid, cudaStream_t st);
int crops_launch(const lwdetr_frame_nv12* frames, int B, const float* boxes, const int32_t* frame_index, int N, const int32_t* count,
                 const CropDesc& d, void* out, int8_t* valid, cudaStream_t st);
// sizes: HOST int32 [B][2] (height, width)
int crop_select_launch(const float* scores, const float* boxes, int B, int k, const int32_t* sizes, float threshold, int32_t* frame_of,
                       int32_t* entry, float* sel_boxes, int32_t* count, cudaStream_t st);
int scatter_rows_launch(int etype, const void* rows, int ld_rows, int D, const int32_t* entry, const int32_t* count, int N, void* out,
                        int num_out, cudaStream_t st);

}  // namespace lwb
