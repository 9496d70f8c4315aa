// Antialiased bilinear resize of raw uint8 HWC frames fused into the patch gather (see resize.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "lwdetr_b200.h"

namespace lwb {

// accepted frames: source sides in [kFrameMinSide, kFrameMaxSide], downscale factor n_in / dst <= kResizeMaxFactor per
// axis (at most 2 * factor + 1 = kResizeMaxTaps taps), any upscale factor, dst sides in [1, run side]
constexpr int kFrameMinSide = 8, kFrameMaxSide = 8192, kResizeMaxFactor = 16, kResizeMaxTaps = 2 * kResizeMaxFactor + 1;

// 0 when every frame is one the kernel runs, else -1 with the broken limit named in *err.  Host only, launches nothing.
int frames_check(const lwdetr_frame* frames, int B, int H, int W, std::string* err);
int frames_check(const lwdetr_frame_nv12* frames, int B, int H, int W, std::string* err);
// true when some frame leaves part of the H x W canvas unfilled (the batch then needs the padding mask)
bool frames_padded(const lwdetr_frame* frames, int B, int H, int W);
bool frames_padded(const lwdetr_frame_nv12* frames, int B, int H, int W);

// frames (HOST array of B descriptors with DEVICE data pointers) -> window-major patch matrix A [B*(H/16)*(W/16), 768] of
// an H x W run size: each frame resized to its (dst_h, dst_w), normalised, placed top-left; the rest of the canvas is 0.
// The descriptors travel as kernel parameters: nothing is copied or allocated, the array is free when the call returns.
int resize_patches_launch(int dtype, const lwdetr_frame* frames, int B, int H, int W, const float* mean, const float* stdv, void* A,
                          cudaStream_t st);
// the same for NV12 frames: each pixel converted to RGB (include/lwdetr_b200.h), then exactly the RGB frame's result
int resize_patches_launch(int dtype, const lwdetr_frame_nv12* frames, int B, int H, int W, const float* mean, const float* stdv, void* A,
                          cudaStream_t st);
// padding mask [B, H, W] (1 = outside the frame's dst_h x dst_w) of the same batch
int frame_mask_launch(const lwdetr_frame* frames, int B, int H, int W, uint8_t* mask, cudaStream_t st);
int frame_mask_launch(const lwdetr_frame_nv12* frames, int B, int H, int W, uint8_t* mask, cudaStream_t st);

}  // namespace lwb
