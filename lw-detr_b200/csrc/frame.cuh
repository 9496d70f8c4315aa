// What the frame readers (resize.cu, crops.cu) share about the two source formats of include/lwdetr_b200.h: the NV12 -> RGB
// coefficient rows and rounding, and the host-side checks of a descriptor's pointers and layout.
#pragma once
#include <stdint.h>

#include <string>

#include "lwdetr_b200.h"

namespace lwb {
namespace {
// NV12 -> RGB rows of include/lwdetr_b200.h: cY, cRv, cGu, cGv, cBu per colorspace; codes 0 and 1 are limited range
__constant__ int kCsc[4][5] = {{1220542, 1673527, -409993, -852492, 2116026},
                               {1220945, 1879825, -223607, -558796, 2215014},
                               {1048576, 1470104, -360853, -748826, 1858077},
                               {1048576, 1651297, -196424, -490864, 1945738}};

__device__ __forceinline__ int shift20(int v) { return min(max((v + (1 << 19)) >> 20, 0), 255); }

// what is wrong with a frame's plane pointers, and (checked after its sides) with its pitches and colour space: "" when nothing
inline std::string pointers_error(const lwdetr_frame& f) { return f.data ? "" : "null data pointer"; }
inline std::string pointers_error(const lwdetr_frame_nv12& f) { return !f.luma ? "null luma pointer" : !f.chroma ? "null chroma pointer" : ""; }
inline std::string layout_error(const lwdetr_frame& f) {
  if (f.pitch_bytes < 3LL * f.width) return "pitch_bytes " + std::to_string(f.pitch_bytes) + " is smaller than 3 * width";
  return "";
}
inline std::string layout_error(const lwdetr_frame_nv12& f) {
  if (f.luma_pitch < f.width) return "luma_pitch " + std::to_string(f.luma_pitch) + " is smaller than width";
  const long long cw = 2LL * ((f.width + 1) / 2);
  if (f.chroma_pitch < cw) return "chroma_pitch " + std::to_string(f.chroma_pitch) + " is smaller than 2 * ceil(width / 2) = " + std::to_string(cw);
  if (f.colorspace < LWDETR_CSC_BT601_LIMITED || f.colorspace > LWDETR_CSC_BT709_FULL)
    return "unknown colorspace " + std::to_string(f.colorspace) + " (LWDETR_CSC_BT601_LIMITED .. LWDETR_CSC_BT709_FULL)";
  return "";
}
}  // namespace
}  // namespace lwb
