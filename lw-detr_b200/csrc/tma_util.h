// Host helper: build CUtensorMap descriptors through the driver entry point (libcuda is never linked).
#pragma once
#include <cuda.h>
#include <string>

namespace lwb {

// swizzle_bytes in {32, 64, 128}; dtype: DT_F16 / DT_BF16 / DT_E4M3 (1-byte elements); rank 2..5; dims/strides/box as in cuTensorMapEncodeTiled
int tma_encode(CUtensorMap* tm, int dtype, int rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, int swizzle_bytes, std::string* err);

}  // namespace lwb
