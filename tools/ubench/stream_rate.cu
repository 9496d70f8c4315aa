// Micro-benchmark: how fast can one launch STREAM a large buffer out of HBM into the SMs, by path?
//   bulk : one producer thread per CTA issues cp.async.bulk (1-D TMA) chunks into a shared-memory ring, consumers only recycle
//          the stages (chunk size x ring depth sweep, 1 or 2 CTAs per SM)
//   ldg  : every thread issues 16-byte ld.global.nc loads (8 in flight per thread), 1024 / 2048 threads per SM
// The buffer (1 GiB) is larger than the L2; every byte is read once.  Motivation: msda.cu stages 51 KB value slabs with
// bulk copies - is its rate the TMA path's limit or the kernel's?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/ubench/stream_rate tools/ubench/stream_rate.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../../lw-detr_b200/csrc/ptx.cuh"
using namespace lwb;

__global__ void __launch_bounds__(160) k_bulk(const uint8_t* src, size_t total, int chunk, int stages, unsigned long long* sink) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + (size_t)stages * chunk);
  uint64_t* empty = full + stages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    fence_mbar_init();
  }
  __syncthreads();
  const size_t nchunks = total / chunk;
  if (warp == 0) {
    if (lane == 0) {
      uint32_t ring = 0;
      for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x, ++ring) {
        const int s = ring % stages;
        mbar_wait(&empty[s], ((ring / stages) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], chunk);
        bulk_load(sm + (size_t)s * chunk, src + c * chunk, chunk, &full[s]);
      }
    }
  } else {
    uint32_t ring = 0;
    unsigned long long acc = 0;
    for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x, ++ring) {
      const int s = ring % stages;
      mbar_wait(&full[s], (ring / stages) & 1);
      acc += *reinterpret_cast<const uint32_t*>(sm + (size_t)s * chunk + threadIdx.x * 4);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    if (acc == 0x1234567) sink[0] = acc;
  }
}

__global__ void __launch_bounds__(1024) k_ldg(const uint4* src, size_t n16, unsigned long long* sink) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t acc = 0;
  for (; i + 7 * stride < n16; i += 8 * stride) {
    uint4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[j].x), "=r"(v[j].y), "=r"(v[j].z), "=r"(v[j].w) : "l"(src + i + j * stride));
#pragma unroll
    for (int j = 0; j < 8; ++j) acc ^= v[j].x ^ v[j].y ^ v[j].z ^ v[j].w;
  }
  if (acc == 0x1234567) sink[0] = acc;
}

int main() {
  const size_t total = 1ull << 30;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  if (sms <= 0) { fprintf(stderr, "no CUDA device\n"); return 1; }
  uint8_t* buf;
  unsigned long long* sink;
  cudaMalloc(&buf, total);
  cudaMalloc(&sink, 8);
  cudaMemset(buf, 1, total);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaFuncSetAttribute(k_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  struct Cfg { int chunk, stages, ctas_per_sm; };
  const Cfg cfgs[] = {{51200, 4, 1}, {51200, 2, 2}, {25600, 8, 1}, {16384, 12, 1}, {8192, 24, 1}, {4096, 48, 1}, {16384, 6, 2}, {8192, 12, 2}, {2048, 48, 2}};
  for (const Cfg& c : cfgs) {
    const size_t smem = (size_t)c.chunk * c.stages + 16 * c.stages + 64;
    for (int rep = 0; rep < 3; ++rep) {
      cudaEventRecord(e0);
      k_bulk<<<sms * c.ctas_per_sm, 160, smem>>>(buf, total, c.chunk, c.stages, sink);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      float ms;
      cudaEventElapsedTime(&ms, e0, e1);
      if (rep == 2) printf("bulk  chunk %6d B x %2d stages x %d CTA/SM (%3zu KB in flight/SM): %7.1f us  %6.2f TB/s  [%s]\n", c.chunk, c.stages, c.ctas_per_sm,
                           smem * c.ctas_per_sm / 1024, ms * 1e3, total / (ms * 1e-3) / 1e12, cudaGetErrorString(cudaGetLastError()));
    }
  }
  for (int tpb : {512, 1024})
    for (int cps : {1, 2}) {
      if (tpb * cps > 2048) continue;
      for (int rep = 0; rep < 3; ++rep) {
        cudaEventRecord(e0);
        k_ldg<<<sms * cps, tpb>>>(reinterpret_cast<const uint4*>(buf), total / 16, sink);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep == 2) printf("ldg   %4d threads x %d CTA/SM, 8 x 16 B in flight per thread: %7.1f us  %6.2f TB/s\n", tpb, cps, ms * 1e3, total / (ms * 1e-3) / 1e12);
      }
    }
  return 0;
}
