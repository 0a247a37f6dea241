// ubench_read.cu — what can a read-mostly kernel pull out of HBM on this GPU?  The roofline denominator of bench.py is
// the driver's COPY bandwidth (MEASURED_PEAKS.json: read + write bytes of a device-to-device copy); update_gso_row is
// read-only, and its reads are 2960 concurrent streams (one per lattice) of 256-byte lines rather than one linear sweep.
//   mode 0: linear sweep, every thread 16-byte loads, grid-stride (the friendliest pattern there is)
//   mode 1: one stream per warp: warp w reads its own contiguous region of `per` bytes in 256-byte lines, 16 lines in
//           flight per warp, 20 warps per SM (k_update_row's geometry: 5920 lattices x 485 KB)
//   mode 2: as 1 with 40 lines in flight per warp
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_read tools/ubench_read.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

__global__ void k_linear(const double2 *p, size_t n, double *out)
{
  double acc = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
  {
    const double2 v = p[i];
    acc += v.x + v.y;
  }
  if (acc == 1.2345e-300)
    *out = acc;
}

template <int DEPTH> __global__ void __launch_bounds__(128, 5) k_streams(const double *p, size_t per_dbl, int nstreams, double *out)
{
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= nstreams)
    return;
  const double *s = p + (size_t)w * per_dbl + lane;
  const size_t lines = per_dbl / 32;
  double acc = 0;
  for (size_t k = 0; k + DEPTH <= lines; k += DEPTH)
  {
    double x[DEPTH];
#pragma unroll
    for (int u = 0; u < DEPTH; u++)
      x[u] = s[(k + u) * 32];
#pragma unroll
    for (int u = 0; u < DEPTH; u++)
      acc += x[u];
  }
  if (acc == 1.2345e-300)
    *out = acc;
}

int main()
{
  const int nstreams = 5920;
  const size_t per = 485632;  // bytes per stream, multiple of 256 (update_gso_row(199): 485 608 algorithmic bytes)
  const size_t bytes = per * nstreams;
  double *buf, *out;
  cudaMalloc(&buf, bytes);
  cudaMalloc(&out, 8);
  cudaMemset(buf, 0, bytes);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  for (int mode = 0; mode < 3; mode++)
  {
    float best = 1e30f;
    for (int rep = 0; rep < 12; rep++)
    {
      cudaEventRecord(e0);
      if (mode == 0)
        k_linear<<<132 * 16, 256>>>((const double2 *)buf, bytes / 16, out);
      else if (mode == 1)
        k_streams<16><<<(nstreams + 3) / 4, 128>>>(buf, per / 8, nstreams, out);
      else
        k_streams<40><<<(nstreams + 3) / 4, 128>>>(buf, per / 8, nstreams, out);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      float ms;
      cudaEventElapsedTime(&ms, e0, e1);
      if (rep >= 2 && ms < best)
        best = ms;
    }
    printf("mode %d: %.4f ms  %.1f GB/s (%s)\n", mode, best, bytes / (best * 1e-3) / 1e9,
           mode == 0 ? "linear sweep, 2.87 GB" : mode == 1 ? "5920 streams x 485 KB, 16 lines in flight per warp" : "5920 streams, 40 lines in flight per warp");
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
