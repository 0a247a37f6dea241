// ubench_lat.cu — dependent-issue latencies that bound the single-lattice LLL chains on the GPU (one warp, clock64):
// fp64 add / mul / sub chains, the shuffle-multiply-subtract step of the triangular solves, shared / L2 loads,
// named and cluster barriers, DSMEM.  Build: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false -O3 -o ubench_lat
#include <cooperative_groups.h>
#include <cstdio>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

constexpr int N = 2048;

__global__ void k_dadd(double *out, double x, double y)
{
  double a = x;
  const long long t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++)
    a = __dadd_rn(a, y);
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / N, out[1] = a;
}
__global__ void k_dmul_dsub(double *out, double x, double y)
{
  double a = x;
  const long long t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++)
    a = __dsub_rn(a, __dmul_rn(a, y));  // mul depends on a, sub depends on mul: the triangle's arithmetic
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / N, out[1] = a;
}
__global__ void k_tri_step(double *out, double x, double y)
{
  double a = x + threadIdx.x;
  const long long t0 = clock64();
#pragma unroll 32
  for (int i = 0; i < N; i++)
  {
    const double rk = __shfl_sync(0xffffffffu, a, i & 31);
    if ((int)(threadIdx.x & 31) > (i & 31))
      a = __dsub_rn(a, __dmul_rn(y, rk));
  }
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / N, out[1] = a;
}
__global__ void k_rnd(double *out, double x, double y)
{
  double a = x;
  const long long t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++)
    a = __dsub_rn(a, __dmul_rn(rint(a), y));
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / N, out[1] = a;
}
__global__ void k_lds_chase(double *out)
{
  __shared__ int nxt[1024];
  for (int i = threadIdx.x; i < 1024; i += blockDim.x)
    nxt[i] = (i * 37 + 11) & 1023;
  __syncthreads();
  int p = threadIdx.x;
  const long long t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; i++)
    p = nxt[p];
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / N, out[1] = p;
}
__global__ void k_l2_chase(double *out, const int *nxt)
{
  int p = threadIdx.x;
  const long long t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < 512; i++)
    p = __ldcg(nxt + p);
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / 512, out[1] = p;
}
__global__ void k_bar(double *out)
{
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++)
    asm volatile("bar.sync 1, 256;" ::: "memory");
  const long long t1 = clock64();
  if (threadIdx.x == 0)
    out[0] = (double)(t1 - t0) / 256;
}
__global__ void __cluster_dims__(4, 1, 1) k_cluster(double *out)
{
  cg::cluster_group cl = cg::this_cluster();
  __shared__ double buf[64];
  buf[threadIdx.x & 63] = threadIdx.x;
  cl.sync();
  const long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++)
    cl.sync();
  const long long t1 = clock64();
  // barrier without the L1 invalidation cooperative_groups' sync implies: raw arrive.release / wait.acquire
  const long long t2 = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++)
  {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
  const long long t3 = clock64();
  // relaxed form (no memory ordering)
#pragma unroll 1
  for (int i = 0; i < 256; i++)
  {
    asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
  }
  const long long t4 = clock64();
  // DSMEM dependent load chain from the next CTA of the cluster
  double *remote = cl.map_shared_rank(buf, (cl.block_rank() + 1) & 3);
  double acc = 0;
  int idx = threadIdx.x & 63;
  const long long t5 = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; i++)
  {
    const double vv = remote[idx];
    idx = ((int)vv + i) & 63;
    acc += vv;
  }
  const long long t6 = clock64();
  cl.sync();
  if (threadIdx.x == 0 && blockIdx.x == 0)
  {
    out[0] = (double)(t1 - t0) / 256, out[1] = (double)(t3 - t2) / 256, out[2] = (double)(t4 - t3) / 256;
    out[3] = (double)(t6 - t5) / 256, out[4] = acc;
  }
}

int main()
{
  double *d, h[8];
  cudaMalloc(&d, 64);
  int *nxt, hn[1 << 16];
  for (int i = 0; i < (1 << 16); i++)
    hn[i] = (i * 4099 + 77) & 0xffff;
  cudaMalloc(&nxt, sizeof(hn));
  cudaMemcpy(nxt, hn, sizeof(hn), cudaMemcpyHostToDevice);
#define RUN(name, call, nout)                                      \
  for (int rep = 0; rep < 2; rep++)                                \
  {                                                                \
    call;                                                          \
    cudaDeviceSynchronize();                                       \
    cudaMemcpy(h, d, 64, cudaMemcpyDeviceToHost);                  \
  }                                                                \
  printf("%-28s", name);                                           \
  for (int q = 0; q < nout; q++)                                   \
    printf(" %8.1f", h[q]);                                        \
  printf("   (%s)\n", cudaGetErrorString(cudaGetLastError()));
  RUN("dadd chain cyc/op", (k_dadd<<<1, 32>>>(d, 1.0, 1e-9)), 1);
  RUN("dmul->dsub chain cyc/step", (k_dmul_dsub<<<1, 32>>>(d, 1.0, 1e-9)), 1);
  RUN("shfl+dmul+dsub tri step", (k_tri_step<<<1, 32>>>(d, 1.0, 1e-9)), 1);
  RUN("rint+dmul+dsub step", (k_rnd<<<1, 32>>>(d, 1.5, 1e-9)), 1);
  RUN("LDS chase cyc/load", (k_lds_chase<<<1, 32>>>(d)), 1);
  RUN("L2 chase cyc/load", (k_l2_chase<<<1, 32>>>(d, nxt)), 1);
  RUN("bar.sync 256 thr", (k_bar<<<1, 256>>>(d)), 1);
  RUN("cluster4: cg sync | arrive.release+wait.acquire | relaxed | DSMEM load", (k_cluster<<<4, 256>>>(d)), 4);
  return 0;
}
