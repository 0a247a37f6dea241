// tma.cuh — Hopper (sm_90a) tensor-copy and mbarrier primitives for the TMA-fed kernel hk_update_R_x32 (hh_api.cu),
// and the host side that encodes its fp64 tensor maps.
//
// Every barrier here is a CTA-local mbarrier in shared memory (the .shared::cluster destinations of the copies are this
// CTA's own shared memory: the kernel is launched without clusters).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

__device__ inline unsigned tma_smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

// COUNT arrivals complete a phase (a compile-time immediate of the PTX instruction)
template <unsigned COUNT> __device__ inline void tma_mbar_init(unsigned long long *bar)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tma_smem_u32(bar)), "n"(COUNT));
}
// after the mbarrier.init of a CTA: make them visible to the other threads and to the async (TMA) proxy
__device__ inline void tma_fence_mbar_init()
{
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ inline void tma_mbar_arrive(unsigned long long *bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tma_smem_u32(bar)) : "memory");
}
// arrive and announce `bytes` of copies that complete on this phase
__device__ inline void tma_mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tma_smem_u32(bar)), "r"(bytes) : "memory");
}
// spin until the phase of parity `parity` has completed
__device__ inline void tma_mbar_wait(unsigned long long *bar, unsigned parity)
{
  asm volatile("{\n\t"
               ".reg .pred p;\n\t"
               "WAIT_%=:\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
               "@p bra DONE_%=;\n\t"
               "bra WAIT_%=;\n\t"
               "DONE_%=:\n\t"
               "}" ::"r"(tma_smem_u32(bar)),
               "r"(parity)
               : "memory");
}
// the same test once, without waiting
__device__ inline bool tma_mbar_test(unsigned long long *bar, unsigned parity)
{
  unsigned ok;
  asm volatile("{\n\t"
               ".reg .pred p;\n\t"
               "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
               "selp.u32 %0, 1, 0, p;\n\t"
               "}"
               : "=r"(ok)
               : "r"(tma_smem_u32(bar)), "r"(parity)
               : "memory");
  return ok != 0;
}

// copies global -> shared memory that complete on `bar` (byte count announced with tma_mbar_expect_tx)
__device__ inline void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, unsigned long long *bar)
{
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::
                   "r"(tma_smem_u32(dst)),
               "l"(map), "r"(c0), "r"(c1), "r"(tma_smem_u32(bar))
               : "memory");
}

// Host: an fp64 tiled tensor map of `rank` (<= 5) dimensions, element strides 1, no interleave, no out-of-bounds NaN
// fill.  cuTensorMapEncodeTiled is a driver function: it is resolved once through the runtime, so the libraries need no
// link-time libcuda.  False when the driver lacks it or rejects the map.
inline bool tma_encode_f64(CUtensorMap *map, void *base, int rank, const cuuint64_t *dims, const cuuint64_t *strides,
                           const cuuint32_t *box, CUtensorMapSwizzle swizzle, CUtensorMapL2promotion promo)
{
  typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const EncodeTiledFn fn = []() -> EncodeTiledFn {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      return (EncodeTiledFn)p;
    return nullptr;
  }();
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  return fn && fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, (cuuint32_t)rank, base, dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
