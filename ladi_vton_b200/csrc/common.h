// Host-side helpers shared by the C-ABI translation units: error reporting and TMA tensor-map encoding.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ladi_b200.h"

typedef __nv_bfloat16 bf16;

// thread-local last error (ladi_last_error); every entry point returns 0 on success, non-zero otherwise,
// and never throws or aborts across the ABI.
void ladi_set_error(const char* fmt, ...);

#define LADI_CHECK(cond, ...)       \
  do {                              \
    if (!(cond)) {                  \
      ladi_set_error(__VA_ARGS__);  \
      return LADI_ERR_INVALID;      \
    }                               \
  } while (0)

#define LADI_CUDA(call)                                                                          \
  do {                                                                                           \
    cudaError_t e__ = (call);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      ladi_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return LADI_ERR_CUDA;                                                                      \
    }                                                                                            \
  } while (0)

// Encodes a bf16 tensor map (rank <= 5), SWIZZLE_128B, zero OOB fill.  dims/box innermost first; strides in BYTES for
// dims 1..rank-1.  Returns 0 on success.
int ladi_encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box, int swizzle_bytes = 128);
// The same for fp32 elements (box[0] * 4 <= 128 bytes under the 128-byte swizzle).
int ladi_encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box);

int ladi_num_sms();
void ladi_count_launch();  // every successful kernel launch of the library (ladi_launch / ladi_launch_cluster) -> ladi_launch_count()
int ladi_pdl_enabled();  // env LADI_PDL=0 disables programmatic dependent launch (A/B timing)
int ladi_conv_pair_default();  // 1 = 2-CTA cluster conv kernels where they apply (env LADI_CONV_2CTA=1); default 0 = single-CTA only

#ifdef __CUDACC__
#include <utility>
// Every kernel of the library is launched through this helper (programmatic stream serialization attribute, see ptx.cuh).
template <typename... KArgs, typename... Args>
inline cudaError_t ladi_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = ladi_pdl_enabled() ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
  if (e == cudaSuccess) ladi_count_launch();
  return e;
}
// Same, as thread-block clusters of `cluster_x` CTAs along x (grid.x must be a multiple of it).
template <typename... KArgs, typename... Args>
inline cudaError_t ladi_launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, unsigned cluster_x, size_t smem, cudaStream_t stream,
                                       Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster_x; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = ladi_pdl_enabled() ? 2 : 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
  if (e == cudaSuccess) ladi_count_launch();
  return e;
}
#endif
