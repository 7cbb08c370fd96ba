// ea_internal.h — declarations shared between the translation units of libea_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <string.h>
#include "../../include/editanything_b200.h"

typedef CUresult (*ea_tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                      const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                      const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// Resolved through cudaGetDriverEntryPoint (no link-time libcuda dependency).
ea_tmap_encode_fn ea_tmap_encode();
void ea_count_launch();
// Per-device caches: cudaFuncSetAttribute and the SM count belong to a DEVICE, not to the process - a process that
// drives a second GPU must set / query them there too.  Tables are indexed by ea_dev() (current device, < EA_MAX_DEV).
#define EA_MAX_DEV 32
static inline int ea_dev() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0) d = 0;
  return d < EA_MAX_DEV ? d : EA_MAX_DEV - 1;
}
int ea_sm_count();   // SMs of the current device (cached per device)
// Remembers the CUDA error behind an EA_ERR_CUDA status (ea_last_error() returns it); returns EA_ERR_CUDA.
int ea_cuda_fail(cudaError_t e, const char* where);

// Programmatic dependent launch (PDL): every kernel of this library calls griddepcontrol.wait before
// it touches global memory, so consecutive launches on a stream may overlap the next kernel's
// prologue (barrier init, tensor-map prefetch, block scheduling) with the tail of
// the previous one.  ea_set_pdl(0) / EA_PDL=0 falls back to plain stream serialisation.
int ea_pdl_enabled();
#ifdef __CUDACC__
#include <utility>
template <typename... KArgs, typename... Args>
static inline cudaError_t ea_launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                            cudaStream_t stream, unsigned cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (ea_pdl_enabled()) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster_x > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster_x;
    at[n].val.clusterDim.y = 1;
    at[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
}
template <typename... KArgs, typename... Args>
static inline cudaError_t ea_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                    cudaStream_t stream, Args&&... args) {
  return ea_launch_cluster(kernel, grid, block, smem, stream, 1u, std::forward<Args>(args)...);
}
#endif
