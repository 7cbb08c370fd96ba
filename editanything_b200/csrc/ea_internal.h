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
static inline cudaError_t ea_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                    cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at;
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &at;
  cfg.numAttrs = ea_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
}
#endif
