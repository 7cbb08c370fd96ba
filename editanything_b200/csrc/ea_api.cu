// ea_api.cu — library bookkeeping for the C ABI declared in include/editanything_b200.h.
#include <atomic>
#include <stdio.h>
#include <stdlib.h>
#include "ea_common.cuh"
#include "ea_internal.h"

static ea_tmap_encode_fn g_encode = nullptr;
static std::atomic<long long> g_launches{0};

static CUresult CUDAAPI encode_unavailable(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                           const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                           const cuuint32_t*, CUtensorMapInterleave,
                                           CUtensorMapSwizzle, CUtensorMapL2promotion,
                                           CUtensorMapFloatOOBfill) {
  return CUDA_ERROR_NOT_INITIALIZED;
}

ea_tmap_encode_fn ea_tmap_encode() {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e == cudaSuccess && fn && qres == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<ea_tmap_encode_fn>(fn);
    else
      g_encode = encode_unavailable;
  }
  return g_encode;
}

static int g_pdl = -1;
int ea_pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("EA_PDL");
    g_pdl = (e && e[0] == '0') ? 0 : 1;
  }
  return g_pdl;
}
extern "C" void ea_set_pdl(int on) { g_pdl = on ? 1 : 0; }

void ea_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

static char g_last_error[256] = "";
int ea_cuda_fail(cudaError_t e, const char* where) {
  snprintf(g_last_error, sizeof(g_last_error), "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
  return EA_ERR_CUDA;
}
extern "C" const char* ea_last_error(void) { return g_last_error; }

int ea_sm_count() {
  static int n_sm[EA_MAX_DEV] = {0};
  const int d = ea_dev();
  if (!n_sm[d]) {
    int n = 0;
    n_sm[d] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d) == cudaSuccess && n > 0) ? n : 132;
  }
  return n_sm[d];
}

extern "C" int ea_version(void) { return 1; }
extern "C" const char* ea_dtype_name(void) {
#ifdef EA_USE_BF16
  return "bfloat16";
#else
  return "float16";
#endif
}
extern "C" const char* ea_strerror(int s) {
  switch (s) {
    case EA_OK: return "ok";
    case EA_ERR_ARG: return "invalid argument";
    case EA_ERR_SHAPE: return "unsupported shape or alignment";
    case EA_ERR_TMAP: return "cuTensorMapEncodeTiled failed";
    case EA_ERR_CUDA: return "CUDA launch/runtime error";
    case EA_ERR_NODRIVER: return "CUDA driver entry point unavailable (no GPU / driver?)";
    default: return "unknown status";
  }
}
extern "C" int ea_init(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { cudaGetLastError(); return EA_ERR_NODRIVER; }
  ea_tmap_encode_fn f = ea_tmap_encode();
  return f == encode_unavailable ? EA_ERR_NODRIVER : EA_OK;
}
extern "C" long long ea_launch_count(void) { return g_launches.load(); }
extern "C" void ea_reset_launch_count(void) { g_launches.store(0); }
