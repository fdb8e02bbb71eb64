// C-ABI glue: version / error / device entry points and the host utilities declared in host_util.h.
#include <cudaTypedefs.h>
#include <stdio.h>
#include <string.h>

#include "../../include/mimo_b200.h"
#include "host_util.h"

namespace mimo {

static thread_local char g_err[512] = "";

int set_error(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}
int set_cuda_error(const char* what, cudaError_t e) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return MIMO_ERR_CUDA;
}

static int g_dev_state = 0;  // 0 unknown, 1 ok, -1 bad
static int g_num_sms = 132;

int ensure_device() {
  if (g_dev_state == 1) return MIMO_OK;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_cuda_error("cudaGetDevice (no CUDA device: this library has no CPU fallback)", e);
    return MIMO_ERR_DEVICE;
  }
  int major = 0, minor = 0, sms = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (major != 9 || minor != 0) {  // sm_90a code (wgmma, setmaxnreg) loads on compute capability 9.0 only
    snprintf(g_err, sizeof(g_err), "device %d is sm_%d%d; mimo_b200 kernels are built for sm_90a only", dev,
             major, minor);
    g_dev_state = -1;
    return MIMO_ERR_DEVICE;
  }
  g_num_sms = sms > 0 ? sms : 132;
  g_dev_state = 1;
  return MIMO_OK;
}
int num_sms() { return g_num_sms; }

static bool g_pdl = false;  // off unless mimo_debug_pdl(1) / MIMO_B200_PDL=1
bool pdl_enabled() { return g_pdl; }

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

int encode_tmap(CUtensorMap* out, int dtype, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
      return set_error(MIMO_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  const CUtensorMapDataType dt =
      dtype == MIMO_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = g_encode(out, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr, bx, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                            : (swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_128B),
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(g_err, sizeof(g_err),
             "cuTensorMapEncodeTiled failed (CUresult %d): rank %d base %p dims [%llu %llu %llu %llu] box [%u %u "
             "%u %u] stride0 %llu",
             static_cast<int>(r), rank, base, (unsigned long long)gdim[0],
             (unsigned long long)(rank > 1 ? gdim[1] : 0), (unsigned long long)(rank > 2 ? gdim[2] : 0),
             (unsigned long long)(rank > 3 ? gdim[3] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0,
             rank > 3 ? bx[3] : 0, (unsigned long long)(rank > 1 ? gstr[0] : 0));
    return MIMO_ERR_CUDA;
  }
  return MIMO_OK;
}

}  // namespace mimo

extern "C" const char* mimo_version(void) { return "mimo_b200 0.1.0 (sm_90a)"; }
extern "C" const char* mimo_last_error(void) { return mimo::g_err; }

extern "C" int mimo_abi_sizeof(int which) {
  switch (which) {
    case 0: return static_cast<int>(sizeof(mimo_epilogue));
    case 1: return static_cast<int>(sizeof(mimo_gemm_params));
    case 2: return static_cast<int>(sizeof(mimo_conv3x3_params));
    case 3: return static_cast<int>(sizeof(mimo_groupnorm_params));
    case 4: return static_cast<int>(sizeof(mimo_attn_params));
    case 5: return static_cast<int>(sizeof(mimo_attn_temporal_params));
    case 6: return static_cast<int>(sizeof(mimo_exchange_params));
  }
  return -1;
}

extern "C" int mimo_device_check(int dev) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    mimo::set_error(MIMO_ERR_DEVICE, "no CUDA device visible; mimo_b200 has no CPU fallback");
    return MIMO_ERR_DEVICE;
  }
  if (dev < 0 || dev >= count) return mimo::set_error(MIMO_ERR_ARG, "mimo_device_check: bad device index");
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) return mimo::set_error(MIMO_ERR_DEVICE, "device is not sm_90 (H100)");
  return MIMO_OK;
}

// ---- peer-shareable memory for mimo_exchange (bootstrap only) ----
extern "C" int mimo_peer_alloc(int64_t bytes, void** ptr, void* handle64) {
  if (!ptr || !handle64 || bytes <= 0) return mimo::set_error(MIMO_ERR_ARG, "mimo_peer_alloc: bad arguments");
  if (int rc = mimo::ensure_device()) return rc;
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, static_cast<size_t>(bytes));
  if (e != cudaSuccess) return mimo::set_cuda_error("mimo_peer_alloc cudaMalloc", e);
  e = cudaMemset(p, 0, static_cast<size_t>(bytes));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    return mimo::set_cuda_error("mimo_peer_alloc", e);
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  memcpy(handle64, &h, 64);
  *ptr = p;
  return MIMO_OK;
}
extern "C" int mimo_peer_open(const void* handle64, void** ptr) {
  if (!ptr || !handle64) return mimo::set_error(MIMO_ERR_ARG, "mimo_peer_open: bad arguments");
  if (int rc = mimo::ensure_device()) return rc;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) return mimo::set_cuda_error("mimo_peer_open cudaIpcOpenMemHandle", e);
  *ptr = p;
  return MIMO_OK;
}
extern "C" int mimo_peer_close(void* ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  return e == cudaSuccess ? MIMO_OK : mimo::set_cuda_error("mimo_peer_close", e);
}
extern "C" int mimo_peer_free(void* ptr) {
  cudaError_t e = cudaFree(ptr);
  return e == cudaSuccess ? MIMO_OK : mimo::set_cuda_error("mimo_peer_free", e);
}

extern "C" int mimo_debug_pdl(int on) {
  mimo::g_pdl = on != 0;
  return 0;
}
