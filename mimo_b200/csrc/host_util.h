// Host-side helpers shared by the C-ABI translation units: error reporting, device checks, TMA tensor-map
// encoding through the driver entry point (no link-time dependency on libcuda, so the library loads — and
// exports its symbols — on a machine without a GPU driver).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace mimo {

int set_error(int code, const char* msg);
int set_cuda_error(const char* what, cudaError_t e);
// MIMO_OK if the current device is sm_90 (cached per process); error otherwise.
int ensure_device();
int num_sms();
// tensor-map element type for one-byte (e4m3) operands; otherwise `dtype` is MIMO_F16 / MIMO_BF16
constexpr int kTmapU8 = 0x100;
// rank-`rank` tiled tensor map, 16-bit (or, with kTmapU8, one-byte) elements, 128-byte swizzle (or 64, 32, 0 = none),
// zero OOB fill.
// dims[0] is the contiguous dimension; strides_bytes[i] is the byte stride of dims[i+1].
int encode_tmap(CUtensorMap* out, int dtype, int rank, const void* base, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128);

inline unsigned div_up(long long a, long long b) { return static_cast<unsigned>((a + b - 1) / b); }

// Programmatic dependent launch (mimo_debug_pdl / MIMO_B200_PDL=1; default OFF): every kernel of the library can be
// launched with programmatic stream serialization; it begins with griddepcontrol.launch_dependents and, after its
// shared-memory prologue, griddepcontrol.wait, so the next kernel's launch latency and prologue overlap the tail
// of the previous one (~14 000 kernel boundaries per clip). Correctness does not depend on it: the wait is a full
// dependency on the previous grid (completion + memory visibility); without the attribute both instructions are no-ops.
// Off by default; kept as a switch for launch-bound regimes.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace mimo
