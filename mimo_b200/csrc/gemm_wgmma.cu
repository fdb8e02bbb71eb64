// Persistent, warp-specialised wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M,N] = epilogue( A[M,K] . W[N,K]^T )          fp16/bf16 operands, fp32 accumulate in registers
//
// One CTA per SM loops over 128 x BN output tiles (static round-robin schedule, n-tile fastest so that CTAs
// running concurrently share A tiles in L2). Every byte that crosses the SM boundary moves by TMA; no thread issues
// a scattered global load or store on the steady-state path. Roles (320 threads: two warpgroups and two warps):
//   warpgroups 0 and 1  : MMA + epilogue    - warpgroup w issues wgmma.m64nBNk16 for tile rows [64 w, 64 w + 64),
//                                             fp32 accumulators in registers. Epilogue per 32-column chunk:
//                                             acc * scale + column constants (bias + per-branch vector, staged in smem
//                                             before the main loop) + residual (smem ring) -> SiLU / GEGLU ->
//                                             64B-swizzled staging buffer shared by both warpgroups -> one TMA store
//   warp 8              : TMA producer      - ring of {A 128x64, W BNx64} 128B-swizzled stages; it runs on into the
//                                             next tile while the MMA warpgroups are in the epilogue of this one
//   warp 9              : residual producer (kRes) - TMA boxes of the residual tensor, 128 rows x 32 columns each, into
//                                             a ring of 8 KiB slots
// Convolution mode replaces the A loads by 4-D TMA boxes {64 ch, TW, TH, TN} over the NHWC input, one box per
// (tap, 64-channel block, source tensor); TMA's out-of-bounds zero fill is the conv's zero padding and also
// the K tail, and the output / residual boxes use the same {TW, TH, TN} footprint (stores are clipped at image
// borders). Two source tensors give the up-blocks' channel concat without materialising it.
// E4M3 mode (mimo_gemm_e4m3, GEMM rows) runs the same roles on fp8 A and W: a K block is 128 one-byte elements, the
// same 128-byte swizzle row and stage bytes, four wgmma.m64nBNk32.e4m3 per block; the epilogue first takes
// acc * a_scale[row] * w_scale[col] in fp32 and then runs the chain above unchanged. mimo_conv3x3_e4m3 is conv mode in
// e4m3 (conv_e4m3_kernel): 128-channel boxes, single source, and a_scale per image of the output pixel.
// The FP8 feed-forward adds two more e4m3 variants of the same body: mimo_gemm_e4m3_geglu_e4m3 (gemm_e4m3_geglu_e4m3_kernel)
// ends the GEGLU epilogue in e4m3 with one scale per row and 128-column block instead of a 16-bit store, and
// mimo_gemm_e4m3_blockscaled (gemm_blockscaled_kernel) reads A with one scale per row and 128-element K block: each K
// block's four wgmma accumulate on their own, and the main loop adds them, times the block's row scale, into the sum.
#include <cuda_runtime.h>

#include <cudaTypedefs.h>

#include <cstdio>
#include <type_traits>

#include "../../include/mimo_b200.h"
#include "host_util.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace mimo {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 x 16-bit = one 128-byte swizzle row
constexpr int kGemmThreads = 320;  // two MMA / epilogue warpgroups, operand producer warp, residual producer warp
constexpr int kChunk = 8192;  // one 128-row x 32-column (64 B) epilogue chunk

struct EpiArgs {
  const void* bias;
  const void* rowvec;
  long long rows_per_group;
  long long ld_rowvec;
  float scale;
  int act;
  float* partial;    // split-K: fp32 accumulators go to partial[split][row][N] instead of the epilogue (else nullptr)
};

struct ConvGeom {
  int conv;  // 0: plain GEMM rows; 1: rows are (n, y, x) footprints
  int H, W, NI;
  int TW, TH, TN;
  int tiles_w, tiles_h;
  int ctot;         // c0 + c1
  int c0;           // channels of source 0 (GEMM mode: K of source 0)
  int kb0, kb1;     // 64-wide K blocks (per tap in conv mode) of source 0 / 1
  int a_bytes;      // bytes one A box deposits in shared memory
  int chunk_bytes;  // bytes one output / residual box moves (TW*TH*TN rows x 64 B)
  int splits;       // split-K factor (1 = off): tile index = (m_tile * n_tiles + n_tile) * splits + split
  int kb_split;     // K blocks per split
  int ntaps;        // 9 (3x3) or 4 (one parity class of nearest-x2 upsample + 3x3, see mimo_conv_up2x)
  signed char tdx[9], tdy[9];  // input offset of tap t relative to the output pixel
};

template <int BN, bool kRes, bool kE4m3 = false, bool kBlockScale = false>
struct GemmCfg {
  // kBlockScale: the K block's 128 fp32 row scales follow W in the stage (512 B, padded to keep stages 1024-B aligned)
  static constexpr int kStageBytes = BM * BK * 2 + BN * BK * 2 + (kBlockScale ? 1024 : 0);
  static constexpr int kNChunk = BN / 32;
  static constexpr int kOutBytes = 2 * kChunk;  // double-buffered staging of the output chunks
  static constexpr int kResSlots = kRes ? 2 : 0;
  static constexpr int kResBytes = kResSlots * kChunk;
  static constexpr int kBarBytes = 512;
  // e4m3 adds [2][256] column and [2][128] row scales (3 KiB). At BN = 256 with a residual that leaves room for 3 stages
  // instead of 4; the engine's e4m3 GEMMs (q|k|v, GEGLU) take no residual and keep 4.
  static constexpr int kFixed = kBarBytes + 2048 /*sbias*/ + (kE4m3 ? 3072 /*column, row scales*/ : 0) + kOutBytes + kResBytes;
  static constexpr int kMaxStages = (BN >= 256) ? 4 : (BN >= 160 ? 5 : (BN >= 128 ? 6 : 8));
  static constexpr int kFit = (227 * 1024 - kFixed) / kStageBytes;
  static constexpr int kStages = kFit < kMaxStages ? kFit : kMaxStages;
  static constexpr int kSmemBytes = kStages * kStageBytes + kFixed;
  static_assert(kStages >= 3, "pipeline too shallow");
};

template <int BN, bool kBf16, bool kRes>
// (registers are reserved per group of 4 warps: 320 threads hold 12 warps' worth, so at most 168 per thread)
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                  const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                  const __grid_constant__ CUtensorMap tmRes, int M, int N, int num_m_tiles, int num_n_tiles,
                  int num_k_blocks, ConvGeom g, EpiArgs ep) {
  constexpr bool kE4m3 = false, kImgScale = false;
  [[maybe_unused]] constexpr const float* a_scale = nullptr;
  [[maybe_unused]] constexpr const float* w_scale = nullptr;
  constexpr bool kOutE4m3 = false, kBlockScale = false;
  [[maybe_unused]] constexpr float* out_scale = nullptr;
  [[maybe_unused]] constexpr long long ld_scale = 0;
  [[maybe_unused]] const CUtensorMap& tmAS = tmA0;
#include "gemm_wgmma_body.cuh"
}

// e4m3 A [M, K] and W [N, K] with one fp32 scale per row of each, 16-bit output: GEMM rows only (g.conv == 0, tmA1 ==
// tmA0 and never read, no split-K)
template <int BN, bool kBf16, bool kRes>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_e4m3_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                 const __grid_constant__ CUtensorMap tmRes, int M, int N, int num_m_tiles, int num_n_tiles,
                 int num_k_blocks, ConvGeom g, EpiArgs ep, const float* __restrict__ a_scale,
                 const float* __restrict__ w_scale) {
  constexpr bool kE4m3 = true, kImgScale = false;
  constexpr bool kOutE4m3 = false, kBlockScale = false;
  [[maybe_unused]] constexpr float* out_scale = nullptr;
  [[maybe_unused]] constexpr long long ld_scale = 0;
  [[maybe_unused]] const CUtensorMap& tmAS = tmA0;
#include "gemm_wgmma_body.cuh"
}

// e4m3 3x3 convolution (g.conv == 1, single source: tmA1 == tmA0 and kb1 == 0, no split-K): as gemm_e4m3_kernel, with
// a_scale one fp32 scale per IMAGE, read for each tile row from the image its output pixel lies in
template <int BN, bool kBf16, bool kRes>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_e4m3_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                 const __grid_constant__ CUtensorMap tmRes, int M, int N, int num_m_tiles, int num_n_tiles,
                 int num_k_blocks, ConvGeom g, EpiArgs ep, const float* __restrict__ a_scale,
                 const float* __restrict__ w_scale) {
  constexpr bool kE4m3 = true, kImgScale = true;
  constexpr bool kOutE4m3 = false, kBlockScale = false;
  [[maybe_unused]] constexpr float* out_scale = nullptr;
  [[maybe_unused]] constexpr long long ld_scale = 0;
  [[maybe_unused]] const CUtensorMap& tmAS = tmA0;
#include "gemm_wgmma_body.cuh"
}

// GEGLU with an e4m3 output (gemm_e4m3_kernel's GEGLU, BN = 256): out_scale[n_tile][row] (row stride ld_scale) is the
// scale of the row's 128 output columns of tile n_tile; tmOut is a one-byte map with 128 x 128 boxes
template <bool kBf16>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_e4m3_geglu_e4m3_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                            const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                            const __grid_constant__ CUtensorMap tmRes, int M, int N, int num_m_tiles, int num_n_tiles,
                            int num_k_blocks, ConvGeom g, EpiArgs ep, const float* __restrict__ a_scale,
                            const float* __restrict__ w_scale, float* __restrict__ out_scale, long long ld_scale) {
  constexpr int BN = 256;
  constexpr bool kRes = false;
  constexpr bool kE4m3 = true, kImgScale = false, kOutE4m3 = true, kBlockScale = false;
  [[maybe_unused]] const CUtensorMap& tmAS = tmA0;
#include "gemm_wgmma_body.cuh"
}

// e4m3 A with one scale per row and 128-element K block (a_scale[kb][row], read through tmAS into the stages), W with one
// per output channel: GEMM rows only (g.conv == 0, tmA1 == tmA0 and never read, no split-K, no GEGLU)
template <int BN, bool kBf16, bool kRes>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_blockscaled_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                        const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
                        const __grid_constant__ CUtensorMap tmRes, const __grid_constant__ CUtensorMap tmAS, int M,
                        int N, int num_m_tiles, int num_n_tiles, int num_k_blocks, ConvGeom g, EpiArgs ep,
                        const float* __restrict__ w_scale) {
  constexpr bool kE4m3 = true, kImgScale = false, kOutE4m3 = false, kBlockScale = true;
  [[maybe_unused]] constexpr const float* a_scale = nullptr;
  [[maybe_unused]] constexpr float* out_scale = nullptr;
  [[maybe_unused]] constexpr long long ld_scale = 0;
#include "gemm_wgmma_body.cuh"
}

// Staging-buffer reuse: the two 8 KiB buffers alternate per chunk. The issuer executes cp.async.bulk.wait_group.read 0
// just BEFORE it joins barrier(i) - after its own math of chunk i, so the time a store needs to drain shared memory hides
// under that math - i.e. after it committed store(i-1); every thread writes buffer (i+1)&1 only after barrier(i), by
// which time stores <= i-1 - including store(i-1), the last reader of that buffer - have finished reading shared memory.

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// split-K reduction + the complete epilogue: out = act((sum_s partial[s] * scale + (bias + rowvec) * scale + residual * scale))
// in the same operation order as the in-kernel epilogue. 8 columns per thread, splits summed in index order.
template <bool kBf16>
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ part, int splits, long long M, int N, const void* __restrict__ bias,
                     const void* __restrict__ rowvec, long long rpg, long long ld_rowvec,
                     const void* __restrict__ res, long long ld_res, float scale, int act, void* __restrict__ out,
                     long long ldo) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  pdl_launch_dependents();
  pdl_wait();
  const int nv = N >> 3;
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= M * nv) return;
  const long long row = idx / nv;
  const int col = static_cast<int>(idx - row * nv) * 8;
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int s = 0; s < splits; ++s) {
    const float4* p = reinterpret_cast<const float4*>(part + (static_cast<long long>(s) * M + row) * N + col);
    const float4 u0 = p[0], u1 = p[1];
    a[0] += u0.x, a[1] += u0.y, a[2] += u0.z, a[3] += u0.w;
    a[4] += u1.x, a[5] += u1.y, a[6] += u1.z, a[7] += u1.w;
  }
  float cst[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  auto add_vec = [&](const T* v, float* dst, bool scaled_fma) {
    const uint4 b = *reinterpret_cast<const uint4*>(v);
    const uint32_t w[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = C::unpack(w[j]);
      if (scaled_fma) {
        dst[2 * j] = fmaf(t.x, scale, dst[2 * j]);
        dst[2 * j + 1] = fmaf(t.y, scale, dst[2 * j + 1]);
      } else {
        dst[2 * j] += t.x;
        dst[2 * j + 1] += t.y;
      }
    }
  };
  if (bias) add_vec(static_cast<const T*>(bias) + col, cst, false);
  if (rowvec) add_vec(static_cast<const T*>(rowvec) + (row / rpg) * ld_rowvec + col, cst, false);
  float f[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = fmaf(a[j], scale, cst[j] * scale);
  if (res) add_vec(static_cast<const T*>(res) + row * ld_res + col, f, true);
  if (act == MIMO_ACT_SILU) {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = silu_f(f[j]);
  }
  uint4 o;
  o.x = C::pack(f[0], f[1]);
  o.y = C::pack(f[2], f[3]);
  o.z = C::pack(f[4], f[5]);
  o.w = C::pack(f[6], f[7]);
  *reinterpret_cast<uint4*>(static_cast<T*>(out) + row * ldo + col) = o;
}

// Runtime -> compile-time selection: f(std::true_type{}) if b, else f(std::false_type{})
template <class F>
static auto with_bool(bool b, F&& f) {
  return b ? f(std::true_type{}) : f(std::false_type{});
}

// Errors that name a kernel family: `fmt` holds one %s for `who`; an ARG error unless a CUDA error `e` is given
static int family_error(const char* fmt, const char* who, cudaError_t e = cudaSuccess) {
  char msg[128];
  snprintf(msg, sizeof(msg), fmt, who);
  return e == cudaSuccess ? set_error(MIMO_ERR_ARG, msg) : set_cuda_error(msg, e);
}

// The tile widths (BN) a kernel family is instantiated at, widest first (pick_bn's tie-break reads them in this order).
// dispatch() calls f(std::integral_constant<int, BN>, kBf16, kRes) (the last two std::bool_constants) for the runtime
// width `bn`, dtype and residual flag, and refuses a width that is not in the list.
template <int... BNs>
struct TileWidths {
  static constexpr int kList[sizeof...(BNs)] = {BNs...};
  static constexpr bool has(int bn) { return ((bn == BNs) || ...); }
  template <class F>
  static int dispatch(const char* who, int bn, int dtype, bool res, F&& f) {
    int rc = MIMO_OK;
    auto at = [&](auto kBN) {
      if (bn != kBN) return false;
      rc = with_bool(dtype == MIMO_BF16,
                     [&](auto kBf16) { return with_bool(res, [&](auto kRes) { return f(kBN, kBf16, kRes); }); });
      return true;
    };
    if ((at(std::integral_constant<int, BNs>{}) || ...)) return rc;
    return family_error("%s: unsupported BN", who);
  }
};

// ptxas (CUDA 12.9, -O3), per thread at the 168-register cap of 320 threads:
//   gemm_e4m3_kernel<192, *, *>: 144-155 registers, no spills
//   gemm_e4m3_kernel<256, f16 / bf16, no residual>: 168 registers, 32 / 16 B spill stores, 36 / 20 B spill loads
//   gemm_e4m3_kernel<256, *, residual>: 168 registers, 32 B spill stores, 48 B spill loads
//   conv_e4m3_kernel<160, *, no residual / residual>: 128 / 144-148 registers, no spills
//   conv_e4m3_kernel<256, *, *>: as gemm_e4m3_kernel<256, *, *> (the engine uses it for 1280 channels at 8 x 8)
//   (gemm_wgmma_kernel<256, *, *>, for comparison: 168 registers, 8 B spill stores, 8-16 B spill loads)
//   gemm_e4m3_geglu_e4m3_kernel<f16 / bf16> (BN 256, e4m3 output): 168 registers, no spills (the 96 B stack frame the
//     spill-free kernels here all have)
//   gemm_blockscaled_kernel<64, *, *>: 91 registers, no spills; <128, *, *>: 146 registers, no spills (two BN / 2
//     accumulators per thread: the running sum and the K block's own)
// e4m3 tile widths: 192 and 256 are the widths pick_bn gives the LN-fed GEMMs of the UNet (q|k|v N = 3 C: 960 / 1920 ->
// 192, 3840 -> 256; GEGLU N = 8 C -> 256).
using Widths16 = TileWidths<256, 192, 160, 128, 64>;  // gemm_wgmma_kernel
using WidthsE4m3 = TileWidths<256, 192>;              // gemm_e4m3_kernel
using WidthsConvE4m3 = TileWidths<256, 160>;          // conv_e4m3_kernel (choice: pick_bn_conv_e4m3)
using WidthsGegluE4m3 = TileWidths<256>;              // gemm_e4m3_geglu_e4m3_kernel, which takes no residual
using WidthsBlockScaled = TileWidths<128, 64>;        // gemm_blockscaled_kernel (choice: pick_bn_blockscaled)

// One launch of a persistent GEMM / conv kernel: min(tiles, SMs) CTAs of kGemmThreads with kSmem bytes of dynamic shared
// memory (the attribute is set on the first launch of each kernel). `who` names the kernel family in error messages.
template <auto kKern, int kSmem, class... A>
static int launch_gemm_kernel(const char* who, int tiles, cudaStream_t st, A... args) {
  static bool attr_done = false;  // per instantiation
  if (!attr_done) {
    const cudaError_t e = cudaFuncSetAttribute(kKern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return family_error("cudaFuncSetAttribute(%s)", who, e);
    attr_done = true;
  }
  const int grid = tiles < num_sms() ? tiles : num_sms();
  cudaError_t e = launch_k(kKern, dim3(grid), dim3(kGemmThreads), kSmem, st, args...);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return family_error("%s launch", who, e);
  return MIMO_OK;
}

static int g_force_bn = 0;

// Tile-width choice: least padded columns first, then the widest tile (fewer A re-reads, higher MMA N).
static int pick_bn(int N, bool geglu, long long m_tiles) {
  if (g_force_bn) return g_force_bn;
  if (geglu) {
    if (N % 256 == 0) return 256;
    if (N % 128 == 0) return 128;
    return 64;
  }
  int best = 64;
  double best_eff = -1.0;
  for (const int bn : Widths16::kList) {
    const int nt = (N + bn - 1) / bn;
    double eff = static_cast<double>(N) / (static_cast<double>(nt) * bn);
    // small problems: prefer enough tiles to occupy the machine
    const long long tiles = m_tiles * nt;
    if (tiles < num_sms() && bn > 64) eff *= 0.5 + 0.5 * static_cast<double>(tiles) / num_sms();
    if (eff > best_eff + 1e-9) {
      best_eff = eff;
      best = bn;
    }
  }
  return best;
}

// e4m3 tile width: pick_bn's rule over the instantiated widths {256, 192} - least padded columns, then the wider; GEGLU
// takes pick_bn's own width (it fixes the weight packing, mimo_gemm_geglu_granule) and must be one of them.
static int pick_bn_e4m3(int N, bool geglu) {
  if (geglu) return pick_bn(N, true, 1 << 20);
  const int pad256 = (N + 255) / 256 * 256 - N, pad192 = (N + 191) / 192 * 192 - N;
  return pad192 < pad256 ? 192 : 256;
}

// e4m3 conv tile widths (conv_e4m3_kernel instantiations): 160 divides every ResBlock width (320, 640, 1280), 256 divides
// 1280. At 1280 BN 256 spills (ptxas report above) and 160 does not; measured on an H100 SXM (700 W) at the 48 images of
// the 512 x 512 CFG window, 256 was faster where its tiles fit one wave and 160's did not (8 x 8: 66 / 68 / 123 us
// against 83 / 85 / 152 us), and at 16 x 16 the two were within 8 % either way (scripts/fp8_conv_bench.py). So: 256 when
// that saves a wave, else the least padded width, 160 on a tie.
static int pick_bn_conv_e4m3(int N, long long m_tiles) {
  if (g_force_bn) return g_force_bn;
  const long long t256 = m_tiles * ((N + 255) / 256), t160 = m_tiles * ((N + 159) / 160);
  if (N % 256 == 0 && t256 <= num_sms() && t160 > num_sms()) return 256;
  const int pad256 = (N + 255) / 256 * 256 - N, pad160 = (N + 159) / 160 * 160 - N;
  return pad256 < pad160 ? 256 : 160;
}

// block-scaled tile widths (gemm_blockscaled_kernel instantiations): the per-block accumulator doubles the accumulator
// registers, so 64 and 128 (ptxas report above). Measured on an H100 SXM (700 W) at the FF-out shapes of the 512 x 512
// CFG window (scripts/fp8_ff_bench.py), 128 was faster at every width, even at N = 320 where it pads to 384 columns
// (290 against 302 us at 64 x 64: 3 column tiles read each A tile 3 times instead of 5): 128, and 64 only for N <= 64.
static int pick_bn_blockscaled(int N) {
  if (g_force_bn) return g_force_bn;
  return N <= 64 ? 64 : 128;
}

// Split-K decision: only when the output tiles would leave more than half of the SMs idle AND every split still gets a
// long K range (>= 16 K blocks = 1024): the deep, small-M convolutions / FF projections of the 8x8 and 16x16 levels when
// the clip's frames are spread over several GPUs. Returns the number of splits (1 = off); a split problem takes the tile
// width a large problem would get, written to `bn`.
static int pick_splits(int& bn, int N, int mt, int nkb, long long M, int64_t ws_bytes) {
  const int bn_wide = pick_bn(N, false, 1 << 20);
  const long long tiles = static_cast<long long>(mt) * ((N + bn_wide - 1) / bn_wide);
  if (tiles * 2 > num_sms() || nkb < 32) return 1;
  long long s = num_sms() / tiles;
  if (s > nkb / 16) s = nkb / 16;
  if (s > 16) s = 16;
  while (s > 1 && s * M * N * 4 > ws_bytes) --s;
  if (s < 2) return 1;
  bn = bn_wide;
  return static_cast<int>(s);
}

static EpiArgs make_epi(const mimo_epilogue& e, int N) {
  EpiArgs a;
  a.bias = e.bias;
  a.rowvec = e.rowvec;
  a.rows_per_group = e.rows_per_group > 0 ? e.rows_per_group : 1;
  if (a.rows_per_group > 0x7fffffffLL) a.rows_per_group = 0x7fffffffLL;  // row counts are ints: same grouping
  a.ld_rowvec = e.ld_rowvec > 0 ? e.ld_rowvec : N;
  a.scale = e.scale;
  a.act = e.act;
  a.partial = nullptr;
  return a;
}

// Split-K is OFF by default: the second kernel and the fp32 partial traffic have to buy back more than the better SM fill,
// and an M-dependent summation order would break the bit-identity of sharded and un-sharded runs. mimo_debug_splitk(1)
// enables the automatic choice (tests/test_kernels_gpu.py keeps it honest).
static int g_splitk = 0;

static int launch_reduce(int dtype, const float* part, int splits, long long M, int N, const mimo_epilogue& e, void* out,
                         long long ldo, cudaStream_t st) {
  const long long total = M * (N / 8);
  const unsigned blocks = div_up(total, 256);
  const long long rpg = e.rows_per_group > 0 ? e.rows_per_group : 1;
  const long long ldr = e.ld_rowvec > 0 ? e.ld_rowvec : N;
  cudaError_t err = dtype == MIMO_BF16
                        ? launch_k(splitk_reduce_kernel<true>, dim3(blocks), dim3(256), 0, st, part, splits, M, N, e.bias,
                                   e.rowvec, rpg, ldr, e.residual, static_cast<long long>(e.ld_res), e.scale, e.act, out, ldo)
                        : launch_k(splitk_reduce_kernel<false>, dim3(blocks), dim3(256), 0, st, part, splits, M, N, e.bias,
                                   e.rowvec, rpg, ldr, e.residual, static_cast<long long>(e.ld_res), e.scale, e.act, out, ldo);
  if (err == cudaSuccess) err = cudaGetLastError();
  if (err != cudaSuccess) return set_cuda_error("split-K reduce launch", err);
  return MIMO_OK;
}

// Geometry of plain GEMM rows: K blocks kb0 of source 0 (K = c0 elements) and kb1 of source 1, 128 x 32 output chunks,
// no split
static ConvGeom gemm_rows(int c0, int kb0, int kb1 = 0) {
  ConvGeom g = {};
  g.c0 = c0;
  g.kb0 = kb0;
  g.kb1 = kb1;
  g.chunk_bytes = kChunk;
  g.splits = 1;
  g.kb_split = kb0 + kb1;
  return g;
}

// Conv geometry: `ntaps` taps at input offsets (tdx, tdy) over [n, h, w] images of c0 (+ c1) channels, in K blocks of kc
// channels of esz bytes each, and the {TW, TH, TN} output footprint of a 128-row tile; no split, so kb_split holds all
// ntaps * (kb0 + kb1) K blocks. Returns the M tiles.
static int conv_geom(ConvGeom& g, int n, int h, int w, int c0, int c1, int kc, int esz, int ntaps,
                     const signed char* tdx, const signed char* tdy) {
  g = {};
  g.conv = 1;
  g.H = h;
  g.W = w;
  g.NI = n;
  g.TW = w < BM ? w : BM;
  g.TH = BM / g.TW;
  if (g.TH > h) g.TH = h;
  if (g.TH < 1) g.TH = 1;
  g.TN = BM / (g.TW * g.TH);
  if (g.TN > n) g.TN = n;
  if (g.TN < 1) g.TN = 1;
  if (g.TN > 1 && g.TH != h) g.TN = 1;  // several images per tile only when a tile spans whole images
  g.tiles_w = (w + g.TW - 1) / g.TW;
  g.tiles_h = (h + g.TH - 1) / g.TH;
  g.ctot = c0 + c1;
  g.c0 = c0;
  g.kb0 = (c0 + kc - 1) / kc;
  g.kb1 = (c1 + kc - 1) / kc;
  const int pixels = g.TW * g.TH * g.TN;
  g.a_bytes = pixels * kc * esz;
  g.chunk_bytes = pixels * 64;
  g.splits = 1;
  g.kb_split = ntaps * (g.kb0 + g.kb1);
  g.ntaps = ntaps;
  for (int t = 0; t < 9; ++t) {
    g.tdx[t] = t < ntaps ? tdx[t] : 0;
    g.tdy[t] = t < ntaps ? tdy[t] : 0;
  }
  return g.tiles_w * g.tiles_h * ((n + g.TN - 1) / g.TN);
}

constexpr signed char kTap3x3Dx[9] = {-1, 0, 1, -1, 0, 1, -1, 0, 1};
constexpr signed char kTap3x3Dy[9] = {-1, -1, -1, 0, 0, 0, 1, 1, 1};

struct Maps {
  CUtensorMap a0, a1, b, out, res;
};

// 2-D map over `rows` rows of `cols` elements (`dtype`: 16-bit, or kTmapU8) that start `pitch` bytes apart
static int rows_map(CUtensorMap* tm, int dtype, const void* base, uint64_t cols, uint64_t rows, uint64_t pitch,
                    uint32_t box_cols, uint32_t box_rows, int swizzle = 128) {
  const uint64_t dim[2] = {cols, rows};
  const uint64_t str[1] = {pitch};
  const uint32_t box[2] = {box_cols, box_rows};
  return encode_tmap(tm, dtype, 2, base, dim, str, box, swizzle);
}

// 4-D map over the NHWC images of g, `c` channels of `dtype` each: pixel (n, y, x) at
// base + ((n * s H + y s) * s W + x s) * pitch elements, i.e. a stride-s view of s times larger images when s > 1. Box
// {box_c, TW, TH, TN}.
static int nhwc_map(CUtensorMap* tm, int dtype, const void* base, const ConvGeom& g, int c, long long pitch,
                    uint32_t box_c, int swizzle, int s = 1) {
  const uint64_t dim[4] = {static_cast<uint64_t>(c), static_cast<uint64_t>(g.W), static_cast<uint64_t>(g.H),
                           static_cast<uint64_t>(g.NI)};
  uint64_t str[3];
  str[0] = static_cast<uint64_t>(s) * pitch * (dtype == kTmapU8 ? 1 : 2);
  str[1] = static_cast<uint64_t>(s) * g.W * str[0];
  str[2] = static_cast<uint64_t>(g.H) * str[1];
  const uint32_t box[4] = {box_c, static_cast<uint32_t>(g.TW), static_cast<uint32_t>(g.TH), static_cast<uint32_t>(g.TN)};
  return encode_tmap(tm, dtype, 4, base, dim, str, box, swizzle);
}

// 16-bit output and (if `residual`) residual maps of GEMM rows: 128-row x 32-column boxes, 64-byte swizzle. Without a
// residual m.res repeats m.out; the kernel does not read it.
static int out_maps_rows(Maps& m, int dtype, void* out, long long ldo, const void* residual, long long ld_res, int cols,
                         int rows) {
  if (int rc = rows_map(&m.out, dtype, out, cols, rows, ldo * 2, 32, BM, 64)) return rc;
  m.res = m.out;
  return residual ? rows_map(&m.res, dtype, residual, cols, rows, ld_res * 2, 32, BM, 64) : MIMO_OK;
}

// The same for conv outputs: {32, TW, TH, TN} boxes; the output may be a stride-s view (nhwc_map), the residual is dense
static int out_maps_nhwc(Maps& m, int dtype, const ConvGeom& g, void* out, long long ldo, int s, const void* residual,
                         long long ld_res, int cout) {
  if (int rc = nhwc_map(&m.out, dtype, out, g, cout, ldo, 32, 64, s)) return rc;
  m.res = m.out;
  return residual ? nhwc_map(&m.res, dtype, residual, g, cout, ld_res, 32, 64) : MIMO_OK;
}

// The 16-bit kernel (mimo_gemm, mimo_conv3x3, mimo_conv_up2x) at tile width bn. With splits > 1 the kernel writes each
// split's fp32 partial sums to `workspace` with its epilogue neutralised, and splitk_reduce_kernel then applies the whole
// epilogue `e` to `out`.
static int launch_16bit(int dtype, int bn, bool res, int splits, const Maps& m, int M, int N, int mt, int nkb,
                        ConvGeom g, const mimo_epilogue& e, void* workspace, void* out, long long ldo, cudaStream_t st) {
  g.splits = splits;
  g.kb_split = (nkb + splits - 1) / splits;
  EpiArgs ep = make_epi(e, N);
  if (splits > 1) {
    ep.bias = ep.rowvec = nullptr;
    ep.act = MIMO_ACT_NONE;
    ep.scale = 1.0f;
    ep.partial = static_cast<float*>(workspace);
  }
  const int nt = (N + bn - 1) / bn;
  const int rc = Widths16::dispatch("gemm", bn, dtype, res, [&](auto kBN, auto kBf16, auto kRes) {
    return launch_gemm_kernel<gemm_wgmma_kernel<kBN, kBf16, kRes>, GemmCfg<kBN, kRes>::kSmemBytes>(
        "gemm", mt * nt, st, m.a0, m.a1, m.b, m.out, m.res, M, N, mt, nt, nkb, g, ep);
  });
  if (rc || splits == 1) return rc;
  return launch_reduce(dtype, ep.partial, splits, M, N, e, out, ldo, st);
}

}  // namespace mimo

using namespace mimo;

extern "C" int mimo_debug_splitk(int mode) {
  g_splitk = mode;
  return 0;
}

extern "C" int mimo_debug_force_bn(int bn) {
  g_force_bn = bn;
  return 0;
}

extern "C" int mimo_gemm_geglu_granule(int32_t N) { return pick_bn(N, true, 1 << 20) / 2; }

extern "C" int mimo_gemm(const mimo_gemm_params* p, void* stream) {
  if (!p || !p->a || !p->w || !p->out) return set_error(MIMO_ERR_ARG, "mimo_gemm: null pointer");
  if (p->M <= 0 || p->N <= 0 || p->K <= 0) return set_error(MIMO_ERR_ARG, "mimo_gemm: empty problem");
  if ((p->K % 8) || (p->lda % 8) || (p->ldw % 8) || (p->N % 8) || (p->ldo % 8))
    return set_error(MIMO_ERR_ARG, "mimo_gemm: K, N, lda, ldw, ldo must be multiples of 8");
  if (p->ep.residual && (p->ep.ld_res % 8)) return set_error(MIMO_ERR_ARG, "mimo_gemm: ld_res % 8 != 0");
  const bool geglu = p->ep.act == MIMO_ACT_GEGLU;
  if (geglu && (p->ep.residual || p->ep.rowvec))
    return set_error(MIMO_ERR_ARG, "mimo_gemm: GEGLU takes neither a residual nor a row vector");
  const int K1 = p->a1 ? p->K1 : 0;
  if (K1 < 0 || (K1 % 8) || (p->a1 && (p->lda1 % 8))) return set_error(MIMO_ERR_ARG, "mimo_gemm: K1/lda1 % 8 != 0");
  // (GEGLU's width does not depend on the SM count, and a GEGLU GEMM is never split)
  if (geglu && (p->N % pick_bn(p->N, true, 0))) return set_error(MIMO_ERR_ARG, "mimo_gemm: GEGLU needs N % tile == 0");
  if (int rc = ensure_device()) return rc;
  const int mt = (p->M + BM - 1) / BM;
  const int kb0 = (p->K + BK - 1) / BK;
  const int kb1 = (K1 + BK - 1) / BK;
  const int nkb = kb0 + kb1;
  int bn = pick_bn(p->N, geglu, mt);
  const int splits = !geglu && g_splitk && p->workspace && !g_force_bn
                         ? pick_splits(bn, p->N, mt, nkb, p->M, p->workspace_bytes)
                         : 1;
  const bool res = p->ep.residual != nullptr && splits == 1;

  Maps m;
  if (int rc = rows_map(&m.a0, p->dtype, p->a, p->K, p->M, p->lda * 2, BK, BM)) return rc;
  m.a1 = m.a0;
  if (K1)
    if (int rc = rows_map(&m.a1, p->dtype, p->a1, K1, p->M, p->lda1 * 2, BK, BM)) return rc;
  if (int rc = rows_map(&m.b, p->dtype, p->w, p->K + K1, p->N, p->ldw * 2, BK, bn)) return rc;
  const int n_out = geglu ? p->N / 2 : p->N;
  if (int rc = out_maps_rows(m, p->dtype, p->out, p->ldo, res ? p->ep.residual : nullptr, p->ep.ld_res, n_out, p->M))
    return rc;
  return launch_16bit(p->dtype, bn, res, splits, m, p->M, p->N, mt, nkb, gemm_rows(p->K, kb0, kb1), p->ep, p->workspace,
                      p->out, p->ldo, static_cast<cudaStream_t>(stream));
}

extern "C" int mimo_gemm_e4m3(const mimo_gemm_e4m3_params* p, void* stream) {
  if (!p || !p->a || !p->w || !p->out || !p->a_scale || !p->w_scale)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: null pointer");
  if (p->M <= 0 || p->N <= 0 || p->K <= 0) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: empty problem");
  if ((p->K % 16) || (p->lda % 16) || (p->ldw % 16))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: K, lda, ldw must be multiples of 16");
  if ((p->N % 8) || (p->ldo % 8)) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: N, ldo must be multiples of 8");
  if ((reinterpret_cast<uintptr_t>(p->a) | reinterpret_cast<uintptr_t>(p->w) | reinterpret_cast<uintptr_t>(p->out) |
       reinterpret_cast<uintptr_t>(p->ep.residual)) % 16)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: a, w, out, residual must be 16-byte aligned");
  if (p->ep.residual && (p->ep.ld_res % 8)) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: ld_res % 8 != 0");
  if (p->workspace || p->workspace_bytes) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: split-K is not supported");
  const bool geglu = p->ep.act == MIMO_ACT_GEGLU;
  if (geglu && (p->ep.residual || p->ep.rowvec))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: GEGLU takes neither a residual nor a row vector");
  const int bn = pick_bn_e4m3(p->N, geglu);
  if (geglu && (p->N % bn)) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: GEGLU needs N % tile == 0");
  if (!WidthsE4m3::has(bn)) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3: GEGLU needs N % 256 == 0");
  if (int rc = ensure_device()) return rc;
  const int mt = (p->M + BM - 1) / BM;
  const int nt = (p->N + bn - 1) / bn;
  const int nkb = (p->K + 2 * BK - 1) / (2 * BK);
  const bool res = p->ep.residual != nullptr && !geglu;

  Maps m;
  if (int rc = rows_map(&m.a0, kTmapU8, p->a, p->K, p->M, p->lda, 2 * BK, BM)) return rc;
  m.a1 = m.a0;
  if (int rc = rows_map(&m.b, kTmapU8, p->w, p->K, p->N, p->ldw, 2 * BK, bn)) return rc;
  const int n_out = geglu ? p->N / 2 : p->N;
  if (int rc = out_maps_rows(m, p->dtype, p->out, p->ldo, res ? p->ep.residual : nullptr, p->ep.ld_res, n_out, p->M))
    return rc;
  const ConvGeom g = gemm_rows(p->K, nkb);
  const EpiArgs ep = make_epi(p->ep, p->N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return WidthsE4m3::dispatch("gemm_e4m3", bn, p->dtype, res, [&](auto kBN, auto kBf16, auto kRes) {
    return launch_gemm_kernel<gemm_e4m3_kernel<kBN, kBf16, kRes>, GemmCfg<kBN, kRes, true>::kSmemBytes>(
        "gemm_e4m3", mt * nt, st, m.a0, m.a1, m.b, m.out, m.res, p->M, p->N, mt, nt, nkb, g, ep, p->a_scale, p->w_scale);
  });
}

// One implicit-GEMM convolution launch: `ntaps` taps at offsets (tdx, tdy) over the [n, h, w, c] input(s); the output
// (and residual) pixel (n, y, x) lives at out + ((n * s h + y s) * s w + x s) * ldo elements, i.e. a strided view of a
// larger image when s > 1.
static int conv_launch(const mimo_conv3x3_params* p, const void* w, int ntaps, const signed char* tdx,
                       const signed char* tdy, void* out, int s, void* stream) {
  const int c1 = p->x1 ? p->c1 : 0;
  ConvGeom g;
  const int mt = conv_geom(g, p->n, p->h, p->w_, p->c0, c1, BK, 2, ntaps, tdx, tdy);
  const int nkb = g.kb_split;
  const long long Mrows = static_cast<long long>(p->n) * p->h * p->w_;
  if (Mrows > 0x7fffffffLL) return set_error(MIMO_ERR_ARG, "mimo_conv: too many pixels");
  int bn = pick_bn(p->cout, false, mt);
  // split-K needs the dense NHWC output (row = pixel index): not for the strided parity classes of mimo_conv_up2x
  const int splits = g_splitk && p->workspace && !g_force_bn && s == 1 && p->ldo == p->cout
                         ? pick_splits(bn, p->cout, mt, nkb, Mrows, p->workspace_bytes)
                         : 1;
  const bool res = p->ep.residual != nullptr && splits == 1;

  Maps m;
  if (int rc = nhwc_map(&m.a0, p->dtype, p->x0, g, p->c0, p->c0, BK, 128)) return rc;
  m.a1 = m.a0;
  if (c1)
    if (int rc = nhwc_map(&m.a1, p->dtype, p->x1, g, c1, c1, BK, 128)) return rc;
  const long long kw = static_cast<long long>(ntaps) * g.ctot;  // weight row: [tap][channel]
  if (int rc = rows_map(&m.b, p->dtype, w, kw, p->cout, kw * 2, BK, bn)) return rc;
  if (int rc = out_maps_nhwc(m, p->dtype, g, out, p->ldo, s, res ? p->ep.residual : nullptr, p->ep.ld_res, p->cout))
    return rc;
  return launch_16bit(p->dtype, bn, res, splits, m, static_cast<int>(Mrows), p->cout, mt, nkb, g, p->ep, p->workspace,
                      out, p->ldo, static_cast<cudaStream_t>(stream));
}

static int conv_check(const mimo_conv3x3_params* p) {
  if (!p || !p->x0 || !p->w || !p->out) return set_error(MIMO_ERR_ARG, "mimo_conv: null pointer");
  if (p->n <= 0 || p->h <= 0 || p->w_ <= 0 || p->cout <= 0 || p->c0 <= 0)
    return set_error(MIMO_ERR_ARG, "mimo_conv: empty problem");
  const int c1 = p->x1 ? p->c1 : 0;
  if ((p->c0 % 8) || (c1 % 8) || (p->cout % 8) || (p->ldo % 8))
    return set_error(MIMO_ERR_ARG, "mimo_conv: channel counts must be multiples of 8");
  if (p->ep.act == MIMO_ACT_GEGLU) return set_error(MIMO_ERR_ARG, "mimo_conv: GEGLU not supported");
  if (p->ep.residual && (p->ep.ld_res % 8)) return set_error(MIMO_ERR_ARG, "mimo_conv: ld_res % 8 != 0");
  return ensure_device();
}

extern "C" int mimo_conv3x3(const mimo_conv3x3_params* p, void* stream) {
  if (int rc = conv_check(p)) return rc;
  return conv_launch(p, p->w, 9, kTap3x3Dx, kTap3x3Dy, p->out, 1, stream);
}

// nearest-x2 upsampling followed by a 3x3 / pad 1 convolution, without the upsampled tensor: output pixel (2y+a, 2x+b)
// only ever sees the 2x2 source neighbourhood {y-1+a, y+a} x {x-1+b, x+b}, so each of the four parity classes (a, b) is a
// 2x2-tap convolution over the SOURCE image whose weights are sums of the 3x3 taps that land on the same source pixel
// (packed by the host: w = [4 classes][cout, 4 * cin], class = 2a + b, tap = 2 iy + ix). 4/9 of the FLOPs, no 4x buffer.
extern "C" int mimo_conv_up2x(const mimo_conv3x3_params* p, void* stream) {
  if (int rc = conv_check(p)) return rc;
  if (p->ep.residual || p->ep.rowvec) return set_error(MIMO_ERR_ARG, "mimo_conv_up2x: bias / activation epilogue only");
  const int ctot = p->c0 + (p->x1 ? p->c1 : 0);
  const size_t esz = 2;
  for (int a = 0; a < 2; ++a)
    for (int b = 0; b < 2; ++b) {
      const signed char dx[4] = {static_cast<signed char>(b - 1), static_cast<signed char>(b),
                                 static_cast<signed char>(b - 1), static_cast<signed char>(b)};
      const signed char dy[4] = {static_cast<signed char>(a - 1), static_cast<signed char>(a - 1),
                                 static_cast<signed char>(a), static_cast<signed char>(a)};
      const char* w = static_cast<const char*>(p->w) + static_cast<size_t>(2 * a + b) * p->cout * 4 * ctot * esz;
      char* out = static_cast<char*>(p->out) + (static_cast<size_t>(a) * 2 * p->w_ + b) * p->ldo * esz;
      if (int rc = conv_launch(p, w, 4, dx, dy, out, 2, stream)) return rc;
    }
  return MIMO_OK;
}

extern "C" int mimo_conv3x3_e4m3(const mimo_conv3x3_e4m3_params* p, void* stream) {
  if (!p || !p->x || !p->w || !p->out || !p->x_scale || !p->w_scale)
    return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: null pointer");
  if (p->n <= 0 || p->h <= 0 || p->w_ <= 0 || p->cout <= 0 || p->c_in <= 0)
    return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: empty problem");
  if (p->c_in % 16) return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: c_in must be a multiple of 16");
  if ((p->cout % 8) || (p->ldo % 8)) return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: cout, ldo must be multiples of 8");
  if ((reinterpret_cast<uintptr_t>(p->x) | reinterpret_cast<uintptr_t>(p->w) | reinterpret_cast<uintptr_t>(p->out) |
       reinterpret_cast<uintptr_t>(p->ep.residual)) % 16)
    return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: x, w, out, residual must be 16-byte aligned");
  if (p->ep.residual && (p->ep.ld_res % 8)) return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: ld_res % 8 != 0");
  if (p->ep.act == MIMO_ACT_GEGLU) return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: GEGLU not supported");
  if (p->workspace || p->workspace_bytes) return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: split-K is not supported");
  const long long Mrows = static_cast<long long>(p->n) * p->h * p->w_;
  if (Mrows > 0x7fffffffLL) return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: too many pixels");
  if (g_force_bn && !WidthsConvE4m3::has(g_force_bn))
    return set_error(MIMO_ERR_ARG, "mimo_conv3x3_e4m3: unsupported BN (160 or 256)");
  if (int rc = ensure_device()) return rc;

  ConvGeom g;
  const int mt = conv_geom(g, p->n, p->h, p->w_, p->c_in, 0, 2 * BK, 1, 9, kTap3x3Dx, kTap3x3Dy);
  const int nkb = g.kb_split;
  const int bn = pick_bn_conv_e4m3(p->cout, mt);
  const int nt = (p->cout + bn - 1) / bn;
  const bool res = p->ep.residual != nullptr;

  Maps m;
  if (int rc = nhwc_map(&m.a0, kTmapU8, p->x, g, p->c_in, p->c_in, 2 * BK, 128)) return rc;
  m.a1 = m.a0;
  if (int rc = rows_map(&m.b, kTmapU8, p->w, 9ull * p->c_in, p->cout, 9ull * p->c_in, 2 * BK, bn)) return rc;
  if (int rc = out_maps_nhwc(m, p->dtype, g, p->out, p->ldo, 1, p->ep.residual, p->ep.ld_res, p->cout)) return rc;
  const EpiArgs ep = make_epi(p->ep, p->cout);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int M = static_cast<int>(Mrows);
  return WidthsConvE4m3::dispatch("conv_e4m3", bn, p->dtype, res, [&](auto kBN, auto kBf16, auto kRes) {
    return launch_gemm_kernel<conv_e4m3_kernel<kBN, kBf16, kRes>, GemmCfg<kBN, kRes, true>::kSmemBytes>(
        "conv_e4m3", mt * nt, st, m.a0, m.a1, m.b, m.out, m.res, M, p->cout, mt, nt, nkb, g, ep, p->x_scale, p->w_scale);
  });
}

// ------------------------------------------------------------------------------------------------
// FP8 feed-forward: GEGLU -> e4m3 blocks, block-scaled e4m3 GEMM
// ------------------------------------------------------------------------------------------------
// (argument checks first, then the device probe, as the other entry points)
extern "C" int mimo_gemm_e4m3_geglu_e4m3(const mimo_gemm_e4m3_geglu_e4m3_params* p, void* stream) {
  if (!p || !p->a || !p->w || !p->out || !p->a_scale || !p->w_scale || !p->out_scale)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: null pointer");
  if (p->M <= 0 || p->N <= 0 || p->K <= 0) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: empty problem");
  if ((p->K % 16) || (p->lda % 16) || (p->ldw % 16) || (p->ldo % 16))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: K, lda, ldw, ldo must be multiples of 16");
  if (p->N % 256) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: N % 256 != 0 (one 128-column block per tile)");
  if (p->ld_scale < p->M || (p->ld_scale % 4))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: ld_scale must be >= M and a multiple of 4");
  if ((reinterpret_cast<uintptr_t>(p->a) | reinterpret_cast<uintptr_t>(p->w) | reinterpret_cast<uintptr_t>(p->out)) % 16)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: a, w, out must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(p->out_scale) % 16)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: out_scale must be 16-byte aligned");
  const int bn = pick_bn(p->N, true, 1 << 20);
  if (!WidthsGegluE4m3::has(bn))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_geglu_e4m3: needs the 256-wide GEGLU tile");
  if (int rc = ensure_device()) return rc;
  const int mt = (p->M + BM - 1) / BM;
  const int nt = p->N / bn;
  const int nkb = (p->K + 2 * BK - 1) / (2 * BK);

  Maps m;
  if (int rc = rows_map(&m.a0, kTmapU8, p->a, p->K, p->M, p->lda, 2 * BK, BM)) return rc;
  m.a1 = m.a0;
  if (int rc = rows_map(&m.b, kTmapU8, p->w, p->K, p->N, p->ldw, 2 * BK, bn)) return rc;
  // output: one-byte elements, 128-row x 128-column boxes (one 128-byte swizzle row per tile row)
  if (int rc = rows_map(&m.out, kTmapU8, p->out, p->N / 2, p->M, p->ldo, 2 * BK, BM)) return rc;
  m.res = m.out;
  const ConvGeom g = gemm_rows(p->K, nkb);
  mimo_epilogue e = {};
  e.bias = p->bias;
  e.scale = 1.0f;
  e.act = MIMO_ACT_GEGLU;
  const EpiArgs ep = make_epi(e, p->N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return WidthsGegluE4m3::dispatch("gemm_e4m3_geglu_e4m3", bn, p->dtype, false, [&](auto kBN, auto kBf16, auto) {
    return launch_gemm_kernel<gemm_e4m3_geglu_e4m3_kernel<kBf16>, GemmCfg<kBN, false, true>::kSmemBytes>(
        "gemm_e4m3_geglu_e4m3", mt * nt, st, m.a0, m.a1, m.b, m.out, m.res, p->M, p->N, mt, nt, nkb, g, ep, p->a_scale,
        p->w_scale, p->out_scale, static_cast<long long>(p->ld_scale));
  });
}

extern "C" int mimo_gemm_e4m3_blockscaled(const mimo_gemm_e4m3_blockscaled_params* p, void* stream) {
  if (!p || !p->a || !p->w || !p->out || !p->a_scale || !p->w_scale)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: null pointer");
  if (p->M <= 0 || p->N <= 0 || p->K <= 0) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: empty problem");
  if (p->K % 128) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: K must be a multiple of 128 (the scale block)");
  if ((p->lda % 16) || (p->ldw % 16))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: lda, ldw must be multiples of 16");
  if ((p->N % 8) || (p->ldo % 8)) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: N, ldo must be multiples of 8");
  if (p->ld_scale < p->M || (p->ld_scale % 4))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: ld_scale must be >= M and a multiple of 4");
  if ((reinterpret_cast<uintptr_t>(p->a) | reinterpret_cast<uintptr_t>(p->w) | reinterpret_cast<uintptr_t>(p->out) |
       reinterpret_cast<uintptr_t>(p->a_scale) | reinterpret_cast<uintptr_t>(p->ep.residual)) % 16)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: a, a_scale, w, out, residual must be 16-byte aligned");
  if (p->ep.residual && (p->ep.ld_res % 8)) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: ld_res % 8 != 0");
  if (p->ep.act == MIMO_ACT_GEGLU) return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: GEGLU not supported");
  if (p->workspace || p->workspace_bytes)
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: split-K is not supported");
  if (g_force_bn && !WidthsBlockScaled::has(g_force_bn))
    return set_error(MIMO_ERR_ARG, "mimo_gemm_e4m3_blockscaled: unsupported BN (64 or 128)");
  if (int rc = ensure_device()) return rc;
  const int bn = pick_bn_blockscaled(p->N);
  const int mt = (p->M + BM - 1) / BM;
  const int nt = (p->N + bn - 1) / bn;
  const int nkb = p->K / (2 * BK);
  const bool res = p->ep.residual != nullptr;

  Maps m;
  if (int rc = rows_map(&m.a0, kTmapU8, p->a, p->K, p->M, p->lda, 2 * BK, BM)) return rc;
  m.a1 = m.a0;
  if (int rc = rows_map(&m.b, kTmapU8, p->w, p->K, p->N, p->ldw, 2 * BK, bn)) return rc;
  if (int rc = out_maps_rows(m, p->dtype, p->out, p->ldo, p->ep.residual, p->ep.ld_res, p->N, p->M)) return rc;
  // row scales: fp32 [K / 128][ld_scale] read as 16-bit pairs, one 128-row (512-byte) box per K block; rows past M
  // are zero-filled
  CUtensorMap tas;
  if (int rc = rows_map(&tas, MIMO_F16, p->a_scale, 2ull * p->M, nkb, p->ld_scale * 4, 2 * BM, 1, 0)) return rc;
  const ConvGeom g = gemm_rows(p->K, nkb);
  const EpiArgs ep = make_epi(p->ep, p->N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return WidthsBlockScaled::dispatch("gemm_blockscaled", bn, p->dtype, res, [&](auto kBN, auto kBf16, auto kRes) {
    return launch_gemm_kernel<gemm_blockscaled_kernel<kBN, kBf16, kRes>, GemmCfg<kBN, kRes, true, true>::kSmemBytes>(
        "gemm_blockscaled", mt * nt, st, m.a0, m.a1, m.b, m.out, m.res, tas, p->M, p->N, mt, nt, nkb, g, ep, p->w_scale);
  });
}
