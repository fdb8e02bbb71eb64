// GroupNorm(+SiLU) and LayerNorm(+positional encoding) over channels-last activations. HBM-bound passes:
// 128-bit loads/stores, fp32 statistics, each thread owns a fixed 8-channel vector so gamma/beta/mean/rstd
// are loaded once and the loop over pixels is pure streaming.
#include <cuda_runtime.h>

#include "../../include/mimo_b200.h"
#include "host_util.h"
#include "ptx.cuh"

namespace mimo {

// ------------------------------------------------------------------------------------------------
// GroupNorm(+SiLU), deterministic: two streaming kernels, no floating-point atomics.
//   pass 1: every block reduces its slab of pixels to per-group (sum, sumsq) in a FIXED order (registers -> shared
//           memory -> one thread per group) and publishes them: part[image][slab][group][2]
//   pass 2: every block sums the slabs' partials of its image in the same fixed order (bit-identical statistics in
//           every block and run to run), then normalises + affine (+ SiLU) with 128-bit loads / stores.
// (A one-pass variant that keeps the slab in registers across a per-image arrival barrier serialises the blocks of an
// image on that barrier, and deadlocks when an image has more slabs than blocks can be resident.)
// ------------------------------------------------------------------------------------------------
struct GnArgs {
  const void* x0;
  const void* x1;
  const void* gamma;
  const void* beta;
  void* out;
  float* part;  // [n][bpi][groups][2] = (sum, sumsq) per slab
  int c0, c1, C, hw, groups, cpg;
  int vecs;  // C / 8
  int P;     // pixels processed side by side by one block
  int pix_per_block;
  int bpi;   // slabs per image
  float eps;
  int silu;
};

template <bool kBf16>
__device__ __forceinline__ uint4 gn_load(const GnArgs& a, long long pix, int cv) {
  using C = Cvt<kBf16>;
  const int ch = cv * 8;
  if (ch < a.c0) {
    return *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.x0) + pix * a.c0 + ch);
  }
  return *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.x1) + pix * a.c1 + (ch - a.c0));
}

constexpr int kGnMaxThreads = 320;

// pass 1: per-(image, slab, group) sum and sum of squares
template <bool kBf16>
__global__ void __launch_bounds__(kGnMaxThreads) gn_stats_kernel(GnArgs a) {
  using C = Cvt<kBf16>;
  __shared__ float4 s_red[kGnMaxThreads];  // per-thread (sumA, sqA, sumB, sqB)
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y;
  const int tid = threadIdx.x;
  const int cv = tid % a.vecs;
  const int pl = tid / a.vecs;
  const bool active = pl < a.P;
  const int ch0 = cv * 8;
  const int gA = ch0 / a.cpg;
  int split = (gA + 1) * a.cpg - ch0;  // channels [0, split) of this vector belong to gA, the rest to gA + 1
  if (split > 8) split = 8;
  float sA = 0.f, qA = 0.f, sB = 0.f, qB = 0.f;
  if (active) {
    const int p_begin = blockIdx.x * a.pix_per_block;
    int p_end = p_begin + a.pix_per_block;
    if (p_end > a.hw) p_end = a.hw;
#pragma unroll 4
    for (int p = p_begin + pl; p < p_end; p += a.P) {
      const uint4 u = gn_load<kBf16>(a, static_cast<long long>(n) * a.hw + p, cv);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = C::unpack(w[j]);
        if (2 * j < split) sA += t.x, qA += t.x * t.x; else sB += t.x, qB += t.x * t.x;
        if (2 * j + 1 < split) sA += t.y, qA += t.y * t.y; else sB += t.y, qB += t.y * t.y;
      }
    }
  }
  s_red[tid] = make_float4(sA, qA, sB, qB);
  __syncthreads();
  for (int g = tid; g < a.groups; g += blockDim.x) {  // fixed order: vectors touching group g, then pixel lanes
    const int v_lo = (g * a.cpg) >> 3;
    const int v_hi = ((g + 1) * a.cpg - 1) >> 3;
    float s = 0.f, q = 0.f;
    for (int v = v_lo; v <= v_hi; ++v) {
      const bool as_a = (v * 8) / a.cpg == g;  // this vector's first group is g (else g is its second group)
      for (int l = 0; l < a.P; ++l) {
        const float4 r = s_red[l * a.vecs + v];
        s += as_a ? r.x : r.z;
        q += as_a ? r.y : r.w;
      }
    }
    float* dst = a.part + ((static_cast<long long>(n) * a.bpi + blockIdx.x) * a.groups + g) * 2;
    dst[0] = s;
    dst[1] = q;
  }
}

// pass 2: image statistics from the slab partials (fixed order), then normalise + affine (+ SiLU)
template <bool kBf16>
__global__ void __launch_bounds__(kGnMaxThreads) gn_apply_kernel(GnArgs a) {
  using C = Cvt<kBf16>;
  __shared__ float s_tot[4][128];
  __shared__ float s_mean[64], s_rstd[64];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y;
  const int tid = threadIdx.x;
  const int g2 = a.groups * 2;
  {
    const int parts = a.bpi >= 16 ? 4 : 1;  // a function of the shape only: the summation order never varies
    const float* src = a.part + static_cast<long long>(n) * a.bpi * g2;
    for (int idx = tid; idx < parts * g2; idx += blockDim.x) {
      const int k = idx % g2, part = idx / g2;
      float acc = 0.f;
      for (int b = part; b < a.bpi; b += parts) acc += src[static_cast<long long>(b) * g2 + k];
      s_tot[part][k] = acc;
    }
    __syncthreads();
    const float inv_cnt = 1.0f / (static_cast<float>(a.hw) * a.cpg);
    for (int g = tid; g < a.groups; g += blockDim.x) {
      float s = 0.f, q = 0.f;
      for (int part = 0; part < parts; ++part) {
        s += s_tot[part][2 * g];
        q += s_tot[part][2 * g + 1];
      }
      const float mean = s * inv_cnt;
      float var = q * inv_cnt - mean * mean;
      var = var < 0.f ? 0.f : var;
      s_mean[g] = mean;
      s_rstd[g] = rsqrtf(var + a.eps);
    }
    __syncthreads();
  }
  const int cv = tid % a.vecs;
  const int pl = tid / a.vecs;
  if (pl >= a.P) return;
  const int ch0 = cv * 8;
  const int gA = ch0 / a.cpg;
  int split = (gA + 1) * a.cpg - ch0;
  if (split > 8) split = 8;
  float sc[8], sh[8];
  {
    const uint4 ug = *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.gamma) + ch0);
    const uint4 ub = *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.beta) + ch0);
    const uint32_t wg[4] = {ug.x, ug.y, ug.z, ug.w};
    const uint32_t wb[4] = {ub.x, ub.y, ub.z, ub.w};
    const float mA = s_mean[gA], rA = s_rstd[gA];
    const float mB = split < 8 ? s_mean[gA + 1] : 0.f, rB = split < 8 ? s_rstd[gA + 1] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 gg = C::unpack(wg[j]);
      const float2 bb = C::unpack(wb[j]);
      const float m0 = 2 * j < split ? mA : mB, r0 = 2 * j < split ? rA : rB;
      const float m1 = 2 * j + 1 < split ? mA : mB, r1 = 2 * j + 1 < split ? rA : rB;
      sc[2 * j] = r0 * gg.x;
      sh[2 * j] = bb.x - m0 * r0 * gg.x;
      sc[2 * j + 1] = r1 * gg.y;
      sh[2 * j + 1] = bb.y - m1 * r1 * gg.y;
    }
  }
  const int p_begin = blockIdx.x * a.pix_per_block;
  int p_end = p_begin + a.pix_per_block;
  if (p_end > a.hw) p_end = a.hw;
#pragma unroll 4
  for (int p = p_begin + pl; p < p_end; p += a.P) {
    const long long pix = static_cast<long long>(n) * a.hw + p;
    const uint4 u = gn_load<kBf16>(a, pix, cv);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = C::unpack(w[j]);
      f[2 * j] = fmaf(t.x, sc[2 * j], sh[2 * j]);
      f[2 * j + 1] = fmaf(t.y, sc[2 * j + 1], sh[2 * j + 1]);
    }
    if (a.silu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = silu_f(f[j]);
    }
    uint4 o;
    o.x = C::pack(f[0], f[1]);
    o.y = C::pack(f[2], f[3]);
    o.z = C::pack(f[4], f[5]);
    o.w = C::pack(f[6], f[7]);
    *reinterpret_cast<uint4*>(static_cast<typename C::T*>(a.out) + pix * a.C + ch0) = o;
  }
}

// launch geometry shared by mimo_groupnorm and mimo_groupnorm_workspace_bytes
struct GnPlan {
  int vecs, P, pix_per_block, bpi, threads;
};
static GnPlan gn_plan(int n, int hw, int C) {
  GnPlan pl;
  pl.vecs = C / 8;
  pl.P = 256 / pl.vecs;
  if (pl.P < 1) pl.P = 1;
  if (pl.P > hw) pl.P = hw;
  pl.threads = ((pl.vecs * pl.P + 31) / 32) * 32;
  int iters = 16;
  // large images: more pixels per block keep the partial table (re-read by every block of pass 2) at <= 128 slabs
  while (static_cast<long long>(hw) > 128LL * pl.P * iters && iters < 4096) iters *= 2;
  pl.pix_per_block = pl.P * iters;
  pl.bpi = static_cast<int>(div_up(hw, pl.pix_per_block));
  (void)n;
  return pl;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row held in registers (C <= 2048)
// ------------------------------------------------------------------------------------------------
constexpr int kLnMaxVec = 8;  // uint4 per lane -> C <= 32 * 8 * 8 = 2048

template <bool kBf16>
__global__ void __launch_bounds__(256)
layernorm_kernel(const void* __restrict__ x, const void* __restrict__ gamma, const void* __restrict__ beta,
                 void* __restrict__ out, long long rows, int Cdim, float eps, const void* __restrict__ pe,
                 long long rows_per_frame, int frames, int pe_off) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  pdl_launch_dependents();
  pdl_wait();
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int vecs = Cdim >> 3;
  const T* xr = static_cast<const T*>(x) + row * Cdim;
  uint4 u[kLnMaxVec];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = lane + i * 32;
    if (v < vecs) {
      u[i] = *reinterpret_cast<const uint4*>(xr + v * 8);
      const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = C::unpack(w[j]);
        sum += t.x + t.y;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / static_cast<float>(Cdim);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = lane + i * 32;
    if (v < vecs) {
      const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = C::unpack(w[j]);
        const float d0 = t.x - mean, d1 = t.y - mean;
        sq += d0 * d0 + d1 * d1;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / static_cast<float>(Cdim) + eps);
  const T* per = nullptr;
  if (pe) per = static_cast<const T*>(pe) + (pe_off + (row / rows_per_frame) % frames) * Cdim;
  T* orow = static_cast<T*>(out) + row * Cdim;
#pragma unroll
  for (int i = 0; i < kLnMaxVec; ++i) {
    const int v = lane + i * 32;
    if (v < vecs) {
      const uint4 ug = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(gamma) + v * 8));
      const uint4 ub = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(beta) + v * 8));
      const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
      const uint32_t wg[4] = {ug.x, ug.y, ug.z, ug.w};
      const uint32_t wb[4] = {ub.x, ub.y, ub.z, ub.w};
      uint32_t wp[4] = {0, 0, 0, 0};
      if (per) {
        const uint4 up = __ldg(reinterpret_cast<const uint4*>(per + v * 8));
        wp[0] = up.x;
        wp[1] = up.y;
        wp[2] = up.z;
        wp[3] = up.w;
      }
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = C::unpack(w[j]);
        const float2 g2 = C::unpack(wg[j]);
        const float2 b2 = C::unpack(wb[j]);
        float y0 = (t.x - mean) * rstd * g2.x + b2.x;
        float y1 = (t.y - mean) * rstd * g2.y + b2.y;
        if (per) {
          // the reference rounds LN's output to the storage type before adding the encoding
          const float2 p2 = C::unpack(wp[j]);
          y0 = C::to_f(C::from_f(y0)) + p2.x;
          y1 = C::to_f(C::from_f(y1)) + p2.y;
        }
        o[j] = C::pack(y0, y1);
      }
      *reinterpret_cast<uint4*>(orow + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// C = 40 L channels (320 / 640 / 1280: every transformer width of the UNet), L = 8 / 16 / 32 lanes per row: each lane
// owns exactly five 8-channel vectors, a warp normalises 32 / L rows at a time and keeps gamma / beta (packed) in
// registers across kLnIter row groups. The generic kernel above spends ~450 instructions per 320-wide row (predicated
// 8-way unroll at 62 % lane use, gamma / beta re-read and unpacked per row, 64-bit frame arithmetic) and is issue-bound
// at 1.9 TB/s; this one needs ~100.
constexpr int kLnIter = 4;

template <bool kBf16, int L>
__global__ void __launch_bounds__(256, 2)
layernorm5_kernel(const void* __restrict__ x, const void* __restrict__ gamma, const void* __restrict__ beta,
                  void* __restrict__ out, int rows, float eps, const void* __restrict__ pe, int rows_per_frame,
                  int frames, int pe_off) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  constexpr int R = 32 / L;       // rows per warp pass
  constexpr int Cdim = 40 * L;
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int sub = lane % L;
  const int rsel = lane / L;
  uint32_t g[5][4], b[5][4];  // packed pairs: unpacking on use is cheaper than 80 fp32 registers (occupancy)
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int v = sub + j * L;
    const uint4 ug = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(gamma) + v * 8));
    const uint4 ub = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(beta) + v * 8));
    g[j][0] = ug.x, g[j][1] = ug.y, g[j][2] = ug.z, g[j][3] = ug.w;
    b[j][0] = ub.x, b[j][1] = ub.y, b[j][2] = ub.z, b[j][3] = ub.w;
  }
  const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
#pragma unroll 1
  for (int it = 0; it < kLnIter; ++it) {
    const int row = (warp_global * kLnIter + it) * R + rsel;
    const bool ok = row < rows;
    const T* xr = static_cast<const T*>(x) + static_cast<long long>(row) * Cdim;
    uint4 u[5];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      u[j] = ok ? *reinterpret_cast<const uint4*>(xr + (sub + j * L) * 8) : make_uint4(0, 0, 0, 0);
      const uint32_t w[4] = {u[j].x, u[j].y, u[j].z, u[j].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 t = C::unpack(w[k]);
        sum += t.x + t.y;
      }
    }
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * (1.0f / Cdim);
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const uint32_t w[4] = {u[j].x, u[j].y, u[j].z, u[j].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 t = C::unpack(w[k]);
        const float d0 = t.x - mean, d1 = t.y - mean;
        sq += d0 * d0 + d1 * d1;
      }
    }
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq * (1.0f / Cdim) + eps);
    if (!ok) continue;
    const T* per = nullptr;
    if (pe) per = static_cast<const T*>(pe) + static_cast<long long>(pe_off + (row / rows_per_frame) % frames) * Cdim;
    T* orow = static_cast<T*>(out) + static_cast<long long>(row) * Cdim;
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const int v = sub + j * L;
      const uint32_t w[4] = {u[j].x, u[j].y, u[j].z, u[j].w};
      uint32_t wp[4] = {0, 0, 0, 0};
      if (per) {
        const uint4 up = __ldg(reinterpret_cast<const uint4*>(per + v * 8));
        wp[0] = up.x;
        wp[1] = up.y;
        wp[2] = up.z;
        wp[3] = up.w;
      }
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 t = C::unpack(w[k]);
        const float2 g2 = C::unpack(g[j][k]);
        const float2 b2 = C::unpack(b[j][k]);
        float y0 = (t.x - mean) * rstd * g2.x + b2.x;
        float y1 = (t.y - mean) * rstd * g2.y + b2.y;
        if (per) {
          // the reference rounds LN's output to the storage type before adding the encoding
          const float2 p2 = C::unpack(wp[k]);
          y0 = C::to_f(C::from_f(y0)) + p2.x;
          y1 = C::to_f(C::from_f(y1)) + p2.y;
        }
        o[k] = C::pack(y0, y1);
      }
      *reinterpret_cast<uint4*>(orow + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

template <bool kBf16>
static void launch_ln5(int L, const void* x, const void* gamma, const void* beta, void* out, int rows, float eps,
                       const void* pe, int rpf, int frames, int pe_off, cudaStream_t st) {
  const int rows_per_block = 8 * kLnIter * (32 / L);
  const unsigned blocks = div_up(rows, rows_per_block);
  if (L == 8)
    launch_k(layernorm5_kernel<kBf16, 8>, dim3(blocks), dim3(256), 0, st, x, gamma, beta, out, rows, eps, pe, rpf, frames, pe_off);
  else if (L == 16)
    launch_k(layernorm5_kernel<kBf16, 16>, dim3(blocks), dim3(256), 0, st, x, gamma, beta, out, rows, eps, pe, rpf, frames, pe_off);
  else
    launch_k(layernorm5_kernel<kBf16, 32>, dim3(blocks), dim3(256), 0, st, x, gamma, beta, out, rows, eps, pe, rpf, frames, pe_off);
}

}  // namespace mimo

using namespace mimo;

static int gn_check(const mimo_groupnorm_params* p, int* Cout) {
  if (!p) return set_error(MIMO_ERR_ARG, "mimo_groupnorm: null params");
  const int c1 = p->x1 ? p->c1 : 0;
  const int C = p->c0 + c1;
  if (p->n <= 0 || p->hw <= 0 || C <= 0 || p->groups <= 0 || p->groups > 64)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm: bad sizes");
  if ((p->c0 % 8) || (c1 % 8) || (C % p->groups) || (C / 8 > kGnMaxThreads))
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm: channels must be multiples of 8, divisible by groups, <= 2560");
  const int cpg = C / p->groups;  // an 8-channel vector may straddle at most two groups
  if (!(cpg >= 8 || cpg == 4)) return set_error(MIMO_ERR_ARG, "mimo_groupnorm: channels per group must be 4 or >= 8");
  *Cout = C;
  return MIMO_OK;
}

extern "C" int64_t mimo_groupnorm_workspace_bytes(const mimo_groupnorm_params* p) {
  int C = 0;
  if (int rc = gn_check(p, &C)) return rc;
  const GnPlan pl = gn_plan(p->n, p->hw, C);
  return static_cast<int64_t>(p->n) * pl.bpi * p->groups * 2 * sizeof(float);
}

extern "C" int mimo_groupnorm(const mimo_groupnorm_params* p, void* stream) {
  int C = 0;
  if (int rc = gn_check(p, &C)) return rc;
  if (!p->x0 || !p->gamma || !p->beta || !p->out || !p->stats)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm: null pointer");
  if (int rc = ensure_device()) return rc;
  const GnPlan pl = gn_plan(p->n, p->hw, C);
  GnArgs a;
  a.x0 = p->x0;
  a.x1 = p->x1;
  a.gamma = p->gamma;
  a.beta = p->beta;
  a.out = p->out;
  a.part = p->stats;
  a.c0 = p->c0;
  a.c1 = p->x1 ? p->c1 : 0;
  a.C = C;
  a.hw = p->hw;
  a.groups = p->groups;
  a.cpg = C / p->groups;
  a.vecs = pl.vecs;
  a.P = pl.P;
  a.pix_per_block = pl.pix_per_block;
  a.bpi = pl.bpi;
  a.eps = p->eps;
  a.silu = p->silu;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 grid(pl.bpi, p->n);
  cudaError_t e;
  if (p->dtype == MIMO_BF16) {
    e = launch_k(gn_stats_kernel<true>, grid, dim3(pl.threads), 0, st, a);
    if (e == cudaSuccess) e = launch_k(gn_apply_kernel<true>, grid, dim3(pl.threads), 0, st, a);
  } else {
    e = launch_k(gn_stats_kernel<false>, grid, dim3(pl.threads), 0, st, a);
    if (e == cudaSuccess) e = launch_k(gn_apply_kernel<false>, grid, dim3(pl.threads), 0, st, a);
  }
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("groupnorm launch", e);
  return MIMO_OK;
}

extern "C" int mimo_layernorm(const void* x, const void* gamma, const void* beta, void* out, int64_t rows,
                              int32_t c, float eps, const void* pe, int64_t rows_per_frame, int32_t frames,
                              int32_t pe_frame_offset, int32_t dtype, void* stream) {
  if (!x || !gamma || !beta || !out) return set_error(MIMO_ERR_ARG, "mimo_layernorm: null pointer");
  if (rows <= 0 || c <= 0 || (c % 8) || c > 32 * 8 * kLnMaxVec)
    return set_error(MIMO_ERR_ARG, "mimo_layernorm: c must be a multiple of 8 and <= 2048");
  if (pe && (rows_per_frame <= 0 || frames <= 0)) return set_error(MIMO_ERR_ARG, "mimo_layernorm: bad pe args");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int L = c == 320 ? 8 : (c == 640 ? 16 : (c == 1280 ? 32 : 0));
  if (L && rows < (1LL << 31) && rows_per_frame < (1LL << 31)) {
    const int rpf = pe ? static_cast<int>(rows_per_frame) : 1;
    if (dtype == MIMO_BF16)
      launch_ln5<true>(L, x, gamma, beta, out, static_cast<int>(rows), eps, pe, rpf, frames, pe_frame_offset, st);
    else
      launch_ln5<false>(L, x, gamma, beta, out, static_cast<int>(rows), eps, pe, rpf, frames, pe_frame_offset, st);
    cudaError_t e5 = cudaGetLastError();
    if (e5 != cudaSuccess) return set_cuda_error("layernorm launch", e5);
    return MIMO_OK;
  }
  const unsigned blocks = div_up(rows, 8);
  if (dtype == MIMO_BF16)
    launch_k(layernorm_kernel<true>, dim3(blocks), dim3(256), 0, st, x, gamma, beta, out, static_cast<long long>(rows), c, eps, pe,
             static_cast<long long>(rows_per_frame), frames, pe_frame_offset);
  else
    launch_k(layernorm_kernel<false>, dim3(blocks), dim3(256), 0, st, x, gamma, beta, out, static_cast<long long>(rows), c, eps, pe,
             static_cast<long long>(rows_per_frame), frames, pe_frame_offset);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("layernorm launch", e);
  return MIMO_OK;
}
