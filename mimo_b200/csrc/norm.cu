// GroupNorm(+SiLU) and LayerNorm(+positional encoding) over channels-last activations. HBM-bound passes:
// 128-bit loads/stores, fp32 statistics, each thread owns a fixed 8-channel vector so gamma/beta/mean/rstd
// are loaded once and the loop over pixels is pure streaming.
#include <cuda_runtime.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/mimo_b200.h"
#include "host_util.h"
#include "ptx.cuh"

namespace mimo {

// ------------------------------------------------------------------------------------------------
// GroupNorm(+SiLU), deterministic: two streaming kernels, no floating-point atomics.
//   pass 1: every block reduces its slab of pixels to per-group (sum, sumsq) of x - K_g in a FIXED order (registers ->
//           shared memory -> one thread per group) and publishes them: part[image][slab][group][2]
//   pass 2: every block sums the slabs' partials of its image in the same fixed order (bit-identical statistics in
//           every block and run to run), then normalises + affine (+ SiLU) with 128-bit loads / stores.
// K_g is one sample of the group (gn_shift). Without it, var = E[x^2] - mean^2 cancels nearly all of fp32's digits once
// |mean| >> std (at mean / std = 300 the output was off by ~1.5 % rel-L2); with it both terms are of the order of the
// variance, as in a two-pass computation, at the cost of a few cached scalar loads per block.
// (A one-pass variant that keeps the slab in registers across a per-image arrival barrier serialises the blocks of an
// image on that barrier, and deadlocks when an image has more slabs than blocks can be resident.)
// ------------------------------------------------------------------------------------------------
struct GnArgs {
  const void* x0;
  const void* x1;
  const void* gamma;
  const void* beta;
  void* out;
  float* part;  // [n][bpi][groups][2] = (sum, sumsq) of x - K_g per slab; window mode: the partial table (below)
  int c0, c1, C, hw, groups, cpg;
  int vecs;  // C / 8
  int P;     // pixels processed side by side by one block
  int pix_per_block;
  int bpi;   // slabs per image
  float eps;
  int silu;
  // window mode only: image n = sample * frames + frame; statistics per sample over every frame of the window
  int frames, samples;
  long long rec;       // floats per (frame, sample) record of the partial table
  const float* stats;  // [samples][groups][2] = (mean, rstd)
};

// the e4m3 output (mimo_groupnorm_e4m3; out is one byte per element). A separate type, so that the 16-bit kernels keep
// their parameter block.
struct GnE4m3Args : GnArgs {
  float* mm;      // [n][bpi][groups][2] = (min, max) of x per slab; per image, also in window mode (never gathered)
  float* qscale;  // [n]: the image's scale amax / 448
};
template <bool kE4m3>
using GnArgsT = std::conditional_t<kE4m3, GnE4m3Args, GnArgs>;

template <bool kBf16>
__device__ __forceinline__ uint4 gn_load(const GnArgs& a, long long pix, int cv) {
  using C = Cvt<kBf16>;
  const int ch = cv * 8;
  if (ch < a.c0) {
    return *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.x0) + pix * a.c0 + ch);
  }
  return *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.x1) + pix * a.c1 + (ch - a.c0));
}

// K_g: image n's first pixel in group g's first channel. Both passes read the same element, so every block shifts by
// the same value.
template <bool kBf16>
__device__ __forceinline__ float gn_shift(const GnArgs& a, int n, int g) {
  using C = Cvt<kBf16>;
  const int ch = g * a.cpg;
  const long long pix = static_cast<long long>(n) * a.hw;
  const typename C::T* p = ch < a.c0 ? static_cast<const typename C::T*>(a.x0) + pix * a.c0 + ch
                                     : static_cast<const typename C::T*>(a.x1) + pix * a.c1 + (ch - a.c0);
  return C::to_f(*p);
}

constexpr int kGnMaxThreads = 320;

// pass 1: per-(image, slab, group) sum and sum of squares. kWindow: the image is frame k of sample s, and the block
// writes slab row 1 + blockIdx.x of record (k, s); the first slab's block also writes the record's K_g row.
// kMinMax (the e4m3 output): also the slab's per-group min / max of x, into a.mm (per image, outside the window table).
template <bool kBf16, bool kWindow = false, bool kMinMax = false>
__global__ void __launch_bounds__(kGnMaxThreads) gn_stats_kernel(GnArgsT<kMinMax> a) {
  using C = Cvt<kBf16>;
  __shared__ float4 s_red[kGnMaxThreads];  // per-thread (sumA, sqA, sumB, sqB); with kMinMax then (loA, hiA, loB, hiB)
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
  [[maybe_unused]] float lA = INFINITY, hA = -INFINITY, lB = INFINITY, hB = -INFINITY;
  if (active) {
    const float kA = gn_shift<kBf16>(a, n, gA), kB = split < 8 ? gn_shift<kBf16>(a, n, gA + 1) : 0.f;
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
        if (2 * j < split) {
          const float d = t.x - kA;
          sA += d, qA += d * d;
        } else {
          const float d = t.x - kB;
          sB += d, qB += d * d;
        }
        if (2 * j + 1 < split) {
          const float d = t.y - kA;
          sA += d, qA += d * d;
        } else {
          const float d = t.y - kB;
          sB += d, qB += d * d;
        }
        if constexpr (kMinMax) {
          if (2 * j < split) lA = fminf(lA, t.x), hA = fmaxf(hA, t.x);
          else lB = fminf(lB, t.x), hB = fmaxf(hB, t.x);
          if (2 * j + 1 < split) lA = fminf(lA, t.y), hA = fmaxf(hA, t.y);
          else lB = fminf(lB, t.y), hB = fmaxf(hB, t.y);
        }
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
    if constexpr (kWindow) {
      const int smp = n / a.frames, k = n - smp * a.frames;
      float* rec = a.part + (static_cast<long long>(k) * a.samples + smp) * a.rec;
      float* dst = rec + (static_cast<long long>(1 + blockIdx.x) * a.groups + g) * 2;
      dst[0] = s;
      dst[1] = q;
      if (blockIdx.x == 0) {
        rec[2 * g] = gn_shift<kBf16>(a, n, g);
        rec[2 * g + 1] = 0.f;
      }
    } else {
      float* dst = a.part + ((static_cast<long long>(n) * a.bpi + blockIdx.x) * a.groups + g) * 2;
      dst[0] = s;
      dst[1] = q;
    }
  }
  if constexpr (kMinMax) {
    __syncthreads();
    s_red[tid] = make_float4(lA, hA, lB, hB);
    __syncthreads();
    for (int g = tid; g < a.groups; g += blockDim.x) {
      const int v_lo = (g * a.cpg) >> 3;
      const int v_hi = ((g + 1) * a.cpg - 1) >> 3;
      float lo = INFINITY, hi = -INFINITY;
      for (int v = v_lo; v <= v_hi; ++v) {
        const bool as_a = (v * 8) / a.cpg == g;
        for (int l = 0; l < a.P; ++l) {
          const float4 r = s_red[l * a.vecs + v];
          lo = fminf(lo, as_a ? r.x : r.z);
          hi = fmaxf(hi, as_a ? r.y : r.w);
        }
      }
      float* dst = a.mm + ((static_cast<long long>(n) * a.bpi + blockIdx.x) * a.groups + g) * 2;
      dst[0] = lo;
      dst[1] = hi;
    }
  }
}

// SiLU's only turning point: its minimum silu(-1.2784645) = -0.27846454
constexpr float kSiluArgMin = -1.2784645f;
constexpr float kSiluMinAbs = 0.27846454f;

// e4m3 output: the image's bound amax on |SiLU(GroupNorm(x))| (include/mimo_b200.h, mimo_groupnorm_e4m3), from the slab
// min / max of pass 1 and the normaliser's mean / rstd. Every block of the image computes the same value (min / max are
// exact in any order); the first writes the scale. Returns 448 / amax (1 for a zero bound) to every thread.
template <bool kBf16>
__device__ float gn_e4m3_inv(const GnE4m3Args& a, int n, const float* s_mean, const float* s_rstd) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  __shared__ float s_lo[64], s_hi[64], s_wmax[kGnMaxThreads / 32], s_inv;
  const int tid = threadIdx.x;
  const long long g2 = 2LL * a.groups;
  for (int g = tid; g < a.groups; g += blockDim.x) {
    const float* src = a.mm + static_cast<long long>(n) * a.bpi * g2 + 2 * g;
    float lo = INFINITY, hi = -INFINITY;
    for (int b = 0; b < a.bpi; ++b) {
      lo = fminf(lo, src[b * g2]);
      hi = fmaxf(hi, src[b * g2 + 1]);
    }
    s_lo[g] = lo;
    s_hi[g] = hi;
  }
  __syncthreads();
  float m = 0.f;
  for (int c = tid; c < a.C; c += blockDim.x) {
    const int g = c / a.cpg;
    // the same products as gn_normalise: y = fmaf(x - mean, rstd * gamma, beta)
    const float sc = s_rstd[g] * C::to_f(static_cast<const T*>(a.gamma)[c]);
    const float bc = C::to_f(static_cast<const T*>(a.beta)[c]);
    const float zl = fmaf(s_lo[g] - s_mean[g], sc, bc), zh = fmaf(s_hi[g] - s_mean[g], sc, bc);
    float bnd = fmaxf(fabsf(silu_f(zl)), fabsf(silu_f(zh)));
    if (fminf(zl, zh) <= kSiluArgMin && fmaxf(zl, zh) >= kSiluArgMin) bnd = fmaxf(bnd, kSiluMinAbs);
    m = fmaxf(m, bnd);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((tid & 31) == 0) s_wmax[tid >> 5] = m;
  __syncthreads();
  if (tid == 0) {
    float amax = 0.f;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) amax = fmaxf(amax, s_wmax[w]);
    s_inv = amax == 0.f ? 1.f : 448.0f / amax;
    if (blockIdx.x == 0) a.qscale[n] = amax == 0.f ? 1.f : amax / 448.0f;
  }
  __syncthreads();
  return s_inv;
}

// normalise + affine (+ SiLU) of image n's slab blockIdx.x, with the per-group mean / rstd in shared memory.
// kE4m3: always SiLU, then cvt.rn.satfinite.e4m3(y * inv) into one-byte elements.
template <bool kBf16, bool kE4m3 = false>
__device__ __forceinline__ void gn_normalise(const GnArgs& a, int n, const float* s_mean, const float* s_rstd,
                                             [[maybe_unused]] float inv = 1.f) {
  using C = Cvt<kBf16>;
  const int tid = threadIdx.x;
  const int cv = tid % a.vecs;
  const int pl = tid / a.vecs;
  if (pl >= a.P) return;
  const int ch0 = cv * 8;
  const int gA = ch0 / a.cpg;
  int split = (gA + 1) * a.cpg - ch0;
  if (split > 8) split = 8;
  // y = (x - mean) * (rstd * gamma) + beta. The folded form x * sc + (beta - mean * sc) cancels: both terms are of the
  // order |mean| * rstd, which reaches 1e6 for a near-constant group at mean 1000 (eps 1e-6), so its fp32 rounding
  // alone moved the output by 0.06. x - mean is exact or nearly so.
  float sc[8], bc[8], mA, mB;
  {
    const uint4 ug = *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.gamma) + ch0);
    const uint4 ub = *reinterpret_cast<const uint4*>(static_cast<const typename C::T*>(a.beta) + ch0);
    const uint32_t wg[4] = {ug.x, ug.y, ug.z, ug.w};
    const uint32_t wb[4] = {ub.x, ub.y, ub.z, ub.w};
    const float rA = s_rstd[gA], rB = split < 8 ? s_rstd[gA + 1] : 0.f;
    mA = s_mean[gA];
    mB = split < 8 ? s_mean[gA + 1] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 gg = C::unpack(wg[j]);
      const float2 bb = C::unpack(wb[j]);
      const float r0 = 2 * j < split ? rA : rB;
      const float r1 = 2 * j + 1 < split ? rA : rB;
      sc[2 * j] = r0 * gg.x;
      bc[2 * j] = bb.x;
      sc[2 * j + 1] = r1 * gg.y;
      bc[2 * j + 1] = bb.y;
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
      f[2 * j] = fmaf(t.x - (2 * j < split ? mA : mB), sc[2 * j], bc[2 * j]);
      f[2 * j + 1] = fmaf(t.y - (2 * j + 1 < split ? mA : mB), sc[2 * j + 1], bc[2 * j + 1]);
    }
    if constexpr (kE4m3) {
      uint32_t q[2];  // elements 4 j .. 4 j + 3 in q[j], lowest address in the lowest byte
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        uint16_t lo, hi;  // cvt packs its first source into the upper byte
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(silu_f(f[4 * j + 1]) * inv), "f"(silu_f(f[4 * j]) * inv));
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(silu_f(f[4 * j + 3]) * inv), "f"(silu_f(f[4 * j + 2]) * inv));
        q[j] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
      }
      *reinterpret_cast<uint2*>(static_cast<uint8_t*>(a.out) + pix * a.C + ch0) = make_uint2(q[0], q[1]);
    } else {
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
}

// pass 2: image statistics from the slab partials (fixed order), then normalise + affine (+ SiLU) (kE4m3: -> e4m3)
template <bool kBf16, bool kE4m3 = false>
__global__ void __launch_bounds__(kGnMaxThreads) gn_apply_kernel(GnArgsT<kE4m3> a) {
  __shared__ float s_tot[4][128];
  __shared__ float s_mean[64], s_rstd[64];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y;
  const int tid = threadIdx.x;
  const int g2 = a.groups * 2;
  {
    // K_g first (the same thread adds the shifted mean below): the load overlaps the partial sums
    for (int g = tid; g < a.groups; g += blockDim.x) s_mean[g] = gn_shift<kBf16>(a, n, g);
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
      const float dmean = s * inv_cnt;  // mean of x - K_g
      float var = q * inv_cnt - dmean * dmean;
      var = var < 0.f ? 0.f : var;
      s_mean[g] += dmean;
      s_rstd[g] = rsqrtf(var + a.eps);
    }
    __syncthreads();
  }
  if constexpr (kE4m3)
    gn_normalise<kBf16, true>(a, n, s_mean, s_rstd, gn_e4m3_inv<kBf16>(a, n, s_mean, s_rstd));
  else
    gn_normalise<kBf16>(a, n, s_mean, s_rstd);
}

// ------------------------------------------------------------------------------------------------
// Window mode (torch.nn.GroupNorm on [b, C, f, h, w]: one set of statistics per sample over all f frames).
// Partial table: one record per (frame k, sample s), frame-major ([f][samples][rec]), so the tables of consecutive
// frame slices concatenate into the table of the whole window. A record holds the K_g row (K_g, 0) of that frame's
// image, then bpi slab rows of (sum, sumsq) of x - K_g; its length is padded to a multiple of 4 floats (16 bytes).
// The reduction kernel adds, per sample and group, each frame's slabs in slab order, then moves the frame's sums to the
// shift of frame 0 and adds them in frame order: the order depends on the frame and slab indices only, so a table
// assembled from any frame-sharding gives bit-identical statistics.
// ------------------------------------------------------------------------------------------------
constexpr int kGnwReduceThreads = 256;
constexpr int kGnwFrameChunk = 16;

// one block per sample: stats[s][g] = (mean, rstd) over `table_frames` frames
__global__ void __launch_bounds__(kGnwReduceThreads) gnw_reduce_kernel(GnArgs a, int table_frames, float* stats) {
  __shared__ float s_tot[kGnwFrameChunk][128];
  pdl_launch_dependents();
  pdl_wait();
  const int smp = blockIdx.x;
  const int tid = threadIdx.x;
  const int g2 = a.groups * 2;
  const long long fstride = static_cast<long long>(a.samples) * a.rec;  // floats between frame k and k + 1
  const float* base = a.part + static_cast<long long>(smp) * a.rec;
  const float cnt = static_cast<float>(a.hw) * a.cpg;  // elements of one group in one frame
  const float k0 = tid < a.groups ? base[2 * tid] : 0.f;
  float S = 0.f, Q = 0.f;
  for (int f0 = 0; f0 < table_frames; f0 += kGnwFrameChunk) {
    const int nf = table_frames - f0 < kGnwFrameChunk ? table_frames - f0 : kGnwFrameChunk;
    for (int idx = tid; idx < nf * g2; idx += blockDim.x) {
      const int fi = idx / g2, k = idx - fi * g2;
      const float* r = base + (f0 + fi) * fstride + g2 + k;
      float acc = 0.f;
#pragma unroll 8
      for (int b = 0; b < a.bpi; ++b) acc += r[static_cast<long long>(b) * g2];
      s_tot[fi][k] = acc;
    }
    __syncthreads();
    if (tid < a.groups) {
      for (int fi = 0; fi < nf; ++fi) {
        const float d = base[(f0 + fi) * fstride + 2 * tid] - k0;  // K_g of this frame relative to frame 0's
        const float sf = s_tot[fi][2 * tid], qf = s_tot[fi][2 * tid + 1];
        // sum over the frame of (x - k0) and (x - k0)^2 from the sums of (x - K_f), (x - K_f)^2
        S += sf + cnt * d;
        Q += qf + d * (2.f * sf + cnt * d);
      }
    }
    __syncthreads();
  }
  if (tid < a.groups) {
    const float inv_cnt = 1.0f / (cnt * static_cast<float>(table_frames));
    const float dmean = S * inv_cnt;
    float var = Q * inv_cnt - dmean * dmean;
    var = var < 0.f ? 0.f : var;
    stats[(static_cast<long long>(smp) * a.groups + tid) * 2] = k0 + dmean;
    stats[(static_cast<long long>(smp) * a.groups + tid) * 2 + 1] = rsqrtf(var + a.eps);
  }
}

template <bool kBf16, bool kE4m3 = false>
__global__ void __launch_bounds__(kGnMaxThreads) gnw_apply_kernel(GnArgsT<kE4m3> a) {
  __shared__ float s_mean[64], s_rstd[64];
  pdl_launch_dependents();
  pdl_wait();
  const int n = blockIdx.y;
  const float* st = a.stats + static_cast<long long>(n / a.frames) * a.groups * 2;
  for (int g = threadIdx.x; g < a.groups; g += blockDim.x) {
    s_mean[g] = st[2 * g];
    s_rstd[g] = st[2 * g + 1];
  }
  __syncthreads();
  if constexpr (kE4m3)  // the window's mean / rstd with this frame's own min / max
    gn_normalise<kBf16, true>(a, n, s_mean, s_rstd, gn_e4m3_inv<kBf16>(a, n, s_mean, s_rstd));
  else
    gn_normalise<kBf16>(a, n, s_mean, s_rstd);
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

// ------------------------------------------------------------------------------------------------
// LayerNorm (+ PE) -> e4m3 rows with one fp32 scale each (the A operand of mimo_gemm_e4m3)
// ------------------------------------------------------------------------------------------------
// L lanes per row, NV 8-channel vectors per lane (C = 320 / 640 / 1280: L = 8 / 16 / 32 and NV = 5, every lane busy; any
// other C: L = 32, NV = 8, predicated). The row's fp32 values stay in registers between the amax and the conversion.
template <bool kBf16, int L, int NV>
__global__ void __launch_bounds__(256)
layernorm_e4m3_kernel(const void* __restrict__ x, const void* __restrict__ gamma, const void* __restrict__ beta,
                      uint8_t* __restrict__ out, float* __restrict__ scale, long long rows, int Cdim, float eps,
                      const void* __restrict__ pe, long long rows_per_frame, int frames, int pe_off) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  constexpr int R = 32 / L;  // rows per warp
  pdl_launch_dependents();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int sub = lane % L;
  const long long row = (static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R + lane / L;
  const bool ok = row < rows;  // no early exit: the lanes of a warp shuffle together
  const int vecs = Cdim >> 3;
  const T* xr = static_cast<const T*>(x) + (ok ? row : 0) * Cdim;
  uint4 u[NV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = sub + i * L;
    u[i] = (ok && v < vecs) ? *reinterpret_cast<const uint4*>(xr + v * 8) : make_uint4(0, 0, 0, 0);
    const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = C::unpack(w[j]);
      sum += t.x + t.y;
    }
  }
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / static_cast<float>(Cdim);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (sub + i * L < vecs) {
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
  for (int o = L / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / static_cast<float>(Cdim) + eps);
  const T* per = (pe && ok) ? static_cast<const T*>(pe) + (pe_off + (row / rows_per_frame) % frames) * Cdim : nullptr;
  float y[NV][8];
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = sub + i * L;
    if (v < vecs) {
      const uint4 ug = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(gamma) + v * 8));
      const uint4 ub = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(beta) + v * 8));
      const uint4 up = per ? __ldg(reinterpret_cast<const uint4*>(per + v * 8)) : make_uint4(0, 0, 0, 0);
      const uint32_t w[4] = {u[i].x, u[i].y, u[i].z, u[i].w};
      const uint32_t wg[4] = {ug.x, ug.y, ug.z, ug.w};
      const uint32_t wb[4] = {ub.x, ub.y, ub.z, ub.w};
      const uint32_t wp[4] = {up.x, up.y, up.z, up.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = C::unpack(w[j]);
        const float2 g2 = C::unpack(wg[j]);
        const float2 b2 = C::unpack(wb[j]);
        float y0 = (t.x - mean) * rstd * g2.x + b2.x;
        float y1 = (t.y - mean) * rstd * g2.y + b2.y;
        if (per) {
          // as mimo_layernorm: LN's output is rounded to the storage type before the encoding is added
          const float2 p2 = C::unpack(wp[j]);
          y0 = C::to_f(C::from_f(y0)) + p2.x;
          y1 = C::to_f(C::from_f(y1)) + p2.y;
        }
        y[i][2 * j] = y0;
        y[i][2 * j + 1] = y1;
        amax = fmaxf(amax, fmaxf(fabsf(y0), fabsf(y1)));
      }
    }
  }
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (!ok) return;
  const float inv = amax == 0.f ? 1.f : 448.0f / amax;
  if (sub == 0) scale[row] = amax == 0.f ? 1.f : amax / 448.0f;
  uint8_t* orow = out + row * Cdim;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = sub + i * L;
    if (v < vecs) {
      uint32_t q[2];  // 8 bytes: elements 4 j .. 4 j + 3 in q[j], lowest address in the lowest byte
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        uint16_t lo, hi;  // cvt packs its first source into the upper byte
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(y[i][4 * j + 1] * inv), "f"(y[i][4 * j] * inv));
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(y[i][4 * j + 3] * inv), "f"(y[i][4 * j + 2] * inv));
        q[j] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
      }
      *reinterpret_cast<uint2*>(orow + v * 8) = make_uint2(q[0], q[1]);
    }
  }
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
  GnArgs a = {};
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

// ---- window mode ----
static int gnw_check(const mimo_groupnorm_window_params* p, const char* who, int* Cout) {
  static thread_local char msg[160];
  auto fail = [&](const char* what) {
    snprintf(msg, sizeof(msg), "%s: %s", who, what);
    return set_error(MIMO_ERR_ARG, msg);
  };
  if (!p) return fail("null params");
  if (p->samples <= 0 || p->frames <= 0 || p->hw <= 0 || p->groups <= 0 || p->groups > 64)
    return fail("bad sizes (samples, frames, hw and groups must be > 0, groups <= 64)");
  if (static_cast<long long>(p->samples) * p->frames > 65535) return fail("samples * frames must be <= 65535");
  const int c1 = p->x1 ? p->c1 : 0;
  const int C = p->c0 + c1;
  if (p->c0 <= 0 || c1 < 0 || (p->c0 % 8) || (c1 % 8) || (C % p->groups) || (C / 8 > kGnMaxThreads))
    return fail("channels must be multiples of 8, divisible by groups, <= 2560");
  const int cpg = C / p->groups;
  if (!(cpg >= 8 || cpg == 4)) return fail("channels per group must be 4 or >= 8");
  if (p->dtype != MIMO_F16 && p->dtype != MIMO_BF16) return fail("dtype must be MIMO_F16 or MIMO_BF16");
  *Cout = C;
  return MIMO_OK;
}

// floats per (frame, sample) record: the K_g row and bpi slab rows of (sum, sumsq), padded to 16 bytes
static long long gnw_rec_floats(const GnPlan& pl, int groups) {
  return (2LL * groups * (pl.bpi + 1) + 3) / 4 * 4;
}

static GnArgs gnw_args(const mimo_groupnorm_window_params* p, int C, const GnPlan& pl) {
  GnArgs a = {};
  a.x0 = p->x0;
  a.x1 = p->x1;
  a.gamma = p->gamma;
  a.beta = p->beta;
  a.out = p->out;
  a.part = p->table;
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
  a.frames = p->frames;
  a.samples = p->samples;
  a.rec = gnw_rec_floats(pl, p->groups);
  a.stats = p->stats;
  return a;
}

static int64_t gnw_table_bytes(const mimo_groupnorm_window_params* p, int C, int frames) {
  const GnPlan pl = gn_plan(p->samples * p->frames, p->hw, C);
  return static_cast<int64_t>(frames) * p->samples * gnw_rec_floats(pl, p->groups) * static_cast<int64_t>(sizeof(float));
}

extern "C" int64_t mimo_groupnorm_window_table_bytes(const mimo_groupnorm_window_params* p) {
  int C = 0;
  if (int rc = gnw_check(p, "mimo_groupnorm_window_table_bytes", &C)) return rc;
  return gnw_table_bytes(p, C, p->frames);
}

// the launches behind the three entry points: partials (pass 1), and/or reduce + normalise (pass 2)
static int gnw_launch(const mimo_groupnorm_window_params* p, int C, bool partials, bool apply, int table_frames,
                      void* stream) {
  const GnPlan pl = gn_plan(p->samples * p->frames, p->hw, C);
  const GnArgs a = gnw_args(p, C, pl);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(pl.bpi, p->samples * p->frames);
  const bool bf = p->dtype == MIMO_BF16;
  cudaError_t e = cudaSuccess;
  if (partials)
    e = bf ? launch_k(gn_stats_kernel<true, true>, grid, dim3(pl.threads), 0, st, a)
           : launch_k(gn_stats_kernel<false, true>, grid, dim3(pl.threads), 0, st, a);
  if (apply && e == cudaSuccess) {
    e = launch_k(gnw_reduce_kernel, dim3(p->samples), dim3(kGnwReduceThreads), 0, st, a, table_frames, p->stats);
    if (e == cudaSuccess)
      e = bf ? launch_k(gnw_apply_kernel<true>, grid, dim3(pl.threads), 0, st, a)
             : launch_k(gnw_apply_kernel<false>, grid, dim3(pl.threads), 0, st, a);
  }
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("groupnorm_window launch", e);
  return MIMO_OK;
}

extern "C" int mimo_groupnorm_window(const mimo_groupnorm_window_params* p, void* stream) {
  const char* who = "mimo_groupnorm_window";
  int C = 0;
  if (int rc = gnw_check(p, who, &C)) return rc;
  if (!p->x0 || !p->gamma || !p->beta || !p->out || !p->table || !p->stats)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_window: null pointer");
  if (p->table_bytes < gnw_table_bytes(p, C, p->frames))
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_window: partial table smaller than mimo_groupnorm_window_table_bytes");
  if (int rc = ensure_device()) return rc;
  return gnw_launch(p, C, true, true, p->frames, stream);
}

extern "C" int mimo_groupnorm_window_partials(const mimo_groupnorm_window_params* p, void* stream) {
  const char* who = "mimo_groupnorm_window_partials";
  int C = 0;
  if (int rc = gnw_check(p, who, &C)) return rc;
  if (!p->x0 || !p->table) return set_error(MIMO_ERR_ARG, "mimo_groupnorm_window_partials: null pointer");
  if (p->table_bytes < gnw_table_bytes(p, C, p->frames))
    return set_error(MIMO_ERR_ARG,
                     "mimo_groupnorm_window_partials: partial table smaller than mimo_groupnorm_window_table_bytes");
  if (int rc = ensure_device()) return rc;
  return gnw_launch(p, C, true, false, 0, stream);
}

extern "C" int mimo_groupnorm_window_apply(const mimo_groupnorm_window_params* p, void* stream) {
  const char* who = "mimo_groupnorm_window_apply";
  int C = 0;
  if (int rc = gnw_check(p, who, &C)) return rc;
  if (p->table_frames < p->frames)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_window_apply: table_frames must be >= frames (the whole window)");
  if (!p->x0 || !p->gamma || !p->beta || !p->out || !p->table || !p->stats)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_window_apply: null pointer");
  if (p->table_bytes < gnw_table_bytes(p, C, p->table_frames))
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_window_apply: partial table smaller than table_frames records");
  if (int rc = ensure_device()) return rc;
  return gnw_launch(p, C, false, true, p->table_frames, stream);
}

// ---- GroupNorm + SiLU -> e4m3 ----
static mimo_groupnorm_window_params gn8_as_window(const mimo_groupnorm_e4m3_params* p) {
  mimo_groupnorm_window_params w = {};
  w.x0 = p->x0;
  w.c0 = p->c0;
  w.x1 = p->x1;
  w.c1 = p->c1;
  w.gamma = p->gamma;
  w.beta = p->beta;
  w.out = p->out;
  w.table = p->table;
  w.table_bytes = p->table_bytes;
  w.samples = p->samples;
  w.frames = p->frames;
  w.table_frames = p->table_frames;
  w.hw = p->hw;
  w.groups = p->groups;
  w.eps = p->eps;
  w.silu = 1;
  w.dtype = p->dtype;
  return w;
}

// work: [images][bpi][groups][2] (min, max) of x, then the per-image partials ([images][bpi][groups][2], FRAME mode) or
// the window statistics ([samples][groups][2], window modes)
static int gn8_sizes(const mimo_groupnorm_e4m3_params* p, int* C, GnPlan* pl, long long* mm_floats, int64_t* work_bytes) {
  if (!p) return set_error(MIMO_ERR_ARG, "mimo_groupnorm_e4m3: null params");
  if (p->mode < MIMO_GN_E4M3_FRAME || p->mode > MIMO_GN_E4M3_WINDOW_APPLY)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_e4m3: unknown mode");
  const mimo_groupnorm_window_params w = gn8_as_window(p);
  if (int rc = gnw_check(&w, "mimo_groupnorm_e4m3", C)) return rc;
  *pl = gn_plan(p->samples * p->frames, p->hw, *C);
  *mm_floats = static_cast<long long>(p->samples) * p->frames * pl->bpi * p->groups * 2;
  const long long rest = p->mode == MIMO_GN_E4M3_FRAME ? *mm_floats : 2LL * p->samples * p->groups;
  *work_bytes = static_cast<int64_t>((*mm_floats + rest) * sizeof(float));
  return MIMO_OK;
}

extern "C" int64_t mimo_groupnorm_e4m3_workspace_bytes(const mimo_groupnorm_e4m3_params* p) {
  int C = 0;
  GnPlan pl;
  long long mmf = 0;
  int64_t wb = 0;
  if (int rc = gn8_sizes(p, &C, &pl, &mmf, &wb)) return rc;
  return wb;
}

extern "C" int mimo_groupnorm_e4m3(const mimo_groupnorm_e4m3_params* p, void* stream) {
  int C = 0;
  GnPlan pl;
  long long mmf = 0;
  int64_t wb = 0;
  if (int rc = gn8_sizes(p, &C, &pl, &mmf, &wb)) return rc;
  const int mode = p->mode;
  const bool window = mode != MIMO_GN_E4M3_FRAME;
  const bool partials = mode != MIMO_GN_E4M3_WINDOW_APPLY, apply = mode != MIMO_GN_E4M3_WINDOW_PARTIALS;
  if (!p->x0 || !p->work || (apply && (!p->gamma || !p->beta || !p->out || !p->scale)) || (window && !p->table))
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_e4m3: null pointer");
  if (p->work_bytes < wb) return set_error(MIMO_ERR_ARG, "mimo_groupnorm_e4m3: work smaller than its workspace bytes");
  if (mode == MIMO_GN_E4M3_WINDOW_APPLY && p->table_frames < p->frames)
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_e4m3: table_frames must be >= frames (the whole window)");
  const mimo_groupnorm_window_params w = gn8_as_window(p);
  const int table_frames = mode == MIMO_GN_E4M3_WINDOW_APPLY ? p->table_frames : p->frames;
  if (window && p->table_bytes < gnw_table_bytes(&w, C, table_frames))
    return set_error(MIMO_ERR_ARG, "mimo_groupnorm_e4m3: partial table smaller than its records");
  if (int rc = ensure_device()) return rc;
  GnE4m3Args a;
  static_cast<GnArgs&>(a) = gnw_args(&w, C, pl);
  a.mm = p->work;
  a.qscale = p->scale;
  float* rest = p->work + mmf;
  if (!window) a.part = rest;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(pl.bpi, p->samples * p->frames);
  const bool bf = p->dtype == MIMO_BF16;
  cudaError_t e = cudaSuccess;
  if (!window) {
    e = bf ? launch_k(gn_stats_kernel<true, false, true>, grid, dim3(pl.threads), 0, st, a)
           : launch_k(gn_stats_kernel<false, false, true>, grid, dim3(pl.threads), 0, st, a);
    if (e == cudaSuccess)
      e = bf ? launch_k(gn_apply_kernel<true, true>, grid, dim3(pl.threads), 0, st, a)
             : launch_k(gn_apply_kernel<false, true>, grid, dim3(pl.threads), 0, st, a);
  } else {
    if (partials)
      e = bf ? launch_k(gn_stats_kernel<true, true, true>, grid, dim3(pl.threads), 0, st, a)
             : launch_k(gn_stats_kernel<false, true, true>, grid, dim3(pl.threads), 0, st, a);
    if (apply && e == cudaSuccess) {
      a.stats = rest;
      e = launch_k(gnw_reduce_kernel, dim3(p->samples), dim3(kGnwReduceThreads), 0, st, static_cast<const GnArgs&>(a),
                   table_frames, rest);
      if (e == cudaSuccess)
        e = bf ? launch_k(gnw_apply_kernel<true, true>, grid, dim3(pl.threads), 0, st, a)
               : launch_k(gnw_apply_kernel<false, true>, grid, dim3(pl.threads), 0, st, a);
    }
  }
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("groupnorm_e4m3 launch", e);
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

extern "C" int mimo_layernorm_e4m3(const void* x, const void* gamma, const void* beta, void* out, float* scale,
                                   int64_t rows, int32_t c, float eps, const void* pe, int64_t rows_per_frame,
                                   int32_t frames, int32_t pe_frame_offset, int32_t dtype, void* stream) {
  if (!x || !gamma || !beta || !out || !scale) return set_error(MIMO_ERR_ARG, "mimo_layernorm_e4m3: null pointer");
  if (rows <= 0 || c <= 0 || (c % 16) || c > 32 * 8 * kLnMaxVec)
    return set_error(MIMO_ERR_ARG, "mimo_layernorm_e4m3: c must be a multiple of 16 and <= 2048");
  if (pe && (rows_per_frame <= 0 || frames <= 0)) return set_error(MIMO_ERR_ARG, "mimo_layernorm_e4m3: bad pe args");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int L = c == 320 ? 8 : (c == 640 ? 16 : (c == 1280 ? 32 : 0));
  const unsigned blocks = div_up(rows, 8LL * (L ? 32 / L : 1));
  uint8_t* o = static_cast<uint8_t*>(out);
  const long long r = rows, rpf = pe ? rows_per_frame : 1;
  cudaError_t e;
#define MIMO_LN_E4M3(BF, LL, NV)                                                                                       \
  e = launch_k(layernorm_e4m3_kernel<BF, LL, NV>, dim3(blocks), dim3(256), 0, st, x, gamma, beta, o, scale, r, c, eps, pe, \
               rpf, frames, pe_frame_offset)
  if (dtype == MIMO_BF16) {
    if (L == 8) MIMO_LN_E4M3(true, 8, 5);
    else if (L == 16) MIMO_LN_E4M3(true, 16, 5);
    else if (L == 32) MIMO_LN_E4M3(true, 32, 5);
    else MIMO_LN_E4M3(true, 32, kLnMaxVec);
  } else {
    if (L == 8) MIMO_LN_E4M3(false, 8, 5);
    else if (L == 16) MIMO_LN_E4M3(false, 16, 5);
    else if (L == 32) MIMO_LN_E4M3(false, 32, 5);
    else MIMO_LN_E4M3(false, 32, kLnMaxVec);
  }
#undef MIMO_LN_E4M3
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("layernorm_e4m3 launch", e);
  return MIMO_OK;
}
