// Layout converters, im2col gather, add / SiLU, and the fused CFG + DDIM / multistep updates. All single coalesced
// passes.
#include <cuda_runtime.h>

#include <cmath>

#include "../../include/mimo_b200.h"
#include "host_util.h"
#include "ptx.cuh"

namespace mimo {

// [b, c, f, h, w] -> [(b f), h, w, cpad]; one thread per output (pixel, 8-channel vector)
template <bool kBf16, typename SrcT>
__global__ void ncfhw_to_nhwc_kernel(const SrcT* __restrict__ src, void* __restrict__ dst, int b, int c, int f,
                                     int h, int w, int cpad) {
  using C = Cvt<kBf16>;
  const long long hw = static_cast<long long>(h) * w;
  const int vecs = cpad / 8;
  const long long total = static_cast<long long>(b) * f * hw * vecs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % vecs);
    const long long pix = i / vecs;  // ((bi * f + fi) * hw + p)
    const long long p = pix % hw;
    const long long nf = pix / hw;
    const int fi = static_cast<int>(nf % f);
    const int bi = static_cast<int>(nf / f);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = cv * 8 + j;
      v[j] = 0.f;
      if (ch < c) {
        const long long s = ((static_cast<long long>(bi) * c + ch) * f + fi) * hw + p;
        if constexpr (sizeof(SrcT) == 4) {
          v[j] = src[s];
        } else {
          v[j] = C::to_f(reinterpret_cast<const typename C::T*>(src)[s]);
        }
      }
    }
    uint4 o;
    o.x = C::pack(v[0], v[1]);
    o.y = C::pack(v[2], v[3]);
    o.z = C::pack(v[4], v[5]);
    o.w = C::pack(v[6], v[7]);
    *reinterpret_cast<uint4*>(static_cast<typename C::T*>(dst) + pix * cpad + cv * 8) = o;
  }
}

// [(b f), h, w, ld] -> [b, c, f, h, w]; one thread per output element (w fastest -> coalesced writes)
template <bool kBf16, typename DstT>
__global__ void nhwc_to_ncfhw_kernel(const void* __restrict__ src, DstT* __restrict__ dst, int b, int c, int f,
                                     int h, int w, int ld) {
  using C = Cvt<kBf16>;
  const long long hw = static_cast<long long>(h) * w;
  const long long total = static_cast<long long>(b) * c * f * hw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = i % hw;
    long long t = i / hw;
    const int fi = static_cast<int>(t % f);
    t /= f;
    const int ch = static_cast<int>(t % c);
    const int bi = static_cast<int>(t / c);
    const float v = C::to_f(static_cast<const typename C::T*>(src)[((static_cast<long long>(bi) * f + fi) * hw + p) * ld + ch]);
    if constexpr (sizeof(DstT) == 4) {
      dst[i] = v;
    } else {
      reinterpret_cast<typename C::T*>(dst)[i] = C::from_f(v);
    }
  }
}

// im2col for 3x3 windows: col[(n, oy, ox), tap * c + ch], optional stride and nearest-upsampled input.
// pad_lo is the number of zero rows/cols before the first input sample (1 for "padding=1"; 0 for the VAE
// encoder's asymmetric F.pad(0,1,0,1) + padding=0 downsample).
template <typename T>
__global__ void im2col3x3_kernel(const T* __restrict__ x, T* __restrict__ col, int n, int h, int w, int c,
                                 int stride, int upshift, int pad_lo, int oh, int ow, long long ldcol) {
  const int vecs = c / 8;
  const long long total = static_cast<long long>(n) * oh * ow * 9 * vecs;
  const int uh = h << upshift, uw = w << upshift;  // logical (upsampled) input size
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % vecs);
    long long t = i / vecs;
    const int tap = static_cast<int>(t % 9);
    const long long opix = t / 9;
    const int ox = static_cast<int>(opix % ow);
    const int oy = static_cast<int>((opix / ow) % oh);
    const long long ni = opix / (static_cast<long long>(ow) * oh);
    const int iy = oy * stride - pad_lo + tap / 3;
    const int ix = ox * stride - pad_lo + tap % 3;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < uh && ix >= 0 && ix < uw) {
      const long long sp = (ni * h + (iy >> upshift)) * w + (ix >> upshift);
      v = *reinterpret_cast<const uint4*>(x + sp * c + cv * 8);
    }
    *reinterpret_cast<uint4*>(col + opix * ldcol + static_cast<long long>(tap) * c + cv * 8) = v;
  }
}

// nearest x2 upsample, channels-last: one thread per output (pixel, 8-channel vector)
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int n, int h, int w, int vecs) {
  const int oh = 2 * h, ow = 2 * w;
  const long long total = static_cast<long long>(n) * oh * ow * vecs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % vecs);
    const long long opix = i / vecs;
    const int ox = static_cast<int>(opix % ow);
    const int oy = static_cast<int>((opix / ow) % oh);
    const long long ni = opix / (static_cast<long long>(ow) * oh);
    out[i] = x[((ni * h + (oy >> 1)) * w + (ox >> 1)) * vecs + cv];
  }
}

// nearest resize to any (oh, ow), channels-last: one thread per output (pixel, 8-channel vector). The source index is
// PyTorch's for F.interpolate(mode="nearest", size=...): floor(d * (float(in) / out)) in fp32, clamped to in - 1.
__global__ void upsample_nearest_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int n, int h, int w,
                                        int oh, int ow, int vecs, float sy, float sx) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(n) * oh * ow * vecs;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % vecs);
    const long long opix = i / vecs;
    const int ox = static_cast<int>(opix % ow);
    const int oy = static_cast<int>((opix / ow) % oh);
    const long long ni = opix / (static_cast<long long>(ow) * oh);
    const int iy = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(oy), sy))), h - 1);
    const int ix = min(static_cast<int>(floorf(__fmul_rn(static_cast<float>(ox), sx))), w - 1);
    out[i] = x[((ni * h + iy) * w + ix) * vecs + cv];
  }
}

// in-place row softmax, one CTA per row, fp32 math
template <bool kBf16>
__global__ void __launch_bounds__(256) softmax_rows_kernel(void* __restrict__ xp, int cols, long long ld) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  __shared__ float red[32];
  T* row = static_cast<T*>(xp) + static_cast<long long>(blockIdx.x) * ld;
  const int vecs = cols / 8;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = C::unpack(w[j]);
      m = fmaxf(m, fmaxf(t.x, t.y));
    }
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < (blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = C::unpack(w[j]);
      s += __expf(t.x - m) + __expf(t.y - m);
    }
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) s += red[i];
  const float inv = 1.0f / s;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(row)[v];
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 t = C::unpack(w[j]);
      o[j] = C::pack(__expf(t.x - m) * inv, __expf(t.y - m) * inv);
    }
    reinterpret_cast<uint4*>(row)[v] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

template <bool kBf16, int kOp>  // 0: add, 1: silu, 2: quick-GELU x * sigmoid(1.702 x) (CLIP's hidden_act)
__global__ void ew_kernel(const void* __restrict__ a, const void* __restrict__ b, void* __restrict__ out,
                          long long nvec) {
  using C = Cvt<kBf16>;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 ua = static_cast<const uint4*>(a)[i];
    uint4 ub = make_uint4(0, 0, 0, 0);
    if (kOp == 0) ub = static_cast<const uint4*>(b)[i];
    const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w};
    const uint32_t wb[4] = {ub.x, ub.y, ub.z, ub.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x = C::unpack(wa[j]);
      if (kOp == 0) {
        const float2 y = C::unpack(wb[j]);
        o[j] = C::pack(x.x + y.x, x.y + y.y);
      } else if (kOp == 1) {
        o[j] = C::pack(silu_f(x.x), silu_f(x.y));
      } else {
        o[j] = C::pack(__fdividef(x.x, 1.0f + __expf(-1.702f * x.x)), __fdividef(x.y, 1.0f + __expf(-1.702f * x.y)));
      }
    }
    static_cast<uint4*>(out)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// The reference's guidance line (pipeline :545-549) on element i, rounded where its torch expression rounds in the storage
// type: (noise_pred / counter).chunk(2) when a per-frame counter is given, then u + g * (c - u). Leaves u and c as the
// divided halves (c is diffusers' noise_pred_text). Shared by every CFG kernel so that they guide identically.
template <bool kBf16>
__device__ __forceinline__ float cfg_guide(float& u, float& c, const typename Cvt<kBf16>::T* cnt, long long i,
                                           long long frame_stride, int frames, float g) {
  using C = Cvt<kBf16>;
  auto rnd = [](float v) { return C::to_f(C::from_f(v)); };
  if (cnt) {
    const float n = C::to_f(cnt[(i / frame_stride) % frames]);
    u = rnd(u / n);
    c = rnd(c / n);
  }
  return rnd(u + rnd(g * rnd(c - u)));
}

// CFG + DDIM (v-prediction). Every intermediate is rounded to the storage type where the reference's torch expression
// would round it (it runs the whole update in the latents' dtype). kNoise: stochastic DDIM (eta > 0): s1a_p is then the
// direction coefficient sqrt(1 - abar_prev - sigma^2), and sigma * noise is added last, as DDIMScheduler.step [3P] does.
template <bool kBf16, bool kNoise>
__global__ void cfg_ddim_kernel(const void* __restrict__ pu, const void* __restrict__ pc,
                                const void* __restrict__ counter, long long frame_stride, int frames,
                                void* __restrict__ lat, long long count, float g, float sa_t, float s1a_t,
                                float sa_p, float s1a_p, const void* __restrict__ noise, float sigma) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  auto rnd = [](float v) { return C::to_f(C::from_f(v)); };
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float u = C::to_f(static_cast<const T*>(pu)[i]);
    float c = C::to_f(static_cast<const T*>(pc)[i]);
    const float v = cfg_guide<kBf16>(u, c, static_cast<const T*>(counter), i, frame_stride, frames, g);
    const float x = C::to_f(static_cast<T*>(lat)[i]);
    // DDIMScheduler.step: alpha terms are fp32 scalars -> products promote to fp32 only for 0-dim tensors'
    // python floats; tensor math stays in the storage dtype
    const float x0 = rnd(rnd(sa_t * x) - rnd(s1a_t * v));
    const float e = rnd(rnd(sa_t * v) + rnd(s1a_t * x));
    const float dir = rnd(s1a_p * e);
    float prev = rnd(rnd(sa_p * x0) + dir);
    if constexpr (kNoise) prev = rnd(prev + rnd(sigma * C::to_f(static_cast<const T*>(noise)[i])));
    static_cast<T*>(lat)[i] = C::from_f(prev);
  }
}

// CFG + one multistep / sigma-space solver step (mimo_cfg_multistep). The guidance lines are cfg_ddim_kernel's, with its
// roundings; m is rounded to the storage type (it is stored as history), the update is fp32 and rounded once. hist_out
// may alias h2: h2[i] is read before hist_out[i] is written, by the same thread, so neither pointer is __restrict__.
template <bool kBf16>
__global__ void cfg_multistep_kernel(const mimo_cfg_multistep_params p, int frames) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  const T* __restrict__ pu = static_cast<const T*>(p.pred_uncond);
  const T* __restrict__ pc = static_cast<const T*>(p.pred_cond);
  const T* __restrict__ cnt = static_cast<const T*>(p.counter);
  const T* __restrict__ h1 = static_cast<const T*>(p.h1);
  const T* __restrict__ nz = static_cast<const T*>(p.noise);
  const T* h2 = static_cast<const T*>(p.h2);
  T* hist = static_cast<T*>(p.hist_out);
  T* __restrict__ lat = static_cast<T*>(p.latents);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < p.count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float u = C::to_f(pu[i]);
    float c = C::to_f(pc[i]);
    const float v = cfg_guide<kBf16>(u, c, cnt, i, p.frame_stride, frames, p.guidance);
    const float x = C::to_f(lat[i]);
    const T mt = C::from_f(fmaf(p.a, x, p.b * v));
    const float m = C::to_f(mt);
    float acc = fmaf(p.c_x, x, p.c_m * m);
    if (h1) acc = fmaf(p.c_1, C::to_f(h1[i]), acc);
    if (h2) acc = fmaf(p.c_2, C::to_f(h2[i]), acc);
    if (nz) acc = fmaf(p.c_n, C::to_f(nz[i]), acc);
    hist[i] = mt;
    lat[i] = C::from_f(acc);
  }
}

// Rescaled CFG (mimo_cfg_rescale), two launches of the same count-only grid. The statistics pass writes one fixed
// partial per CTA (sum and sum of squares of the text half and of the guided value, fp64); the apply pass has every CTA
// add all partials in the same fixed order, so each derives bit-identical statistics with no atomics and no host sync.
constexpr int kRescaleThreads = 256;
constexpr long long kRescaleElemsPerCta = 4096;
constexpr int kRescaleMaxCtas = 256;  // the apply pass re-reads at most 256 x 32 B of partials per CTA

static inline int cfg_rescale_ctas(long long count) {
  const long long b = (count + kRescaleElemsPerCta - 1) / kRescaleElemsPerCta;
  return static_cast<int>(b < 1 ? 1 : (b > kRescaleMaxCtas ? kRescaleMaxCtas : b));
}

// sums s[0..3] over the CTA: fixed xor-shuffle tree per warp, then every thread adds the warp totals in warp order
__device__ __forceinline__ void cta_sum4(double (&s)[4], double (*red)[kRescaleThreads / 32]) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < 4; ++k) red[k][threadIdx.x >> 5] = s[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    s[k] = 0.0;
    for (int w = 0; w < kRescaleThreads / 32; ++w) s[k] += red[k][w];
  }
}

template <bool kBf16>
__global__ void __launch_bounds__(kRescaleThreads) cfg_rescale_stats_kernel(const mimo_cfg_rescale_params p,
                                                                              int frames) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  __shared__ double red[4][kRescaleThreads / 32];
  const T* __restrict__ pu = static_cast<const T*>(p.pred_uncond);
  const T* __restrict__ pc = static_cast<const T*>(p.pred_cond);
  const T* __restrict__ cnt = static_cast<const T*>(p.counter);
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < p.count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float u = C::to_f(pu[i]);
    float c = C::to_f(pc[i]);
    const double g = cfg_guide<kBf16>(u, c, cnt, i, p.frame_stride, frames, p.guidance);
    const double t = c;
    s[0] += t;
    s[1] = fma(t, t, s[1]);
    s[2] += g;
    s[3] = fma(g, g, s[3]);
  }
  cta_sum4(s, red);
  if (threadIdx.x == 0) {
    double* part = static_cast<double*>(p.workspace) + 4LL * blockIdx.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) part[k] = s[k];
  }
}

// out = phi * rnd(cfg * r) + (1 - phi) * cfg, r = rnd(rnd(std(text)) / rnd(std(cfg))) (r = 1 when std(cfg) rounds to 0),
// each product and the sum rounded to the storage type: diffusers' rescale_noise_cfg [3P] evaluated by PyTorch in that
// type. w1 / w0 are phi and 1 - phi, computed in double and cast to fp32 as PyTorch casts a Python scalar.
template <bool kBf16>
__global__ void __launch_bounds__(kRescaleThreads) cfg_rescale_apply_kernel(const mimo_cfg_rescale_params p,
                                                                              int frames, int parts, float w1,
                                                                              float w0) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  auto rnd = [](float v) { return C::to_f(C::from_f(v)); };
  __shared__ double red[4][kRescaleThreads / 32];
  const T* __restrict__ pu = static_cast<const T*>(p.pred_uncond);
  const T* __restrict__ pc = static_cast<const T*>(p.pred_cond);
  const T* __restrict__ cnt = static_cast<const T*>(p.counter);
  T* __restrict__ out = static_cast<T*>(p.out);
  const double* __restrict__ part = static_cast<const double*>(p.workspace);
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int j = threadIdx.x; j < parts; j += blockDim.x)
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] += part[4LL * j + k];
  cta_sum4(s, red);
  // unbiased variance (torch.std's default); a constant input may cancel to a tiny negative value
  const double n = static_cast<double>(p.count);
  const double var_t = fmax((s[1] - s[0] * s[0] / n) / (n - 1.0), 0.0);
  const double var_g = fmax((s[3] - s[2] * s[2] / n) / (n - 1.0), 0.0);
  const float std_t = rnd(static_cast<float>(sqrt(var_t)));
  const float std_g = rnd(static_cast<float>(sqrt(var_g)));
  const float r = std_g == 0.f ? 1.f : rnd(__fdiv_rn(std_t, std_g));
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < p.count;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float u = C::to_f(pu[i]);
    float c = C::to_f(pc[i]);
    const float g = cfg_guide<kBf16>(u, c, cnt, i, p.frame_stride, frames, p.guidance);
    out[i] = C::from_f(__fadd_rn(rnd(__fmul_rn(w1, rnd(__fmul_rn(g, r)))), rnd(__fmul_rn(w0, g))));
  }
}

// Latent frame interpolation (pipeline interpolate_latents, :294-334): one CTA per frame pair (i, i + 1) of
// src [4, F, hw] (the [1, 4, F, h, w] latents); writes dst frames i*k (a copy of frame i) and i*k + j, j = 1 .. k-1, of
// dst [4, (F-1)*k + 1, hw]; the last CTA also copies frame F-1. Weights: t = j / k and 1 - t in double, as the reference's
// Python floats are, then cast to fp32 as PyTorch does for a scalar operand. method 0 (linear): (1 - t) * v0 + t * v1,
// each product rounded to the storage type, then the sum - PyTorch's rounding points for that expression. method 1
// (slerp): |v0|^2, |v1|^2 and v0.v1 are fp32 sums in a fixed order (per-thread strided, then a fixed shuffle / shared
// memory tree: deterministic); |cos| > 0.9995 takes the linear path, else (sin((1-t) theta) v0 + sin(t theta) v1) /
// sin(theta) in fp32 with precise acosf / sinf, rounded once at the store.
template <bool kBf16>
__global__ void __launch_bounds__(256) interpolate_frames_kernel(const void* __restrict__ srcp, void* __restrict__ dstp,
                                                                 int frames, long long hw, int k, int method) {
  using C = Cvt<kBf16>;
  using T = typename C::T;
  auto rnd = [](float v) { return C::to_f(C::from_f(v)); };
  const T* src = static_cast<const T*>(srcp);
  T* dst = static_cast<T*>(dstp);
  const int i = blockIdx.x;
  const long long fo = static_cast<long long>(frames - 1) * k + 1;
  bool slerp = method == 1;
  float theta = 0.f, sin_theta = 1.f;
  if (slerp) {
    __shared__ float red[3][8];
    float s00 = 0.f, s11 = 0.f, s01 = 0.f;
    for (int c = 0; c < 4; ++c) {
      const T* a = src + (static_cast<long long>(c) * frames + i) * hw;
      for (long long p = threadIdx.x; p < hw; p += blockDim.x) {
        const float x0 = C::to_f(a[p]), x1 = C::to_f(a[p + hw]);
        s00 = fmaf(x0, x0, s00);
        s11 = fmaf(x1, x1, s11);
        s01 = fmaf(x0, x1, s01);
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      s00 += __shfl_xor_sync(0xffffffffu, s00, o);
      s11 += __shfl_xor_sync(0xffffffffu, s11, o);
      s01 += __shfl_xor_sync(0xffffffffu, s01, o);
    }
    if ((threadIdx.x & 31) == 0) {
      red[0][threadIdx.x >> 5] = s00;
      red[1][threadIdx.x >> 5] = s11;
      red[2][threadIdx.x >> 5] = s01;
    }
    __syncthreads();
    s00 = s11 = s01 = 0.f;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {
      s00 += red[0][w];
      s11 += red[1][w];
      s01 += red[2][w];
    }
    const float cosv = __fdiv_rn(s01, __fmul_rn(sqrtf(s00), sqrtf(s11)));
    // the branch is taken on the device (no host sync): the call stays capturable in a graph. NaN (a zero frame)
    // fails the test and propagates, as in the reference.
    slerp = !(fabsf(cosv) > 0.9995f);
    if (slerp) {
      theta = acosf(cosv);
      sin_theta = sinf(theta);
    }
  }
  for (int c = 0; c < 4; ++c) {
    const T* a = src + (static_cast<long long>(c) * frames + i) * hw;
    T* o = dst + (static_cast<long long>(c) * fo + static_cast<long long>(i) * k) * hw;
    for (long long p = threadIdx.x; p < hw; p += blockDim.x) {
      const T v0 = a[p], v1 = a[p + hw];
      const float x0 = C::to_f(v0), x1 = C::to_f(v1);
      o[p] = v0;
      for (int j = 1; j < k; ++j) {
        const double t = static_cast<double>(j) / k;
        const float wa = static_cast<float>(1.0 - t), wb = static_cast<float>(t);
        float y;
        if (slerp) {
          y = __fdiv_rn(__fadd_rn(__fmul_rn(sinf(__fmul_rn(wa, theta)), x0), __fmul_rn(sinf(__fmul_rn(wb, theta)), x1)),
                        sin_theta);
        } else {
          y = rnd(__fmul_rn(wa, x0)) + rnd(__fmul_rn(wb, x1));
        }
        o[static_cast<long long>(j) * hw + p] = C::from_f(y);
      }
      if (i == frames - 2) o[static_cast<long long>(k) * hw + p] = v1;
    }
  }
}

static inline unsigned ew_grid(long long n, int threads) {
  long long b = (n + threads - 1) / threads;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<unsigned>(b);
}

}  // namespace mimo

using namespace mimo;

#define MIMO_CHECK_LAUNCH(what)                                  \
  do {                                                           \
    cudaError_t e__ = cudaGetLastError();                        \
    if (e__ != cudaSuccess) return set_cuda_error(what, e__);    \
  } while (0)

extern "C" int mimo_ncfhw_to_nhwc(const void* src, void* dst, int32_t b, int32_t c, int32_t f, int32_t h,
                                  int32_t w, int32_t cpad, int32_t src_is_f32, int32_t dtype, void* stream) {
  if (!src || !dst || b <= 0 || c <= 0 || f <= 0 || h <= 0 || w <= 0 || cpad < c || (cpad % 8))
    return set_error(MIMO_ERR_ARG, "mimo_ncfhw_to_nhwc: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(b) * f * h * w * (cpad / 8);
  const unsigned grid = ew_grid(total, 256);
  if (src_is_f32) {
    if (dtype == MIMO_BF16)
      ncfhw_to_nhwc_kernel<true, float><<<grid, 256, 0, st>>>(static_cast<const float*>(src), dst, b, c, f, h, w, cpad);
    else
      ncfhw_to_nhwc_kernel<false, float><<<grid, 256, 0, st>>>(static_cast<const float*>(src), dst, b, c, f, h, w, cpad);
  } else {
    if (dtype == MIMO_BF16)
      ncfhw_to_nhwc_kernel<true, uint16_t><<<grid, 256, 0, st>>>(static_cast<const uint16_t*>(src), dst, b, c, f, h, w, cpad);
    else
      ncfhw_to_nhwc_kernel<false, uint16_t><<<grid, 256, 0, st>>>(static_cast<const uint16_t*>(src), dst, b, c, f, h, w, cpad);
  }
  MIMO_CHECK_LAUNCH("ncfhw_to_nhwc launch");
  return MIMO_OK;
}

extern "C" int mimo_nhwc_to_ncfhw(const void* src, void* dst, int32_t b, int32_t c, int32_t f, int32_t h,
                                  int32_t w, int32_t ld, int32_t dst_is_f32, int32_t dtype, void* stream) {
  if (!src || !dst || b <= 0 || c <= 0 || f <= 0 || h <= 0 || w <= 0 || ld < c)
    return set_error(MIMO_ERR_ARG, "mimo_nhwc_to_ncfhw: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(b) * c * f * h * w;
  const unsigned grid = ew_grid(total, 256);
  if (dst_is_f32) {
    if (dtype == MIMO_BF16)
      nhwc_to_ncfhw_kernel<true, float><<<grid, 256, 0, st>>>(src, static_cast<float*>(dst), b, c, f, h, w, ld);
    else
      nhwc_to_ncfhw_kernel<false, float><<<grid, 256, 0, st>>>(src, static_cast<float*>(dst), b, c, f, h, w, ld);
  } else {
    if (dtype == MIMO_BF16)
      nhwc_to_ncfhw_kernel<true, uint16_t><<<grid, 256, 0, st>>>(src, static_cast<uint16_t*>(dst), b, c, f, h, w, ld);
    else
      nhwc_to_ncfhw_kernel<false, uint16_t><<<grid, 256, 0, st>>>(src, static_cast<uint16_t*>(dst), b, c, f, h, w, ld);
  }
  MIMO_CHECK_LAUNCH("nhwc_to_ncfhw launch");
  return MIMO_OK;
}

extern "C" int mimo_im2col3x3(const void* x, void* col, int32_t n, int32_t h, int32_t w, int32_t c,
                              int32_t stride, int32_t upshift, int32_t pad_lo, int64_t ldcol, int32_t dtype,
                              void* stream) {
  (void)dtype;  // 16-bit payload either way
  if (!x || !col || n <= 0 || h <= 0 || w <= 0 || c <= 0 || (c % 8) || stride < 1 || stride > 2 || upshift < 0 ||
      upshift > 1 || pad_lo < 0 || pad_lo > 1 || ldcol < 9LL * c || (ldcol % 8))
    return set_error(MIMO_ERR_ARG, "mimo_im2col3x3: bad arguments");
  if (int rc = ensure_device()) return rc;
  const int uh = h << upshift, uw = w << upshift;
  // output size of a 3x3 window: pad_lo = 1 -> "padding 1"; pad_lo = 0 -> input padded by one at the far edge
  const int oh = (uh + 2 * pad_lo - 3 + (pad_lo ? 0 : 1)) / stride + 1;
  const int ow = (uw + 2 * pad_lo - 3 + (pad_lo ? 0 : 1)) / stride + 1;
  const long long total = static_cast<long long>(n) * oh * ow * 9 * (c / 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  im2col3x3_kernel<uint16_t><<<ew_grid(total, 256), 256, 0, st>>>(
      static_cast<const uint16_t*>(x), static_cast<uint16_t*>(col), n, h, w, c, stride, upshift, pad_lo, oh, ow,
      ldcol);
  MIMO_CHECK_LAUNCH("im2col3x3 launch");
  return MIMO_OK;
}

extern "C" int mimo_upsample2x(const void* x, void* out, int32_t n, int32_t h, int32_t w, int32_t c, int32_t dtype,
                               void* stream) {
  (void)dtype;
  if (!x || !out || n <= 0 || h <= 0 || w <= 0 || c <= 0 || (c % 8)) return set_error(MIMO_ERR_ARG, "mimo_upsample2x: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(n) * 4 * h * w * (c / 8);
  upsample2x_kernel<<<ew_grid(total, 256), 256, 0, st>>>(static_cast<const uint4*>(x), static_cast<uint4*>(out), n, h, w, c / 8);
  MIMO_CHECK_LAUNCH("upsample2x launch");
  return MIMO_OK;
}

extern "C" int mimo_upsample_nearest(const void* x, void* out, int32_t n, int32_t h, int32_t w, int32_t oh, int32_t ow,
                                     int32_t c, int32_t dtype, void* stream) {
  if (!x || !out) return set_error(MIMO_ERR_ARG, "mimo_upsample_nearest: null pointer");
  if (n <= 0 || h <= 0 || w <= 0 || oh <= 0 || ow <= 0 || c <= 0 || (c % 8))
    return set_error(MIMO_ERR_ARG, "mimo_upsample_nearest: sizes must be positive and c a multiple of 8");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15)
    return set_error(MIMO_ERR_ARG, "mimo_upsample_nearest: x and out must be 16-byte aligned");
  if (dtype != MIMO_F16 && dtype != MIMO_BF16) return set_error(MIMO_ERR_ARG, "mimo_upsample_nearest: bad dtype");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(n) * oh * ow * (c / 8);
  // the same fp32 quotient PyTorch's kernel uses (compute_scales_value without a scale factor: in / out)
  const float sy = static_cast<float>(h) / static_cast<float>(oh);
  const float sx = static_cast<float>(w) / static_cast<float>(ow);
  cudaError_t e = launch_k(upsample_nearest_kernel, dim3(ew_grid(total, 256)), dim3(256), 0, st,
                           static_cast<const uint4*>(x), static_cast<uint4*>(out), n, h, w, oh, ow, c / 8, sy, sx);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("upsample_nearest launch", e);
  return MIMO_OK;
}

extern "C" int mimo_softmax_rows(void* x, int64_t rows, int32_t cols, int64_t ld, int32_t dtype, void* stream) {
  if (!x || rows <= 0 || cols <= 0 || (cols % 8) || (ld % 8) || rows > 0x7fffffffLL)
    return set_error(MIMO_ERR_ARG, "mimo_softmax_rows: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == MIMO_BF16)
    softmax_rows_kernel<true><<<static_cast<unsigned>(rows), 256, 0, st>>>(x, cols, ld);
  else
    softmax_rows_kernel<false><<<static_cast<unsigned>(rows), 256, 0, st>>>(x, cols, ld);
  MIMO_CHECK_LAUNCH("softmax_rows launch");
  return MIMO_OK;
}

extern "C" int mimo_add(const void* a, const void* b, void* out, int64_t count, int32_t dtype, void* stream) {
  if (!a || !b || !out || count <= 0 || (count % 8)) return set_error(MIMO_ERR_ARG, "mimo_add: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long nvec = count / 8;
  if (dtype == MIMO_BF16)
    ew_kernel<true, 0><<<ew_grid(nvec, 256), 256, 0, st>>>(a, b, out, nvec);
  else
    ew_kernel<false, 0><<<ew_grid(nvec, 256), 256, 0, st>>>(a, b, out, nvec);
  MIMO_CHECK_LAUNCH("add launch");
  return MIMO_OK;
}

extern "C" int mimo_silu(const void* x, void* out, int64_t count, int32_t dtype, void* stream) {
  if (!x || !out || count <= 0 || (count % 8)) return set_error(MIMO_ERR_ARG, "mimo_silu: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long nvec = count / 8;
  if (dtype == MIMO_BF16)
    ew_kernel<true, 1><<<ew_grid(nvec, 256), 256, 0, st>>>(x, nullptr, out, nvec);
  else
    ew_kernel<false, 1><<<ew_grid(nvec, 256), 256, 0, st>>>(x, nullptr, out, nvec);
  MIMO_CHECK_LAUNCH("silu launch");
  return MIMO_OK;
}

extern "C" int mimo_quick_gelu(const void* x, void* out, int64_t count, int32_t dtype, void* stream) {
  if (!x || !out || count <= 0 || (count % 8)) return set_error(MIMO_ERR_ARG, "mimo_quick_gelu: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long nvec = count / 8;
  if (dtype == MIMO_BF16)
    ew_kernel<true, 2><<<ew_grid(nvec, 256), 256, 0, st>>>(x, nullptr, out, nvec);
  else
    ew_kernel<false, 2><<<ew_grid(nvec, 256), 256, 0, st>>>(x, nullptr, out, nvec);
  MIMO_CHECK_LAUNCH("quick_gelu launch");
  return MIMO_OK;
}

extern "C" int mimo_cfg_ddim_step(const void* pred_uncond, const void* pred_cond, const void* counter_or_null,
                                  int64_t frame_stride, void* latents, int64_t count, float guidance,
                                  float sqrt_a_t, float sqrt_1ma_t, float sqrt_a_prev, float sqrt_1ma_prev,
                                  int32_t dtype, void* stream) {
  if (!pred_uncond || !pred_cond || !latents || count <= 0)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_ddim_step: bad arguments");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // counter (if given) holds one value per frame; latents are [1, 4, F, h, w] so the frame index of element i is
  // (i / frame_stride) % frames with frames = count / (4 * frame_stride)
  int frames = 1;
  if (counter_or_null) {
    if (frame_stride <= 0 || count % (4 * frame_stride)) return set_error(MIMO_ERR_ARG, "mimo_cfg_ddim_step: bad frame_stride");
    frames = static_cast<int>(count / (4 * frame_stride));
  }
  if (dtype == MIMO_BF16)
    cfg_ddim_kernel<true, false><<<ew_grid(count, 256), 256, 0, st>>>(pred_uncond, pred_cond, counter_or_null,
                                                                     frame_stride, frames, latents, count, guidance,
                                                                     sqrt_a_t, sqrt_1ma_t, sqrt_a_prev, sqrt_1ma_prev,
                                                                     nullptr, 0.f);
  else
    cfg_ddim_kernel<false, false><<<ew_grid(count, 256), 256, 0, st>>>(pred_uncond, pred_cond, counter_or_null,
                                                                      frame_stride, frames, latents, count, guidance,
                                                                      sqrt_a_t, sqrt_1ma_t, sqrt_a_prev, sqrt_1ma_prev,
                                                                      nullptr, 0.f);
  MIMO_CHECK_LAUNCH("cfg_ddim launch");
  return MIMO_OK;
}

extern "C" int mimo_cfg_ddim_step_noise(const void* pred_uncond, const void* pred_cond, const void* counter_or_null,
                                        int64_t frame_stride, void* latents, int64_t count, float guidance,
                                        float sqrt_a_t, float sqrt_1ma_t, float sqrt_a_prev, float dir_coef,
                                        const void* noise, float sigma, int32_t dtype, void* stream) {
  if (!pred_uncond || !pred_cond || !latents || !noise || count <= 0)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_ddim_step_noise: null pointer or count <= 0");
  if (dtype != MIMO_F16 && dtype != MIMO_BF16) return set_error(MIMO_ERR_ARG, "mimo_cfg_ddim_step_noise: bad dtype");
  if (!(sigma >= 0.f) || !(dir_coef >= 0.f))  // also refuses NaN (sqrt of a negative variance)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_ddim_step_noise: sigma and dir_coef must be >= 0");
  int frames = 1;
  if (counter_or_null) {
    if (frame_stride <= 0 || count % (4 * frame_stride))
      return set_error(MIMO_ERR_ARG, "mimo_cfg_ddim_step_noise: bad frame_stride");
    frames = static_cast<int>(count / (4 * frame_stride));
  }
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == MIMO_BF16)
    cfg_ddim_kernel<true, true><<<ew_grid(count, 256), 256, 0, st>>>(pred_uncond, pred_cond, counter_or_null,
                                                                    frame_stride, frames, latents, count, guidance,
                                                                    sqrt_a_t, sqrt_1ma_t, sqrt_a_prev, dir_coef,
                                                                    noise, sigma);
  else
    cfg_ddim_kernel<false, true><<<ew_grid(count, 256), 256, 0, st>>>(pred_uncond, pred_cond, counter_or_null,
                                                                     frame_stride, frames, latents, count, guidance,
                                                                     sqrt_a_t, sqrt_1ma_t, sqrt_a_prev, dir_coef,
                                                                     noise, sigma);
  MIMO_CHECK_LAUNCH("cfg_ddim_noise launch");
  return MIMO_OK;
}

extern "C" int mimo_cfg_multistep(const mimo_cfg_multistep_params* p, void* stream) {
  if (!p || !p->pred_uncond || !p->pred_cond || !p->latents || !p->hist_out)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: null pointer");
  if (p->count <= 0) return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: count <= 0");
  if (p->dtype != MIMO_F16 && p->dtype != MIMO_BF16) return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: bad dtype");
  const float sc[8] = {p->guidance, p->a, p->b, p->c_x, p->c_m, p->c_1, p->c_2, p->c_n};
  for (float s : sc)
    if (!std::isfinite(s)) return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: non-finite coefficient");
  if ((!p->h1 && p->c_1 != 0.f) || (!p->h2 && p->c_2 != 0.f) || (!p->noise && p->c_n != 0.f))
    return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: null h1 / h2 / noise with a non-zero coefficient");
  const void* h = p->hist_out;
  if (h == p->latents || h == p->pred_uncond || h == p->pred_cond || h == p->h1 || h == p->noise)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: hist_out aliases latents, pred_uncond, pred_cond, h1 or noise");
  int frames = 1;
  if (p->counter) {
    if (p->frame_stride <= 0 || p->count % (4 * p->frame_stride))
      return set_error(MIMO_ERR_ARG, "mimo_cfg_multistep: bad frame_stride");
    frames = static_cast<int>(p->count / (4 * p->frame_stride));
  }
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (p->dtype == MIMO_BF16)
    cfg_multistep_kernel<true><<<ew_grid(p->count, 256), 256, 0, st>>>(*p, frames);
  else
    cfg_multistep_kernel<false><<<ew_grid(p->count, 256), 256, 0, st>>>(*p, frames);
  MIMO_CHECK_LAUNCH("cfg_multistep launch");
  return MIMO_OK;
}

extern "C" int64_t mimo_cfg_rescale_workspace_bytes(const mimo_cfg_rescale_params* p) {
  if (!p) return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale_workspace_bytes: null params");
  if (p->count < 2) return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale_workspace_bytes: count < 2");
  return 4LL * static_cast<long long>(sizeof(double)) * cfg_rescale_ctas(p->count);
}

extern "C" int mimo_cfg_rescale(const mimo_cfg_rescale_params* p, void* stream) {
  if (!p || !p->pred_uncond || !p->pred_cond || !p->out || !p->workspace)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: null pointer");
  if (p->count < 2) return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: count < 2 (the standard deviation is unbiased)");
  if (p->dtype != MIMO_F16 && p->dtype != MIMO_BF16) return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: bad dtype");
  if (!std::isfinite(p->guidance)) return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: non-finite guidance");
  if (!(p->phi >= 0.0 && p->phi <= 1.0)) return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: phi must be in [0, 1]");
  int frames = 1;
  if (p->counter) {
    if (p->frame_stride <= 0 || p->count % (4 * p->frame_stride))
      return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: bad frame_stride");
    frames = static_cast<int>(p->count / (4 * p->frame_stride));
  }
  const int parts = cfg_rescale_ctas(p->count);
  if (p->workspace_bytes < 4LL * static_cast<long long>(sizeof(double)) * parts ||
      (reinterpret_cast<uintptr_t>(p->workspace) & 15))
    return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: workspace smaller than mimo_cfg_rescale_workspace_bytes or "
                                   "not 16-byte aligned");
  const void* o = p->out;
  if (o == p->pred_uncond || o == p->pred_cond || o == p->counter || o == p->workspace)
    return set_error(MIMO_ERR_ARG, "mimo_cfg_rescale: out aliases pred_uncond, pred_cond, counter or workspace");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float w1 = static_cast<float>(p->phi), w0 = static_cast<float>(1.0 - p->phi);
  if (p->dtype == MIMO_BF16) {
    cfg_rescale_stats_kernel<true><<<parts, kRescaleThreads, 0, st>>>(*p, frames);
    cfg_rescale_apply_kernel<true><<<parts, kRescaleThreads, 0, st>>>(*p, frames, parts, w1, w0);
  } else {
    cfg_rescale_stats_kernel<false><<<parts, kRescaleThreads, 0, st>>>(*p, frames);
    cfg_rescale_apply_kernel<false><<<parts, kRescaleThreads, 0, st>>>(*p, frames, parts, w1, w0);
  }
  MIMO_CHECK_LAUNCH("cfg_rescale launch");
  return MIMO_OK;
}

extern "C" int mimo_interpolate_frames(const void* src, void* dst, int32_t frames, int64_t hw, int32_t k, int32_t method,
                                       int32_t dtype, void* stream) {
  if (!src || !dst || src == dst) return set_error(MIMO_ERR_ARG, "mimo_interpolate_frames: null or aliased pointers");
  if (frames < 2 || hw <= 0 || k < 2 || (method != 0 && method != 1))
    return set_error(MIMO_ERR_ARG, "mimo_interpolate_frames: need frames >= 2, hw > 0, k >= 2, method 0 or 1");
  if (dtype != MIMO_F16 && dtype != MIMO_BF16) return set_error(MIMO_ERR_ARG, "mimo_interpolate_frames: bad dtype");
  if (int rc = ensure_device()) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == MIMO_BF16)
    interpolate_frames_kernel<true><<<frames - 1, 256, 0, st>>>(src, dst, frames, hw, k, method);
  else
    interpolate_frames_kernel<false><<<frames - 1, 256, 0, st>>>(src, dst, frames, hw, k, method);
  MIMO_CHECK_LAUNCH("interpolate_frames launch");
  return MIMO_OK;
}
