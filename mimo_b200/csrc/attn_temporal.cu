// Motion-module temporal self-attention: for every (batch b, pixel p, head h) an Fq x F attention over the
// frame axis (F <= 32, head dim d a multiple of 8).
//
// The problems are tiny (24 x 24 x 40) but there are 65 536 of them per call at the 64x64 level, so the kernel is
// organised around memory: one CTA stages the Q, K and V rows of all frames of one pixel (for a group of heads) in
// shared memory with 128-bit loads — every row is a contiguous C-element segment, so the reference's
// "(b f) d c <-> (b d) f c" transposes never materialise — and one warp per head then runs the attention on tensor
// cores with warp-level mma.sync.m16n8k16 (a 24-row problem cannot fill a 64-row wgmma tile): S = Q K^T from
// ldmatrix fragments, fp32 softmax in the accumulator registers, P re-used in registers as the A operand of P V,
// V read with ldmatrix.trans. Outputs are staged through shared memory for 128-bit stores.
//
// Frame sharding: with the clip's frames split over G GPUs the queries are the Fq local frames while K/V cover all
// F frames, stored as G chunks of frames_per_chunk frames each (the all-gathered per-rank buffers):
//   kv_row(b, f, p) = (f / fpc) * chunk_stride_rows + (b * fpc + f % fpc) * hw + p
#include <cuda_runtime.h>

#include "../../include/mimo_b200.h"
#include "host_util.h"
#include "ptx.cuh"

namespace mimo {

struct TemporalArgs {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  long long ld_q, ld_kv, ld_out, chunk_stride_rows;
  int Fq, F, fpc, hw, heads, d;
  int dpad;    // d rounded up to 16 (K dimension of Q K^T)
  int hg;      // heads per CTA
  int pitch;   // smem row pitch in elements: hg * dpad + 8 (the +8 keeps ldmatrix rows on distinct banks)
  float scale_log2;
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
template <bool kBf16>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (kBf16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

// D / HG > 0: head dim and heads per CTA fixed at compile time (the UNet's three levels: 40x8, 80x4, 160x2), which
// turns the row pitch and every fragment address into immediates; D = 0: generic (runtime) geometry.
template <bool kBf16, int D, int HG>
__global__ void __launch_bounds__(1024) attn_temporal_kernel(TemporalArgs a_in) {
  pdl_launch_dependents();
  pdl_wait();
  TemporalArgs a = a_in;
  if constexpr (D > 0) {
    a.d = D;
    a.dpad = (D + 15) / 16 * 16;
    a.hg = HG;
    a.pitch = HG * ((D + 15) / 16 * 16) + 8;
  }
  using C = Cvt<kBf16>;
  using T = typename C::T;
  extern __shared__ uint4 smem_qkv[];
  T* sq = reinterpret_cast<T*>(smem_qkv);           // [32][pitch]
  T* sk = sq + 32 * a.pitch;                         // [32][pitch]
  T* sv = sk + 32 * a.pitch;                         // [32][pitch]
  const int groups = a.heads / a.hg;
  const int hg0 = (blockIdx.x % groups) * a.hg;      // first head of this CTA
  const int bp = blockIdx.x / groups;
  const int b = bp / a.hw;
  const int p = bp % a.hw;
  const int d = a.d, dpad = a.dpad, pitch = a.pitch;
  const int dv = d / 8;                              // 16-byte vectors per head row
  const int vec_row = a.hg * dv;

  // ---- stage Q (Fq rows), K, V (F rows) of this pixel with 16-byte cp.async ----
  // A warp takes whole frames; a lane's vectors inside the row segment do not depend on the frame, so their
  // (head, piece) split - the only divisions - is done once. (The first version recomputed three divisions and a
  // 64-bit row product per 16-byte vector: ~18k warp instructions per CTA, issue-bound at 2 TB/s.)
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    int soff[4], goff[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int v = lane + 32 * j;
      const int hh = v / dv, pc = v - hh * dv;
      soff[j] = v < vec_row ? hh * dpad + pc * 8 : -1;
      goff[j] = (hg0 + hh) * d + pc * 8;
    }
    for (int f = warp; f < a.F; f += nwarps) {
      const long long kvrow = static_cast<long long>(f / a.fpc) * a.chunk_stride_rows +
                              (static_cast<long long>(b) * a.fpc + f % a.fpc) * a.hw + p;
      const T* kr = static_cast<const T*>(a.k) + kvrow * a.ld_kv;
      const T* vr = static_cast<const T*>(a.v) + kvrow * a.ld_kv;
      const T* qr = static_cast<const T*>(a.q) + ((static_cast<long long>(b) * a.Fq + f) * a.hw + p) * a.ld_q;
      const bool has_q = f < a.Fq;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (soff[j] >= 0) {
          cp_async16(sk + f * pitch + soff[j], kr + goff[j]);
          cp_async16(sv + f * pitch + soff[j], vr + goff[j]);
          if (has_q) cp_async16(sq + f * pitch + soff[j], qr + goff[j]);
        }
      }
    }
  }
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    if (dpad > d) {  // zero the K-dimension padding of Q and K (d = 40 -> 48): lane = head, warp strides the rows
      const int padv = (dpad - d) / 8;
      for (int f = warp; f < 32; f += nwarps)
        for (int hh = lane; hh < a.hg; hh += 32)
          for (int pc = 0; pc < padv; ++pc) {
            *reinterpret_cast<uint4*>(sq + f * pitch + hh * dpad + d + pc * 8) = make_uint4(0, 0, 0, 0);
            *reinterpret_cast<uint4*>(sk + f * pitch + hh * dpad + d + pc * 8) = make_uint4(0, 0, 0, 0);
          }
    }
    // V rows beyond F multiply probabilities that are exactly 0: they must be finite -> zero them
    for (int f = a.F + warp; f < 32; f += nwarps)
      for (int pc = lane; pc < pitch / 8; pc += 32) *reinterpret_cast<uint4*>(sv + f * pitch + pc * 8) = make_uint4(0, 0, 0, 0);
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  const int hh = threadIdx.x >> 5;  // head within the group
  const int lane = threadIdx.x & 31;
  if (hh >= a.hg) return;
  const int g = lane >> 2, t = lane & 3;
  const int MT = (a.Fq + 15) >> 4;  // 16-row query tiles
  const int NT = (a.F + 7) >> 3;    // 8-key tiles
  const bool ragged = (a.F & 7) != 0;
  const T* qh = sq + hh * dpad;
  const T* kh = sk + hh * dpad;
  const T* vh = sv + hh * dpad;

  // ---- S = Q K^T ----
  float s[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[mt][nt][e] = 0.f;
  for (int ks = 0; ks < dpad / 16; ++ks) {
    uint32_t af[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
      if (mt < MT) ldsm_x4(af[mt], qh + (mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * pitch + ks * 16 + (lane >> 4) * 8);
#pragma unroll
    for (int np = 0; np < 2; ++np) {  // pairs of key tiles
      if (np * 2 < NT) {
        uint32_t bf[4];
        ldsm_x4(bf, kh + (np * 16 + (lane & 7) + (lane >> 4) * 8) * pitch + ks * 16 + ((lane >> 3) & 1) * 8);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          if (mt < MT) {
            mma16816<kBf16>(s[mt][np * 2], af[mt], bf[0], bf[1]);
            if (np * 2 + 1 < NT) mma16816<kBf16>(s[mt][np * 2 + 1], af[mt], bf[2], bf[3]);
          }
        }
      }
    }
  }

  // ---- softmax over the F keys (rows g and g + 8 of each query tile live in this thread's quad) ----
  float inv_sum[2][2];
  uint32_t pf[2][2][4];  // P as A fragments: [query tile][16-key step]
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {  // half 0: row g, half 1: row g + 8
      float m = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        if (nt < NT) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = s[mt][nt][half * 2 + e];
            v *= a.scale_log2;
            if (ragged && nt == NT - 1 && nt * 8 + 2 * t + e >= a.F) v = -INFINITY;
            m = fmaxf(m, v);
          }
        }
      }
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
      float sum = 0.f;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        if (nt < NT) {  // key tiles beyond NT keep their zero accumulators: P = 0 there
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float& v = s[mt][nt][half * 2 + e];
            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(v) : "f"(v - m));  // ex2(-inf) = 0 for the masked keys
            sum += v;
          }
        }
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      inv_sum[mt][half] = 1.0f / sum;
    }
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      pf[mt][kk][0] = C::pack(s[mt][2 * kk][0], s[mt][2 * kk][1]);
      pf[mt][kk][1] = C::pack(s[mt][2 * kk][2], s[mt][2 * kk][3]);
      pf[mt][kk][2] = C::pack(s[mt][2 * kk + 1][0], s[mt][2 * kk + 1][1]);
      pf[mt][kk][3] = C::pack(s[mt][2 * kk + 1][2], s[mt][2 * kk + 1][3]);
    }
  }

  // ---- O = P V, eight output channels at a time; results overwrite this head's (already consumed) Q columns ----
  __syncwarp();
  T* oh = sq + hh * dpad;
  const int KK = (a.F + 15) >> 4;
  for (int nd = 0; nd < dv; ++nd) {
    uint32_t bv[4];
    ldsm_x4_trans(bv, vh + lane * pitch + nd * 8);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      if (mt < MT) {
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        mma16816<kBf16>(o, pf[mt][0], bv[0], bv[1]);
        if (KK > 1) mma16816<kBf16>(o, pf[mt][1], bv[2], bv[3]);
        *reinterpret_cast<uint32_t*>(oh + (mt * 16 + g) * pitch + nd * 8 + 2 * t) =
            C::pack(o[0] * inv_sum[mt][0], o[1] * inv_sum[mt][0]);
        *reinterpret_cast<uint32_t*>(oh + (mt * 16 + g + 8) * pitch + nd * 8 + 2 * t) =
            C::pack(o[2] * inv_sum[mt][1], o[3] * inv_sum[mt][1]);
      }
    }
  }
  __syncwarp();
  {
    const int lf = lane / dv, lpc = lane - lf * dv, fstep = 32 / dv;  // 32 / dv frames per pass, one vector per lane
    if (lf < fstep) {
      for (int f = lf; f < a.Fq; f += fstep) {
        const long long row = (static_cast<long long>(b) * a.Fq + f) * a.hw + p;
        *reinterpret_cast<uint4*>(static_cast<T*>(a.out) + row * a.ld_out + (hg0 + hh) * d + lpc * 8) =
            *reinterpret_cast<const uint4*>(oh + f * pitch + lpc * 8);
      }
    }
  }
}

}  // namespace mimo

using namespace mimo;

extern "C" int mimo_attn_temporal(const mimo_attn_temporal_params* p, void* stream) {
  if (!p || !p->q || !p->k || !p->v || !p->out) return set_error(MIMO_ERR_ARG, "mimo_attn_temporal: null pointer");
  const int fpc = p->frames_per_chunk > 0 ? p->frames_per_chunk : p->kv_frames;
  if (p->batch <= 0 || p->q_frames <= 0 || p->kv_frames <= 0 || p->kv_frames > 32 || p->q_frames > 32 || p->hw <= 0 ||
      p->heads <= 0 || p->heads > 32 || p->d <= 0 || (p->d % 8) || p->d > 256 || (p->ld_q % 8) || (p->ld_kv % 8) || (p->ld_out % 8) ||
      (p->kv_frames % fpc))
    return set_error(MIMO_ERR_ARG, "mimo_attn_temporal: need frames <= 32, heads <= 32, d % 8 == 0, kv_frames % chunk == 0");
  if (int rc = ensure_device()) return rc;
  TemporalArgs a;
  a.q = p->q;
  a.k = p->k;
  a.v = p->v;
  a.out = p->out;
  a.ld_q = p->ld_q;
  a.ld_kv = p->ld_kv;
  a.ld_out = p->ld_out;
  a.chunk_stride_rows = p->chunk_stride_rows;
  a.Fq = p->q_frames;
  a.F = p->kv_frames;
  a.fpc = fpc;
  a.hw = p->hw;
  a.heads = p->heads;
  a.d = p->d;
  a.dpad = (p->d + 15) / 16 * 16;
  a.scale_log2 = p->scale * 1.4426950408889634f;
  // heads per CTA: as many as keep the Q/K/V staging under ~100 KB (several CTAs per SM)
  int hg = p->heads;
  auto smem_for = [&](int h) { return static_cast<size_t>(3) * 32 * (h * a.dpad + 8) * 2; };
  while (hg > 1 && (hg % 2 == 0) && smem_for(hg) > 100 * 1024) hg /= 2;
  if (smem_for(hg) > 227 * 1024) return set_error(MIMO_ERR_ARG, "mimo_attn_temporal: head dim too large");
  a.hg = hg;
  a.pitch = hg * a.dpad + 8;
  const size_t smem = smem_for(hg);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int threads = hg * 32;
  const long long nblk = static_cast<long long>(p->batch) * p->hw * (p->heads / hg);
  if (nblk > 0x7fffffffLL) return set_error(MIMO_ERR_ARG, "mimo_attn_temporal: grid too large");
  const unsigned grid = static_cast<unsigned>(nblk);
  cudaError_t e;
  static bool attr_done[8] = {};  // per kernel instantiation
  auto launch = [&](void (*kern)(TemporalArgs), int id) -> cudaError_t {
    if (!attr_done[id]) {
      cudaError_t ea = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
      if (ea != cudaSuccess) return ea;
      attr_done[id] = true;
    }
    return launch_k(kern, dim3(grid), dim3(threads), smem, st, a);
  };
  const bool bf = p->dtype == MIMO_BF16;
  if (a.d == 40 && hg == 8)
    e = bf ? launch(attn_temporal_kernel<true, 40, 8>, 0) : launch(attn_temporal_kernel<false, 40, 8>, 1);
  else if (a.d == 80 && hg == 4)
    e = bf ? launch(attn_temporal_kernel<true, 80, 4>, 2) : launch(attn_temporal_kernel<false, 80, 4>, 3);
  else if (a.d == 160 && hg == 2)
    e = bf ? launch(attn_temporal_kernel<true, 160, 2>, 4) : launch(attn_temporal_kernel<false, 160, 2>, 5);
  else
    e = bf ? launch(attn_temporal_kernel<true, 0, 0>, 6) : launch(attn_temporal_kernel<false, 0, 0>, 7);
  if (e != cudaSuccess) return set_cuda_error("attn_temporal attr", e);
  e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("attn_temporal launch", e);
  return MIMO_OK;
}
