// Spatial self-attention with the reference-image bank: flash attention on wgmma.
//
// One CTA = 128 query rows (64 from d = 160 on, see AttnCfg) of one (frame-sample n, head h). The key/value sequence
// is [self tokens | bank tokens of branch bank_index[n]] (bank skipped when bank_index[n] < 0: the unconditional CFG
// half attends to itself only, which is what src/models/mutual_self_attention.py:177-197 computes by running attn1 a
// second time). Roles: each MMA warpgroup owns 64 query rows and, per 128-key tile:
//     S  = Q K^T         wgmma m64n128k16 (d rounded to 16 / 16 steps), Q and K tiles K-major, fp32 S in registers
//     P  = exp2(S*c - m) online max / sum in fp32 (a row lives in the 4 lanes of a quad), P converted in registers to
//                        the A fragments of the next MMA - it never touches shared memory
//     O += P V           wgmma m64n(d rounded to 16)k16, A = P from registers, V tile as an MN-major B operand
// and one thread of the warp after the MMA warpgroups issues the TMA loads.
// Q/K/V tiles arrive by 4-D TMA boxes straight out of the fused QKV activation buffer ([token, 3C] rows, head
// slices addressed by a tensor-map dimension); head dims 40/80/160 are zero-filled up to 64-element chunks by
// TMA's out-of-bounds handling, so no padded copies exist in HBM.
#include <cuda_runtime.h>

#include "../../include/mimo_b200.h"
#include "attn_common.h"
#include "host_util.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace mimo {

// Registers are reserved per group of 4 warps. With two MMA warpgroups (+ the TMA warp = 12 warps' worth) a thread may
// hold 168 registers: enough for S (64) + O (d/2) below d = 160. From d = 160 on a CTA has ONE MMA warpgroup (64 query
// rows, 8 warps' worth, up to 255 registers), so O, S and P stay in registers without spills, and the smaller Q tile
// leaves room for a second K/V stage.
template <int DP>
struct AttnCfg {
  static constexpr int NCH = (DP + 63) / 64;                   // 64-column chunks of Q / K / V
  static constexpr int NWG = DP >= 160 ? 1 : 2;                // MMA warpgroups, 64 query rows each
  static constexpr int QROWS = 64 * NWG;                       // query rows per CTA
  static constexpr int kThreads = 128 * NWG + 32;              // + the TMA warp (warp 4 * NWG)
  static constexpr int kQChunk = QROWS * 128;                  // one 64-column chunk of the Q tile
  static constexpr int kQBytes = NCH * kQChunk;
  static constexpr int kKVStageBytes = 2 * NCH * kChunkBytes;  // K chunks then V chunks
  static constexpr int kFit = (227 * 1024 - 1024 - 256 - kQBytes) / kKVStageBytes;
  static constexpr int KVST = kFit < 3 ? kFit : 3;             // K/V stages that fit next to Q
  static constexpr int kSmemBytes = kQBytes + KVST * kKVStageBytes + 1024 + 256;
  static_assert(KVST >= 1, "K/V tile does not fit");
};

template <int DP, bool kBf16>
__global__ void __launch_bounds__(AttnCfg<DP>::kThreads, 1)
attn_spatial_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmBK,
                    const __grid_constant__ CUtensorMap tmBV, AttnArgs a) {
  using Cfg = AttnCfg<DP>;
  using C = Cvt<kBf16>;
  constexpr int NCH = Cfg::NCH, KVST = Cfg::KVST, kProd = 4 * Cfg::NWG;  // kProd: the TMA warp
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + Cfg::kQBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + KVST * Cfg::kKVStageBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + KVST;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // provably warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int q_tile = blockIdx.x;
  const int h = blockIdx.y;
  const int n = blockIdx.z;
  pdl_launch_dependents();
  pdl_wait();
  const int bidx = __shfl_sync(0xffffffffu, a.bank_index ? a.bank_index[n] : -1, 0);
  const int T = a.n_self_tiles + (bidx >= 0 ? a.n_bank_tiles : 0);

  if (warp == kProd && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    if (bidx >= 0) {
      tma_prefetch_desc(&tmBK);
      tma_prefetch_desc(&tmBV);
    }
  }
  if (warp == kProd && lane == 1) {
    mbar_init(q_full, 1);
    for (int s = 0; s < KVST; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], kProd);  // lane 0 of each MMA warp, once its P.V has read the stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kProd && lane == 0) {
    // ===================== TMA producer =====================
    mbar_expect_tx(q_full, Cfg::kQBytes);
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) tma_load_4d(sQ + ch * Cfg::kQChunk, &tmQ, q_full, ch * 64, h, q_tile * Cfg::QROWS, n);
    for (int j = 0; j < T; ++j) {
      const int stage = j % KVST;
      const uint32_t phase = (j / KVST) & 1u;
      mbar_wait(&kv_empty[stage], phase ^ 1u);
      uint8_t* sk = sKV + stage * Cfg::kKVStageBytes;
      uint8_t* sv = sk + NCH * kChunkBytes;
      mbar_expect_tx(&kv_full[stage], Cfg::kKVStageBytes);
      const bool bank = j >= a.n_self_tiles;
      const int row0 = (bank ? j - a.n_self_tiles : j) * BKV;
      const int img = bank ? bidx : n;
      const CUtensorMap* mk = bank ? &tmBK : &tmK;
      const CUtensorMap* mv = bank ? &tmBV : &tmV;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        tma_load_4d(sk + ch * kChunkBytes, mk, &kv_full[stage], ch * 64, h, row0, img);
        tma_load_4d(sv + ch * kChunkBytes, mv, &kv_full[stage], ch * 64, h, row0, img);
      }
    }
  } else if (warp < kProd) {
    // ===================== MMA / softmax / epilogue =====================
    const int wg = warp >> 2;  // query rows [64 wg, 64 wg + 64) of the tile
    // accumulator layout (S and O alike): this thread holds rows rbase and rbase + 8; fragment j (8 columns) holds
    // columns 8 j + q2, + 1 in [4 j], [4 j + 1] (row rbase) and [4 j + 2], [4 j + 3] (row rbase + 8)
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int q2 = (lane & 3) * 2;
    const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);
    float o[DP / 2];
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    mbar_wait(q_full, 0);
    for (int j = 0; j < T; ++j) {
      const int stage = j % KVST;
      const bool bank = j >= a.n_self_tiles;
      const int len = bank ? a.lb : a.lq;
      const int row0 = (bank ? j - a.n_self_tiles : j) * BKV;
      int valid = len - row0;
      if (valid > BKV) valid = BKV;
      mbar_wait(&kv_full[stage], (j / KVST) & 1u);
      const uint32_t k_addr = smem_u32(sKV + stage * Cfg::kKVStageBytes);
      const uint32_t v_addr = k_addr + NCH * kChunkBytes;

      float s[BKV / 2];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < DP / 16; ++ks) {
        const uint32_t off = (ks & 3) * 32;
        Wgmma<BKV, kBf16>::ss(s, make_smem_desc_sw128(q_addr + (ks >> 2) * Cfg::kQChunk + off, 16, 1024),
                              make_smem_desc_sw128(k_addr + (ks >> 2) * kChunkBytes + off, 16, 1024), ks != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);

      // row maximum over the valid keys (a row is spread over the 4 lanes of a quad)
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int jn = 0; jn < BKV / 8; ++jn)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (8 * jn + q2 + (e & 1) < valid)
            mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * jn + e]);
          else
            s[4 * jn + e] = -INFINITY;
        }
      float alpha[2], m_new[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        m_new[r] = fmaxf(m[r], mx[r] * a.scale_log2);
        alpha[r] = exp2f(m[r] - m_new[r]);
      }
      // probabilities -> A fragments of P.V: k-step kk covers keys [16 kk, 16 kk + 16) = S fragments 2 kk, 2 kk + 1
      uint32_t pa[BKV / 16][4];
      float rowsum[2] = {0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int e = 8 * kk + 2 * i;  // i: (row, keys 0-7), (row + 8, keys 0-7), (row, keys 8-15), (row + 8, keys 8-15)
          const int r = i & 1;
          const float p0 = exp2f(fmaf(s[e], a.scale_log2, -m_new[r]));
          const float p1 = exp2f(fmaf(s[e + 1], a.scale_log2, -m_new[r]));
          rowsum[r] += p0 + p1;
          pa[kk][i] = C::pack(p0, p1);
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        l[r] = l[r] * alpha[r] + rowsum[r];
        m[r] = m_new[r];
      }
      if (j > 0) {
#pragma unroll
        for (int i = 0; i < DP / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk) {
        // B = V: MN-major, 16 keys = 2 KiB further down; 64-column chunks kChunkBytes apart
        Wgmma<DP, kBf16>::rs(o, pa[kk], make_smem_desc_sw128(v_addr + kk * 2048, kChunkBytes, 1024),
                             (j | kk) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      if (lane == 0) mbar_arrive(&kv_empty[stage]);
    }
    // epilogue: O / l -> global
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
      l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
      const float inv_l = 1.0f / l[r];
      const int qrow = q_tile * Cfg::QROWS + rbase + 8 * r;
      if (qrow < a.lq) {
        typename C::T* orow =
            static_cast<typename C::T*>(a.out) + (static_cast<long long>(n) * a.lq + qrow) * a.ld_out + h * a.d;
#pragma unroll
        for (int jn = 0; jn < DP / 8; ++jn)
          if (8 * jn + q2 < a.d)
            *reinterpret_cast<uint32_t*>(orow + 8 * jn + q2) = C::pack(o[4 * jn + 2 * r] * inv_l, o[4 * jn + 2 * r + 1] * inv_l);
      }
    }
  }
}

static int attn_tmap(CUtensorMap* m, int dtype, const void* base, int d, int heads, int len, int nimg, long long ld,
                     uint32_t rows = BKV);

template <int DP, bool kBf16>
static int launch_attn(const mimo_attn_params* p, const CUtensorMap& k, const CUtensorMap& v, const CUtensorMap& bk,
                       const CUtensorMap& bv, const AttnArgs& a, cudaStream_t st) {
  using Cfg = AttnCfg<DP>;
  auto kern = attn_spatial_kernel<DP, kBf16>;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_cuda_error("cudaFuncSetAttribute(attn)", e);
    attr_done = true;
  }
  CUtensorMap q;  // Q boxes cover the CTA's query rows
  if (int rc = attn_tmap(&q, p->dtype, p->q, p->d, p->heads, p->lq, p->n, p->ld_qkv, Cfg::QROWS)) return rc;
  const dim3 grid((p->lq + Cfg::QROWS - 1) / Cfg::QROWS, p->heads, p->n);
  cudaError_t e = launch_k(kern, grid, dim3(Cfg::kThreads), Cfg::kSmemBytes, st, q, k, v, bk, bv, a);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("attn launch", e);
  return MIMO_OK;
}

static int attn_tmap(CUtensorMap* m, int dtype, const void* base, int d, int heads, int len, int nimg, long long ld,
                     uint32_t rows) {
  const uint64_t dims[4] = {static_cast<uint64_t>(d), static_cast<uint64_t>(heads), static_cast<uint64_t>(len),
                            static_cast<uint64_t>(nimg)};
  const uint64_t str[3] = {static_cast<uint64_t>(d) * 2, static_cast<uint64_t>(ld) * 2,
                           static_cast<uint64_t>(len) * ld * 2};
  const uint32_t box[4] = {64, 1, rows, 1};
  return encode_tmap(m, dtype, 4, base, dims, str, box);
}

}  // namespace mimo

using namespace mimo;

extern "C" int mimo_attn_spatial(const mimo_attn_params* p, void* stream) {
  if (!p || !p->q || !p->k || !p->v || !p->out) return set_error(MIMO_ERR_ARG, "mimo_attn_spatial: null pointer");
  if (p->n <= 0 || p->lq <= 0 || p->heads <= 0 || p->d <= 0 || (p->d % 8) || p->d > 192 || (p->ld_qkv % 8) ||
      (p->ld_out % 8))
    return set_error(MIMO_ERR_ARG, "mimo_attn_spatial: need d % 8 == 0, d <= 192, leading dims % 8 == 0");
  const bool has_bank = p->bank_index && p->bank_k && p->bank_v && p->lb > 0;
  if (has_bank && (p->ld_bank % 8)) return set_error(MIMO_ERR_ARG, "mimo_attn_spatial: ld_bank % 8 != 0");
  if (int rc = ensure_device()) return rc;

  AttnArgs a;
  a.lq = p->lq;
  a.lb = has_bank ? p->lb : 0;
  a.heads = p->heads;
  a.d = p->d;
  a.dp = (p->d + 15) / 16 * 16;
  a.n_self_tiles = (p->lq + BKV - 1) / BKV;
  a.n_bank_tiles = has_bank ? (p->lb + BKV - 1) / BKV : 0;
  a.scale_log2 = p->scale * 1.4426950408889634f;
  a.bank_index = has_bank ? p->bank_index : nullptr;
  a.out = p->out;
  a.ld_out = p->ld_out;

  CUtensorMap tk, tv, tbk, tbv;
  if (int rc = attn_tmap(&tk, p->dtype, p->k, p->d, p->heads, p->lq, p->n, p->ld_qkv)) return rc;
  if (int rc = attn_tmap(&tv, p->dtype, p->v, p->d, p->heads, p->lq, p->n, p->ld_qkv)) return rc;
  if (has_bank) {
    const int nb = p->nb > 0 ? p->nb : 1;
    if (int rc = attn_tmap(&tbk, p->dtype, p->bank_k, p->d, p->heads, p->lb, nb, p->ld_bank)) return rc;
    if (int rc = attn_tmap(&tbv, p->dtype, p->bank_v, p->d, p->heads, p->lb, nb, p->ld_bank)) return rc;
  } else {
    tbk = tk;
    tbv = tv;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // one instantiation per head dim rounded up to 16 (the P.V instruction's N)
  switch (a.dp) {
#define MIMO_ATTN_DP(DP) \
  case DP:               \
    return p->dtype == MIMO_BF16 ? launch_attn<DP, true>(p, tk, tv, tbk, tbv, a, st) \
                                 : launch_attn<DP, false>(p, tk, tv, tbk, tbv, a, st);
    MIMO_ATTN_DP(16) MIMO_ATTN_DP(32) MIMO_ATTN_DP(48) MIMO_ATTN_DP(64) MIMO_ATTN_DP(80) MIMO_ATTN_DP(96)
    MIMO_ATTN_DP(112) MIMO_ATTN_DP(128) MIMO_ATTN_DP(144) MIMO_ATTN_DP(160) MIMO_ATTN_DP(176) MIMO_ATTN_DP(192)
#undef MIMO_ATTN_DP
  }
  return set_error(MIMO_ERR_ARG, "mimo_attn_spatial: unsupported head dim");
}
