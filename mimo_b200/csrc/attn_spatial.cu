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
//
// Schedule with two MMA warpgroups, two K/V stages and registers for a second S tile (DP <= 80, kLook): a warpgroup
// issues S(j+1) = Q K(j+1)^T and O += P(j) V(j) back to back, runs the softmax of S(j+1) while both MMAs run, and
// rescales O once P(j) V(j) has landed. The two warpgroups take turns at issuing (named barriers 1 and 2), so one's
// softmax runs while the other's MMAs occupy the tensor cores. Each row still computes O(j) = O(j-1) alpha(j) + P(j) V(j)
// in the same order as the plain loop (S, softmax, rescale, P V per tile) that DP = 96 ... 144 and the one-warpgroup
// path run.
#include <cuda_runtime.h>

#include "../../include/mimo_b200.h"
#include "attn_common.h"
#include "host_util.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace mimo {

// Registers are reserved per group of 4 warps. With two MMA warpgroups (+ the TMA warp = 12 warps' worth) a thread may
// hold 168 registers: enough for S (64) + O (d/2) below d = 160, and up to d = 80 for the lookahead's S(j+1) (64) +
// P(j) (32) + O (ptxas -v: 0 spills). From d = 160 on a CTA has ONE MMA warpgroup (64 query rows, 8 warps' worth, up to
// 255 registers), so O, S and P stay in registers without spills, and the smaller Q tile leaves room for a second K/V
// stage.
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
  static constexpr int KVST = kFit < 4 ? kFit : 4;             // K/V stages that fit next to Q
  // S(j+1) is loaded while stage j still feeds P(j) V(j): the lookahead needs two stages, and registers (above)
  static constexpr bool kLook = NWG == 2 && KVST >= 2 && DP <= 80;
  static constexpr int kSmemBytes = kQBytes + KVST * kKVStageBytes + 1024 + 256;
  static_assert(KVST >= 1, "K/V tile does not fit");
};

// One online-softmax step on an S tile: row maxima over the tile's valid keys (kMask: the tile holds fewer than BKV
// keys, the others become -inf), the new running max m, alpha = the factor for the previous O and l, l updated, and P
// converted to the A fragments of P.V (k-step kk covers keys [16 kk, 16 kk + 16) = S fragments 2 kk, 2 kk + 1).
// Accumulator layout (S and O alike): this thread holds rows rbase and rbase + 8; fragment j (8 columns) holds columns
// 8 j + q2, + 1 in [4 j], [4 j + 1] (row rbase) and [4 j + 2], [4 j + 3] (row rbase + 8).
template <bool kMask, bool kBf16>
__device__ __forceinline__ void softmax_tile(float (&s)[BKV / 2], int valid, int q2, float scale_log2, float (&m)[2],
                                             float (&l)[2], float (&alpha)[2], uint32_t (&pa)[BKV / 16][4]) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int jn = 0; jn < BKV / 8; ++jn)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (!kMask || 8 * jn + q2 + (e & 1) < valid)
        mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * jn + e]);
      else
        s[4 * jn + e] = -INFINITY;
    }
  float m_new[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    m_new[r] = fmaxf(m[r], mx[r] * scale_log2);
    alpha[r] = ex2_ftz(m[r] - m_new[r]);
  }
  float rowsum[2] = {0.f, 0.f};
#pragma unroll
  for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = 8 * kk + 2 * i;  // i: (row, keys 0-7), (row + 8, keys 0-7), (row, keys 8-15), (row + 8, keys 8-15)
      const int r = i & 1;
      const float p0 = ex2_ftz(fmaf(s[e], scale_log2, -m_new[r]));
      const float p1 = ex2_ftz(fmaf(s[e + 1], scale_log2, -m_new[r]));
      rowsum[r] += p0 + p1;
      pa[kk][i] = Cvt<kBf16>::pack(p0, p1);
    }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] = l[r] * alpha[r] + rowsum[r];
    m[r] = m_new[r];
  }
}

template <bool kBf16>
__device__ __forceinline__ void softmax_step(float (&s)[BKV / 2], int valid, int q2, float scale_log2, float (&m)[2],
                                             float (&l)[2], float (&alpha)[2], uint32_t (&pa)[BKV / 16][4]) {
  if (valid < BKV)  // only the ragged last tile of the self or bank keys
    softmax_tile<true, kBf16>(s, valid, q2, scale_log2, m, l, alpha, pa);
  else
    softmax_tile<false, kBf16>(s, valid, q2, scale_log2, m, l, alpha, pa);
}

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

  if (warp == kProd) {
    if (lane != 0) return;
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
    return;
  }
  // ===================== MMA / softmax / epilogue =====================
  const int wg = warp >> 2;  // query rows [64 wg, 64 wg + 64) of the tile
  const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int q2 = (lane & 3) * 2;
  const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);
  const float scale_log2 = a.scale_log2;
  // keys of tile j that exist (the last self tile and the last bank tile may be ragged)
  auto tile_valid = [&](int j) {
    const bool bank = j >= a.n_self_tiles;
    const int valid = (bank ? a.lb : a.lq) - (bank ? j - a.n_self_tiles : j) * BKV;
    return valid < BKV ? valid : BKV;
  };
  auto kv_addr = [&](int j) { return smem_u32(sKV + (j % KVST) * Cfg::kKVStageBytes); };
  auto wait_kv = [&](int j) { mbar_wait(&kv_full[j % KVST], (j / KVST) & 1u); };
  auto issue_s = [&](float (&s)[BKV / 2], uint32_t k_addr) {
#pragma unroll
    for (int ks = 0; ks < DP / 16; ++ks) {
      const uint32_t off = (ks & 3) * 32;
      Wgmma<BKV, kBf16>::ss(s, make_smem_desc_sw128(q_addr + (ks >> 2) * Cfg::kQChunk + off, 16, 1024),
                            make_smem_desc_sw128(k_addr + (ks >> 2) * kChunkBytes + off, 16, 1024), ks != 0 ? 1u : 0u);
    }
  };
  float o[DP / 2];
  auto issue_pv = [&](const uint32_t (&pa)[BKV / 16][4], uint32_t v_addr, bool first) {
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      // B = V: MN-major, 16 keys = 2 KiB further down; 64-column chunks kChunkBytes apart
      Wgmma<DP, kBf16>::rs(o, pa[kk], make_smem_desc_sw128(v_addr + kk * 2048, kChunkBytes, 1024),
                           (!first || kk != 0) ? 1u : 0u);
    }
  };
  auto release = [&](int j) {
    if (lane == 0) mbar_arrive(&kv_empty[j % KVST]);
  };
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, alpha[2];
  float s[BKV / 2];
  uint32_t pa[BKV / 16][4];
  mbar_wait(q_full, 0);

  if constexpr (Cfg::kLook) {
    // turns at issuing MMAs: warpgroup wg waits on barrier 1 + wg and hands over on the other's; warpgroup 1 hands
    // the first turn to warpgroup 0 and skips its hand-over after its last turn, so every phase completes
    const int bar_mine = 1 + wg, bar_other = 2 - wg;
    if (wg == 1) bar_arrive(bar_other, 256);
    wait_kv(0);
    bar_sync(bar_mine, 256);
    wgmma_fence();
    issue_s(s, kv_addr(0));
    wgmma_commit();
    bar_arrive(bar_other, 256);
    wgmma_wait<0>();
    reg_fence(s);
    softmax_step<kBf16>(s, tile_valid(0), q2, scale_log2, m, l, alpha, pa);
    for (int j = 0; j + 1 < T; ++j) {
      wait_kv(j + 1);
      bar_sync(bar_mine, 256);
      wgmma_fence();
      issue_s(s, kv_addr(j + 1));
      wgmma_commit();
      issue_pv(pa, kv_addr(j) + NCH * kChunkBytes, j == 0);
      wgmma_commit();
      bar_arrive(bar_other, 256);
      uint32_t pn[BKV / 16][4];
      wgmma_wait<1>();
      reg_fence(s);
      softmax_step<kBf16>(s, tile_valid(j + 1), q2, scale_log2, m, l, alpha, pn);
      wgmma_wait<0>();
      reg_fence(o);
      release(j);
#pragma unroll
      for (int i = 0; i < DP / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      // P(j+1) replaces P(j). The byte permute (= pn) reads P(j) after the wait: ptxas ends a register's life at the
      // wgmma that reads it, and a plain copy let the softmax reuse P(j)'s registers while P(j) V(j) was still running,
      // which ptxas answers by serializing every wgmma of the kernel.
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
#pragma unroll
        for (int i = 0; i < 4; ++i) pa[kk][i] = __byte_perm(pa[kk][i], pn[kk][i], 0x7654);
    }
    // last tile: P(T-1) V(T-1) alone; warpgroup 1 keeps its turn (see above)
    bar_sync(bar_mine, 256);
    wgmma_fence();
    issue_pv(pa, kv_addr(T - 1) + NCH * kChunkBytes, T == 1);
    wgmma_commit();
    if (wg == 0) bar_arrive(bar_other, 256);
    wgmma_wait<0>();
    reg_fence(o);
    release(T - 1);
  } else {
    for (int j = 0; j < T; ++j) {
      wait_kv(j);
      wgmma_fence();
      issue_s(s, kv_addr(j));
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      softmax_step<kBf16>(s, tile_valid(j), q2, scale_log2, m, l, alpha, pa);
      if (j > 0) {
#pragma unroll
        for (int i = 0; i < DP / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
      }
      wgmma_fence();
      issue_pv(pa, kv_addr(j) + NCH * kChunkBytes, j == 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      release(j);
    }
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
