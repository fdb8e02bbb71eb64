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
#include <cuda_runtime.h>

#include <cudaTypedefs.h>

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

template <int BN, bool kRes>
struct GemmCfg {
  static constexpr int kStageBytes = BM * BK * 2 + BN * BK * 2;
  static constexpr int kNChunk = BN / 32;
  static constexpr int kOutBytes = 2 * kChunk;  // double-buffered staging of the output chunks
  static constexpr int kResSlots = kRes ? 2 : 0;
  static constexpr int kResBytes = kResSlots * kChunk;
  static constexpr int kBarBytes = 512;
  static constexpr int kFixed = kBarBytes + 2048 /*sbias*/ + kOutBytes + kResBytes;
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
  using Cfg = GemmCfg<BN, kRes>;
  using C = Cvt<kBf16>;
  using T = typename C::T;
  constexpr int NCHUNK = Cfg::kNChunk;
  extern __shared__ __align__(1024) uint8_t smem[];  // 128B-swizzled tiles need 1024-byte alignment
  uint8_t* sOut = smem + Cfg::kStages * Cfg::kStageBytes;  // [2 buffers][8 KiB]
  uint8_t* sRes = sOut + Cfg::kOutBytes;                    // [kResSlots][8 KiB]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sRes + Cfg::kResBytes);
  uint64_t* full_bar = bars;        // kStages (<= 8)
  uint64_t* empty_bar = bars + 8;   // kStages
  uint64_t* res_full = bars + 16;   // kResSlots (<= 2)
  uint64_t* res_empty = bars + 18;  // kResSlots
  float* sbias = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + Cfg::kBarBytes);  // [2][256]

  pdl_launch_dependents();
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // provably warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const int num_tiles = num_m_tiles * num_n_tiles * g.splits;
  // tile -> (output tile, K range): with split-K several CTAs share an output tile and each takes kb_split K blocks
  auto decode = [&](int tile, int& m_tile, int& n_tile, int& split, int& kb_begin, int& kb_cnt) {
    const int mn = tile / g.splits;
    split = tile - mn * g.splits;
    m_tile = mn / num_n_tiles;
    n_tile = mn - m_tile * num_n_tiles;
    kb_begin = split * g.kb_split;
    kb_cnt = num_k_blocks - kb_begin;
    if (kb_cnt > g.kb_split) kb_cnt = g.kb_split;
  };

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA0);
    tma_prefetch_desc(&tmA1);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmOut);
    if (kRes) tma_prefetch_desc(&tmRes);
  }
  if (warp == 9 && lane == 0) {
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // lane 0 of each MMA warp, once its wgmma group has read the stage
    }
    for (int s = 0; s < Cfg::kResSlots; ++s) {
      mbar_init(&res_full[s], 1);
      mbar_init(&res_empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // everything above touched only shared memory / the kernel parameters

  // tile -> coordinates of its first output row / pixel
  auto tile_origin = [&](int m_tile, int& x0, int& y0, int& n0) {
    if (g.conv) {
      x0 = (m_tile % g.tiles_w) * g.TW;
      y0 = ((m_tile / g.tiles_w) % g.tiles_h) * g.TH;
      n0 = (m_tile / (g.tiles_w * g.tiles_h)) * g.TN;
    } else {
      x0 = y0 = n0 = 0;
    }
  };

  // Producer warps run their loops with all 32 lanes (uniform control flow) and elect one lane for the TMA
  // instructions: addresses then live in uniform registers.
  if (warp == 8) {
    // ===================== TMA producer (operands) =====================
    // (all index arithmetic is incremental: one division per tile, only under split-K)
    uint32_t stage = 0, phase = 0;
    const int kb_per_tap = g.kb0 + g.kb1;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_tile, n_tile, split, kb_begin, kb_cnt;
      decode(tile, m_tile, n_tile, split, kb_begin, kb_cnt);
      int x0, y0, n0;
      tile_origin(m_tile, x0, y0, n0);
      // conv: k-block inside the tap, tap index / offsets, tap * ctot
      int tap = kb_per_tap > 0 ? kb_begin / kb_per_tap : 0;
      int rem = kb_begin - tap * kb_per_tap;
      int dx = g.tdx[tap], dy = g.tdy[tap], tap_k = tap * g.ctot;
      for (int kbl = 0, kb = kb_begin; kbl < kb_cnt; ++kbl, ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        uint8_t* sa = smem + stage * Cfg::kStageBytes;
        uint8_t* sb = sa + BM * BK * 2;
        if (elect_one()) {
          if (!g.conv) {
            mbar_expect_tx(&full_bar[stage], BM * BK * 2 + BN * BK * 2);
            if (kb < g.kb0) {  // A = [A0 | A1] along K (virtual concat for the up-block shortcut GEMMs)
              tma_load_2d(sa, &tmA0, &full_bar[stage], kb * BK, m_tile * BM);
              tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n_tile * BN);
            } else {
              tma_load_2d(sa, &tmA1, &full_bar[stage], (kb - g.kb0) * BK, m_tile * BM);
              tma_load_2d(sb, &tmB, &full_bar[stage], g.c0 + (kb - g.kb0) * BK, n_tile * BN);
            }
          } else {
            mbar_expect_tx(&full_bar[stage], g.a_bytes + BN * BK * 2);
            int kcoord;
            if (rem < g.kb0) {
              tma_load_4d(sa, &tmA0, &full_bar[stage], rem * BK, x0 + dx, y0 + dy, n0);
              kcoord = tap_k + rem * BK;
            } else {
              tma_load_4d(sa, &tmA1, &full_bar[stage], (rem - g.kb0) * BK, x0 + dx, y0 + dy, n0);
              kcoord = tap_k + g.c0 + (rem - g.kb0) * BK;
            }
            tma_load_2d(sb, &tmB, &full_bar[stage], kcoord, n_tile * BN);
          }
        }
        __syncwarp();
        if (++rem == kb_per_tap) {
          rem = 0;
          tap_k += g.ctot;
          if (++tap == g.ntaps) tap = 0;
          dx = g.tdx[tap];
          dy = g.tdy[tap];
        }
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
    }
  } else if (warp == 9) {
    // ===================== TMA producer (residual chunks) =====================
    if constexpr (kRes) {
      uint32_t k = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_tile = tile / num_n_tiles;  // (a residual never comes with split-K: splits == 1 here)
        const int n_tile = tile % num_n_tiles;
        int x0, y0, n0;
        tile_origin(m_tile, x0, y0, n0);
        for (int c = 0; c < NCHUNK; ++c, ++k) {
          const uint32_t slot = k % Cfg::kResSlots;
          mbar_wait(&res_empty[slot], ((k / Cfg::kResSlots) & 1u) ^ 1u);
          if (elect_one()) {
            mbar_expect_tx(&res_full[slot], g.chunk_bytes);
            const int col = n_tile * BN + c * 32;  // boxes beyond N are zero-filled (keeps the slot sequence uniform)
            if (g.conv)
              tma_load_4d(sRes + slot * kChunk, &tmRes, &res_full[slot], col, x0, y0, n0);
            else
              tma_load_2d(sRes + slot * kChunk, &tmRes, &res_full[slot], col, m_tile * BM);
          }
          __syncwarp();
        }
      }
    }
  } else if (warp < 8) {
    // ===================== MMA + epilogue (warpgroups 0, 1) =====================
    const int wg = warp >> 2;    // tile rows [64 wg, 64 wg + 64)
    const int ct = threadIdx.x;  // 0..255
    // wgmma accumulator layout: warp w of the warpgroup holds rows 16 w + lane / 4 (+ 8); fragment j (8 columns)
    // holds columns 8 j + 2 (lane % 4) (+ 1) in acc[4 j + {0, 1}] (row) and acc[4 j + {2, 3}] (row + 8)
    const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int q2 = (lane & 3) * 2;
    const bool issuer = ct == 0;
    const int sw[2] = {(rbase >> 1) & 3, ((rbase + 8) >> 1) & 3};  // 64-byte swizzle: 16-byte piece ^= addr bits [7:8]
    const bool do_silu = ep.act == MIMO_ACT_SILU;
    // (32-bit arithmetic: M, the pixel count and rows_per_group all fit an int; 64-bit divisions cost ~1 us here)
    const uint32_t rpg = static_cast<uint32_t>(ep.rows_per_group);
    float acc[BN / 2];
    uint32_t stage = 0, phase = 0, lt = 0, oc = 0, rc = 0;

    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++lt) {
      int m_tile, n_tile, split, kb_begin, kb_cnt;
      decode(tile, m_tile, n_tile, split, kb_begin, kb_cnt);
      int x0, y0, n0;
      tile_origin(m_tile, x0, y0, n0);
      // first / last group touched by a tile (uniform per tile)
      auto tile_groups = [&](int mt, uint32_t& gf, uint32_t& gl) {
        if (!g.conv) {
          const uint32_t m0 = static_cast<uint32_t>(mt) * BM;
          uint32_t m1 = m0 + BM - 1;
          if (m1 > static_cast<uint32_t>(M) - 1) m1 = static_cast<uint32_t>(M) - 1;
          gf = m0 / rpg;
          gl = m1 / rpg;
        } else {
          int tx, ty, tn;
          tile_origin(mt, tx, ty, tn);
          int n1 = tn + g.TN - 1;
          if (n1 > g.NI - 1) n1 = g.NI - 1;
          const uint32_t hw = static_cast<uint32_t>(g.H) * g.W;
          gf = (static_cast<uint32_t>(tn) * hw) / rpg;
          gl = (static_cast<uint32_t>(n1 + 1) * hw - 1) / rpg;
        }
      };
      // column constants of a tile: bias (+ the per-branch vector when the whole tile shares one group)
      const int ce = ct;  // one column per MMA-warpgroup thread (BN <= 256)
      auto load_consts = [&](int t) -> float {
        float v = 0.f;
        const int mt = (t / g.splits) / num_n_tiles, nt = (t / g.splits) % num_n_tiles;
        const int col = nt * BN + ce;
        if (ce < BN && col < N) {
          if (ep.bias) v = C::to_f(static_cast<const T*>(ep.bias)[col]);
          if (ep.rowvec) {
            uint32_t gf, gl;
            tile_groups(mt, gf, gl);
            if (gf == gl) v += C::to_f(static_cast<const T*>(ep.rowvec)[static_cast<long long>(gf) * ep.ld_rowvec + col]);
          }
        }
        return ep.act == MIMO_ACT_GEGLU ? v : v * ep.scale;  // y = acc * scale + (bias + vec) * scale
      };
      float* sb = sbias + (lt & 1u) * 256;
      if (ct < BN) sb[ct] = load_consts(tile);  // the loads fly under the main loop

      // ---- main loop: one wgmma group per k-block; the stage of k-block i - 1 is released once group i is issued ----
      uint32_t prev_stage = 0;
      for (int kb = 0; kb < kb_cnt; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint64_t da = make_smem_desc_sw128(sa + wg * (64 * 128), 16, 1024);
        const uint64_t db = make_smem_desc_sw128(sa + BM * BK * 2, 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // advance 16 elements (32 B) along K inside the 128-B swizzle row: +2 in the (addr >> 4) field
          Wgmma<BN, kBf16>::ss(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        }
        prev_stage = stage;
        if (++stage == Cfg::kStages) {
          stage = 0;
          phase ^= 1u;
        }
      }
      wgmma_wait<0>();
      reg_fence(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      // ---- rows of this thread; which group(s) of the per-branch vector they belong to ----
      long long row[2];
      bool row_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rbase + 8 * h;
        if (!g.conv) {
          row[h] = static_cast<long long>(m_tile) * BM + r;
          row_ok[h] = row[h] < M;
        } else {
          const int x = r % g.TW, y = (r / g.TW) % g.TH, n = r / (g.TW * g.TH);
          row_ok[h] = (n < g.TN) && (x0 + x < g.W) && (y0 + y < g.H) && (n0 + n < g.NI);
          row[h] = (static_cast<long long>(n0 + n) * g.H + (y0 + y)) * g.W + (x0 + x);
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");  // MMA warpgroups only: column constants visible

      if (ep.partial) {
        // split-K: raw fp32 accumulators of this K range -> partial[split][row][N]; the reduction kernel sums the
        // splits in a fixed order and applies the whole epilogue (deterministic: no atomics)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h]) continue;
          float* prow = ep.partial + (static_cast<long long>(split) * M + row[h]) * N;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_tile * BN + 8 * j + q2;
            if (col < N) *reinterpret_cast<float2*>(prow + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
        }
        continue;
      }

      // one 32-column chunk: tile columns [32 c, 32 c + 32) of both rows -> staging buffer -> TMA store
      auto stage_and_store = [&](uint8_t* obuf, int col0) {
        fence_proxy_async_smem();
        if (issuer) tma_store_wait_read0();  // see "Staging-buffer reuse" below
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (issuer) {
          if (g.conv)
            tma_store_4d(&tmOut, obuf, col0, x0, y0, n0);
          else
            tma_store_2d(&tmOut, obuf, col0, m_tile * BM);
          tma_store_commit();
        }
      };

      if (ep.act != MIMO_ACT_GEGLU) {
        const float scale = ep.scale;
        bool rv_uniform = false;
        if (ep.rowvec) {
          uint32_t gf, gl;
          tile_groups(m_tile, gf, gl);
          rv_uniform = gf == gl;
        }
        const bool need_rv = ep.rowvec != nullptr && !rv_uniform;  // uniform per tile
        // mode 0: no column constants, unit scale, no residual -> accumulators are packed as they are;
        //      1: y = acc * scale + consts (+ residual);  2: as 1, plus per-row vectors (tile straddles groups)
        const int mode = (!kRes && !do_silu && !need_rv && ep.bias == nullptr && ep.rowvec == nullptr && scale == 1.0f)
                             ? 0 : (need_rv ? 2 : 1);
        const T* rv[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          rv[h] = (need_rv && row_ok[h])
                      ? static_cast<const T*>(ep.rowvec) + static_cast<long long>(static_cast<uint32_t>(row[h]) / rpg) * ep.ld_rowvec
                      : nullptr;
#pragma unroll
        for (int c = 0; c < NCHUNK; ++c) {
          uint8_t* obuf = sOut + (oc & 1u) * kChunk;
          ++oc;
          const int col0 = n_tile * BN + c * 32;
          [[maybe_unused]] uint32_t rslot = 0;
          if constexpr (kRes) {
            const uint32_t k = rc++;
            rslot = k % Cfg::kResSlots;
            mbar_wait(&res_full[rslot], (k / Cfg::kResSlots) & 1u);
          }
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * c + jj;
            const float2 cst0 = *reinterpret_cast<const float2*>(sb + c * 32 + 8 * jj + q2);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = rbase + 8 * h;
              const int off = r * 64 + ((jj ^ sw[h]) << 4) + q2 * 2;
              float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
              if (mode != 0) {
                float c0 = cst0.x, c1 = cst0.y;
                // the per-row vector joins the column constants FIRST, as load_consts() pre-sums them when a tile lies
                // inside one group
                if (mode == 2 && rv[h] && col0 + 8 * jj + q2 < N) {
                  const float2 t = C::unpack(__ldg(reinterpret_cast<const unsigned int*>(rv[h] + col0 + 8 * jj + q2)));
                  c0 = fmaf(t.x, scale, c0);
                  c1 = fmaf(t.y, scale, c1);
                }
                f0 = fmaf(f0, scale, c0);
                f1 = fmaf(f1, scale, c1);
              }
              if constexpr (kRes) {
                const float2 t = C::unpack(*reinterpret_cast<const uint32_t*>(sRes + rslot * kChunk + off));
                f0 = fmaf(t.x, scale, f0);
                f1 = fmaf(t.y, scale, f1);
              }
              if (do_silu) {
                f0 = silu_f(f0);
                f1 = silu_f(f1);
              }
              *reinterpret_cast<uint32_t*>(obuf + off) = C::pack(f0, f1);
            }
          }
          if constexpr (kRes) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&res_empty[rslot]);
          }
          stage_and_store(obuf, col0);
        }
      } else {
        // GEGLU: tile columns [0, BN/2) are values, [BN/2, BN) the matching gates (same thread, BN/16 fragments on)
        constexpr int HALF = BN / 2;
#pragma unroll
        for (int c = 0; c < HALF / 32; ++c) {
          uint8_t* obuf = sOut + (oc & 1u) * kChunk;
          ++oc;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * c + jj, jg = j + HALF / 8;
            const float2 cv = *reinterpret_cast<const float2*>(sb + c * 32 + 8 * jj + q2);
            const float2 cg = *reinterpret_cast<const float2*>(sb + HALF + c * 32 + 8 * jj + q2);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = rbase + 8 * h;
              const float f0 = (acc[4 * j + 2 * h] + cv.x) * gelu_erf_fast(acc[4 * jg + 2 * h] + cg.x);
              const float f1 = (acc[4 * j + 2 * h + 1] + cv.y) * gelu_erf_fast(acc[4 * jg + 2 * h + 1] + cg.y);
              *reinterpret_cast<uint32_t*>(obuf + r * 64 + ((jj ^ sw[h]) << 4) + q2 * 2) = C::pack(f0, f1);
            }
          }
          stage_and_store(obuf, n_tile * HALF + c * 32);
        }
      }
    }
    if (issuer) tma_store_wait_all();
  }
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

// Split-K decision: only when the output tiles would leave more than half of the SMs idle AND every split still gets a
// long K range (>= 16 K blocks = 1024): the deep, small-M convolutions / FF projections of the 8x8 and 16x16 levels when
// the clip's frames are spread over several GPUs. Returns the number of splits (1 = off).
static int pick_splits(long long tiles, int nkb, long long M, int N, int64_t ws_bytes) {
  if (tiles * 2 > num_sms() || nkb < 32) return 1;
  long long s = num_sms() / tiles;
  if (s > nkb / 16) s = nkb / 16;
  if (s > 16) s = 16;
  while (s > 1 && s * M * N * 4 > ws_bytes) --s;
  return s < 2 ? 1 : static_cast<int>(s);
}

struct Maps {
  CUtensorMap a0, a1, b, out, res;
};

template <int BN, bool kBf16, bool kRes>
static int launch_cfg(const Maps& m, int M, int N, int mt, int nt, int nkb, const ConvGeom& g, const EpiArgs& ep,
                      cudaStream_t st) {
  using Cfg = GemmCfg<BN, kRes>;
  auto kern = gemm_wgmma_kernel<BN, kBf16, kRes>;
  static bool attr_done = false;  // per instantiation
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_cuda_error("cudaFuncSetAttribute(gemm)", e);
    attr_done = true;
  }
  const int tiles = mt * nt;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  cudaError_t e = launch_k(kern, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, st, m.a0, m.a1, m.b, m.out, m.res, M, N, mt,
                           nt, nkb, g, ep);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error("gemm launch", e);
  return MIMO_OK;
}

template <bool kBf16>
static int launch_bn(int bn, bool res, const Maps& m, int M, int N, int mt, int nt, int nkb, const ConvGeom& g,
                     const EpiArgs& ep, cudaStream_t st) {
  switch (bn) {
    case 64:
      return res ? launch_cfg<64, kBf16, true>(m, M, N, mt, nt, nkb, g, ep, st)
                 : launch_cfg<64, kBf16, false>(m, M, N, mt, nt, nkb, g, ep, st);
    case 128:
      return res ? launch_cfg<128, kBf16, true>(m, M, N, mt, nt, nkb, g, ep, st)
                 : launch_cfg<128, kBf16, false>(m, M, N, mt, nt, nkb, g, ep, st);
    case 160:
      return res ? launch_cfg<160, kBf16, true>(m, M, N, mt, nt, nkb, g, ep, st)
                 : launch_cfg<160, kBf16, false>(m, M, N, mt, nt, nkb, g, ep, st);
    case 192:
      return res ? launch_cfg<192, kBf16, true>(m, M, N, mt, nt, nkb, g, ep, st)
                 : launch_cfg<192, kBf16, false>(m, M, N, mt, nt, nkb, g, ep, st);
    case 256:
      return res ? launch_cfg<256, kBf16, true>(m, M, N, mt, nt, nkb, g, ep, st)
                 : launch_cfg<256, kBf16, false>(m, M, N, mt, nt, nkb, g, ep, st);
  }
  return set_error(MIMO_ERR_ARG, "gemm: unsupported BN");
}

static int g_force_bn = 0;

// Tile-width choice: least padded columns first, then the widest tile (fewer A re-reads, higher MMA N).
int pick_bn(int N, bool geglu, long long m_tiles) {
  if (g_force_bn) return g_force_bn;
  if (geglu) {
    if (N % 256 == 0) return 256;
    if (N % 128 == 0) return 128;
    return 64;
  }
  const int cands[5] = {256, 192, 160, 128, 64};
  int best = 64;
  double best_eff = -1.0;
  for (int i = 0; i < 5; ++i) {
    const int bn = cands[i];
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
  if (int rc = ensure_device()) return rc;
  const int mt = (p->M + BM - 1) / BM;
  const int K1 = p->a1 ? p->K1 : 0;
  if (K1 < 0 || (K1 % 8) || (p->a1 && (p->lda1 % 8))) return set_error(MIMO_ERR_ARG, "mimo_gemm: K1/lda1 % 8 != 0");
  const int kb0 = (p->K + BK - 1) / BK;
  const int kb1 = (K1 + BK - 1) / BK;
  const int nkb = kb0 + kb1;
  int bn = pick_bn(p->N, geglu, mt);
  int splits = 1;
  if (!geglu && g_splitk && p->workspace && !g_force_bn) {
    const int bn_wide = pick_bn(p->N, false, 1 << 20);  // the tile width a large problem would get
    splits = pick_splits(static_cast<long long>(mt) * ((p->N + bn_wide - 1) / bn_wide), nkb, p->M, p->N, p->workspace_bytes);
    if (splits > 1) bn = bn_wide;
  }
  if (geglu && (p->N % bn)) return set_error(MIMO_ERR_ARG, "mimo_gemm: GEGLU needs N % tile == 0");
  const int nt = (p->N + bn - 1) / bn;
  const bool res = p->ep.residual != nullptr && !geglu && splits == 1;

  Maps m;
  const uint64_t adim[2] = {static_cast<uint64_t>(p->K), static_cast<uint64_t>(p->M)};
  const uint64_t astr[1] = {static_cast<uint64_t>(p->lda) * 2};
  const uint32_t abox[2] = {BK, BM};
  if (int rc = encode_tmap(&m.a0, p->dtype, 2, p->a, adim, astr, abox)) return rc;
  m.a1 = m.a0;
  if (K1) {
    const uint64_t a1dim[2] = {static_cast<uint64_t>(K1), static_cast<uint64_t>(p->M)};
    const uint64_t a1str[1] = {static_cast<uint64_t>(p->lda1) * 2};
    if (int rc = encode_tmap(&m.a1, p->dtype, 2, p->a1, a1dim, a1str, abox)) return rc;
  }
  const uint64_t bdim[2] = {static_cast<uint64_t>(p->K + K1), static_cast<uint64_t>(p->N)};
  const uint64_t bstr[1] = {static_cast<uint64_t>(p->ldw) * 2};
  const uint32_t bbox[2] = {BK, static_cast<uint32_t>(bn)};
  if (int rc = encode_tmap(&m.b, p->dtype, 2, p->w, bdim, bstr, bbox)) return rc;
  // output / residual: 128-row x 32-column boxes, 64-byte swizzle
  const int n_out = geglu ? p->N / 2 : p->N;
  const uint64_t odim[2] = {static_cast<uint64_t>(n_out), static_cast<uint64_t>(p->M)};
  const uint64_t ostr[1] = {static_cast<uint64_t>(p->ldo) * 2};
  const uint32_t obox[2] = {32, BM};
  if (int rc = encode_tmap(&m.out, p->dtype, 2, p->out, odim, ostr, obox, 64)) return rc;
  m.res = m.out;
  if (res) {
    const uint64_t rstr[1] = {static_cast<uint64_t>(p->ep.ld_res) * 2};
    if (int rc = encode_tmap(&m.res, p->dtype, 2, p->ep.residual, odim, rstr, obox, 64)) return rc;
  }

  ConvGeom g = {};
  g.kb0 = kb0;
  g.kb1 = kb1;
  g.c0 = p->K;
  g.chunk_bytes = kChunk;
  g.splits = splits;
  g.kb_split = (nkb + splits - 1) / splits;
  EpiArgs ep = make_epi(p->ep, p->N);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (splits > 1) {
    ep.bias = ep.rowvec = nullptr;
    ep.act = MIMO_ACT_NONE;
    ep.scale = 1.0f;
    ep.partial = static_cast<float*>(p->workspace);
  }
  const int rc = p->dtype == MIMO_BF16 ? launch_bn<true>(bn, res, m, p->M, p->N, mt, nt, nkb, g, ep, st)
                                       : launch_bn<false>(bn, res, m, p->M, p->N, mt, nt, nkb, g, ep, st);
  if (rc || splits == 1) return rc;
  return launch_reduce(p->dtype, ep.partial, splits, p->M, p->N, p->ep, p->out, p->ldo, st);
}

// One implicit-GEMM convolution launch: `ntaps` taps at offsets (tdx, tdy) over the [n, h, w, c] input(s); the output
// (and residual) pixel (n, y, x) lives at out + ((n * oh + y * sy) * ow + x * sx) * ldo elements, i.e. a strided view of a
// larger image when (sx, sy) != (1, 1).
static int conv_launch(const mimo_conv3x3_params* p, const void* w, int ntaps, const signed char* tdx,
                       const signed char* tdy, void* out, int sx, int sy, int ow, int oh, void* stream) {
  const int c1 = p->x1 ? p->c1 : 0;
  ConvGeom g = {};
  g.conv = 1;
  g.H = p->h;
  g.W = p->w_;
  g.NI = p->n;
  g.TW = p->w_ < BM ? p->w_ : BM;
  g.TH = BM / g.TW;
  if (g.TH > p->h) g.TH = p->h;
  if (g.TH < 1) g.TH = 1;
  g.TN = BM / (g.TW * g.TH);
  if (g.TN > p->n) g.TN = p->n;
  if (g.TN < 1) g.TN = 1;
  if (g.TN > 1 && g.TH != p->h) g.TN = 1;  // several images per tile only when a tile spans whole images
  g.tiles_w = (p->w_ + g.TW - 1) / g.TW;
  g.tiles_h = (p->h + g.TH - 1) / g.TH;
  const int tiles_n = (p->n + g.TN - 1) / g.TN;
  g.ctot = p->c0 + c1;
  g.c0 = p->c0;
  g.kb0 = (p->c0 + BK - 1) / BK;
  g.kb1 = (c1 + BK - 1) / BK;
  g.a_bytes = g.TW * g.TH * g.TN * BK * 2;
  g.chunk_bytes = g.TW * g.TH * g.TN * 64;
  g.ntaps = ntaps;
  for (int t = 0; t < 9; ++t) {
    g.tdx[t] = t < ntaps ? tdx[t] : 0;
    g.tdy[t] = t < ntaps ? tdy[t] : 0;
  }
  const int mt = g.tiles_w * g.tiles_h * tiles_n;
  const int nkb = ntaps * (g.kb0 + g.kb1);
  const long long Mrows = static_cast<long long>(p->n) * p->h * p->w_;
  if (Mrows > 0x7fffffffLL) return set_error(MIMO_ERR_ARG, "mimo_conv: too many pixels");
  int bn = pick_bn(p->cout, false, mt);
  int splits = 1;
  // split-K needs the dense NHWC output (row = pixel index): not for the strided parity classes of mimo_conv_up2x
  if (g_splitk && p->workspace && !g_force_bn && sx == 1 && sy == 1 && p->ldo == p->cout) {
    const int bn_wide = pick_bn(p->cout, false, 1 << 20);
    splits = pick_splits(static_cast<long long>(mt) * ((p->cout + bn_wide - 1) / bn_wide), nkb, Mrows, p->cout,
                         p->workspace_bytes);
    if (splits > 1) bn = bn_wide;
  }
  g.splits = splits;
  g.kb_split = (nkb + splits - 1) / splits;
  const int nt = (p->cout + bn - 1) / bn;
  const bool res = p->ep.residual != nullptr && splits == 1;

  Maps m;
  auto nhwc_map = [&](CUtensorMap* tm, const void* base, int c, long long pitch, uint32_t box_c, int swz, int px,
                      int py, int iw, int ih) {
    // pixel (n, y, x) at base + ((n * ih + y * py) * iw + x * px) * pitch elements
    const uint64_t dim[4] = {static_cast<uint64_t>(c), static_cast<uint64_t>(p->w_), static_cast<uint64_t>(p->h),
                             static_cast<uint64_t>(p->n)};
    const uint64_t str[3] = {static_cast<uint64_t>(px) * pitch * 2, static_cast<uint64_t>(py) * iw * pitch * 2,
                             static_cast<uint64_t>(ih) * iw * pitch * 2};
    const uint32_t box[4] = {box_c, static_cast<uint32_t>(g.TW), static_cast<uint32_t>(g.TH),
                             static_cast<uint32_t>(g.TN)};
    return encode_tmap(tm, p->dtype, 4, base, dim, str, box, swz);
  };
  if (int rc = nhwc_map(&m.a0, p->x0, p->c0, p->c0, BK, 128, 1, 1, p->w_, p->h)) return rc;
  m.a1 = m.a0;
  if (c1)
    if (int rc = nhwc_map(&m.a1, p->x1, c1, c1, BK, 128, 1, 1, p->w_, p->h)) return rc;
  {
    const uint64_t dim[2] = {static_cast<uint64_t>(ntaps) * g.ctot, static_cast<uint64_t>(p->cout)};
    const uint64_t str[1] = {static_cast<uint64_t>(ntaps) * g.ctot * 2};
    const uint32_t box[2] = {BK, static_cast<uint32_t>(bn)};
    if (int rc = encode_tmap(&m.b, p->dtype, 2, w, dim, str, box)) return rc;
  }
  if (int rc = nhwc_map(&m.out, out, p->cout, p->ldo, 32, 64, sx, sy, ow, oh)) return rc;
  m.res = m.out;
  if (res)
    if (int rc = nhwc_map(&m.res, p->ep.residual, p->cout, p->ep.ld_res, 32, 64, 1, 1, p->w_, p->h)) return rc;

  EpiArgs ep = make_epi(p->ep, p->cout);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (splits > 1) {
    ep.bias = ep.rowvec = nullptr;
    ep.act = MIMO_ACT_NONE;
    ep.scale = 1.0f;
    ep.partial = static_cast<float*>(p->workspace);
  }
  const int rc = p->dtype == MIMO_BF16
                     ? launch_bn<true>(bn, res, m, static_cast<int>(Mrows), p->cout, mt, nt, nkb, g, ep, st)
                     : launch_bn<false>(bn, res, m, static_cast<int>(Mrows), p->cout, mt, nt, nkb, g, ep, st);
  if (rc || splits == 1) return rc;
  return launch_reduce(p->dtype, ep.partial, splits, Mrows, p->cout, p->ep, out, p->ldo, st);
}

static int conv_check(const mimo_conv3x3_params* p, const char* who) {
  if (!p || !p->x0 || !p->w || !p->out) return set_error(MIMO_ERR_ARG, "mimo_conv: null pointer");
  if (p->n <= 0 || p->h <= 0 || p->w_ <= 0 || p->cout <= 0 || p->c0 <= 0)
    return set_error(MIMO_ERR_ARG, "mimo_conv: empty problem");
  const int c1 = p->x1 ? p->c1 : 0;
  if ((p->c0 % 8) || (c1 % 8) || (p->cout % 8) || (p->ldo % 8))
    return set_error(MIMO_ERR_ARG, "mimo_conv: channel counts must be multiples of 8");
  if (p->ep.act == MIMO_ACT_GEGLU) return set_error(MIMO_ERR_ARG, "mimo_conv: GEGLU not supported");
  if (p->ep.residual && (p->ep.ld_res % 8)) return set_error(MIMO_ERR_ARG, "mimo_conv: ld_res % 8 != 0");
  (void)who;
  return ensure_device();
}

extern "C" int mimo_conv3x3(const mimo_conv3x3_params* p, void* stream) {
  if (int rc = conv_check(p, "mimo_conv3x3")) return rc;
  static const signed char dx[9] = {-1, 0, 1, -1, 0, 1, -1, 0, 1};
  static const signed char dy[9] = {-1, -1, -1, 0, 0, 0, 1, 1, 1};
  return conv_launch(p, p->w, 9, dx, dy, p->out, 1, 1, p->w_, p->h, stream);
}

// nearest-x2 upsampling followed by a 3x3 / pad 1 convolution, without the upsampled tensor: output pixel (2y+a, 2x+b)
// only ever sees the 2x2 source neighbourhood {y-1+a, y+a} x {x-1+b, x+b}, so each of the four parity classes (a, b) is a
// 2x2-tap convolution over the SOURCE image whose weights are sums of the 3x3 taps that land on the same source pixel
// (packed by the host: w = [4 classes][cout, 4 * cin], class = 2a + b, tap = 2 iy + ix). 4/9 of the FLOPs, no 4x buffer.
extern "C" int mimo_conv_up2x(const mimo_conv3x3_params* p, void* stream) {
  if (int rc = conv_check(p, "mimo_conv_up2x")) return rc;
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
      if (int rc = conv_launch(p, w, 4, dx, dy, out, 2, 2, 2 * p->w_, 2 * p->h, stream)) return rc;
    }
  return MIMO_OK;
}
