// Body of the GEMM / conv kernels of gemm_wgmma.cu (see the description at the top of that file). Not a header: the
// kernels there include it as their whole body, so the 16-bit kernel is compiled from the same statements with the e4m3
// steps removed by `if constexpr (kE4m3)`, and keeps its parameter list and generated code. In scope at the include:
// the template parameters BN, kBf16, kRes, the constants kE4m3, kImgScale, kOutE4m3 and kBlockScale, the kernel parameters
// tmA0, tmA1, tmB, tmOut, tmRes, M, N, num_m_tiles, num_n_tiles, num_k_blocks, g, ep, and a_scale, w_scale (fp32 scales of
// A and W, used when kE4m3: a_scale per A row, or with kImgScale per image of a convolution), out_scale and ld_scale
// (kOutE4m3: the GEGLU output is e4m3 with one scale per row and 128-column block, out_scale[n_tile][row]), and tmAS
// (kBlockScale: A has one scale per row and 128-element K block, a_scale[kb][row], fetched into each pipeline stage
// through tmAS; a_scale itself is not read).
  using Cfg = GemmCfg<BN, kRes, kE4m3, kBlockScale>;
  constexpr int kBKel = kE4m3 ? 2 * BK : BK;  // elements per K block (one 128-byte swizzle row either way)
  constexpr int kConvKel = kImgScale ? kBKel : BK;  // channels per conv K block (gemm_e4m3_kernel runs GEMM rows only)
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
    if constexpr (kBlockScale) tma_prefetch_desc(&tmAS);
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
            mbar_expect_tx(&full_bar[stage], BM * BK * 2 + BN * BK * 2 + (kBlockScale ? BM * 4 : 0));
            if constexpr (kBlockScale)  // the K block's 128 row scales, behind W in the stage
              tma_load_2d(sb + BN * BK * 2, &tmAS, &full_bar[stage], 2 * m_tile * BM, kb);  // (fp32 as 16-bit pairs)
            if (kb < g.kb0) {  // A = [A0 | A1] along K (virtual concat for the up-block shortcut GEMMs)
              tma_load_2d(sa, &tmA0, &full_bar[stage], kb * kBKel, m_tile * BM);
              tma_load_2d(sb, &tmB, &full_bar[stage], kb * kBKel, n_tile * BN);
            } else {
              tma_load_2d(sa, &tmA1, &full_bar[stage], (kb - g.kb0) * BK, m_tile * BM);
              tma_load_2d(sb, &tmB, &full_bar[stage], g.c0 + (kb - g.kb0) * BK, n_tile * BN);
            }
          } else {
            mbar_expect_tx(&full_bar[stage], g.a_bytes + BN * BK * 2);
            int kcoord;
            // e4m3: a channel count of 64 mod 128 (320, 960) leaves half a block in each tap; TMA zero-fills the A box
            // past the channels, while the W box reads on into the next tap's weights (finite e4m3 bytes): they meet
            // zeros only, so the sum is exact, at 384 / 320 of the MMA work for 320 channels
            if (rem < g.kb0) {
              tma_load_4d(sa, &tmA0, &full_bar[stage], rem * kConvKel, x0 + dx, y0 + dy, n0);
              kcoord = tap_k + rem * kConvKel;
            } else {
              tma_load_4d(sa, &tmA1, &full_bar[stage], (rem - g.kb0) * kConvKel, x0 + dx, y0 + dy, n0);
              kcoord = tap_k + g.c0 + (rem - g.kb0) * kConvKel;
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
      if constexpr (kE4m3) {
        // behind sbias: [2][256] column scales, then [2][128] row scales
        float* sws = sbias + 512 + (lt & 1u) * 256;
        float* sas = sbias + 1024 + (lt & 1u) * 128;
        const int col = n_tile * BN + ct;
        if (ct < BN) sws[ct] = col < N ? __ldg(w_scale + col) : 0.f;
        if constexpr (kBlockScale) {
          // (row scales come with each K block)
        } else if constexpr (kImgScale) {
          // conv: one scale per image; tile row ct lies in image n0 + ct / (TW TH) of the {TW, TH, TN} footprint
          const int img = n0 + ct / (g.TW * g.TH);
          if (ct < BM) sas[ct] = img < g.NI ? __ldg(a_scale + img) : 0.f;
        } else {
          const int r = m_tile * BM + ct;
          if (ct < BM) sas[ct] = r < M ? __ldg(a_scale + r) : 0.f;
        }
      }

      // ---- main loop: one wgmma group per k-block; the stage of k-block i - 1 is released once group i is issued ----
      // kBlockScale: each k-block's group accumulates into blk on its own; once it has completed, acc += blk * row scale
      // of that block (the two rows of this thread), and the stage is released
      if constexpr (kBlockScale) {
        float blk[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < kb_cnt; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          uint8_t* st = smem + stage * Cfg::kStageBytes;
          const uint32_t sa = smem_u32(st);
          const uint64_t da = make_smem_desc_sw128(sa + wg * (64 * 128), 16, 1024);
          const uint64_t db = make_smem_desc_sw128(sa + BM * BK * 2, 16, 1024);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) WgmmaE4m3<BN>::ss(blk, da + 2 * k, db + 2 * k, k != 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(blk);
          const float* srs = reinterpret_cast<const float*>(st + BM * BK * 2 + BN * BK * 2);
          const float s0 = srs[rbase], s1 = srs[rbase + 8];
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            acc[4 * j] = fmaf(blk[4 * j], s0, acc[4 * j]);
            acc[4 * j + 1] = fmaf(blk[4 * j + 1], s0, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(blk[4 * j + 2], s1, acc[4 * j + 2]);
            acc[4 * j + 3] = fmaf(blk[4 * j + 3], s1, acc[4 * j + 3]);
          }
          if (++stage == Cfg::kStages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      } else {
        uint32_t prev_stage = 0;
        for (int kb = 0; kb < kb_cnt; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
          const uint64_t da = make_smem_desc_sw128(sa + wg * (64 * 128), 16, 1024);
          const uint64_t db = make_smem_desc_sw128(sa + BM * BK * 2, 16, 1024);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            // advance 32 B along K (16 16-bit / 32 e4m3 elements) inside the 128-B swizzle row: +2 in the (addr >> 4) field
            if constexpr (kE4m3)
              WgmmaE4m3<BN>::ss(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
            else
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
      }

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
      // e4m3: acc * a_scale[row] * w_scale[col] is taken where each accumulator is first read below (a separate pass over
      // all BN / 2 accumulators spills at BN = 256). Split-K (ep.partial) never runs in e4m3.
      [[maybe_unused]] const float* sws = sbias + 512 + (lt & 1u) * 256;
      [[maybe_unused]] float ascale[2];
      if constexpr (kE4m3 && !kBlockScale) {
        const float* sas = sbias + 1024 + (lt & 1u) * 128;
        ascale[0] = sas[rbase];
        ascale[1] = sas[rbase + 8];
      }

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

      if (!kOutE4m3 && ep.act != MIMO_ACT_GEGLU) {
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
              if constexpr (kBlockScale) {  // (the row scales are in the sum already)
                const float2 ws = *reinterpret_cast<const float2*>(sws + c * 32 + 8 * jj + q2);
                f0 = f0 * ws.x;
                f1 = f1 * ws.y;
              } else if constexpr (kE4m3) {
                const float2 ws = *reinterpret_cast<const float2*>(sws + c * 32 + 8 * jj + q2);
                f0 = f0 * ascale[h] * ws.x;
                f1 = f1 * ascale[h] * ws.y;
              }
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
      } else if constexpr (kOutE4m3) {
        // GEGLU -> e4m3 (BN = 256): the tile's 128 output columns are one scale block. Each row's 128 values lie in the
        // accumulators of one quad (32 per thread); they replace the value accumulators, then the row's amax is a
        // register max and two quad shuffles, ahead of any byte. Staging: the whole 16 KiB of sOut as 128 rows of one
        // 128-byte swizzle row each, one TMA store per tile.
        constexpr int HALF = BN / 2;
        static_assert(HALF == 128, "e4m3 GEGLU output: one 128-column scale block per tile");
        float amax[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < HALF / 8; ++j) {
          const int jg = j + HALF / 8;
          const float2 cv = *reinterpret_cast<const float2*>(sb + 8 * j + q2);
          const float2 cg = *reinterpret_cast<const float2*>(sb + HALF + 8 * j + q2);
          const float2 wv = *reinterpret_cast<const float2*>(sws + 8 * j + q2);
          const float2 wg = *reinterpret_cast<const float2*>(sws + HALF + 8 * j + q2);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float v0 = acc[4 * j + 2 * h] * ascale[h] * wv.x, v1 = acc[4 * j + 2 * h + 1] * ascale[h] * wv.y;
            const float g0 = acc[4 * jg + 2 * h] * ascale[h] * wg.x, g1 = acc[4 * jg + 2 * h + 1] * ascale[h] * wg.y;
            const float f0 = (v0 + cv.x) * gelu_erf_fast(g0 + cg.x);
            const float f1 = (v1 + cv.y) * gelu_erf_fast(g1 + cg.y);
            acc[4 * j + 2 * h] = f0;
            acc[4 * j + 2 * h + 1] = f1;
            amax[h] = fmaxf(amax[h], fmaxf(fabsf(f0), fabsf(f1)));
          }
        }
        float inv[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          amax[h] = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 1));
          amax[h] = fmaxf(amax[h], __shfl_xor_sync(0xffffffffu, amax[h], 2));
          inv[h] = amax[h] == 0.f ? 1.f : 448.0f / amax[h];
          if ((lane & 3) == 0 && row_ok[h])
            out_scale[static_cast<long long>(n_tile) * ld_scale + row[h]] = amax[h] == 0.f ? 1.f : amax[h] / 448.0f;
        }
        // the previous tile's store has finished reading sOut before anyone writes it
        if (issuer) tma_store_wait_read0();
        asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
        for (int j = 0; j < HALF / 8; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = rbase + 8 * h;
            uint16_t q;
            asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;"
                : "=h"(q) : "f"(acc[4 * j + 2 * h + 1] * inv[h]), "f"(acc[4 * j + 2 * h] * inv[h]));
            *reinterpret_cast<uint16_t*>(sOut + r * 128 + (((j >> 1) ^ (r & 7)) << 4) + (j & 1) * 8 + q2) = q;
          }
        }
        stage_and_store(sOut, n_tile * HALF);
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
              if constexpr (kE4m3) {
                const float2 wv = *reinterpret_cast<const float2*>(sws + c * 32 + 8 * jj + q2);
                const float2 wg = *reinterpret_cast<const float2*>(sws + HALF + c * 32 + 8 * jj + q2);
                const float v0 = acc[4 * j + 2 * h] * ascale[h] * wv.x, v1 = acc[4 * j + 2 * h + 1] * ascale[h] * wv.y;
                const float g0 = acc[4 * jg + 2 * h] * ascale[h] * wg.x, g1 = acc[4 * jg + 2 * h + 1] * ascale[h] * wg.y;
                const float f0 = (v0 + cv.x) * gelu_erf_fast(g0 + cg.x);
                const float f1 = (v1 + cv.y) * gelu_erf_fast(g1 + cg.y);
                *reinterpret_cast<uint32_t*>(obuf + r * 64 + ((jj ^ sw[h]) << 4) + q2 * 2) = C::pack(f0, f1);
              } else {
                const float f0 = (acc[4 * j + 2 * h] + cv.x) * gelu_erf_fast(acc[4 * jg + 2 * h] + cg.x);
                const float f1 = (acc[4 * j + 2 * h + 1] + cv.y) * gelu_erf_fast(acc[4 * jg + 2 * h + 1] + cg.y);
                *reinterpret_cast<uint32_t*>(obuf + r * 64 + ((jj ^ sw[h]) << 4) + q2 * 2) = C::pack(f0, f1);
              }
            }
          }
          stage_and_store(obuf, n_tile * HALF + c * 32);
        }
      }
    }
    if (issuer) tma_store_wait_all();
  }
