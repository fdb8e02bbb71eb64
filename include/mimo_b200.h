/* mimo_b200 — C ABI of the H100 (sm_90a) denoising-engine kernels.
 *
 * The reference (menyifang/MIMO) has no FFI layer: every op on its hot path is a PyTorch library call made
 * from src/models/*.py. Each entry point below replaces one of those call sites (cited per function as
 * reference file:line) and is what a ctypes binding in the reference's modules would call; see INTEGRATION.md.
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer unless stated; tensors are dense,
 *    "channels-last": activations are [rows, C] with rows = (frame-sample, y, x) flattened, C contiguous.
 *  - `stream` is a cudaStream_t (CUstream) passed as void*; kernels are enqueued, never synchronised, never
 *    allocate: all entry points are CUDA-graph capturable.
 *  - dtype: 0 = fp16, 1 = bf16 storage; accumulation and all epilogue math are fp32.
 *  - return 0 on success, negative on error; mimo_last_error() gives the thread-local message.
 *  - there is no CPU fallback: on a machine without an sm_90 device every compute entry point fails.
 */
#ifndef MIMO_B200_H_
#define MIMO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MIMO_OK 0
#define MIMO_ERR_ARG (-1)
#define MIMO_ERR_CUDA (-2)
#define MIMO_ERR_DEVICE (-3)

#define MIMO_F16 0
#define MIMO_BF16 1

#define MIMO_ACT_NONE 0
#define MIMO_ACT_SILU 1
/* GEGLU: weight rows are packed per output tile as [value rows | gate rows]; out has N/2 columns.
 * Packing granule (rows of value, then rows of gate) is returned by mimo_gemm_geglu_granule(). */
#define MIMO_ACT_GEGLU 2

const char* mimo_version(void);
const char* mimo_last_error(void);
/* 0 if device `dev` is sm_90; MIMO_ERR_DEVICE otherwise (also when there is no CUDA device at all). */
int mimo_device_check(int dev);
/* sizeof() of the parameter structs as compiled into the library (0 epilogue, 1 gemm, 2 conv3x3, 3 groupnorm,
 * 4 attn, 5 attn_temporal, 6 exchange, 7 cfg_multistep, 8 groupnorm_window, 9 gemm_e4m3, 10 groupnorm_e4m3,
 * 11 conv3x3_e4m3, 12 gemm_e4m3_geglu_e4m3, 13 gemm_e4m3_blockscaled, 14 cfg_rescale): lets a binding verify its struct
 * mirrors before the first call. */
int mimo_abi_sizeof(int which);

/* Fused epilogue shared by GEMM and conv:  out = act((acc + bias[c] + rowvec[row / rows_per_group][c]
 *                                                      + residual[row][c]) * scale)                      */
typedef struct {
  const void* bias;       /* [N] or NULL                                                              */
  const void* rowvec;     /* [ceil(M / rows_per_group), ld_rowvec] or NULL (time embedding / folded cross-attn) */
  int64_t rows_per_group; /* rows sharing one rowvec row (f*H*W for per-CFG-branch vectors)            */
  int64_t ld_rowvec;      /* row stride of rowvec in elements (0 = N)                                  */
  const void* residual;   /* [M, ld_res] or NULL                                                      */
  int64_t ld_res;
  float scale; /* 1 / output_scale_factor                                                  */
  int act;     /* MIMO_ACT_*                                                               */
} mimo_epilogue;

/* out[M,N] = epilogue(A[M,K] . W[N,K]^T).  wgmma GEMM, TMA-fed, fp32 accumulate in registers.
 * Replaces: torch.nn.Linear / 1x1 Conv2d call sites — to_q/k/v/to_out (diffusers Attention, constructed at
 * src/models/attention.py:321-345, src/models/motion_module.py:282-292), FeedForward/GEGLU
 * (src/models/attention.py:359, motion_module.py:235), proj_in/proj_out (src/models/transformer_3d.py:64-66,
 * 93-95; motion_module.py:122,144), conv_shortcut (src/models/resnet.py:213-215), time_emb_proj (resnet.py:179).
 * Requirements: K % 8 == 0, lda/ldw % 8 == 0, N % 8 == 0, 16-byte aligned bases. */
typedef struct {
  const void* a;
  int64_t lda;
  const void* a1; /* optional second A source: A = [a | a1] along K (virtual concat), or NULL */
  int64_t lda1;
  const void* w;
  int64_t ldw;
  void* out;
  int64_t ldo;
  int32_t M, N, K; /* K = columns of `a`   */
  int32_t K1;      /* columns of `a1` (0 if a1 == NULL); w is [N, K + K1] */
  int32_t dtype;
  mimo_epilogue ep;
  /* optional scratch (device, 16-byte aligned, contents irrelevant, may be shared by all calls of a stream): lets small-M /
   * long-K problems split the K loop over several CTAs (fp32 partials, summed in a fixed order by a second kernel:
   * deterministic). NULL = never split. (Disabled by default inside the library - see
   * csrc/gemm_wgmma.cu.) */
  void* workspace;
  int64_t workspace_bytes;
} mimo_gemm_params;
int mimo_gemm(const mimo_gemm_params* p, void* stream);
/* number of value rows (== gate rows) per packed GEGLU tile for a packed width N (N = 2 * out features) */
int mimo_gemm_geglu_granule(int32_t N);

/* FP8 form of mimo_gemm for projections fed by mimo_layernorm_e4m3:
 *   out[M,N] = epilogue((A[M,K] . W[N,K]^T)[m][n] * a_scale[m] * w_scale[n])
 * A and W are e4m3 (OCP E4M3FN, one byte per element, both K-major), a_scale / w_scale fp32; accumulation in fp32. The
 * product with the two scales is taken in fp32 in that order, then the mimo_epilogue chain runs as in mimo_gemm (bias,
 * residual, act NONE or GEGLU, scale); out, bias, rowvec and residual are `dtype` (fp16 / bf16).
 * Replaces, when the caller opts into FP8: the q|k|v projection after norm1 (src/models/attention.py:329-345 ->
 * mutual_self_attention.py:154-197), the GEGLU up-projection after norm3 (attention.py:359-360), and the motion module's
 * q|k|v after its norms + PE (motion_module.py:230, 277-292) and its GEGLU after ff_norm (motion_module.py:235-236).
 * Requirements: GEMM rows only (no second A source, no split-K: workspace must be NULL), K % 16 == 0, lda / ldw % 16 == 0
 * (bytes), N % 8 == 0, ldo % 8 == 0, 16-byte aligned a / w / out / residual, non-NULL scales; GEGLU needs N % 256 == 0. */
typedef struct {
  const void* a;        /* [M, lda] e4m3 */
  int64_t lda;
  const float* a_scale; /* [M] */
  const void* w;        /* [N, ldw] e4m3 (GEGLU: packed as for mimo_gemm) */
  int64_t ldw;
  const float* w_scale; /* [N] */
  void* out;
  int64_t ldo;
  int32_t M, N, K;
  int32_t dtype; /* of out / bias / rowvec / residual */
  mimo_epilogue ep;
  void* workspace; /* must be NULL (split-K is not supported in e4m3) */
  int64_t workspace_bytes;
} mimo_gemm_e4m3_params;
int mimo_gemm_e4m3(const mimo_gemm_e4m3_params* p, void* stream);

/* mimo_gemm_e4m3 with act = GEGLU whose output is e4m3 with one fp32 scale per (row, 128-column block): the A operand of
 * mimo_gemm_e4m3_blockscaled. With v the fp32 GEGLU values of a row's block - (acc * a_scale * w_scale + bias) of the value
 * column times gelu of the gate column's, exactly as mimo_gemm_e4m3 computes them, without a rounding to 16 bits:
 *   amax = max |v|;  inv = 448 / amax, out_scale[block][row] = amax / 448 (IEEE divisions);  out = cvt.rn.satfinite.e4m3(v * inv)
 * and inv = out_scale = 1 when amax == 0: the per-row rule of mimo_layernorm_e4m3, applied to each 128-column block. One
 * GEGLU tile (256 packed weight rows) writes exactly one block of each of its rows, so the block's amax is known before
 * any of its bytes is written. out_scale is block-major, [N / 256][ld_scale]: a tile's 128 scales are one contiguous run.
 * Replaces, when the caller opts into the FP8 feed-forward output projection, the GEGLU of diffusers' FeedForward
 * (src/models/attention.py:359-360, motion_module.py:235-236) ahead of mimo_gemm_e4m3_blockscaled.
 * Requirements as mimo_gemm_e4m3 with GEGLU and a bias, and N % 256 == 0 (the 256-wide tile, weights packed with
 * mimo_gemm_geglu_granule(N) == 128), ldo % 16 == 0 (bytes), ld_scale >= M and ld_scale % 4 == 0, no residual, no row
 * vector, scale 1. */
typedef struct {
  const void* a;        /* [M, lda] e4m3 */
  int64_t lda;
  const float* a_scale; /* [M] */
  const void* w;        /* [N, ldw] e4m3, GEGLU-packed */
  int64_t ldw;
  const float* w_scale; /* [N] */
  const void* bias;     /* [N] `dtype`, GEGLU-packed */
  void* out;            /* [M, ldo] e4m3, N / 2 columns */
  int64_t ldo;
  float* out_scale;     /* [N / 256, ld_scale] */
  int64_t ld_scale;
  int32_t M, N, K;
  int32_t dtype; /* of bias */
} mimo_gemm_e4m3_geglu_e4m3_params;
int mimo_gemm_e4m3_geglu_e4m3(const mimo_gemm_e4m3_geglu_e4m3_params* p, void* stream);

/* e4m3 GEMM with one fp32 scale per (row of A, 128-element K block) - fine-grained activation scaling - and one per
 * output channel of W:
 *   out[M,N] = epilogue((sum_kb a_scale[kb][m] * (A_kb . W_kb^T)[m][n]) * w_scale[n])
 * Each K block's partial product is accumulated in fp32 on its own and added, times its row scale, into the fp32 sum
 * (blocks in order, one fma each); w_scale is taken where the epilogue first reads the sum, then the mimo_epilogue chain
 * runs as in mimo_gemm (bias, rowvec, residual, act NONE or SILU, scale); out, bias, rowvec and residual are `dtype`.
 * Replaces, when the caller opts into the FP8 feed-forward output projection, FeedForward's ff.net.2 Linear(4C, C)
 * (src/models/attention.py:359-360, motion_module.py:235-236), fed by mimo_gemm_e4m3_geglu_e4m3.
 * Requirements: K % 128 == 0, lda / ldw % 16 == 0 (bytes), N % 8 == 0, ldo % 8 == 0, 16-byte aligned a / w / out /
 * residual, non-NULL scales, a_scale [K / 128][ld_scale] with ld_scale >= M and ld_scale % 4 == 0, no GEGLU, no split-K
 * (workspace must be NULL). */
typedef struct {
  const void* a;        /* [M, lda] e4m3 */
  int64_t lda;
  const float* a_scale; /* [K / 128, ld_scale] */
  int64_t ld_scale;
  const void* w;        /* [N, ldw] e4m3 */
  int64_t ldw;
  const float* w_scale; /* [N] */
  void* out;
  int64_t ldo;
  int32_t M, N, K;
  int32_t dtype; /* of out / bias / rowvec / residual */
  mimo_epilogue ep;
  void* workspace; /* must be NULL */
  int64_t workspace_bytes;
} mimo_gemm_e4m3_blockscaled_params;
int mimo_gemm_e4m3_blockscaled(const mimo_gemm_e4m3_blockscaled_params* p, void* stream);

/* 3x3 / stride 1 / pad 1 convolution as implicit GEMM: the A operand is fetched tap by tap with 4-D TMA boxes
 * over the NHWC input (out-of-bounds = zero padding), optionally from two tensors (virtual channel concat).
 * Weights packed [Cout, 9 * (c0 + c1)], K index = tap * (c0 + c1) + channel, tap = ky * 3 + kx.
 * Replaces: InflatedConv3d.forward (src/models/resnet.py:9-17) inside ResnetBlock3D (resnet.py:217-247), conv_in /
 * conv_out (src/models/unet_3d_edit_bkfill.py:89-91, 249-251), Upsample3D's conv (resnet.py:88), and the
 * torch.cat([h, skip]) feeding up-block ResBlocks (src/models/unet_3d_blocks.py:697, 827).
 * Requirements: c0 % 8 == 0, c1 % 8 == 0, cout % 8 == 0. */
typedef struct {
  const void* x0;
  int32_t c0;
  const void* x1; /* NULL if single source */
  int32_t c1;
  const void* w;
  void* out;
  int64_t ldo;
  int32_t n, h, w_, cout;
  int32_t dtype;
  mimo_epilogue ep;
  void* workspace; /* as in mimo_gemm_params */
  int64_t workspace_bytes;
} mimo_conv3x3_params;
int mimo_conv3x3(const mimo_conv3x3_params* p, void* stream);
/* Upsample3D (src/models/resnet.py:53-90): nearest x2 (H, W) followed by the 3x3 / pad 1 conv, WITHOUT materialising
 * the upsampled tensor. x0 is the [n, h, w, c0] source, out the [n, 2h, 2w, cout] result (row stride ldo). Output pixel
 * (2y+a, 2x+b) only sees source rows {y-1+a, y+a} and columns {x-1+b, x+b}: four 2x2-tap implicit-GEMM convolutions (one
 * per parity class) whose weights are the sums of the 3x3 taps that land on the same source pixel - 4/9 of the FLOPs.
 * w: [4 classes (2a+b)][cout, 4 * c0], K index = (2*iy + ix) * c0 + channel, packed by the host
 * (mimo_b200.ops.pack_conv_up2x_weight). Epilogue: bias / scale / SiLU only. */
int mimo_conv_up2x(const mimo_conv3x3_params* p, void* stream);

/* FP8 form of mimo_conv3x3 for convolutions fed by mimo_groupnorm_e4m3:
 *   out[n, y, x, o] = epilogue((sum_{tap, c} X[n, y + dy, x + dx, c] * W[o, tap * c_in + c]) * x_scale[n] * w_scale[o])
 * X and W are e4m3 (OCP E4M3FN), x_scale one fp32 scale per image (a tap never leaves its image, and padding is zero, so
 * the scale factors out of every output pixel's sum), w_scale one per output channel; accumulation in fp32. The product
 * with the two scales is taken in fp32 in that order, then the mimo_epilogue chain runs as in mimo_conv3x3 (bias, rowvec,
 * residual, act NONE or SILU, scale); out, bias, rowvec and residual are `dtype` (fp16 / bf16).
 * Replaces, when the caller opts into FP8 convolutions, ResnetBlock3D's conv1 and conv2 (InflatedConv3d,
 * src/models/resnet.py:9-17, called at resnet.py:222 and :239). Single source (mimo_groupnorm_e4m3 writes the up blocks'
 * channel concat). Requirements: c_in % 16 == 0, cout % 8 == 0, ldo % 8 == 0, 16-byte aligned x / w / out / residual,
 * non-NULL scales, no GEGLU, no split-K (workspace must be NULL). */
typedef struct {
  const void* x;        /* [n, h, w_, c_in] e4m3 */
  const float* x_scale; /* [n] */
  int32_t c_in;
  const void* w;        /* [cout, 9 * c_in] e4m3, K index = tap * c_in + channel as in mimo_conv3x3 */
  const float* w_scale; /* [cout] */
  void* out;
  int64_t ldo;
  int32_t n, h, w_, cout;
  int32_t dtype; /* of out / bias / rowvec / residual */
  mimo_epilogue ep;
  void* workspace; /* must be NULL */
  int64_t workspace_bytes;
} mimo_conv3x3_e4m3_params;
int mimo_conv3x3_e4m3(const mimo_conv3x3_e4m3_params* p, void* stream);

/* im2col gather for the convolutions the TMA path does not cover (stride 2, nearest-x2 upsampled input):
 * col[(n,oy,ox), tap*c + ch] = x[n, (oy*stride-1+ky) >> up, (ox*stride-1+kx) >> up, ch], zero outside.
 * Replaces: Downsample3D (src/models/resnet.py:112-120), F.interpolate in Upsample3D (resnet.py:70-73),
 * PoseGuider's stride-2 convs (src/models/pose_guider.py:31-36). */
int mimo_im2col3x3(const void* x, void* col, int32_t n, int32_t h, int32_t w, int32_t c, int32_t stride,
                   int32_t upshift, int32_t pad_lo, int64_t ldcol, int32_t dtype, void* stream);

/* GroupNorm over channels-last activations, optional SiLU, optional two-source virtual concat. Deterministic: a
 * statistics pass publishes per-slab partial sums, the normalisation pass adds them in a fixed order (no floating-point
 * atomics; bit-identical run to run). stats: workspace of mimo_groupnorm_workspace_bytes(p) bytes, 16-byte aligned,
 * contents irrelevant. Replaces InflatedGroupNorm / nn.GroupNorm + F.silu
 * (src/models/resnet.py:20-28, 220-221, 231, 237; transformer_3d.py:58-60,124; motion_module.py:119-121,156). */
typedef struct {
  const void* x0;
  int32_t c0;
  const void* x1;
  int32_t c1;
  const void* gamma;
  const void* beta; /* [c0 + c1] */
  void* out;        /* [n, hw, c0 + c1] */
  float* stats;
  int32_t n, hw, groups;
  float eps;
  int32_t silu;
  int32_t dtype;
} mimo_groupnorm_params;
int mimo_groupnorm(const mimo_groupnorm_params* p, void* stream);
/* bytes of `stats` workspace mimo_groupnorm needs for these sizes (pointers in *p are ignored); < 0 on bad sizes */
int64_t mimo_groupnorm_workspace_bytes(const mimo_groupnorm_params* p);

/* GroupNorm with statistics over a whole window of frames: torch.nn.GroupNorm applied to [b, C, f, h, w], which the
 * reference builds for ResnetBlock3D norm1 / norm2 and conv_norm_out when use_inflated_groupnorm is False
 * (src/models/resnet.py:155-163, 185-192; unet_3d_edit_bkfill.py:236-247). x is [samples, frames, hw, c0 (+ c1)]
 * channels-last (image = sample * frames + frame); every sample gets one mean / variance per group over all frames.
 * Deterministic and shard-invariant: a statistics pass writes a partial table with one record per (frame, sample),
 * frame-major, so the tables of consecutive frame slices (e.g. the ranks of a frame-sharded window) concatenate into the
 * table of the whole window; the normalisation pass adds the records in an order fixed by frame and slab index only.
 *   mimo_groupnorm_window          both passes on x (x holds the whole window: table_frames is ignored)
 *   mimo_groupnorm_window_partials writes the `frames` records of x's frames into table (gamma/beta/out/stats unused)
 *   mimo_groupnorm_window_apply    normalises x's frames from a table of table_frames >= frames records
 * Same channel rules and SiLU / two-source concat as mimo_groupnorm. All three are graph-capturable. */
typedef struct {
  const void* x0;
  int32_t c0;
  const void* x1; /* NULL if single source */
  int32_t c1;
  const void* gamma;
  const void* beta;    /* [c0 + c1] */
  void* out;           /* [samples, frames, hw, c0 + c1] */
  float* table;        /* partial table, 16-byte aligned */
  int64_t table_bytes; /* size of `table`: >= mimo_groupnorm_window_table_bytes per frames it holds */
  float* stats;        /* scratch of samples * groups * 2 floats (apply / one call), contents irrelevant */
  int32_t samples, frames, table_frames, hw, groups;
  float eps;
  int32_t silu;
  int32_t dtype;
} mimo_groupnorm_window_params;
int mimo_groupnorm_window(const mimo_groupnorm_window_params* p, void* stream);
int mimo_groupnorm_window_partials(const mimo_groupnorm_window_params* p, void* stream);
int mimo_groupnorm_window_apply(const mimo_groupnorm_window_params* p, void* stream);
/* bytes of the partial table of x's `frames` frames (pointers and table_frames ignored); < 0 on bad sizes. The table of
 * a window sharded into G equal frame slices is G times the slice's. */
int64_t mimo_groupnorm_window_table_bytes(const mimo_groupnorm_window_params* p);

/* GroupNorm + SiLU with an e4m3 output and one fp32 scale per image: the A operand of mimo_conv3x3_e4m3.
 * Replaces, when the caller opts into FP8 convolutions, ResnetBlock3D's norm1 / norm2 + SiLU ahead of conv1 / conv2
 * (src/models/resnet.py:217-240; InflatedGroupNorm resnet.py:20-28, or nn.GroupNorm over the window, resnet.py:155-163).
 * The scale is an upper bound on the image's amax, built before any output is written. For image i and group g, with
 * lo_g / hi_g the min / max of x over the image's elements of the group, mean_g / rstd_g the normaliser's statistics
 * (the image's own, or the sample's window statistics), and for each channel c of g
 *   z_lo = (lo_g - mean_g) * (rstd_g * gamma_c) + beta_c,  z_hi likewise with hi_g  (one fma each, as the normaliser)
 *   B_c = max(|silu(z_lo)|, |silu(z_hi)|, and 0.27846454 when [min(z_lo, z_hi), max(z_lo, z_hi)] holds -1.2784645)
 *   amax_i = max_c B_c;  scale[i] = amax_i / 448,  out = cvt.rn.satfinite.e4m3(silu(y) * (448 / amax_i))  (IEEE divisions)
 * and scale[i] = 1, multiplier 1 when amax_i == 0. SiLU's only turning point is its minimum at -1.2784645, so B_c bounds
 * |silu| over [z_lo, z_hi]: nothing saturates except by rounding. mimo_b200.ops.e4m3_image_scales states the rule on the
 * host. x, gamma, beta are `dtype`; out is [samples * frames, hw, c0 + c1] bytes (image = sample * frames + frame).
 * Modes (the window modes keep mimo_groupnorm_window's partial table and its format; min / max never enter the table, so
 * a frame-sharded window exchanges exactly what the 16-bit GroupNorm exchanges):
 *   MIMO_GN_E4M3_FRAME          statistics per image (`table` unused)
 *   MIMO_GN_E4M3_WINDOW         statistics per sample over its `frames` frames, both passes (table of `frames` records)
 *   MIMO_GN_E4M3_WINDOW_PARTIALS the `frames` records of x's frames into `table`, the min / max into `work`
 *   MIMO_GN_E4M3_WINDOW_APPLY   normalise x's frames from a table of table_frames >= frames records, with the min / max
 *                               the partials call left in `work`
 * work: scratch of mimo_groupnorm_e4m3_workspace_bytes(p) bytes, 16-byte aligned (kept between PARTIALS and APPLY).
 * Requirements: as mimo_groupnorm_window; silu is implied. All modes are graph-capturable. */
#define MIMO_GN_E4M3_FRAME 0
#define MIMO_GN_E4M3_WINDOW 1
#define MIMO_GN_E4M3_WINDOW_PARTIALS 2
#define MIMO_GN_E4M3_WINDOW_APPLY 3
typedef struct {
  const void* x0;
  int32_t c0;
  const void* x1; /* NULL if single source */
  int32_t c1;
  const void* gamma;
  const void* beta;    /* [c0 + c1] */
  void* out;           /* [samples * frames, hw, c0 + c1] e4m3 */
  float* scale;        /* [samples * frames] */
  float* work;
  int64_t work_bytes;
  float* table;        /* window modes: partial table as in mimo_groupnorm_window */
  int64_t table_bytes;
  int32_t mode;
  int32_t samples, frames, table_frames, hw, groups;
  float eps;
  int32_t dtype;
} mimo_groupnorm_e4m3_params;
int mimo_groupnorm_e4m3(const mimo_groupnorm_e4m3_params* p, void* stream);
/* bytes of `work` for these sizes and mode (pointers ignored); < 0 on bad sizes */
int64_t mimo_groupnorm_e4m3_workspace_bytes(const mimo_groupnorm_e4m3_params* p);

/* LayerNorm over the last dim; optional additive per-frame vector AFTER the affine (the motion module's
 * sinusoidal positional encoding): out[r] = LN(x[r]) * gamma + beta + pe[pe_frame_offset + (r / rows_per_frame) % frames]
 * (pe_frame_offset = first global frame of this rank's shard).
 * Replaces nn.LayerNorm (src/models/attention.py:329-360; motion_module.py:230,236) and PositionalEncoding.forward
 * (motion_module.py:277-279). */
int mimo_layernorm(const void* x, const void* gamma, const void* beta, void* out, int64_t rows, int32_t c,
                   float eps, const void* pe, int64_t rows_per_frame, int32_t frames, int32_t pe_frame_offset,
                   int32_t dtype, void* stream);
/* mimo_layernorm with an e4m3 output and one fp32 scale per row: the A operand of mimo_gemm_e4m3. With y the row's fp32
 * LN(+PE) values (with a PE, LN's output is rounded to `dtype` before the encoding is added, as in mimo_layernorm):
 *   amax = max |y|;  inv = 448 / amax, scale[r] = amax / 448 (IEEE divisions);  out[r] = cvt.rn.satfinite.e4m3(y * inv)
 * and inv = scale[r] = 1 when amax == 0. out is [rows, c] bytes, scale [rows] fp32; x, gamma, beta, pe are `dtype`.
 * Replaces, when the caller opts into FP8, the nn.LayerNorm (+ PositionalEncoding) call sites ahead of mimo_gemm_e4m3's
 * projections (attention.py:329-360; motion_module.py:230, 236, 277-279). Requirements as mimo_layernorm, and c % 16 == 0. */
int mimo_layernorm_e4m3(const void* x, const void* gamma, const void* beta, void* out, float* scale, int64_t rows,
                        int32_t c, float eps, const void* pe, int64_t rows_per_frame, int32_t frames,
                        int32_t pe_frame_offset, int32_t dtype, void* stream);

/* Spatial self-attention with the reference-image bank (flash attention, wgmma QK^T and PV, online softmax).
 * q/k/v: [n, lq, heads, d] slices of a fused QKV buffer (row stride ld_qkv elements). bank_k/bank_v:
 * [nb, lb, heads, d] with row stride ld_bank; frame-sample i attends to [self keys | bank keys of branch
 * bank_index[i]] when bank_index[i] >= 0, and to self keys only when bank_index[i] < 0 (the unconditional half).
 * Replaces hacked_basic_transformer_inner_forward's attn1 calls (src/models/mutual_self_attention.py:154-197)
 * -> diffusers Attention/AttnProcessor2_0 -> F.scaled_dot_product_attention. */
typedef struct {
  const void* q;
  const void* k;
  const void* v;
  int64_t ld_qkv;
  const void* bank_k;
  const void* bank_v;
  int64_t ld_bank;
  int32_t lb;                /* bank tokens per feature map */
  int32_t nb;                /* number of bank feature maps (CFG branches written by the reference UNet) */
  const int32_t* bank_index; /* DEVICE [n], values in [-1, nb), or NULL (= no bank) */
  void* out;
  int64_t ld_out;
  int32_t n, lq, heads, d;
  float scale;
  int32_t dtype;
} mimo_attn_params;
int mimo_attn_spatial(const mimo_attn_params* p, void* stream);

/* Temporal self-attention of the motion module: for every (batch b, pixel p, head) a q_frames x kv_frames attention
 * over the frame axis. Query rows are ordered ((b * q_frames + f) * hw + p). Keys/values cover all kv_frames frames
 * and may live in several chunks of frames_per_chunk frames (the per-rank buffers of a frame-sharded clip after the
 * all-gather): kv_row(b, f, p) = (f / frames_per_chunk) * chunk_stride_rows + (b * frames_per_chunk + f %
 * frames_per_chunk) * hw + p. Single GPU: q_frames == kv_frames == frames_per_chunk, chunk_stride_rows = 0.
 * Replaces VersatileAttention.forward (src/models/motion_module.py:353-390), including its two
 * "(b f) d c <-> (b d) f c" transposes. */
typedef struct {
  const void* q;
  int64_t ld_q;
  const void* k;
  const void* v;
  int64_t ld_kv;
  void* out;
  int64_t ld_out;
  int64_t chunk_stride_rows;
  int32_t batch, q_frames, kv_frames, frames_per_chunk;
  int32_t hw, heads, d;
  float scale;
  int32_t dtype;
} mimo_attn_temporal_params;
int mimo_attn_temporal(const mimo_attn_temporal_params* p, void* stream);

/* Frame-shard <-> pixel-shard exchange of the motion module over NVLink PEER MEMORY (one process per GPU, G GPUs in a
 * frame group, this GPU is member r). Each GPU pulls its share directly from its peers' source buffers (IPC-mapped
 * device pointers, see mimo_peer_*), synchronised by epoch flags in peer memory; no collective library and no host
 * work on the data path, CUDA-graph capturable. Tokens are channels-last rows of C elements.
 *   mode 0 (frames -> pixels): src on every peer is [b, fl, hw, C] (its fl frames of the window); dst becomes
 *           [b, G*fl, hw/G, C]: ALL frames of this GPU's pixel shard  (before VersatileAttention, motion_module.py:353-390)
 *   mode 1 (pixels -> frames): src on every peer is [b, G*fl, hw/G, C]; dst becomes [b, fl, hw, C] (+ residual, same
 *           layout as dst): the motion module's output for this GPU's frames (motion_module.py:181-183)
 *   mode 2 (all-gather): src on every peer is [b*fl*hw, C]; dst becomes [G, b*fl*hw, C]
 * peer_src[s] / peer_ready[s]: peer s's source buffer / its array of MIMO_MAX_PEERS uint32 flags (zero-initialised once),
 * as mapped into THIS process; index r is this GPU's own buffer / flags. ctl: two uint32 of local device memory,
 * initialised to {1, 0} once per group, never touched by the host afterwards. All members must issue the same sequence
 * of exchanges. A peer that does not show up within timeout_ms (0 = 30 s) traps the kernel. */
#define MIMO_MAX_PEERS 8
typedef struct {
  const void* peer_src[MIMO_MAX_PEERS];
  void* peer_ready[MIMO_MAX_PEERS];
  void* ctl;
  void* dst;
  const void* residual; /* mode 1 only, or NULL */
  int32_t mode, G, r;
  int32_t b, fl, hw, C;
  int32_t dtype;
  int32_t max_blocks; /* 0 = 2 per SM */
  int32_t timeout_ms;
} mimo_exchange_params;
int mimo_exchange(const mimo_exchange_params* p, void* stream);
/* Peer-shareable device memory for mimo_exchange: cudaMalloc'd, zero-filled, exported as a 64-byte CUDA IPC handle;
 * mimo_peer_open maps another process's buffer into this process for the CURRENT device (peer access is enabled on
 * first use). Bootstrap only (the handles travel over whatever the host uses, e.g. torch.distributed objects). */
int mimo_peer_alloc(int64_t bytes, void** ptr, void* handle64);
int mimo_peer_open(const void* handle64, void** ptr);
int mimo_peer_close(void* ptr);
int mimo_peer_free(void* ptr);

/* Elementwise / layout helpers (each one coalesced pass). */
/* [b, c, f, h, w] (reference layout) -> [(b f), h, w, cpad] channels-last, zero-padding channels c..cpad */
int mimo_ncfhw_to_nhwc(const void* src, void* dst, int32_t b, int32_t c, int32_t f, int32_t h, int32_t w,
                       int32_t cpad, int32_t src_is_f32, int32_t dtype, void* stream);
/* [(b f), h, w, ld] channels-last (first c channels) -> [b, c, f, h, w] */
int mimo_nhwc_to_ncfhw(const void* src, void* dst, int32_t b, int32_t c, int32_t f, int32_t h, int32_t w,
                       int32_t ld, int32_t dst_is_f32, int32_t dtype, void* stream);
/* nearest-neighbour x2 upsampling of [n, h, w, c] -> [n, 2h, 2w, c] (F.interpolate in Upsample3D, resnet.py:70-73) */
int mimo_upsample2x(const void* x, void* out, int32_t n, int32_t h, int32_t w, int32_t c, int32_t dtype, void* stream);
/* nearest-neighbour resize of [n, h, w, c] -> [n, oh, ow, c] to any size, bit-identical to F.interpolate(mode="nearest",
 * size=(oh, ow)): source row min(floor(oy * (float(h) / oh)), h - 1) in fp32, columns alike. Replaces the forwarded-size
 * interpolation of Upsample3D / Upsample2D (src/models/resnet.py:75-77) that the UNets run when a latent side is not a
 * multiple of 8 (src/models/unet_3d_edit_bkfill.py:427-435, 544-545; unet_2d_condition.py:946-955, 1269-1270).
 * Requirements: c % 8 == 0, 16-byte aligned x and out. */
int mimo_upsample_nearest(const void* x, void* out, int32_t n, int32_t h, int32_t w, int32_t oh, int32_t ow, int32_t c,
                          int32_t dtype, void* stream);
/* in-place row softmax of x[rows, cols] (leading dim ld), fp32 math: the VAE mid-block attention (1 head, d=512) is
 * run as GEMM -> softmax -> GEMM (diffusers AttnProcessor2_0 on UNetMidBlock2D's Attention). */
int mimo_softmax_rows(void* x, int64_t rows, int32_t cols, int64_t ld, int32_t dtype, void* stream);
/* out = a + b (same shape, count elements) */
int mimo_add(const void* a, const void* b, void* out, int64_t count, int32_t dtype, void* stream);
/* out = silu(x) */
int mimo_silu(const void* x, void* out, int64_t count, int32_t dtype, void* stream);

/* out = x * sigmoid(1.702 x): CLIP's quick_gelu (transformers CLIPMLP [3P]; the image encoder of pipeline :378-385) */
int mimo_quick_gelu(const void* x, void* out, int64_t count, int32_t dtype, void* stream);

/* Scene compositing of run_edit.py:282-300, one frame, one pass (all images uint8 [H, W, 3] on the device):
 *   res = canvas * mask + bk * (1 - mask);  [res = res * (1 - occ/255) + vid * (occ/255)];  [out = prev * (1 - factor)
 *   + res * factor];  out -> uint8 by truncation. mask: float32 [H, W] feather mask placed on the full frame; occ: uint8
 *   [H, W] or NULL (then vid is NULL too); prev: the frame composited from the previous, overlapping clip or NULL.
 * Intermediate types follow numpy's promotion in the reference, so the bytes are identical. */
int mimo_composite_frame(const void* canvas, const void* bk, const float* mask, const void* occ, const void* vid,
                         const void* prev, double factor, void* out, int64_t pixels, void* stream);

/* Classifier-free guidance + DDIM (v-prediction, eta = 0) update, one pass:
 *   eps = (pred_u + g * (pred_c - pred_u)) / counter ; x0 = sa_t * x - s1a_t * v ; e = sa_t * v + s1a_t * x ;
 *   x_prev = sa_p * x0 + s1a_p * e.   latents/pred_* are [count]; math in fp32, stored in `dtype`.
 * Replaces pipeline_pose2vid_long_edit_bkfill_roiclip.py:545-553 (+ diffusers DDIMScheduler.step). */
int mimo_cfg_ddim_step(const void* pred_uncond, const void* pred_cond, const void* counter_or_null,
                       int64_t frame_stride, void* latents, int64_t count, float guidance, float sqrt_a_t,
                       float sqrt_1ma_t, float sqrt_a_prev, float sqrt_1ma_prev, int32_t dtype, void* stream);

/* mimo_cfg_ddim_step for stochastic DDIM (eta > 0): the same update with the direction coefficient passed in, plus
 * noise, as diffusers DDIMScheduler.step [3P] computes it with eta > 0:
 *   x_prev = sa_p * x0 + dir_coef * e + sigma * noise,   dir_coef = sqrt(1 - abar_prev - sigma^2),
 *   sigma = eta * sqrt((1 - abar_prev) / (1 - abar_t) * (1 - abar_t / abar_prev)).
 * noise is [count] in `dtype` (the caller's draw, randn_tensor(model_output.shape, generator)). Each product and sum is
 * rounded to `dtype` where the torch expression rounds it. Replaces pipeline :128-147, :421, :551-553 with eta > 0.
 * Requirements: sigma >= 0, dir_coef >= 0. */
int mimo_cfg_ddim_step_noise(const void* pred_uncond, const void* pred_cond, const void* counter_or_null,
                             int64_t frame_stride, void* latents, int64_t count, float guidance, float sqrt_a_t,
                             float sqrt_1ma_t, float sqrt_a_prev, float dir_coef, const void* noise, float sigma,
                             int32_t dtype, void* stream);

/* Classifier-free guidance + one step of a multistep / sigma-space solver (DPM-Solver++ orders 1-3, Euler,
 * Euler-ancestral; v-prediction), one pass. Per element, with v the guided prediction exactly as in mimo_cfg_ddim_step
 * (same roundings: the reference's torch ops at pipeline :545-549):
 *   m  = rnd(a * x + b * v)                                   the solver's model quantity, written to hist_out
 *   x' = c_x * x + c_m * m + c_1 * h1 + c_2 * h2 + c_n * noise  in fp32, rounded once at the store into latents
 * h1 / h2 are the m of the previous two steps. The host computes the eight scalars per step (host/scheduler.py:
 * multistep_coefficients). Replaces pipeline :519-521, :545-553 with a DPMSolverMultistepScheduler,
 * EulerDiscreteScheduler or EulerAncestralDiscreteScheduler [3P]. */
typedef struct {
  const void* pred_uncond; /* [count]                                                                      */
  const void* pred_cond;   /* [count]                                                                      */
  const void* counter;     /* [F] window count per frame (as mimo_cfg_ddim_step), or NULL                  */
  int64_t frame_stride;    /* h * w: latents are [1, 4, F, h, w]; needed with counter                      */
  void* latents;           /* [count], updated in place                                                    */
  int64_t count;
  void* hist_out;          /* [count] receives m; may alias h2 (each element is read before it is written)  */
  const void* h1;          /* [count] or NULL (then c_1 must be 0)                                         */
  const void* h2;          /* [count] or NULL (then c_2 must be 0)                                         */
  const void* noise;       /* [count] or NULL (then c_n must be 0)                                         */
  float guidance;
  float a, b;              /* m = a * x + b * v                                                            */
  float c_x, c_m, c_1, c_2, c_n;
  int32_t dtype;
} mimo_cfg_multistep_params;
/* Requirements: finite scalars; hist_out distinct from latents, pred_*, h1 and noise. Graph-capturable. */
int mimo_cfg_multistep(const mimo_cfg_multistep_params* p, void* stream);

/* Rescaled classifier-free guidance (Lin et al. 2023, arXiv 2305.08891 §3.4; diffusers rescale_noise_cfg [3P]) at the
 * point where diffusers' pipelines apply it in the reference's loop: after the guidance line, before the scheduler step
 * (pipeline_pose2vid_long_edit_bkfill_roiclip.py:545-553). With text = pred_cond / counter and cfg the guided prediction,
 * both computed exactly as mimo_cfg_ddim_step computes them:
 *   r   = rnd(rnd(std(text)) / rnd(std(cfg)))        std unbiased over all `count` elements (the whole clip); r = 1 when
 *                                                    rnd(std(cfg)) is 0 (diffusers would give NaN)
 *   out = rnd(rnd(phi * rnd(cfg * r)) + rnd((1 - phi) * cfg))   phi and 1 - phi in double, cast to fp32
 * rnd rounds to `dtype`, where PyTorch rounds that expression on 16-bit tensors. The sums behind the two std are fp64, one
 * fixed partial per CTA in `workspace`, added in a fixed order by a grid whose size depends on `count` only: repeated
 * calls, graph replays and every rank of a sharded run give the same bits. No host synchronisation; graph-capturable.
 * Two kernel launches. The scheduler step then runs on (out, out, guidance 1, no counter), which passes out through. */
typedef struct {
  const void* pred_uncond; /* [count]                                                                      */
  const void* pred_cond;   /* [count]                                                                      */
  const void* counter;     /* [F] window count per frame (as mimo_cfg_ddim_step), or NULL                  */
  int64_t frame_stride;    /* h * w: latents are [1, 4, F, h, w]; needed with counter                      */
  void* out;               /* [count] in `dtype`; distinct from every input                               */
  int64_t count;           /* >= 2                                                                         */
  void* workspace;         /* mimo_cfg_rescale_workspace_bytes(p) bytes, 16-byte aligned, contents irrelevant  */
  int64_t workspace_bytes;
  double phi;              /* guidance_rescale, in [0, 1]                                                  */
  float guidance;          /* finite                                                                       */
  int32_t dtype;
} mimo_cfg_rescale_params;
int mimo_cfg_rescale(const mimo_cfg_rescale_params* p, void* stream);
/* bytes of `workspace` mimo_cfg_rescale needs for p->count (pointers in *p are ignored); < 0 on a bad count */
int64_t mimo_cfg_rescale_workspace_bytes(const mimo_cfg_rescale_params* p);

/* Latent frame interpolation (pipeline interpolate_latents, :294-334, with the methods of src/pipelines/utils.py):
 * src [1, 4, F, h, w] -> dst [1, 4, (F-1)*k + 1, h, w] (hw = h * w): frame i goes to i*k, and k-1 frames
 * interp(v_i, v_{i+1}, j / k) fill the gap. method 0 = linear, (1 - t) * v0 + t * v1 rounded where PyTorch rounds it
 * (bit-identical to the torch expression on CUDA); method 1 = slerp: cos from fp32 sums over the pair's 4*hw elements in a
 * fixed order (deterministic), |cos| > 0.9995 -> linear, else fp32 great-circle formula rounded once. The branch is taken
 * on the device (graph-capturable). One CTA per frame pair. Requirements: F >= 2, k >= 2, src and dst distinct. */
int mimo_interpolate_frames(const void* src, void* dst, int32_t frames, int64_t hw, int32_t k, int32_t method,
                            int32_t dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MIMO_B200_H_ */
