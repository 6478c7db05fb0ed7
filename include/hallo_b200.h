/*
 * hallo_b200 -- C ABI of the sm_90a kernels behind the Hallo denoising hot path.
 *
 * The reference (fudan-generative-vision/hallo) has no FFI/operator layer of its own: its
 * hot path is Python classes over torch library calls (SURVEY.md section 8b).  This header is
 * therefore the boundary the build introduces (SURVEY.md 8b "B2"); every entry point names the
 * reference code whose arithmetic it replaces.
 *
 * Conventions
 *   - plain pointers + sizes, no torch types; every pointer is a DEVICE pointer unless noted;
 *   - the caller owns every buffer (inputs, outputs, workspaces); the library never allocates
 *     or frees device memory;
 *   - all activations are "channels-last token matrices": row = (frame, pixel), column = channel;
 *   - every call is asynchronous on `stream` and re-entrant; returns 0 on success or a
 *     negative hb_status; never throws;
 *   - dtype selects the storage / tensor-core input type (fp32 accumulate everywhere).
 */
#ifndef HALLO_B200_H_
#define HALLO_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* hb_stream_t; /* cudaStream_t */

enum hb_status {
  HB_OK = 0,
  HB_ERR_BAD_SHAPE = -1,   /* dimension not supported by the kernel (alignment, head dim ...) */
  HB_ERR_BAD_DTYPE = -2,
  HB_ERR_CUDA = -3,        /* a CUDA runtime / driver call failed; see hallo_b200_last_error() */
  HB_ERR_NULL = -4,
  HB_ERR_DEVICE_TRAP = -5  /* a kernel recorded a barrier timeout in the device error word */
};

enum hb_dtype { HB_F16 = 0, HB_BF16 = 1 };

/* ------------------------------------------------------------------------------------------
 * Library info
 * ---------------------------------------------------------------------------------------- */
int hallo_b200_abi_version(void);
/* sizeof(hb_gemm_params) / sizeof(hb_attention_params) as compiled into the library: a binding written in another
 * language asserts its own struct size against these before the first call (a short struct would be read past). */
int hallo_b200_sizeof_gemm_params(void);
int hallo_b200_sizeof_attention_params(void);
const char* hallo_b200_last_error(void);
/* Reads and clears the device-side error word written by a kernel that timed out on a barrier. */
int hallo_b200_device_error(unsigned int* code_out);
/* Number of kernel launches issued by this library since the last reset (bench.py gpu_launches). */
int64_t hallo_b200_launch_count(int reset);
/* Kernel-selection switches (A/B measurements; results are identical up to rounding whatever the setting).  Each
 * option starts from the environment variable HALLO_B200_<NAME> (upper case) or its default and can be changed at run
 * time; unknown names return HB_ERR_BAD_SHAPE / -1.
 *   "xattn_tc"    cross-attention on wgmma tensor cores (0: CUDA-core kernel)                        (default 1)
 *   "tattn_mma"   temporal attention on warp-level tensor-core MMAs (0: CUDA cores)                   (default 1)
 *   "gn_fused"    one-launch GroupNorm when a (frame, group) slab fits shared memory                  (default 1)
 *   "gemm_splitk" split the K loop of a GEMM / conv whose tiles fill less than half of the SMs over several CTAs
 *                 (fp32 partials in the caller's workspace, fixed summation order); 1 = for K >= 2048, a value
 *                 n > 1 = for K >= 64 n                                                                  (default 1)
 *   "pdl"         programmatic dependent launch: a kernel's prologue overlaps the tail of its predecessor     (default 0) */
int hallo_b200_set_option(const char* name, int value);
int hallo_b200_get_option(const char* name);

/* ------------------------------------------------------------------------------------------
 * hallo_b200_gemm -- C = epilogue(A * W^T) on wgmma tensor cores, TMA-fed, register accumulators.
 *
 * Replaces every nn.Linear / 1x1 conv / 3x3 conv on the path:
 *   to_q/to_k/to_v/to_out           diffusers Attention used at hallo/models/attention.py:479-503,
 *                                   703-761, hallo/models/motion_module.py:464-482
 *   FeedForward (GEGLU)             hallo/models/attention.py:517,777; motion_module.py:383
 *   proj_in / proj_out (1x1)        hallo/models/transformer_3d.py:197-203,236-251;
 *                                   hallo/models/motion_module.py:290-313
 *   zero_conv_{full,face,lip}       hallo/models/attention.py:854-890
 *   InflatedConv3d 3x3 (+shortcut)  hallo/models/resnet.py:50-66, 385-410, 166-183, 250
 *
 *   A  : [M, K] row-major (lda), optionally split along K into two sources (A for k < K1,
 *        A2 for k >= K1) -- the UNet skip-connection channel concat without a copy
 *        (hallo/models/unet_3d_blocks.py:1131,1373).
 *   W  : [N, K] row-major (torch Linear layout; conv weights packed [Cout][tap][Cin]).
 *   conv3x3 == 1: A is an NHWC image batch [img_n, img_h, img_w, Cin]; M = img_n*img_h*img_w,
 *        K = 9*Cin; stride 1, zero padding 1 (TMA out-of-bounds fill).
 *   conv3x3 == 2: stride-2 conv (Downsample3D, resnet.py:232-252).  A holds the 4 phase planes
 *        written by hallo_b200_phase_split: [4*img_n, img_h, img_w, Cin] where img_h/img_w are
 *        the OUTPUT height/width; M = img_n*img_h*img_w.
 *   conv3x3 == 3: stride-2 conv with zero padding (0, 1) on each axis -- diffusers Downsample2D(padding=0), the VAE
 *        encoder's downsampler: output o reads input rows 2o, 2o+1, 2o+2 (conv3x3 == 2 reads 2o-1 .. 2o+1).  Same
 *        phase-plane input and img_h / img_w (OUTPUT size) as conv3x3 == 2; the input height / width are 2 img_h /
 *        2 img_w, and the bottom / right pad comes from the TMA out-of-bounds fill.
 *        A conv takes bias / group_bias / row_scale / residual only (no activation, GEGLU, LayerNorm fold, stats_out).
 *   epilogue, in this order (each optional):
 *        v  = acc + bias[col] + group_bias[row / rows_per_group][col]
 *        v  = v_even * gelu_erf(v_odd)           (HB_EPI_GEGLU: W rows interleaved value/gate,
 *                                                 output has N/2 columns)
 *        v  = v * row_scale[row] * alpha + residual[row][col]
 *   Constraints: K % 64 == 0 (K1 % 64 == 0, Cin % 64 == 0); lda/ldw/ldc/ldr % 8 == 0.
 *   Tile: 128 x 160 output tiles, or 128 x 128 when N is a multiple of 128 but not of 160 (N = 128, 256, 512, 1536 ...:
 *        a 160-wide tile would leave up to 37.5 % of its MMA columns empty).  Chosen from N alone; no option.
 * ---------------------------------------------------------------------------------------- */
enum hb_epi_flags {
  HB_EPI_GEGLU = 1,
  HB_EPI_SILU = 2, /* v = silu(v) right after the bias adds */
  HB_EPI_RELU = 4  /* v = max(v, 0) right after the bias adds (AudioProjModel, hallo/models/audio_proj.py:117-119) */
};

typedef struct {
  int32_t dtype;
  int32_t M, N, K;
  const void* A;
  int64_t lda;
  const void* A2; /* NULL when unused */
  int64_t lda2;
  int32_t K1;
  const void* W;
  int64_t ldw;
  void* C;
  int64_t ldc;
  const void* bias;       /* [N] */
  const void* group_bias; /* [ceil(M/rows_per_group), ld_group_bias] */
  int64_t ld_group_bias;
  int32_t rows_per_group;
  const void* row_scale; /* [M] */
  const void* residual;  /* [M, ldr] */
  int64_t ldr;
  float alpha;
  int32_t flags;
  int32_t conv3x3;
  int32_t img_n, img_h, img_w;
  /* LayerNorm folded into the GEMM (nn.LayerNorm -> nn.Linear chains of attention.py / motion_module.py):
   *   LN(x) W^T = rstd_r * (x (W diag(gamma))^T - mu_r * colsum_n) + (W beta + b)_n
   * W must already hold W*diag(gamma), bias W*beta + b.  ln_stats: fp32 [M,2] = (sum, sum of squares) of each A row,
   * accumulated by the producing GEMM through stats_out; ln_colsum: fp32 [N] row sums of the packed W.  NULL = off. */
  const float* ln_stats;
  const float* ln_colsum;
  float ln_eps;
  /* fp32 [M,2]: atomically accumulates (sum, sum of squares) of every output row over the stored columns (zeroed by
   * the caller) -- feeds the next folded LayerNorm.  NULL = off. */
  float* stats_out;
  /* Output-row scatter (multi-GPU, see "Peer memory" below): NULL = rows go to C + row*ldc.  Direct-store epilogue
   * only; residual must be NULL. */
  const struct hb_row_scatter* scatter;
  /* Split-K scratch (option "gemm_splitk"): device memory owned by the caller, zero-filled once, never shared by two
   * GEMMs that may run concurrently (one per engine / stream).  When the tiles of a launch cover less than half of
   * the SMs and K >= 2048, the K loop is divided over several CTAs per tile; CTAs 1.. write fp32 partial tiles here
   * and CTA 0 adds them in split order (deterministic) before its epilogue.  hallo_b200_gemm_workspace_bytes() is
   * the size that never limits the split; a smaller buffer lowers the split count, NULL / 0 turns it off. */
  void* workspace;
  long long workspace_bytes;
} hb_gemm_params;

/* Output row r of the GEMM is split as s = r / seg, q = r % seg, d = s / segs_per_dest, i = s % segs_per_dest and
 * stored at  base[d] + ((i * seg_stride + row0 + q) * ldc + col) elements  -- base[d] is a buffer of destination rank
 * d (peer-mapped with hallo_b200_peer_open, or local).  Used by the motion module's proj_out (motion_module.py:312)
 * of a frame-sharded window: the GEMM runs on (all frames x this rank's pixel slice) and its epilogue writes every
 * (frame, pixel) row straight into the frame owner's buffer over NVLink -- the transfer IS the epilogue's store. */
typedef struct hb_row_scatter {
  void* base[16];
  int32_t seg;
  int32_t segs_per_dest;
  int64_t seg_stride;
  int64_t row0;
} hb_row_scatter;

int hallo_b200_gemm(const hb_gemm_params* p, hb_stream_t stream);
long long hallo_b200_gemm_workspace_bytes(void);
/* split factor the most recent hallo_b200_gemm call of this process used (1 = unsplit): tests / diagnostics */
int hallo_b200_gemm_last_splits(void);
/* The split-K decision itself (host arithmetic, no device needed): `tiles` output tiles of 128 x bn on `sm_units` SMs
 * (hallo_b200_gemm passes the device's SM count, cta_group 1 and the tile width it picked, 160 or 128), reduction length K, the caller's workspace
 * size and the value of option
 * "gemm_splitk" (0 = off, 1 = default threshold K >= 2048, n > 1 = K >= 64 n).  Returns the split factor, 1 = unsplit. */
int hallo_b200_gemm_choose_splits(int tiles, int sm_units, int K, int cta_group, int bn, long long workspace_bytes,
                                  int option_value);

/* ------------------------------------------------------------------------------------------
 * hallo_b200_attention -- fused softmax(Q K^T / sqrt(d)) V on wgmma, flash-style.
 *
 * Replaces diffusers Attention/AttnProcessor2_0 SDPA at
 *   hallo/models/mutual_self_attention.py:253-286  spatial self-attention with ReferenceNet KV concat
 *                                                  (and the uncond-half recomputation, Q3)
 *   hallo/models/attention.py:828-831              audio-block self-attention
 *
 *   Q, K, V : token matrices [frames*L, ld*], head h occupies columns [h*head_dim, (h+1)*head_dim)
 *             (they may be column slices of one fused QKV projection buffer).
 *   Kref/Vref: [ref_frames*L, ld*ref] reference tokens, projected once per window.
 *   ref_index: int32 [frames] on the device; frame n attends to its own L keys and, when
 *             ref_index[n] >= 0, additionally to the L keys of reference frame ref_index[n]
 *             (the reference tiles CFG halves over the batch: ref_index[n] = n % 2 for cond
 *             frames, -1 for uncond frames -- SURVEY quirk Q9).  NULL = plain self-attention.
 *   O       : [frames*L, ldo], same head layout.
 *   head_dim in {40, 80, 160, 512}; scale = head_dim^-0.5; no mask, no dropout.  Scores and softmax in fp32.
 *   Checked before anything runs: Q, K, V, O non-NULL, and Kref, Vref non-NULL with ref_frames >= 1 when ref_index
 *             is given (HB_ERR_NULL); 1 <= heads <= 256, L >= 1, frames >= 1, every ld* a multiple of 8, Q / K / V /
 *             Kref / Vref 16-byte aligned, O 4-byte aligned (the kernels store O as 32-bit pairs) (HB_ERR_BAD_SHAPE).
 *   head_dim 512 (the VAE mid-block attention, diffusers Attention(heads=1) over the (h/8)(w/8) tokens of a frame):
 *             heads == 1 and no reference keys; L may be any length.  The V / O columns are split over 4 CTAs of
 *             128 columns, each of which recomputes the 512-wide Q K^T.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int32_t dtype;
  int32_t head_dim, heads;
  int32_t L, frames;
  const void* Q;
  int64_t ldq;
  const void* K;
  int64_t ldk;
  const void* V;
  int64_t ldv;
  const void* Kref;
  int64_t ldkref;
  const void* Vref;
  int64_t ldvref;
  int32_t ref_frames;
  const int32_t* ref_index;
  void* O;
  int64_t ldo;
} hb_attention_params;

int hallo_b200_attention(const hb_attention_params* p, hb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * HBM-bound helpers (csrc/aux.cu)
 * ---------------------------------------------------------------------------------------- */
/* nn.LayerNorm(C, eps) per token row; optional `+ pe[pe_index[(row / L) % frames]]` after the norm
 * (PositionalEncoding of hallo/models/motion_module.py:426-461, applied at :585-586).
 * pe: fp32 [max_len, C] or NULL; pe_index: int32 [frames] or NULL (identity). */
int hallo_b200_layernorm(int dtype, const void* x, int64_t ldx, void* out, int64_t ldo, const void* gamma,
                         const void* beta, int rows, int C, float eps, const float* pe,
                         const int32_t* pe_index, int L, int frames, hb_stream_t stream);

/* Per-frame GroupNorm over channels-last frames [N, HW, C1(+C2)] (InflatedGroupNorm, resnet.py:88-101;
 * transformer_3d.py:197; motion_module.py:290), optional SiLU (resnet.py:386-387, 399).
 * x2/C2: second channel-concatenated source (UNet skip connection) or NULL/0.
 * stats_ws: fp32 workspace of N*ceil(HW/64)*G*2 + N*2*(C1+C2) floats (per-chunk group sums -- summed in a fixed order, no
 * atomics: results are bitwise reproducible -- then per-channel scale/shift).  Output frame n -> (n / fpb_in) * fpb_out + frame_off + n % fpb_in
 * (fpb_in <= 0: identity) -- used to drop frames into the 18-frame temporal buffer. */
int hallo_b200_groupnorm(int dtype, const void* x1, int C1, const void* x2, int C2, int N, int HW, int G,
                         const void* gamma, const void* beta, float eps, int silu, void* out,
                         float* stats_ws, int fpb_in, int fpb_out, int frame_off, hb_stream_t stream);

/* softmax(q k^T / sqrt d) v against n_keys in {4, 32} keys per (kv-frame, head, region):
 * image-token cross-attention (mutual_self_attention.py:289-303) and the three audio cross-attentions
 * (attention.py:854-890).  Frame n reads keys of kv-frame n / kv_frame_div.  Region r reads Q columns
 * at r*q_region_stride, K/V columns at r*kv_region_stride, writes O columns at r*o_region_stride.
 * Q and O must be 16-byte aligned (the CUDA-core kernel moves 8 elements per access); otherwise HB_ERR_BAD_SHAPE,
 * whichever kernel the "xattn_tc" option selects. */
int hallo_b200_cross_attention(int dtype, const void* Q, int64_t ldq, int q_region_stride, const void* K,
                               const void* V, int64_t ldkv, int kv_region_stride, void* O, int64_t ldo,
                               int o_region_stride, int frames, int L, int heads, int head_dim, int n_keys,
                               int kv_frame_div, int regions, hb_stream_t stream);

/* Temporal self-attention over the frame axis at every pixel (VersatileAttention,
 * motion_module.py:579-609).  Q: [batch*Fq*L, ldq]; K/V: [batch*Fk*L, ldkv]; Fk <= 32. */
int hallo_b200_temporal_attention(int dtype, const void* Q, int64_t ldq, const void* K, const void* V,
                                  int64_t ldkv, void* O, int64_t ldo, int batch, int Fq, int Fk, int L,
                                  int heads, int head_dim, hb_stream_t stream);

/* F.interpolate(scale 2, nearest) on NHWC (Upsample3D, resnet.py:166-183). */
int hallo_b200_upsample2x(int dtype, const void* x, void* out, int N, int H, int W, int C, hb_stream_t stream);
/* space-to-depth phase planes feeding the stride-2 conv (conv3x3 == 2). */
int hallo_b200_phase_split(int dtype, const void* x, void* out, int N, int H, int W, int C, hb_stream_t stream);
/* im2col of the fp32 latents for conv_in (unet_3d.py:603): out [batch*F*H*W, 64].  latents are
 * [1, Cl, F, H, W] shared by both CFG halves (face_animate.py:398) or, with per_half_latents != 0,
 * [batch, Cl, F, H, W]. */
int hallo_b200_im2col_latent(int dtype, const float* latents, void* out, int batch, int Cl, int F, int H,
                             int W, int per_half_latents, hb_stream_t stream);
/* im2col for a 3x3 stem conv over a small-channel fp32 NCHW image x [N, Cl, H, W] (9 Cl <= 64): out [N*H*W, 64],
 * column (kh*3 + kw)*Cl + c of row (n, h, w) = y_c at pixel (h + kh - 1, w + kw - 1), 0 outside the image (columns
 * >= 9 Cl are 0), where y = mat (scale x) + bias per pixel.  mat: fp32 [Cl, Cl] row-major or NULL (identity); bias:
 * fp32 [Cl] or NULL (0).  The affine map is applied before the zero padding: the VAE decoder's post_quant_conv (1x1
 * with bias) in front of its padded conv_in, which no folded weight reproduces at the border; with mat = bias = NULL
 * it is the plain im2col of the encoder's RGB conv_in. */
int hallo_b200_im2col_affine(int dtype, const float* x, void* out, int N, int Cl, int H, int W, const float* mat,
                             const float* bias, float scale, hb_stream_t stream);
/* diffusers Timesteps(dim, flip_sin_to_cos=True, shift 0) for t = t_table[*step] (unet_3d.py:565-587). */
int hallo_b200_timestep_embed(int dtype, const float* t_table, const int32_t* step, void* out, int rows,
                              int dim, hb_stream_t stream);
/* CFG combine + DDIM v-prediction update on fp32 latents [1, Cl, F, HW] (face_animate.py:415-420).
 * coef: fp32 [n_steps, 4] = sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev). */
int hallo_b200_cfg_ddim_step(int dtype, const void* model_out, int64_t ldm, float* latents, const float* coef,
                             const int32_t* step, float guidance, int Cl, int F, int HW, float* v_out,
                             hb_stream_t stream);
/* CFG combine + DPM-Solver++ (order 1 or 2, data prediction) v-prediction update on fp32 latents [1, Cl, F, HW].
 * coef: fp32 [n_steps, 5] = alpha, sigma, a, b, c; with v = v_u + guidance (v_c - v_u) and x0 = alpha x - sigma v,
 * x <- a x + b x0 + c x0_hist, then x0_hist <- x0.  x0_hist: fp32, shaped like latents; it is not read on rows with
 * c == 0, so step 0 of a schedule needs no initialised history. */
int hallo_b200_cfg_multistep_step(int dtype, const void* model_out, int64_t ldm, float* latents, float* x0_hist,
                                  const float* coef, const int32_t* step, float guidance, int Cl, int F, int HW,
                                  hb_stream_t stream);
/* CFG combine + ancestral Euler (Euler-a) v-prediction update on fp32 latents y [1, Cl, F, HW] in the VP form.
 * coef: fp32 [n_steps, 5] = alpha, sigma, a, b, d; with v = v_u + guidance (v_c - v_u) and x0 = alpha y - sigma v,
 * y <- a y + b x0 + d z.  noise: [n_steps, Cl, F, HW] in the model dtype; z is its slice of the current step. */
int hallo_b200_cfg_ancestral_step(int dtype, const void* model_out, int64_t ldm, float* latents, const void* noise,
                                  const float* coef, const int32_t* step, float guidance, int Cl, int F, int HW,
                                  hb_stream_t stream);
/* CFG combine + UniPC (bh1 / bh2, order 1 or 2, data prediction) v-prediction update on fp32 latents [1, Cl, F, HW].
 * coef: fp32 [n_steps, 10] = alpha, sigma, kx, kL, k0, k1, k2, pc, p0, p1; with v = v_u + guidance (v_c - v_u) and
 * m = alpha x - sigma v (the data estimate at the sample the UNet saw), the corrector c = kx x + kL last_sample + k0 m
 * + k1 x0_hist + k2 x0_hist2 (kx = 1, the rest 0 where it does not run), then x <- pc c + p0 m + p1 x0_hist,
 * last_sample <- c, x0_hist2 <- x0_hist, x0_hist <- m.  last_sample, x0_hist, x0_hist2: fp32, shaped like latents; a
 * term whose coefficient is 0 does not read its buffer, so step 0 of a schedule needs no initialised state. */
int hallo_b200_cfg_unipc_step(int dtype, const void* model_out, int64_t ldm, float* latents, float* last_sample,
                              float* x0_hist, float* x0_hist2, const float* coef, const int32_t* step, float guidance,
                              int Cl, int F, int HW, hb_stream_t stream);
/* Three-branch CFG combine with a separate audio guidance scale, in place on model_out [3*F*HW, ldm] (rows uncond,
 * cond, cond with zero audio tokens; first Cl columns valid): v = v_u + guidance (v_r - v_u) + audio_guidance
 * (v_c - v_r) in fp32, written back as 0 over the uncond rows and v (rounded to the model dtype) over the cond rows.
 * Any cfg_*_step above then applies the scheduler update to v when it is called on the same buffer with
 * guidance = 1.  With audio_guidance == guidance this is the two-branch combine up to that one rounding. */
int hallo_b200_cfg_guide3_step(int dtype, void* model_out, int64_t ldm, float guidance, float audio_guidance, int Cl,
                               int F, int HW, hb_stream_t stream);
/* Guidance rescale (diffusers rescale_noise_cfg) over a whole window, possibly frame-sharded over ranks, in three
 * stream-ordered calls on model_out [nb*F*HW, ldm] (nb = 2: rows uncond, cond; nb = 3: uncond, cond, cond with zero
 * audio tokens; first Cl columns valid).  v_cfg is the fp32 combine of cfg_*_step (nb = 2) or cfg_guide3_step
 * (nb = 3) with the same guidance / audio_guidance; the "text" prediction is always the cond rows, v_c.
 *   stats : partials [HB_RESCALE_PARTIALS, 4] fp64 <- per-CTA (sum v_c, sum v_c^2, sum v_cfg, sum v_cfg^2) of this
 *           rank's elements.
 *   reduce: the 4 totals of the partials (summed in a fixed order) are stored to each of dst[0 .. n_dst) (host array
 *           of device pointers: this rank's slot in every rank's totals table, or copies).
 *   apply : totals [n_ranks, 4] fp64, summed in rank order, over n = n_ranks*Cl*F*HW elements (every rank holds F
 *           frames) give the unbiased std_t = std(v_c) and std_g = std(v_cfg), and
 *             v = rescale * v_cfg * std_t / std_g + (1 - rescale) * v_cfg,
 *           written as 0 over the uncond rows and v (rounded to the model dtype) over the cond rows, so any cfg_*_step
 *           then applies the scheduler update to v with guidance = 1.  Where std_g is 0 (up to the rounding of the
 *           fp64 sums, var(v_cfg) <= 1e-12 mean(v_cfg^2)) v = v_cfg is written instead of NaN.  rescale in [0, 1].
 * No atomics: equal inputs give bitwise-equal outputs, and ranks holding equal totals apply the same factor. */
#define HB_RESCALE_PARTIALS 256
int hallo_b200_cfg_rescale_stats(int dtype, const void* model_out, int64_t ldm, int nb, float guidance,
                                 float audio_guidance, int Cl, int F, int HW, double* partials, hb_stream_t stream);
int hallo_b200_cfg_rescale_reduce(const double* partials, double* const* dst /* host array */, int n_dst,
                                  hb_stream_t stream);
int hallo_b200_cfg_rescale_apply(int dtype, void* model_out, int64_t ldm, int nb, float guidance, float audio_guidance,
                                 float rescale, const double* totals, int n_ranks, int Cl, int F, int HW,
                                 hb_stream_t stream);
int hallo_b200_advance_step(int32_t* step, int n_steps, hb_stream_t stream);
/* channels-last [B*F*HW, ld] (first C columns) -> fp32 [B, C, F, HW] (the reference's output layout). */
int hallo_b200_tokens_to_bcfhw(int dtype, const void* x, int64_t ld, float* out, int B, int C, int F, int HW,
                               hb_stream_t stream);
/* out = a + b over n elements (n % 8 == 0, 16-byte aligned): the residual add that closes a frame-sharded motion
 * module (motion_module.py:313-315) once the peers' proj_out rows have landed. */
int hallo_b200_add(int dtype, const void* a, const void* b, void* out, int64_t n, hb_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Peer memory (multi-GPU, one process per GPU): the temporal attention of the motion modules
 * (hallo/models/motion_module.py:579-609) mixes all frames of a pixel, everything else on the path is
 * per-frame.  A frame-sharded window therefore swaps frame <-> pixel ownership around each motion
 * module; the swap is FUSED into the producing kernels: the GroupNorm-apply that feeds the module and
 * the module's proj_out GEMM store their rows directly into the destination rank's buffer over
 * NVLink (peer-mapped device memory), two flag barriers per module replace the collectives.
 *
 * The one exception to "the library never allocates": exchange buffers must be cudaMalloc'ed
 * allocations of their own to be exportable through CUDA IPC, so the library owns them.
 * ---------------------------------------------------------------------------------------- */
#define HB_MAX_PEERS 16
#define HB_IPC_HANDLE_BYTES 64
int hallo_b200_peer_alloc(int64_t bytes, void** ptr_out);                 /* cudaMalloc + zero fill */
int hallo_b200_peer_free(void* ptr);
int hallo_b200_peer_export(void* ptr, void* handle_out /* HB_IPC_HANDLE_BYTES, host */);
int hallo_b200_peer_open(const void* handle /* host */, void** ptr_out);  /* maps another process's allocation */
int hallo_b200_peer_close(void* ptr);
/* Barrier over n ranks through flag words in peer memory.  flags[r] points at rank r's flag array (>= n uint32,
 * zero-initialised; flags[me] is local, the others peer-mapped).  epoch: local device counter (uint32, starts 0),
 * incremented by every call -- kept on the device so that a captured CUDA graph replays correctly.  Everything the
 * calling stream wrote to peer memory before the barrier is visible to the peers' kernels after it.  A rank that
 * waits longer than ~20 s records HB_ERR_DEVICE_TRAP in the device error word instead of hanging the GPU. */
int hallo_b200_peer_barrier(void* const* flags /* host array of n device pointers */, int n, int me,
                            uint32_t* epoch, hb_stream_t stream);
/* hallo_b200_groupnorm whose output rows are scattered by pixel: pixel p of (remapped) frame n_out goes to
 * out_peers[p / seg] + ((n_out * seg + p % seg) * C) elements, seg = HW / n_dest -- the frame -> pixel swap in front of
 * a motion module (motion_module.py:290-296), fused into the GroupNorm's store. */
int hallo_b200_groupnorm_scatter(int dtype, const void* x1, int C1, int N, int HW, int G, const void* gamma,
                                 const void* beta, float eps, void* const* out_peers /* host array */, int n_dest,
                                 float* stats_ws, int fpb_in, int fpb_out, int frame_off, hb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* HALLO_B200_H_ */
