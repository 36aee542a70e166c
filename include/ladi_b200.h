/* ladi_b200.h -- C ABI of libladi_b200.so: hand-written sm_90a (H100) kernels for the LaDI-VTON try-on hot path.
 *
 * The reference (miccunifi/ladi-vton) has no FFI of its own: it is pure Python and every GPU operation on its hot path is
 * a PyTorch/cuDNN/cuBLAS library call made from `StableDiffusionTryOnePipeline.__call__`
 * (src/vto_pipelines/tryon_pipe.py:494-765 of the reference).  This header is the boundary a maintainer binds (ctypes, see
 * INTEGRATION.md) to replace those library calls.  Each entry point names the reference call-site(s) it replaces.
 *
 * Conventions
 *  - plain pointers and sizes only; all pointers are CALLER-OWNED DEVICE pointers (e.g. torch.Tensor.data_ptr());
 *  - activations are NHWC bf16 (`pitch` = elements between consecutive pixels, multiple of 8 => 16-byte aligned rows);
 *  - `stream` is a cudaStream_t passed as void*; nothing allocates, synchronises or uses an implicit stream, so every call
 *    is CUDA-graph capturable;
 *  - return 0 (LADI_OK) on success; otherwise an error code, with a thread-local message in ladi_last_error();
 *    no exceptions/aborts cross the ABI;
 *  - there is NO CPU fallback: without a CUDA device every compute entry point returns LADI_ERR_CUDA.
 */
#ifndef LADI_B200_H
#define LADI_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define LADI_API __attribute__((visibility("default")))
#else
#define LADI_API
#endif

#define LADI_OK 0
#define LADI_ERR_INVALID 1
#define LADI_ERR_CUDA 2

#define LADI_ACT_NONE 0
#define LADI_ACT_SILU 1
#define LADI_ACT_GEGLU 2
#define LADI_ACT_GELU 3 /* GELU(erf): CLIP encoder-layer MLP and the adapter's projection MLP (inversion_adapter.py:12-20) */
#define LADI_ACT_RELU 4 /* warping module: ConvNet_TPS.py:32-42,93-105, unet_parts.py:15-22 */

LADI_API const char* ladi_last_error(void);
LADI_API int ladi_abi_version(void);
/* number of kernels this process has launched (or recorded into a CUDA graph under capture) through the library so far */
LADI_API long long ladi_launch_count(void);

/* ---- implicit-GEMM convolution / GEMM (wgmma + TMA) ----------------------------------------------------------------
 * Replaces nn.Conv2d (3x3 s1 p1, 3x3 s2, 1x1) and nn.Linear of: diffusers ResnetBlock2D / Transformer2DModel /
 * Downsample2D / Upsample2D inside UNet2DConditionModel.forward (call-site tryon_pipe.py:732), the VAE Encoder/Decoder
 * (src/models/vae.py:99-119, 183-212; AutoencoderKL.py:151,163) and EMASC (src/models/emasc.py:25-40).
 *
 * out[n,y,x,:] = epilogue( sum_{tap,src,c} in_src[n, y*stride+ky-pad_lo, x*stride+kx-pad_lo, c] * W[:, k(tap,src,c)]
 *                          + sum_{sc,c} sc[n,y,x,c] * W[:, k(sc,c)] )
 * The sources are concatenated along channels (UNet skip `torch.cat([x, skip], 1)`, diffusers CrossAttnUpBlock2D) WITHOUT
 * materialising the concat; the optional `sc` sources are the ResnetBlock2D 1x1 `conv_shortcut` folded into the same
 * accumulation.  Weight layout: bf16 [c_out][k_total], K order = for tap(ky,kx) row-major: for src: channels padded to a
 * multiple of 64 (zero weights in the padding); then for sc: channels padded to 64.  k_total = 64 * (#K blocks).
 * A GEMM out[M,N] = A[M,K] W[N,K]^T is ksize=1, n=1, h_out=1, w_out=M, src_c=K.
 * epilogue: +bias[c] (or +bias[row] if bias_per_row; bias += *step_ptr * bias_step_stride when step_ptr != NULL),
 *           act (SiLU, or GEGLU on interleaved (value,gate) column pairs -> c_out/2 outputs), +residual, *row_scale[row]. */
typedef struct ladi_conv_desc {
  int n, h_out, w_out, c_out;
  int h_in, w_in;            /* 0 => h_out*stride, w_out*stride */
  int ksize, stride, pad_lo; /* ksize 1|3, stride 1|2, pad_lo = top/left padding (1; 0 for the VAE (0,1,0,1) downsample) */
  int n_src;
  const void* src[2];
  int src_c[2];
  int src_pitch[2];
  int n_sc;
  const void* sc[2];
  int sc_c[2];
  int sc_pitch[2];
  const void* weight;
  int k_total;
  int weight_pitch;          /* elements between weight rows (>= k_total, multiple of 8) */
  const float* bias;
  int bias_per_row;
  int bias_step_stride;
  const int* step_ptr;
  const void* residual;
  int residual_pitch;
  const float* row_scale;
  int act;
  void* out;
  int out_pitch;
  int out_fp32;
  int force_bn;              /* 0 = the library chooses the N tile (and may split K); else this N tile, one of {32,64,128,160,192,256},
                                without split-K (tests / tuning) */
  int force_direct_epilogue; /* accepted and ignored (kept for ABI compatibility): the store path, staged through shared memory or from
                                the accumulator fragment, is chosen from the rest of the descriptor */
  void* splitk_ws;           /* optional fp32 workspace: enables split-K for few-tile / long-K shapes (NULL = never split) */
  int64_t splitk_ws_bytes;
  int pair_mode;             /* CTA pairs (2-CTA clusters on two M tiles of one N tile; each CTA loads half of the B tile and multicasts
                                it to both): 0 = library default (single CTAs; env LADI_CONV_2CTA=1 pairs where the shape allows), 1 = force
                                (error if the shape cannot pair), 2 = never */
  /* LayerNorm folded into the GEMMs on either side of it (BasicTransformerBlock.norm1/2/3 of the UNet, call-site tryon_pipe.py:732):
   * the PRODUCER of the normalised tensor also writes, per output row and 32-column chunk, {sum, sum of squares} of what it stores
   * (rowstat_out: fp32 [rows][c_out/32][2]); the CONSUMER multiplies the RAW tensor with W' = W diag(gamma) and corrects in its epilogue:
   * out[r,c] = rstd_r * (acc[r,c] - mean_r * ln_colsum[c]) + bias[c], bias = W beta (+ the linear's own bias); the LayerNorm pass and its
   * HBM round trip disappear.  ln_stats is the producer's rowstat_out for this GEMM's A rows (normalised width = src_c[0], %% 64 == 0). */
  float* rowstat_out;
  const float* ln_stats;
  const float* ln_colsum;    /* fp32 [c_out]: row sums of the bf16 weight actually multiplied */
  float ln_eps;
  /* nearest-2x upsample fused into the 3x3 convolution that follows it (diffusers Upsample2D: F.interpolate(scale_factor=2) + conv;
   * UNet up blocks and VAE decoder vae.py:142-174): src = the HALF-resolution tensor [n, h_out/2, w_out/2, C]; each output parity
   * (y&1, x&1) is a 2x2-tap convolution of it with merged weights (weights.pack_conv_up2x: [4 parities * c_out][4 taps * Cpad]),
   * 4/9 of the multiply-adds of the materialised form and no intermediate tensor.  ksize 3, stride 1, bf16 output. */
  int up2x;
} ladi_conv_desc;
/* Placement rules (LADI_ERR_INVALID, naming the operand, when broken): sources and shortcuts 16-byte aligned with pitches that are
 * multiples of 8; bf16 out and residual 4-byte aligned, fp32 out 8-byte aligned; out_pitch >= the output width (c_out, c_out/2 for
 * GEGLU), residual_pitch >= c_out; rowstat_out 8-byte and ln_stats 16-byte aligned.
 * Store paths, chosen per call from the descriptor (ladi_conv2d_plan names the one a call takes):
 *  - staged (16-byte stores through shared memory): bf16 out, N tile <= 128, no pair / split-K / LayerNorm fold / row statistics,
 *    c_out, output width and out_pitch multiples of 8, out 16-byte aligned, residual 16-byte aligned with residual_pitch % 8 == 0,
 *    a per-column bias 8-byte aligned with an even bias_step_stride;
 *  - split-K (fp32 partials in splitk_ws, then a reduce pass): only when c_out, out_pitch and residual_pitch are multiples of 4, out
 *    and residual 8-byte aligned, bias 16-byte aligned with bias_step_stride % 4 == 0 and splitk_ws 16-byte aligned; otherwise the
 *    call runs unsplit, which is not an error;
 *  - fragment (stores from the accumulator): every other valid descriptor. */
LADI_API int ladi_conv2d_bf16(const ladi_conv_desc* d, void* stream);
/* The plan ladi_conv2d_bf16 would run for `d` on a device with `sms` SMs (sms <= 0: the current device's count): N tile, split-K
 * factor and K blocks per split, CTA pairs (the cluster count is the launch's, from the occupancy API), staged epilogue, pipeline
 * stages, tile grid and total K blocks.  The same validation and decision code as the launch; it dereferences no pointer and needs no
 * device, so it also answers on a machine without a GPU. */
typedef struct ladi_conv_plan {
  int bn, splits, kb_per_split, pair, staged, stages, tiles_m, tiles_n, total_kb;
} ladi_conv_plan;
LADI_API int ladi_conv2d_plan(const ladi_conv_desc* d, int sms, ladi_conv_plan* out);

/* ---- fused multi-head attention, head_dim 64 (flash-style: S and O live in registers, online softmax in exp2) -------
 * Replaces diffusers CrossAttention.forward for attn1 (self) and attn2 (cross, 77 text tokens) of every
 * BasicTransformerBlock in the UNet (torch SDPA / xformers in the reference, src/inference.py:143-147).
 * element (b, i, h, e) of q is q[b*q_batch_stride + i*q_pitch + h*64 + e]; same for k, v, out.  No mask. */
typedef struct ladi_attn_desc {
  int batch, heads, nq, nkv;
  const void* q; int q_pitch; int64_t q_batch_stride;
  const void* k; int k_pitch; int64_t k_batch_stride;
  const void* v; int v_pitch; int64_t v_batch_stride;
  void* out; int out_pitch; int64_t out_batch_stride;
  float scale;               /* softmax(scale * q k^T) */
  int variant;               /* accepted values 0, 1, 2, 4, 5, 6, 8 (8 needs nkv <= 128); sm_90a runs one kernel for all of them */
  void* trace;               /* unused (NULL) */
  int head_dim;              /* ladi_attention_d512_bf16 only: 0 or 512 (the VAE), or 256 (reduced-width test models) */
} ladi_attn_desc;
/* Placement rules of both attention entry points (LADI_ERR_INVALID when broken): q, k, v 16-byte aligned with batch strides that are
 * multiples of 8 (TMA: 16-byte global addresses and strides), every pitch a multiple of 8 and >= the head columns (heads*64, or
 * head_dim), out 4-byte aligned (it is stored as bf16 pairs) with an even out_batch_stride. */
LADI_API int ladi_attention_bf16(const ladi_attn_desc* d, void* stream);
/* The same for ONE head of width 512: the VAE mid-block AttentionBlock (src/models/vae.py:81-90,112 encoder; :142-150,187 decoder;
 * N = h*w tokens: 3072 at 512x384, 12288 at 1024x768).  heads must be 1, pitches >= head_dim; `variant` / `trace` ignored.  Flash-style:
 * the N x N score matrix is never written (the reference's baddbmm + softmax + bmm materialises it per sample). */
LADI_API int ladi_attention_d512_bf16(const ladi_attn_desc* d, void* stream);
/* The launch ladi_attention_bf16 (wide = 0) or ladi_attention_d512_bf16 (wide != 0) runs for `d` on a device with `sms` SMs (sms <= 0:
 * the current device's count).  head_dim 64 is attention_d64_kernel: persistent, grid_x = min(n_items, sms) CTAs, where an item is one
 * (query tile, head, image), numbered query tile fastest, and CTA c runs items c, c + grid_x, ...  (items_min / items_max per CTA).
 * head_dim 512 / 256 is attention_kernel<D>: one CTA per (query tile, 128-column output slice, image), n_items = grid_x*grid_y*grid_z.
 * q_tile / kv_tile are the query rows and keys of one tile, stages the K / V ring depth (D = 64: K and V tile pairs; wide: 64-column
 * chunks), consumers the warpgroups that each own 64 query rows of a tile; idle_consumers_last_q_tile of them have no row in the
 * last query tile.  The same validation and policy code as the launches; it dereferences no pointer and needs no device. */
typedef struct ladi_attn_plan {
  int head_dim;
  int grid_x, grid_y, grid_z;
  int q_tile, kv_tile, stages, consumers;
  int n_q_tiles, n_kv_tiles, n_items;
  int items_min, items_max;
  int idle_consumers_last_q_tile;
  int smem_bytes;
} ladi_attn_plan;
LADI_API int ladi_attention_plan(const ladi_attn_desc* d, int wide, int sms, ladi_attn_plan* out);

/* ---- normalisation ---------------------------------------------------------------------------------------------------
 * GroupNorm(+SiLU) over the channel-concat of up to two NHWC sources (diffusers ResnetBlock2D.norm1/norm2,
 * Transformer2DModel.norm, conv_norm_out; VAE conv_norm_out vae.py:115-116,200-201), two passes:
 *   stats: partial sums per (image, pixel chunk, group) -> ws[n][chunks][groups][2] fp32 (chunks returned by the query);
 *   apply: y = (x-mean)*rstd*gamma+beta, optional SiLU, optional "+ add" AFTER the activation (vae.py:204-205), bf16 out
 *          of pitch out_pitch holding the concatenated, normalised tensor. */
LADI_API int ladi_groupnorm_chunks(int hw);
LADI_API int ladi_groupnorm_stats(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                         float* ws, void* stream);
LADI_API int ladi_groupnorm_apply(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                         const float* ws, const float* gamma, const float* beta, float eps, int silu, const void* add,
                         int add_pitch, void* out, int out_pitch, void* stream);
/* Placement rules (LADI_ERR_INVALID, naming the operand, when broken).  Both passes: x0 16-byte aligned, c0 > 0, c0 and pitch0
 * multiples of 8 with pitch0 >= c0; c1 >= 0, and when c1 > 0 x1 16-byte aligned with c1 and pitch1 multiples of 8, pitch1 >= c1;
 * n > 0, hw > 0; ws non-null; groups <= 64 dividing c0 + c1 <= 2560.  Apply also: gamma and beta non-null (read as scalars); out
 * 16-byte aligned with out_pitch % 8 == 0 and >= c0 + c1; add (optional) 16-byte aligned with add_pitch % 8 == 0 and >= c0 + c1. */
/* The grids the two passes launch for these arguments on a device with `sms` SMs (sms <= 0: the current device's count): pixel
 * chunks per image; group splits (gsplit: blockIdx.z of the stats pass, each owning block_channels channels); the stats block's
 * 16-byte channel lanes (lanes_v) and pixel lanes (k); pixels per chunk; the apply pass's pixels per block and block count; its
 * cursor step of dp pixels plus dv vectors per 256 elements; the threads per group (slices) folding the chunk partials.  The same
 * validation and decision code as the launches; it dereferences no pointer and needs no device. */
typedef struct ladi_gn_plan {
  int chunks, gsplit, block_channels, lanes_v, k, px_per_chunk, px_per_block, apply_blocks, dv, dp, slices;
} ladi_gn_plan;
LADI_API int ladi_groupnorm_plan(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                         const float* ws, const float* gamma, const float* beta, float eps, int silu, const void* add,
                         int add_pitch, const void* out, int out_pitch, int sms, ladi_gn_plan* plan);
/* LayerNorm over the last dim (BasicTransformerBlock.norm1/2/3; inversion adapter LayerNorms).  Two-pass statistics per row (mean,
 * then the sum of squared deviations).  Placement rules (LADI_ERR_INVALID, naming the operand): x, out, gamma and beta 16-byte aligned;
 * c a multiple of 8, <= 2048, with c / 8 = T * VPL for T in {4, 8, 16, 32} and VPL <= 8; x_pitch and out_pitch multiples of 8 and
 * >= c; rows > 0. */
LADI_API int ladi_layernorm(const void* x, int x_pitch, int rows, int c, const float* gamma, const float* beta, float eps, void* out,
                   int out_pitch, void* stream);
/* The LayerNorm launch for these arguments: T lanes per row, VPL 16-byte vectors per lane, rows per 256-thread block, blocks.  `sms` is
 * accepted like ladi_groupnorm_plan's; this plan does not depend on it.  Dereferences no pointer, needs no device. */
typedef struct ladi_ln_plan {
  int T, vpl, rows_per_block, blocks;
} ladi_ln_plan;
LADI_API int ladi_layernorm_plan(const void* x, int x_pitch, int rows, int c, const float* gamma, const float* beta, float eps,
                         const void* out, int out_pitch, int sms, ladi_ln_plan* plan);
/* Row softmax fp32 -> bf16 (VAE mid-block AttentionBlock: softmax in fp32, Appendix A.5). */
LADI_API int ladi_softmax_rows(const float* s, int rows, int cols, int s_pitch, float scale, void* out, int out_pitch, void* stream);

/* CLS-row attention of the inversion adapter's CLIP ViT-H encoder layer (16 heads, head_dim 80, 257 tokens): only token 0 of the
 * layer output is consumed (src/models/inversion_adapter.py:22-28), so only the CLS query is attended.
 * q0 [batch, heads*head_dim] bf16, kv [batch, tokens, >= 2*heads*head_dim] bf16 (K columns then V columns) -> out [batch, heads*head_dim].
 * Placement rules (LADI_ERR_INVALID, naming the operand): kv 4-byte aligned with an even kv_pitch >= 2*heads*head_dim (K is read as
 * bf16 pairs); q_pitch and out_pitch >= heads*head_dim; head_dim even.  Image b's K/V rows start at kv + b*tokens*kv_pitch.  The
 * (head_dim + tokens) fp32 values of one block and its 16 bytes of static reduction slots must fit 48 KB: tokens <= 12204 at head_dim 80. */
LADI_API int ladi_cls_attention(const void* q0, int q_pitch, const void* kv, int kv_pitch, int batch, int tokens, int heads, int head_dim,
                       float scale, void* out, int out_pitch, void* stream);
/* The launch ladi_cls_attention runs for these arguments (ladi_sa_plan below): chunks = rows_per_block = 1 (one block per head and
 * image, for the CLS row), its dynamic shared memory, never an opt-in.  `sms` is accepted like the other plan queries'; this plan does
 * not depend on it.  The same validation code as the launch; dereferences no pointer, needs no device. */
typedef struct ladi_sa_plan {
  int chunks, rows_per_block, smem_bytes, smem_optin;
} ladi_sa_plan;
LADI_API int ladi_cls_attention_plan(const void* q0, int q_pitch, const void* kv, int kv_pitch, int batch, int tokens, int heads,
                            int head_dim, float scale, const void* out, int out_pitch, int sms, ladi_sa_plan* plan);

/* ---- pointwise glue ------------------------------------------------------------------------------------------------- *
 * Every entry point below returns LADI_ERR_INVALID, naming the operand, for a null operand, an extent <= 0 or a placement its rules
 * exclude; nothing is launched then. */
/* out = a + b (bf16, equal pitch-free dense [count]); VAE decoder `sample += int_feat` (vae.py:193).  count a multiple of 8; a, b and
 * out 16-byte aligned (8-element vectors). */
LADI_API int ladi_add_bf16(const void* a, const void* b, void* out, int64_t count, void* stream);
/* nearest 2x upsample NHWC (diffusers Upsample2D F.interpolate(scale_factor=2, mode="nearest")).  Dense, c a multiple of 8; x and out
 * 16-byte aligned. */
LADI_API int ladi_upsample2x_nhwc(const void* x, int n, int h, int w, int c, void* out, void* stream);
/* NCHW fp32 [n,c,h*f,w*f] -> NHWC bf16 [n,h,w,pitch] channels [c_off, c_off+c): nearest sampling every f-th pixel
 * (F.interpolate default mode, tryon_pipe.py:434-436), times `scale`, optionally gated by (gate[n,0,..] < 0.5) -- the
 * `masked_image = image * (mask < 0.5)` of diffusers prepare_mask_and_masked_image (call-site tryon_pipe.py:630).  f >= 1,
 * c_off >= 0 and out_pitch >= c_off + c. */
LADI_API int ladi_nchw_f32_to_nhwc_bf16(const float* x, int n, int c, int h, int w, int f, float scale, const float* gate, void* out,
                               int out_pitch, int c_off, void* stream);
/* NHWC (bf16 or fp32) -> NCHW fp32, channels [c_off, c_off+c) of an NHWC tensor of given pitch: c_off >= 0, x_pitch >= c_off + c. */
LADI_API int ladi_nhwc_to_nchw_f32(const void* x, int x_is_fp32, int n, int c, int h, int w, int x_pitch, int c_off, float* out,
                          void* stream);
/* DiagonalGaussianDistribution.sample * scaling_factor (vae.py:330-348; tryon_pipe.py:647,462):
 * moments NHWC fp32 [n,h,w,2*cz] -> latents NCHW fp32 [n,cz,h,w] = (mean + exp(0.5*clamp(logvar,-30,20))*noise) * scale; m_pitch >= 2*cz.
 * A NaN logvar stays NaN through the clamp, as torch.clamp keeps it. */
LADI_API int ladi_posterior_sample(const float* moments, int m_pitch, const float* noise_nchw, int n, int cz, int h, int w, float scale,
                          float* out_nchw, void* stream);
/* mask (1 - m) rows for EMASC mask_features (src/utils/data_utils.py:9-14): mask NCHW fp32 [n,1,H,W] nearest-resized by
 * integer factor f to [n, H/f, W/f] and written as 1-m (fp32 per output pixel). */
LADI_API int ladi_inv_mask_rows(const float* mask, int n, int H, int W, int f, float* out, void* stream);
/* bilinear /8 downsample, align_corners=False, no antialias (tryon_pipe.py:632-634), NCHW fp32 -> NCHW fp32. */
LADI_API int ladi_bilinear_down8(const float* x, int n, int c, int H, int W, float* out, void* stream);
/* One DDIM step with classifier-free guidance and re-assembly of the next UNet input (tryon_pipe.py:715,735-741 +
 * DDIMScheduler.step): eps NHWC fp32 [cfg?2B:B, h, w, eps_pitch] (first 4 channels), latents NCHW fp32 [B,4,h,w] updated
 * in place; unet_in NHWC bf16 [cfg?2B:B, h, w, in_pitch] channels 0..3 rewritten for both halves.  coef = device table
 * [steps][8] = {1/sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-sigma_t^2), sigma_t, 0, 0, 0}, indexed by *step_ptr, which is
 * then incremented by the last block when advance != 0.  noise: NCHW fp32 [B,4,h,w] variance noise of the eta > 0 (stochastic)
 * DDIM update, x_prev += sigma_t * noise; NULL for eta = 0.  eps_pitch >= 4 and in_pitch >= 4; advance != 0 needs step_ptr (the
 * counter it advances; with step_ptr NULL the call reads coefficient row 0 and cannot advance). */
LADI_API int ladi_ddim_cfg_step(const float* eps, int eps_pitch, float* latents, void* unet_in, int in_pitch, int B, int h, int w,
                       int cfg, float guidance, const float* coef, int* step_ptr, int advance, const float* noise, void* stream);
/* diffusers prepare_mask_and_masked_image, tensor branch (called at tryon_pipe.py:630), without host synchronisation: range checks
 * image in [-1,1] / mask in [0,1] recorded in flags[0] / flags[1] (device int32[2], OR-ed; the pipeline reads them once, with the result)
 * and the IN-PLACE binarisation of the caller's mask at 0.5.  image fp32 [n_image], mask fp32 [n_mask], both dense. */
LADI_API int ladi_check_binarise(const float* image, long long n_image, float* mask, long long n_mask, int* flags, void* stream);
/* (x/2+0.5).clamp(0,1) NHWC bf16/fp32 [n,h,w,pitch] (first 3 channels) -> NHWC fp32 [n,h,w,3] (tryon_pipe.py:356-358); x_pitch >= 3.
 * NaN stays NaN, as torch.clamp keeps it. */
LADI_API int ladi_image_out(const void* x, int x_is_fp32, int n, int h, int w, int x_pitch, float* out, void* stream);
/* The same clamp followed by numpy_to_pil's (x * 255).round().astype(uint8) (DiffusionPipeline.numpy_to_pil, called at
 * tryon_pipe.py:760; round-half-to-even like numpy): NHWC uint8 [n,h,w,3], so output_type="pil" moves a quarter of the bytes to the host.
 * x_pitch >= 3.  NaN gives 0 (numpy's NaN -> uint8 cast has no defined value). */
LADI_API int ladi_image_out_u8(const void* x, int x_is_fp32, int n, int h, int w, int x_pitch, unsigned char* out, void* stream);
/* The EMASC trainer's reconstruction writer (src/utils/image_from_pipe.py:252-258: `(x + 1) / 2`, then torchvision.utils.save_image's
 * `mul(255).add_(0.5).clamp_(0, 255).to(uint8)`): t = (x + 1) * 0.5, u = fl(fl(t * 255) + 0.5) with two roundings (no FMA), clamp to
 * [0, 255], truncate.  x NHWC fp32 [n,h,w,pitch] (first 3 channels, as ladi_vae_decode_emasc writes it) -> NHWC uint8 [n,h,w,3];
 * x_pitch >= 3.  NaN gives 0. */
LADI_API int ladi_image_save_u8(const float* x, int n, int h, int w, int x_pitch, unsigned char* out, void* stream);
/* Sinusoidal timestep embedding of the UNet (diffusers get_timestep_embedding, flip_sin_to_cos, the input of time_embedding.linear_1; SURVEY App. A.2)
 * for n timesteps (device fp32 [n]), written as a (hi, lo) pair of bf16 column blocks: out bf16 [n, 2*k_pad], hi at columns [0, channels),
 * lo = bf16(e - hi) at [k_pad, k_pad + channels), zeros elsewhere (k_pad = channels rounded up to 64: the K layout of the packed [W | W] weight). */
LADI_API int ladi_timestep_embedding(const float* timesteps, int n, int channels, int k_pad, void* out, void* stream);
/* ---- dataset tensorisation edge (SURVEY.md 8(f) row 3): src/utils/posemap.py:6-35 kpoint_to_heatmap for n_maps key-points
 * (keypoints fp32 [n_maps,2] = (x, y) in pixels; the reference calls it per sample and joint with sigma 9, src/dataset/vitonhd.py:277-287):
 * out fp32 [n_maps,h,w] = exp(-|p - k|^2 / sigma^2) / (max + eps), all zeros for a key-point with no coordinate > 0. */
LADI_API int ladi_pose_heatmaps(const float* keypoints, int n_maps, int h, int w, float sigma, float* out, void* stream);

/* ---- text / vision conditioning front-end (SURVEY.md 8(f) row 1; not on the per-step path) ------------------------------------
 * Exact softmax attention for short sequences and any head width that is a multiple of 8 (<= 128), optional causal mask:
 * the CLIP text transformer driven by src/utils/encode_text_word_embedding.py:41-54 (77 causal tokens, 16 x 64) and the CLIP ViT-H
 * vision tower called at src/inference.py:269-273 (257 tokens, 16 x 80).  q/k/v/out: bf16 [batch, n, heads*head_dim] views with
 * row pitches and batch strides in elements (multiples of 8).  nkv <= 1024; causal needs nq == nkv.  Placement rules
 * (LADI_ERR_INVALID, naming the operand): k and v 16-byte aligned (rows are read as 16-byte vectors), q and out 4-byte aligned (bf16
 * pairs); every pitch >= heads*head_dim; for batch > 1 out_batch_stride >= nq*out_pitch (output images may not overlap; input images
 * may).  K and V of one (image, head), the 8 warps' query rows and probabilities must fit 200 KB of shared memory: at head_dim 128,
 * nkv <= 365; 1024 keys need head_dim <= 40. */
LADI_API int ladi_attention_small(const void* q, const void* k, const void* v, void* out, int batch, int heads, int nq, int nkv,
                         int head_dim, int q_pitch, int k_pitch, int v_pitch, int out_pitch, long long q_batch_stride,
                         long long k_batch_stride, long long v_batch_stride, long long out_batch_stride, float scale, int causal,
                         void* stream);
/* The launch ladi_attention_small runs for these arguments on a device with `sms` SMs (sms <= 0: the current device's): query-row
 * chunks per (head, image) (blockIdx.x), query rows per 8-warp block (warp w takes rows w, w + 8, ... of its block), dynamic shared
 * memory bytes, and whether they exceed the 48 KB a launch gets without raising the kernel's limit (smem_optin).  The same validation
 * and policy code as the launch; it dereferences no pointer and needs no device. */
LADI_API int ladi_attention_small_plan(const void* q, const void* k, const void* v, const void* out, int batch, int heads, int nq, int nkv,
                              int head_dim, int q_pitch, int k_pitch, int v_pitch, int out_pitch, long long q_batch_stride,
                              long long k_batch_stride, long long v_batch_stride, long long out_batch_stride, float scale,
                              int causal, int sms, ladi_sa_plan* plan);
/* out[row,:] = (src[row] >= 0 ? tok[src[row],:] : word_emb[-src[row]-1,:]) + pos[row % seq,:]  (bf16 tables, fp32 sum):
 * token_embedding + the '$' -> pseudo-word-embedding substitution + position_embedding of
 * src/utils/encode_text_word_embedding.py:27-38 (the index list `src` is built on the host from input_ids).  c and out_pitch
 * multiples of 8; tok, pos, out and word_emb (NULL when no row is negative) 16-byte aligned. */
LADI_API int ladi_clip_embed(const int* src, const void* tok, const void* word_emb, const void* pos, void* out, int rows, int seq, int c,
                    int out_pitch, void* stream);
/* pixels NCHW fp32 [n,ch,h,w] -> bf16 rows [n*(h/patch)*(w/patch), k_pad], column (c*patch+ky)*patch+kx, zero padding columns:
 * the im2col of CLIPVisionEmbeddings.patch_embedding (14x14 stride-14 convolution, no bias), followed by one ladi_conv2d_bf16 GEMM. */
LADI_API int ladi_patchify(const float* pixels, void* out, int n, int ch, int h, int w, int patch, int k_pad, void* stream);
/* x[b,0,:] = cls + pos[0,:]; x[b,1+i,:] = patch[b*n_patches+i,:] + pos[1+i,:]  (CLIPVisionEmbeddings.forward), all bf16.  c and
 * patch_pitch multiples of 8, patch_pitch >= c; patch, cls, pos and out 16-byte aligned; n <= 65535 (one grid.y slice per image). */
LADI_API int ladi_vit_assemble(const void* patch, int patch_pitch, const void* cls, const void* pos, void* out, int n, int n_patches, int c,
                      void* stream);

/* ---- cloth-warping front-end (SURVEY.md 8(f) row 2): ConvNet_TPS + refinement U-Net, src/inference.py:236-266 -----------------
 * torchvision resize(x, (oh, ow), BILINEAR, antialias=True) of an NCHW fp32 tensor, written as channels [c_off, c_off+c) of an NHWC
 * bf16 tensor (inference.py:239-247: cloth / im_mask / pose_map -> 256x192; the agnostic concat is built in place). */
LADI_API int ladi_resize_aa(const float* x, int n, int c, int h, int w, int oh, int ow, void* out, int out_pitch, int c_off, void* stream);
/* src/inference.py:265-271: torchvision resize((cloth + 1) / 2, (oh, ow), antialias=True).clamp(0, 1) followed by the CLIP image
 * processor's per-channel (v - mean) / std (AutoProcessor call, :267): x NCHW fp32 in [-1,1] -> out NCHW fp32 [n,c,oh,ow], the
 * `pixel_values` of the vision tower.  quantise != 0: v = floor(v * 255) / 255 first (a processor that round-trips through uint8). */
LADI_API int ladi_clip_preprocess(const float* x, int n, int c, int h, int w, int oh, int ow, const float* mean, const float* stdev,
                         int quantise, float* out, void* stream);
/* NHWC bf16 [n,h,w,c] -> [n,h/2,w/2,4c], channel (sy*2+sx)*c+ch <- pixel (2y+sy, 2x+sx): the 4x4 stride-2 pad-1 convolutions of
 * FeatureExtraction / FeatureRegression (ConvNet_TPS.py:31-38,93-97) become 3x3 stride-1 pad-1 ladi_conv2d_bf16 calls. */
LADI_API int ladi_space_to_depth2(const void* x, int n, int h, int w, int c, int x_pitch, void* out, int out_pitch, void* stream);
/* in place x[row,c] = x[row,c]*scale[c] + shift[c]: eval-mode BatchNorm2d that follows a ReLU (ConvNet_TPS.py:33,39,41).  c and pitch
 * multiples of 8; x, scale and shift 16-byte aligned (scale / shift are read as float4). */
LADI_API int ladi_channel_affine(void* x, long long rows, int c, int pitch, const float* scale, const float* shift, void* stream);
/* FeatureL2Norm (ConvNet_TPS.py:58-66), in place over the channel dimension of NHWC bf16 rows.  c and pitch multiples of 8; x 16-byte
 * aligned. */
LADI_API int ladi_l2norm_channels(void* x, long long rows, int c, int pitch, void* stream);
/* FeatureCorrelation (ConvNet_TPS.py:69-81): out NHWC bf16 [n,h,w,h*w], out[b,yB,xB,xA*h+yA] = <B[b,yB,xB,:], A[b,yA,xA,:]>.  Dense
 * inputs, c a multiple of 8; feat_a and feat_b 16-byte aligned; out_pitch >= h*w. */
LADI_API int ladi_feature_correlation(const void* feat_a, const void* feat_b, int n, int h, int w, int c, void* out, int out_pitch, void* stream);
/* points = tanh(theta) (ConvNet_TPS.py:122); grid = target_coordinate_repr @ (inverse_kernel @ [points; 0]) (TPSGridGen.forward,
 * :183-193).  theta fp32 [n, >= 2*n_ctrl]; inverse_kernel [(n_ctrl+3)^2]; target_coordinate_repr [n_points, n_ctrl+3];
 * points fp32 [n, n_ctrl, 2]; grid fp32 [n, n_points, 2].  1 <= n_ctrl <= 64, theta_pitch >= 2*n_ctrl, n <= 65535 (one grid.y slice
 * per image). */
LADI_API int ladi_tps_grid(const float* theta, int theta_pitch, const float* inverse_kernel, const float* target_coordinate_repr, int n, int n_ctrl,
                  int n_points, float* points, float* grid, void* stream);
/* inference.py:252-257: antialiased-bilinear resize of low_grid fp32 [n,gh,gw,2] to (h,w) fused with F.grid_sample(cloth, grid,
 * bilinear, padding_mode='border', align_corners=False); cloth NCHW fp32 [n,c,h,w] -> channels [c_off,c_off+c) of NHWC bf16 out. */
LADI_API int ladi_warp_grid_sample(const float* low_grid, int gh, int gw, const float* cloth, int n, int c, int h, int w, void* out, int out_pitch,
                          int c_off, void* stream);
/* fp32 forms of ladi_resize_aa and ladi_warp_grid_sample: the same arithmetic, written unrounded as NCHW fp32 [n, c, oh, ow] / [n, c, h, w]
 * (the bf16 forms store the round-to-nearest bf16 of exactly these values).  The TPS trainer's validation (src/train_tps.py:43-92) reads
 * the TPS-only warped cloth and the VGG loss's resized inputs in fp32.  x, low_grid, cloth and out 4-byte aligned. */
LADI_API int ladi_resize_aa_f32(const float* x, int n, int c, int h, int w, int oh, int ow, float* out, void* stream);
LADI_API int ladi_warp_grid_sample_f32(const float* low_grid, int gh, int gw, const float* cloth, int n, int c, int h, int w, float* out,
                                       void* stream);
/* nn.MaxPool2d(2) / nn.Upsample(scale_factor=2, bilinear, align_corners=True) on NHWC bf16 (unet_parts.py:31-34,47).  Dense, c a
 * multiple of 8; x and out 16-byte aligned.  The max pool returns NaN for a window holding a NaN, as nn.MaxPool2d does. */
LADI_API int ladi_maxpool2_nhwc(const void* x, int n, int h, int w, int c, void* out, void* stream);
LADI_API int ladi_upsample2x_bilinear_ac(const void* x, int n, int h, int w, int c, void* out, void* stream);
/* NHWC fp32 [n,h,w,pitch] (first c channels) -> NCHW fp32 clamped to [lo,hi] (inference.py:262 warped_cloth.clamp(-1,1)); NaN stays
 * NaN, as torch.clamp keeps it. */
LADI_API int ladi_nhwc_f32_to_nchw_clamp(const float* x, int n, int c, int h, int w, int x_pitch, float lo, float hi, float* out, void* stream);

/* ---- image-quality metrics (csrc/metrics.cu; the engine form of src/utils/val_metrics.py:105-225, which runs clean-fid's FID / KID
 * Inception and torchmetrics' SSIM, LPIPS and Inception Score).  Every kernel reduces in a fixed order: two runs give the same bits. ---
 * im2col of a kh x kw / (sh, sw) / (ph, pw) convolution (nn.Conv2d of torchvision's Inception-v3 and AlexNet where ladi_conv2d_bf16's
 * ksize-3 rules do not apply: 3-channel stems, 11x11/4, 5x5, 1x7, 7x1, 1x3, 3x1, valid 3x3): bf16 rows [n*oh*ow, k_pad], column
 * (ky*kw + kx)*c + ch, zeros in columns [kh*kw*c, k_pad); then one ladi_conv2d_bf16 GEMM (ksize 1).  x_is_f32_nchw = 0: x NHWC bf16 of
 * channel pitch `pitch` (c % 8 == 0), shift = scale = NULL.  x_is_f32_nchw = 1: x NCHW fp32 pixels, each in-image pixel becomes
 * (x - shift[ch]) / scale[ch] BEFORE the zero padding (LPIPS ScalingLayer ahead of AlexNet's padded 11x11 conv, lpips/pretrained_networks;
 * the FID Inception's (x - 128) / 128).  ladi_patchify is the special case patch = stride, no padding.  Placement rules (LADI_ERR_INVALID,
 * naming the operand): NHWC form x and out 16-byte aligned; pixel form x, shift and scale 4-byte aligned, out 2-byte aligned. */
LADI_API int ladi_im2col_bf16(const void* x, int x_is_f32_nchw, int n, int c, int h, int w, int pitch, int kh, int kw, int sh, int sw, int ph,
                              int pw, const float* shift, const float* scale, void* out, int k_pad, void* stream);
/* torch max_pool2d / avg_pool2d (ceil_mode=False) on NHWC bf16 (c, pitches and c_off multiples of 8): window k, stride s, padding p,
 * output [n, (h+2p-k)/s+1, (w+2p-k)/s+1] written to channels [c_off, c_off+c) of `out` (pitch out_pitch) -- an Inception branch writes
 * straight into its Mixed_* concatenation.  Modes: MAX (padding never wins), AVG (count_include_pad=True, torchvision InceptionA/C/E),
 * AVG_EXCLUDE_PAD (count_include_pad=False, the FID blocks of pytorch-fid / torch-fidelity), GLOBAL_AVG_F32 (adaptive_avg_pool2d(x, 1):
 * `out` is fp32 [n, out_pitch], k / s / p ignored -- the Inception pool3 features).  Placement rules (LADI_ERR_INVALID, naming the
 * operand): window modes x and out 16-byte aligned; GLOBAL_AVG_F32 x 2-byte and out 4-byte aligned. */
#define LADI_POOL_MAX 0
#define LADI_POOL_AVG 1
#define LADI_POOL_AVG_EXCLUDE_PAD 2
#define LADI_POOL_GLOBAL_AVG_F32 3
LADI_API int ladi_pool2d_bf16(const void* x, int n, int h, int w, int c, int x_pitch, int k, int s, int p, int mode, void* out, int out_pitch,
                              int c_off, void* stream);
/* One LPIPS layer (lpips.LPIPS.forward, version 0.1; torchmetrics LearnedPerceptualImagePatchSimilarity): feature pairs fa, fb NHWC bf16
 * [n, h, w, pitch]; per pixel n_a = a / (sqrt(sum_c a^2) + 1e-10), n_b likewise, d = sum_c lin[c] * (n_a - n_b)^2 (the 1x1 C -> 1 `lin`
 * conv, no bias, fp32 weights); acc[b] += mean over the h*w pixels of d.  Called once per AlexNet tap, acc (fp32 [n]) ends as the LPIPS
 * distance of each pair.  Placement rules (LADI_ERR_INVALID, naming the operand): fa, fb 2-byte aligned, lin and acc 4-byte aligned. */
LADI_API int ladi_lpips_layer(const void* fa, const void* fb, int n, int h, int w, int c, int pitch, const float* lin, float* acc, void* stream);
/* SSIM of torchmetrics StructuralSimilarityIndexMeasure(data_range=1.0) per image: x, y NCHW fp32; gaussian window 11 wide, sigma 1.5
 * (separable), C1 = 0.01^2, C2 = 0.03^2; the mean over channels and the (h-10) x (w-10) positions whose window lies inside the image
 * (torchmetrics reflect-pads by 5 and crops 5, which is the same).  fp32 throughout; ws: fp32 [n * ladi_ssim_partials(h, w)] of tile sums;
 * out fp32 [n].  h, w >= 11, n <= 65535 (one grid.z slice per image).  x, y, ws and out 4-byte aligned (LADI_ERR_INVALID otherwise). */
LADI_API int ladi_ssim_partials(int h, int w);
LADI_API int ladi_ssim_f32(const float* x, const float* y, int n, int c, int h, int w, float* ws, float* out, void* stream);
/* The Inception Score input of torchmetrics InceptionScore(normalize=True): (x * 255).byte() then torch-fidelity's TF1-style bilinear resize
 * (source coordinate o * in/out, no half-pixel offset, upper neighbour clamped): x NCHW fp32 in [0, 1] -> out NCHW fp32 [n, c, oh, ow].
 * x and out 4-byte aligned (LADI_ERR_INVALID otherwise). */
LADI_API int ladi_resize_tf1_u8(const float* x, int n, int c, int h, int w, int oh, int ow, float* out, void* stream);
/* fp32 forms of the metric networks (metrics.py, precision="tf32": fp32 NHWC activations, every convolution a TF32 tensor-core GEMM
 * with fp32 accumulation, as cuDNN runs the reference's fp32 convolutions by default on Ampere and Hopper).
 * ladi_gemm_tf32: out[m, c_off + j] = relu?(sum_k a[m, k] w[j, k] + bias[j]) for j < n; a fp32 [m, a_pitch], w fp32 [n, w_pitch] (the
 * K-major [c_out, K] convolution weight), bias fp32 [n] or NULL, relu 0 | 1, out fp32 of row pitch out_pitch (a block's NHWC
 * concatenation; columns outside [c_off, c_off + n) untouched).  Both operands are rounded to TF32 to nearest (cvt.rna: 10 explicit
 * mantissa bits, ties away from zero) inside the kernel, so each product is within 2^-10 relative of the fp32 operands' product;
 * the sum is fp32 in K order (two runs give the same bits).  Columns k..a_pitch of `a` and k..w_pitch of `w` are never read (a K padded to a
 * multiple of 4 with zeros is the packed layout).  Placement rules (LADI_ERR_INVALID, naming the operand): a and w 16-byte aligned with
 * pitches >= k that are multiples of 4; n, c_off and out_pitch multiples of 4 with c_off + n <= out_pitch; out 16-byte aligned; bias 4-byte
 * aligned; at most 65535 tiles of 128 rows (m <= 8388480).
 * ladi_im2col_f32, ladi_pool2d_f32, ladi_lpips_layer_f32: ladi_im2col_bf16, ladi_pool2d_bf16 and ladi_lpips_layer on fp32 activations,
 * with 4 in place of 8 in the channel, pitch, k_pad and c_off rules; the pixel form's out is fp32 (no rounding after the fp32 affine)
 * and 4-byte aligned; lpips fa / fb 4-byte aligned.  GLOBAL_AVG_F32 reads fp32 x (4-byte aligned). */
LADI_API int ladi_gemm_tf32(const float* a, int m, int k, int a_pitch, const float* w, int n, int w_pitch, const float* bias, int relu, float* out,
                            int out_pitch, int c_off, void* stream);
LADI_API int ladi_im2col_f32(const float* x, int x_is_nchw_pixels, int n, int c, int h, int w, int pitch, int kh, int kw, int sh, int sw, int ph,
                             int pw, const float* shift, const float* scale, float* out, int k_pad, void* stream);
LADI_API int ladi_pool2d_f32(const float* x, int n, int h, int w, int c, int x_pitch, int k, int s, int p, int mode, float* out, int out_pitch,
                             int c_off, void* stream);
LADI_API int ladi_lpips_layer_f32(const float* fa, const float* fb, int n, int h, int w, int c, int pitch, const float* lin, float* acc,
                                  void* stream);
/* nn.L1Loss (mean) of two fp32 row-pitched tensors, accumulated on the device: *acc += weight * sum|a - b| / (rows * cols) over
 * a[r * a_pitch + j], b[r * b_pitch + j], j < cols (the columns past `cols` are never read).  The VGG loss's taps (GEMM output rows) and
 * NCHW images (rows = n*c*h, cols = w).  Two launches: per-block partial sums into ws (fp32, LADI_L1_MEAN_WS floats), then one block that
 * sums them in a fixed tree; the grid depends on the shape only, so two runs give the same bits.  Operands 4-byte aligned (16-byte
 * alignment with cols and pitches multiples of 4 takes the float4 path). */
#define LADI_L1_MEAN_WS 1024
LADI_API int ladi_l1_mean_f32(const float* a, int a_pitch, const float* b, int b_pitch, long long rows, int cols, float weight, float* ws,
                              float* acc, void* stream);

/* ================================================================================================================================
 * Module-level ABI (SURVEY.md section 8(b)): an opaque per-device engine handle + one entry point per module of the try-on path.
 * What a non-Python host binds to run the reference's objects without re-writing their forward passes:
 *   unet(x, t, encoder_hidden_states).sample           tryon_pipe.py:732 (diffusers UNet2DConditionModel.forward)   -> ladi_unet_forward
 *   vae.encode(x) -> (posterior moments, 6 skips)      tryon_pipe.py:640,457; AutoencoderKL.py:145-157; vae.py:99-119 -> ladi_vae_encode
 *   vae.decode(z, intermediate_features, int_layers)   tryon_pipe.py:352-353; AutoencoderKL.py:159-188; vae.py:183-212 -> ladi_vae_decode_emasc
 *   emasc(features) + mask_features(features, mask)    tryon_pipe.py:684-685; emasc.py:37-40; data_utils.py:4-16     -> ladi_emasc_forward
 *   inversion_adapter(clip_features)                   src/inference.py:276; inversion_adapter.py:22-28              -> ladi_inversion_adapter_forward
 *   the denoising loop                                 tryon_pipe.py:713-747                                         -> ladi_denoise_loop
 * Rules: all pointers are caller-owned device pointers; activations NHWC bf16 (channel pitch = multiple of 8); the caller supplies the
 * activation workspace (ladi_workspace_bytes) and the stream; no call allocates, synchronises or uses an implicit stream, so every call is
 * CUDA-graph capturable.  ladi_engine_create allocates the two scratch buffers all calls share (64 MB split-K partials, 16 MB GroupNorm
 * statistics) and ladi_engine_destroy frees them.  One handle per (device, stream); calls on one handle are not concurrent. */
typedef struct ladi_engine ladi_engine;

/* one packed weight: name (the key the Python packer uses, e.g. "down_blocks.0.resnets.0.w1"), device pointer, rows x cols
 * (bf16 matrices: cols = K = row pitch, layouts as documented at ladi_conv_desc; fp32 vectors: rows = 1) */
typedef struct ladi_weight {
  const char* name;
  const void* ptr;
  int rows, cols;
} ladi_weight;

typedef struct ladi_engine_config {
  /* UNet2DConditionModel (SD-2-inpainting layout, hubconf.py:30-33) */
  int unet_channels[4];        /* block_out_channels */
  int unet_heads[4];           /* attention_head_dim = head COUNT per level in SD-2 configs (head width is always 64) */
  int unet_down_attn[4];       /* down block i is a CrossAttnDownBlock2D */
  int unet_up_attn[4];         /* up block i is a CrossAttnUpBlock2D */
  int unet_layers_per_block;
  int unet_in_channels, unet_out_channels;
  float unet_norm_eps;
  int norm_groups;             /* GroupNorm groups (32), UNet and VAE */
  int fuse_upsample;           /* 1: upsampler weights are packed for the sub-pixel form (ladi_conv_desc.up2x) */
  /* AutoencoderKL (LaDI-VTON fork, src/models/AutoencoderKL.py) */
  int vae_channels[4];
  int vae_layers_per_block, vae_latent_channels, vae_in_channels, vae_out_channels;
  /* EMASC (hubconf.py:40-53) */
  int emasc_scales;
  int emasc_in[8], emasc_out[8], emasc_stride[8];   /* per scale: channels in / out, resolution divisor of the feature (1, 1, 2, 4, 8) */
  /* InversionAdapter (hubconf.py:16-27) */
  int adapter_dim, adapter_heads, adapter_mlp, adapter_hidden, adapter_out;
  int plan_only;               /* 1: no device: the handle only answers ladi_workspace_bytes / ladi_engine_trace (tests, tooling) */
} ladi_engine_config;

LADI_API int ladi_engine_create(const ladi_engine_config* cfg, const ladi_weight* table, int n_weights, ladi_engine** out);
LADI_API int ladi_engine_destroy(ladi_engine* engine);
#define LADI_Q_TEMB_TOTAL 0 /* columns of the per-step bias table (sum of the resnets' widths) */
#define LADI_Q_KV_TOTAL 1   /* columns of the text K/V buffer (sum over cross-attention layers of 2C) */
#define LADI_Q_IN_PITCH 2   /* channel pitch of the UNet input buffer (in_channels rounded up to 8) */
LADI_API int ladi_engine_query(const ladi_engine* engine, int what);

#define LADI_MODULE_UNET 0        /* (batch = UNet batch, height = latent h, width = latent w) */
#define LADI_MODULE_VAE_ENCODE 1  /* (batch, image height, image width) */
#define LADI_MODULE_VAE_DECODE 2  /* (batch, latent h, latent w) */
#define LADI_MODULE_EMASC 3       /* (batch, image height, image width) */
#define LADI_MODULE_ADAPTER 4     /* (batch, height = tokens, width ignored) */
#define LADI_MODULE_UNET_PLAN 5   /* ladi_unet_plan_steps: (batch = number of timesteps, height / width ignored) */
/* bytes of caller workspace one call of `module` needs at this shape (a walk of the module body with the allocator only); -1 on error */
LADI_API int64_t ladi_workspace_bytes(ladi_engine* engine, int module, int batch, int height, int width);
/* the launch sequence of the last ladi_workspace_bytes walk, one op per line (tooling / the CPU test that pins it to the Python sequencing) */
LADI_API const char* ladi_engine_trace(const ladi_engine* engine);

/* eps = unet(x, t, ctx):  x_in NHWC bf16 [batch, h, w, in_pitch] (first in_channels valid; channel order latents4, mask1, masked4,
 * pose18, cloth4, tryon_pipe.py:724-726); step_ptr device int32[2] = {row of `steps` to use, 0}; steps fp32 [n_steps][temb_total] =
 * conv1.bias + time_emb_proj(silu(time_embedding(t_s))) per resnet (step-invariant, built once per call); ctx_kv bf16
 * [batch, ctx_tokens, kv_total] = the text context already projected by every cross-attention layer's to_k / to_v;
 * eps_out NHWC fp32 [batch, h, w, 4]. */
LADI_API int ladi_unet_forward(ladi_engine* engine, const void* x_in, const int* step_ptr, const float* steps, const void* ctx_kv, int batch, int lat_h,
                               int lat_w, int ctx_tokens, void* eps_out, void* workspace, int64_t workspace_bytes, void* stream);
/* The two step-invariant tables ladi_unet_forward reads (the reference recomputes both inside every forward, tryon_pipe.py:732):
 *   steps  fp32 [n][temb_total] = conv1.bias + time_emb_proj(silu(time_embedding(t_s))) for every resnet, from the n timesteps (device fp32 [n],
 *          the scheduler's `timesteps`, tryon_pipe.py:650-651); needs ladi_workspace_bytes(engine, LADI_MODULE_UNET_PLAN, n, 0, 0) of workspace;
 *   ctx_kv bf16 [rows = batch * ctx_tokens][kv_total] = the text context (bf16 [rows][ctx_dim]) through every cross-attention layer's to_k / to_v. */
LADI_API int ladi_unet_plan_steps(ladi_engine* engine, const float* timesteps, int n, float* steps_out, void* workspace, int64_t workspace_bytes, void* stream);
LADI_API int ladi_unet_plan_context(ladi_engine* engine, const void* ctx, int rows, int ctx_dim, void* ctx_kv_out, void* stream);
/* x NHWC bf16 [batch, H, W, 8] (3 valid channels) -> posterior moments NHWC fp32 [batch, H/8, W/8, 2*latent] (quant_conv folded in) and the
 * retained encoder features (vae.py:100-109): skips[1] (= skips[2]) [batch,H,W,C0], skips[3] [batch,H/2,W/2,C0], skips[4] [.., /4, C1],
 * skips[5] [.., /8, C2]; skips[0] is unused (the input itself); a null entry (or skips == NULL) keeps that feature in the workspace. */
LADI_API int ladi_vae_encode(ladi_engine* engine, const void* x_nhwc8, int batch, int height, int width, float* moments, void* const* skips,
                             void* workspace, int64_t workspace_bytes, void* stream);
/* z NHWC bf16 [batch, h, w, 8] (latents / scaling_factor, 4 valid channels) + the EMASC outputs feats[0..n_feats) in the reference's list
 * order with their encoder layer indices int_layers[] (vae.py:183-212; n_feats = 0: plain decode) -> image NHWC fp32 [batch, 8h, 8w, 4]. */
LADI_API int ladi_vae_decode_emasc(ladi_engine* engine, const void* z_nhwc8, int batch, int lat_h, int lat_w, const void* const* feats, int n_feats,
                                   const int* int_layers, float* image_out, void* workspace, int64_t workspace_bytes, void* stream);
/* per scale i: outs[i] = conv(silu(conv(feats[i]))) * inv_masks[i] (fp32 per output pixel = 1 - nearest-resized mask; NULL: no
 * masking); feats / outs NHWC bf16 at resolution (height, width) / emasc_stride[i].  The form of each scale is read from the weight table
 * (emasc.py:20-33): with `emasc.<i>.w1/b1` and `emasc.<i>.w2/b2` it is the nonlinear form above; without `emasc.<i>.w2` it is the linear
 * form, outs[i] = conv(feats[i]) * inv_masks[i] with `emasc.<i>.w1/b1`.  The kernel size comes from the packed width of `emasc.<i>.w1`:
 * cols / (64 * ceil(emasc_in[i] / 64)) taps, 9 -> 3x3 with padding 1, 1 -> 1x1 with padding 0; any other width is rejected. */
LADI_API int ladi_emasc_forward(ladi_engine* engine, const void* const* feats, const float* const* inv_masks, int batch, int height, int width,
                                void* const* outs, void* workspace, int64_t workspace_bytes, void* stream);
/* feats bf16 [batch, tokens, adapter_dim] (CLIP ViT-H last_hidden_state) -> out bf16 [batch, adapter_out].  The number of encoder layers
 * L is read from the weight table (inversion_adapter.py:9): layers 0..L-2 are `adapter.enc<l>.{ln1,qkv,o,ln2,fc1,fc2}` (full pre-LN
 * CLIP layers over all tokens, attention on ladi_attention_small, tokens <= 1024), counted from l = 0 while `adapter.enc<l>.ln1.0`
 * exists; the last layer keeps the names `adapter.{ln1,kv,q,o,ln2,fc1,fc2}` and runs on the CLS row only. */
LADI_API int ladi_inversion_adapter_forward(ladi_engine* engine, const void* feats, int batch, int tokens, void* out, void* workspace,
                                            int64_t workspace_bytes, void* stream);
/* n_steps x (ladi_unet_forward + ladi_ddim_cfg_step) enqueued on `stream`: unet_in NHWC bf16 [cfg ? 2*batch : batch, h, w, in_pitch] with
 * the static channels already written, latents NCHW fp32 [batch,4,h,w], step_ptr device int32[2] zeroed by the caller (advances on the
 * device: no host sync in the loop), coef fp32 [n_steps][8] (see ladi_ddim_cfg_step), eps_scratch fp32 [cfg ? 2*batch : batch, h, w, 4]. */
LADI_API int ladi_denoise_loop(ladi_engine* engine, void* unet_in, float* latents, int* step_ptr, const float* steps, const float* coef, const void* ctx_kv,
                               int batch, int lat_h, int lat_w, int ctx_tokens, int cfg, float guidance, int n_steps, float* eps_scratch, void* workspace,
                               int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif
