/* b200svd — C ABI of the H100-native (sm_90a) StreamingSVD denoiser kernels (libb200svd.so).
 *
 * The reference (Picsart-AI-Research/StreamingT2V, pure Python) has no FFI: its seam for this path is the
 * nn.Module call `StreamingWrapper.forward(x, t, c, **kwargs)` (code/models/diffusion/wrappers.py:23-78).  Every
 * entry point below replaces one class of eager-PyTorch library calls that the reference makes underneath that
 * seam; the citation on each function names the reference call sites it stands in for.  The Python host
 * (streamingt2v_b200/) binds these with ctypes (see INTEGRATION.md) and mirrors the reference module interface.
 *
 * Conventions
 *   - plain C: raw device pointers, integer sizes, a CUDA stream passed as void* (cudaStream_t).
 *   - PyTorch (or any allocator) owns all memory; the library borrows pointers for the duration of a call.
 *   - every function enqueues work on `stream` and returns without synchronising.
 *   - return value 0 = success; non-zero = failure, message via b200svd_last_error() (thread local).
 *   - activations are bf16, channel-last: [frames, H, W, C] == [(b t), (h w), c] token rows.
 *   - no CPU fallback, no backend dispatch: sm_90a only.
 */
#ifndef B200SVD_H
#define B200SVD_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SVD_MAX_TAPS 12

enum { B200SVD_ACT_NONE = 0, B200SVD_ACT_SILU = 1, B200SVD_ACT_GELU = 2, B200SVD_ACT_GEGLU = 3 };

/* ---- library ------------------------------------------------------------------------------------------- */
const char* b200svd_last_error(void);
int b200svd_version(void);
/* 0 if the current device is sm_90 and the driver entry points resolve, else error. */
int b200svd_init(int device);

/* ---- multi-tap tensor-core GEMM (wgmma + TMA) ------------------------------------------------------------
 * out[row, n] = s_acc * act( sum_{tap, k} A_tap[row, k] * W[tap, n, k] + bias[n] + fvec[row / rows_per_frame, n] )
 *               + s1 * res1[row, n] + s2 * res2[row, n]
 *
 * One kernel covers: nn.Linear (attention.py:94-120, 262-351; video_attention.py; openaimodel.py emb_layers),
 * 3x3 Conv2d stride 1/2 (openaimodel.py:107-207, 257-305), (3,1,1) Conv3d of the time_stack
 * (video_model.py:46-59) — the A operand is addressed through a rank-5 TMA view of the channel-last activation,
 * each tap is a coordinate offset in that view (out-of-bounds = zero padding), and all taps accumulate into one
 * register accumulator.  The epilogue carries the reference's elementwise neighbours: bias, per-frame embedding add
 * (openaimodel.py:346-352), GEGLU (attention.py:94-101), residual adds and AlphaBlender (util.py:358-370).
 */
typedef struct {
  /* A operand: bf16 tensor viewed as rank-5 (dim0 = channels, contiguous). strides in BYTES for dims 1..4. */
  const void* a_ptr;
  uint64_t a_dims[5];
  uint64_t a_strides[4];
  uint32_t a_box[5]; /* a_box[0] must be 64; product of a_box[1..4] must be 128 */
  /* weights: bf16 [taps][n][k], k contiguous */
  const void* w_ptr;
  uint32_t n, k, taps;
  int32_t tap_off[B200SVD_MAX_TAPS][5]; /* per-tap coordinate offset in the A view (dim0 = channel offset) */
  /* output-pixel space (m1 fastest); boxes are powers of two with product 128 */
  uint32_t m_ext[3];
  uint32_t m_box[3];
  uint32_t m_adim[3]; /* which A dim (1..4) each m dim walks */
  /* output addressing: row = m1*out_rs[0] + m2*out_rs[1] + m3*out_rs[2]; element (row, col) at out + row*ldo + col */
  int64_t out_rs[3];
  void* out;
  int64_t ldo;
  int32_t out_fp32; /* 0: bf16 output, 1: fp32 output */
  /* epilogue */
  const float* bias;       /* [n] or NULL */
  const float* fvec;       /* [frames][ldf] fp32 or NULL */
  int64_t ldf;
  uint32_t rows_per_frame; /* frame index = row / rows_per_frame */
  int32_t act;             /* B200SVD_ACT_* ; GEGLU halves the output width (weights must be tile-interleaved) */
  float s_acc;
  const void* res1; /* bf16 [rows][ld1] or NULL */
  int64_t ld1;
  float s1;
  const void* res2;
  int64_t ld2;
  float s2;
  int32_t bn; /* N tile: 32, 64, 128, 160 or 256 (0 = choose) */
  /* optional: GroupNorm statistics of the OUTPUT taken in the epilogue (the consumer's gn_stats pass over the
   * activation disappears; GroupNorm32, util.py:274-276).  Every 32-row quadrant of every 128-row M tile ("slot" =
   * 4 * M-tile index + quadrant) writes, per output channel, the sum and the sum of squares over its valid rows to
   * gn_part[slot][gn_ld][2] (fp32) and the sample index of its rows (row / gn_rows, -1 if the quadrant is empty) to
   * gn_slot_sample[slot].  The caller guarantees that all valid rows of a quadrant belong to one sample, that the
   * epilogue is activation-free with bf16 output (else the call fails), and reduces the partials with
   * b200svd_gn_stats_partials.  NULL gn_part = off. */
  float* gn_part;
  int32_t* gn_slot_sample;
  int64_t gn_ld;     /* channels per slot row of gn_part (>= n) */
  uint32_t gn_rows;  /* output rows per GroupNorm sample */
} b200svd_gemm_params;

int b200svd_gemm(const b200svd_gemm_params* p, void* stream);

/* Kept for ABI compatibility (no reference counterpart): records a CTA-pair tile mode 0..3 and returns the previous
 * one.  sm_90 has no CTA-pair MMA; every launch uses single-CTA tiles whatever the mode.  Other values only query. */
int b200svd_gemm_pair_mode(int mode);

/* ---- FlashAttention forward, head dim 64 (wgmma + TMA) -----------------------------------------------------
 * Spatial self-attention core of BasicTransformerBlock.attn1 (attention.py:320-351 SDPA / :427-446 xformers).
 * qkv: [(n s), ldqkv] bf16, columns [q | k | v] each heads*64 wide (output of the fused QKV projection);
 * out: [(n s), ldo] bf16.  softmax(q k^T * scale) v per (frame, head). */
int b200svd_flash_attn(const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s, int heads, float scale,
                       void* stream);

/* ---- FlashAttention forward, head dim 80 (wgmma + TMA) -----------------------------------------------------
 * Self-attention of the OpenCLIP ViT-H/14 image tower of the SVD conditioner (open_clip ResidualAttentionBlock,
 * nn.MultiheadAttention with 16 heads of 80; encoders/modules.py:697-729).  Same contract as b200svd_flash_attn with
 * head dim 80: qkv [(n s), ldqkv] bf16, columns [q | k | v] each heads*80 wide (the in_proj output), out [(n s), ldo]
 * bf16.  qkv and out 16-byte aligned, leading dims multiples of 8, ldqkv >= 3*heads*80, ldo >= heads*80. */
int b200svd_flash_attn_d80(const void* qkv, int64_t ldqkv, void* out, int64_t ldo, int n, int s, int heads,
                           float scale, void* stream);

/* ---- CLIP image preprocessing + patch gather (ViT-H/14) ------------------------------------------------------
 * FrozenOpenCLIPImageEmbedder.preprocess (encoders/modules.py:624-636): kornia resize to 224x224 (antialias Gaussian
 * blur with reflect borders, then bicubic align_corners=True), (x+1)/2, CLIP mean/std normalisation; written as the
 * A operand of the 14x14/stride-14 patch GEMM.  x: [n][3][h][w] fp32 contiguous; out: bf16 [(n*256)][ldp], column
 * (kh*14 + kw)*3 + c, columns 588..ldp-1 zero (ldp multiple of 8, >= 592).  taps_y / taps_x: HOST arrays of the
 * normalised 1-D Gaussian taps (odd counts <= 63, reflect padding ky/2 < h, kx/2 < w); {1.0f} = no blur. */
int b200svd_clip_preprocess(const float* x, int n, int h, int w, void* out, int64_t ldp, const float* taps_y, int ky,
                            const float* taps_x, int kx, void* stream);

/* Kept for ABI compatibility (no reference counterpart): records a softmax variant 3..5 and returns the previous one.
 * The sm_90 kernel has a single softmax organisation whatever the variant.  Other values only query. */
int b200svd_flash_attn_variant(int v);

/* ---- small-sequence attention, head dim 64, one warp per (batch, pixel, head) -----------------------------
 * Temporal self-attention (video_attention.py:145-148), CAM cross-frame attention (cam/conditioning.py:65-68),
 * temporal cross-attention over APM tokens (video_attention.py:150-154).  Row addressing:
 *   q/out row(b,i,s) = (b*lq + i)*s_pixels + s ;  k/v row(b,j,s) = (b*lk + j)*s_pixels + s  (kv_per_pixel = 1)
 *                                                  k/v row(b,j)   =  b*lk + j               (kv_per_pixel = 0) */
int b200svd_small_attn(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                       int64_t ldo, int b, int s_pixels, int heads, int lq, int lk, int kv_per_pixel, float scale,
                       void* stream);

/* ---- per-pixel attention over frames on the tensor cores (wgmma), head dim 64, K/V per pixel ------------
 * Same contract as b200svd_small_attn with kv_per_pixel = 1: temporal self-attention (video_attention.py:145-148)
 * and CAM cross-frame attention (cam/conditioning.py:65-68).  One CTA = 4 pixels x 1 head; frames are gathered by
 * TMA through their row stride, scores are block-diagonal in a 64 x 64 wgmma tile per two pixels. */
int b200svd_pixel_attn(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                       int64_t ldo, int b, int s_pixels, int heads, int lq, int lk, float scale, void* stream);

/* ---- GroupNorm(32) / LayerNorm, channel-last bf16, fp32 statistics ----------------------------------------
 * GroupNorm32 (diffusionmodules/util.py:274-276), Normalize (attention.py:132-135), CAM joint norm over
 * (C/32,F,H,W) (cam/conditioning.py:57-59: pass n = B, p = F*H*W), nn.LayerNorm (attention.py:528-530,
 * video_attention.py:59-102, controlnet.py:113-118).
 * x: [n][p][c] rows (stride ldx).  sums: n*32*2 doubles (sum, sum of squares).  The reduction is deterministic
 * (fixed order, no floating-point atomics): scratch holds per-chunk partials (b200svd_gn_scratch_doubles doubles),
 * counters is n int32 zero-initialised once by the caller (left zero by every call). */
int64_t b200svd_gn_scratch_doubles(int64_t n, int64_t p, int c);
int b200svd_gn_stats(const void* x, int64_t ldx, int64_t n, int64_t p, int c, void* sums, void* scratch,
                     void* counters, void* stream);
int b200svd_gn_apply(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t n, int64_t p, int c, const void* sums,
                     const float* gamma, const float* beta, float eps, int apply_silu, void* stream);
/* y = LN(x [+ fvec[row / rows_per_frame]]) ; if xsum != NULL also writes xsum = bf16(x + fvec). */
int b200svd_layernorm(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int c, const float* gamma,
                      const float* beta, float eps, const float* fvec, int64_t ldf, int rows_per_frame, void* xsum,
                      int64_t ldxs, int apply_silu, void* stream);

/* ---- layout / glue kernels ---------------------------------------------------------------------------------
 * nchw_to_nhwc: wrappers.py:33 (cat of latents + concat cond) at the module seam; src [n][c_src][hw] fp32 with an
 *   explicit frame stride -> dst[(n*hw + p)*ldd + c_off + c] bf16.
 * nhwc_to_nchw: output of VideoUNet.out (video_model.py:618) back to [n][c][hw] fp32.
 * upsample2x: Upsample nearest (openaimodel.py:138-155).  timestep_embed: util.py:207-231.
 * add_silu: out = bf16(silu(a + b)) for emb = time_embed + label_emb followed by emb_layers' SiLU
 *   (video_model.py:561-567, openaimodel.py:282-288).  add_rows: ControlNet Merger addition (controlnet.py:23-48).
 * apm_mix: BasicTransformerBlockWithAPM context mix (attention.py:612-620). */
int b200svd_nchw_to_nhwc(const float* src, int64_t src_frame_stride, int n, int c_src, int64_t hw, void* dst,
                         int64_t ldd, int c_off, void* stream);
int b200svd_nhwc_to_nchw(const void* src, int src_is_fp32, int64_t lds, int n, int c, int64_t hw, float* dst,
                         void* stream);
int b200svd_upsample2x(const void* x, void* y, int n, int h, int w, int c, void* stream);
int b200svd_timestep_embed(const float* t, int n, int dim, float max_period, void* out, int64_t ldo, void* stream);
int b200svd_add_silu(const float* a, const float* b, void* out, int64_t total, int apply_silu, void* stream);
int b200svd_copy2d(const void* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int cols, void* stream);
int b200svd_add_rows(void* dst, int64_t ldd, const void* src, int64_t lds, int64_t rows, int64_t src_rows, int cols,
                     void* stream);
/* VAE decoder AttnBlock (diffusionmodules/model.py:180-195, one head of width C): row softmax of fp32 scores to
 * bf16 probabilities, and a bf16 transpose that turns V into the K-major operand of the P.V GEMM. */
int b200svd_softmax_rows(const float* in, int64_t lds, void* out, int64_t ldo, int64_t rows, int cols, void* stream);
int b200svd_transpose(const void* in, int64_t ldi, void* out, int64_t ldo, int rows, int cols, void* stream);
int b200svd_apm_mix(const float* ctx, int n, int l, int d, const float* w, const float* wb, const float* ln_g,
                    const float* ln_b, const float* alpha, void* out, void* stream);

/* ---- sampler arithmetic around the seam (SURVEY.md section 8 rows a19-a21; fp32, NCHW latents) -----------------
 * The reference has no FFI here; these replace the per-step elementwise torch ops of
 *   Denoiser.forward + VScalingWithEDMcNoise   sgm/modules/diffusionmodules/denoiser.py:23-39, denoiser_scaling.py:51-59
 *   LinearPredictionGuider                     .../guiders.py:60-99 (doubled batch: rows [0,rows) unconditional,
 *                                              [rows,2*rows) conditional)
 *   EulerEDMSampler.sampler_step (gamma = 0)   .../sampling.py:82-103,211-215
 * prepare: xin2[2*rows*chw] = cat([x, x]) * c_in.
 * step:    x_next = x + (next_sigma - sigma) * (x - denoised) / sigma with
 *          denoised = D_u + scale[t] * (D_c - D_u), D_* = net_* * c_out + x * c_skip, t = row % num_frames;
 *          scale = num_frames device floats (torch.linspace(min_scale, max_scale, num_frames)). */
int b200svd_sampler_prepare(const float* x, float* xin2, int64_t rows, int64_t chw, float c_in, void* stream);
int b200svd_sampler_step(const float* net, const float* x, float* x_next, int64_t rows, int64_t chw, int num_frames,
                         const float* scale, float c_skip, float c_out, float sigma, float next_sigma, void* stream);

/* GroupNorm statistics from the epilogue partials of b200svd_gemm (see gn_part above): sums[n][32][2] doubles, the
 * same output as b200svd_gn_stats, reduced in a fixed order (deterministic).  scratch / counters as for
 * b200svd_gn_stats (scratch >= n * chunks * 64 doubles with chunks = ceil(n_slots / 64)). */
int b200svd_gn_stats_partials(const float* gn_part, const int32_t* gn_slot_sample, int64_t n_slots, int64_t gn_ld,
                              int c, int64_t n, void* sums, void* scratch, void* counters, void* stream);

/* ---- enhance stage: one DDIM step of one randomized-blending chunk (SURVEY.md section 8 row a24, loop part) -------
 * Replaces, per chunk and step, the guidance combine, `DDIMScheduler.step` (eta = 0; diffusers==0.30.2, restated —
 * parity unpinned) and the blended write `latents_denoised[:, :, start+offset : start+cs] = chunk[:, :, offset:]` of
 * code/i2v_enhance/pipeline_i2vgen_xl.py:868-903.  fp32, batch 1, layout [C][frames][hw]:
 *   noise [cfg ? 2 : 1][C][cs][hw] (unconditional first), lat [C][lat_frames][hw] read at frames lat_start + f,
 *   out [C][out_frames][hw] written at frames out_start + f for offset <= f < cs.
 *   e = u + guidance (t - u);  v-prediction: x0 = sqrt(a_t) x - sqrt(1-a_t) e, eps = sqrt(a_t) e + sqrt(1-a_t) x;
 *   epsilon: x0 = (x - sqrt(1-a_t) e) / sqrt(a_t), eps = e;  out = sqrt(a_prev) x0 + sqrt(1-a_prev) eps. */
int b200svd_ddim_blend_step(const float* noise, const float* lat, float* out, int channels, int cs, int64_t hw,
                            int lat_frames, int lat_start, int out_frames, int out_start, int offset, int cfg,
                            float guidance, float alpha_t, float alpha_prev, int v_pred, void* stream);

/* ---- frames for the media container (SURVEY.md section 8 row f4, on-device part) ---------------------------------
 * float NCHW in [vmin, vmax] -> uint8 NHWC with the arithmetic of the reference's `torch2np`
 * (code/lib/farancia/libimage/iimage.py:21-39; `IImage(chunk, vmin=0, vmax=255)` at utils/result_processor.py:24):
 * out = uint8(255 * (clip(x, vmin, vmax) - vmin) / (vmax - vmin)), truncating.  The device->host copy of a chunk
 * shrinks from 4 to 1 byte per sample. */
int b200svd_frames_to_uint8(const float* x, void* out, int64_t n, int c, int64_t hw, float vmin, float vmax,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SVD_H */
