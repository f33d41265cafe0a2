/*
 * idiff_b200.h -- C ABI of libidiff_b200.so: the sm_90a (H100) kernels behind the
 * InstanceDiffusion sampling hot path.
 *
 * The reference (frank-xwang/InstanceDiffusion) is pure Python/PyTorch and has no FFI; its
 * seam is the set of nn.Module classes resolved by dotted path (ldm/util.py:71-84).  Each entry
 * point below replaces the arithmetic of one (group of) reference call site(s); the Python
 * mirror modules in instancediffusion_b200/ldm/... call these through ctypes with raw device
 * pointers (tensor.data_ptr()) and the current CUDA stream.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; idiff_last_error() gives the text.
 *   - nothing here allocates device memory or synchronises; all work is enqueued on `stream`
 *     (a cudaStream_t passed as void*).  Buffers are caller-owned.
 *   - activations are fp16, token-major / NHWC: a (B,H,W,C) image is the (B*H*W, C) row-major
 *     matrix the transformer blocks see, so the reference's NCHW<->(B,HW,C) rearranges vanish.
 *   - weights are fp16 [out_features, in_features] row-major (conv3x3: [Cout, 3, 3, Cin]).
 */
#ifndef IDIFF_B200_H
#define IDIFF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* idiff_last_error(void);
int idiff_version(void);

/* 16-bit storage type of the loaded library.  The same sources are compiled twice: libidiff_b200.so
 * stores activations / weights as IEEE fp16 (the reference's torch.autocast type, inference.py:94) and
 * libidiff_b200_bf16.so (-DIDIFF_STORAGE_BF16=1) as bfloat16 (BASELINE.json configs[3]).  Every entry
 * point below has the same name, arguments and meaning in both; wherever a comment or a name says
 * "fp16" / "f16" it means "the 16-bit storage type of this library".  Accumulators, normalisation
 * statistics, biases, the sampler state and all fp32 arguments are fp32 in both. */
#define IDIFF_DTYPE_F16 0
#define IDIFF_DTYPE_BF16 1
int idiff_storage_dtype(void);

/* Batch-invariant mode (process-wide, per library build; off by default).  While it is on, every image's
 * output of every entry point below is a function of that image's inputs and the weights only: launch
 * geometry that shapes a reduction depends on the per-image shape, never on the batch size, the total row
 * count or the SM count.  In particular idiff_gemm runs data-parallel (no stream-K) with a tile width that
 * depends on N and the epilogue family only, LayerNorm statistics (ln_stats_out) are taken over the stored
 * 16-bit values, and GroupNorm / ScaleU reduce in a fixed number of pixel chunks per image.  Returns the
 * previous setting. */
int idiff_set_batch_invariant(int on);

/* ---------------------------------------------------------------------------------------------
 * idiff_gemm: out = epilogue(A . W^T) on wgmma tensor cores (TMA-staged 128B-swizzled tiles,
 * fp32 accumulation in registers).  Replaces every nn.Linear / 1x1 conv / 3x3 conv of the path:
 *   attention.py:41 (GEGLU proj), :62 (FF out), :121-125,175-179 (to_q/k/v/to_out), :297 (fuser
 *   linear), :354,363 (proj_in/proj_out 1x1); openaimodel.py:186,213 (ResBlock conv3x3), :109
 *   (Upsample conv), :134 (Downsample conv), :205 (emb_layers), :361-363 (time_embed), :464 (out);
 *   text_grounding_net.py:75-81 (UniFusion MLPs).
 * conv3x3 (conv_h > 0): A is the NHWC activation (conv_b, conv_h, conv_w, conv_cin), gathered
 * tap by tap with 4-D TMA boxes and hardware zero fill at the borders (no im2col buffer);
 * W is [N, 9*conv_cin] with k = (ky*3+kx)*conv_cin + c; stride 1, padding 1.
 * ------------------------------------------------------------------------------------------- */
#define IDIFF_EPI_GEGLU 1       /* W rows interleaved per 128: [value(128) | gate(128)]; out has N/2 cols:
                                   (value+b)*gelu_erf(gate+b)            (attention.py:41-43)   */
#define IDIFF_EPI_SILU 2        /* x -> x*sigmoid(x) after bias                                   */
#define IDIFF_OUT_F32_NCHW 4    /* out is fp32 (B, N, H*W): the eps layout the samplers consume   */
#define IDIFF_EPI_GELU 8        /* x -> exact (erf) GELU after bias: ConvNeXt pwconv1 (convnext.py:31,42) */

typedef struct {
  const void* a;        /* fp16 [M, K] (lda)            | conv: fp16 NHWC activation            */
  const void* w;        /* fp16 [N, K] (ldw)                                                    */
  void* out;            /* fp16 [M, N or N/2] (ldo)     | fp32 NCHW with IDIFF_OUT_F32_NCHW      */
  const float* bias;    /* [N] or NULL                                                          */
  const void* rowadd;   /* fp16 [M / rows_per_batch, N] (row stride ldra) added per batch (ResBlock
                           emb, openaimodel.py:246-256) or NULL                                 */
  const void* residual; /* fp16 [M, N_out] (ldr) or NULL: out = residual + gate * (...)         */
  float gate;           /* scale * tanh(alpha) of GatedSelfAttentionDense; 1 for plain residual */
  int M, N, K;
  int lda, ldw, ldo, ldr, ldra;
  int rows_per_batch;
  int flags;
  int conv_b, conv_h, conv_w, conv_cin;
  void* workspace;      /* optional stream-K scratch of this call (>= idiff_gemm_workspace_bytes(), 256B aligned,
                           zero-initialised once by the caller, then owned by the library between calls on ONE
                           stream); NULL = the process-wide default of idiff_set_gemm_workspace, if any        */
  long workspace_bytes;
  /* LayerNorm folded across two GEMMs (attention.py:333-338 norm1/2/3, :309-310 fuser norms).  LN(x) W^T + b
     = rstd_r (x W'^T - mean_r colsum(W')) + (W beta + b) with W' = W * gamma: the GEMM reads the
     un-normalised residual stream, the row statistics come from the GEMM that wrote it.
     Producer (any plain linear layer): ln_stats_out != NULL receives, per output row, the partial
       (sum, sum of squares) of the stored row over each column slot: float2 [idiff_gemm_ln_slots(args)][M].
     Consumer (plain or GEGLU, K <= 2560): ln_stats_in != NULL = the producer's buffer over this GEMM's A
       rows (ln_slots_in slots, summed in slot order), w = fp16(W * gamma), ln_colsum[n] = sum_k w[n,k]
       (fp32), bias = W beta + b, ln_eps the LayerNorm epsilon. */
  void* ln_stats_out;
  const void* ln_stats_in;
  const float* ln_colsum;
  int ln_slots_in;
  float ln_eps;
  /* Per-batch-entry residual gate (batched forwards of requests with different fuser scales): NULL, or fp32
     [number of batch entries] -- with a residual, out = residual + gate * gate_b[b] * (...), b = row / rows_per_batch
     (conv: the image).  Needs residual != NULL and combines with bias and ln_stats_out only (no rowadd, SiLU /
     GELU, ln_stats_in); NULL leaves the epilogue as above. */
  const float* gate_b;
} idiff_gemm_args;
int idiff_gemm(const idiff_gemm_args* args, void* stream);
/* number of column slots a producer GEMM with these arguments writes to ln_stats_out (depends on the
   tile plan; <= 64) */
int idiff_gemm_ln_slots(const idiff_gemm_args* args);
/* per-row (sum, sum of squares) of an fp16 [rows, channels] matrix as ONE slot: float2 [rows] -- the entry
   point of the folded LayerNorm when the stream was not written by idiff_gemm (module-level calls) */
int idiff_row_stats(const void* x, void* stats, int rows, int channels, void* stream);
/* Stream-K scratch (fp32 partial tiles + flags) for load-balancing GEMMs whose tile count is not a
 * multiple of the SM count.  Caller-owned device memory of at least idiff_gemm_workspace_bytes().
 * Preferred: pass it per call in idiff_gemm_args.workspace (one buffer per stream -- GEMMs in flight on
 * different streams must not share flags).  idiff_set_gemm_workspace registers a process-wide default
 * for callers that use a single stream (zeroed by the call, synchronous).  Without any scratch every
 * GEMM runs data-parallel. */
long idiff_gemm_workspace_bytes(void);
int idiff_set_gemm_workspace(void* ptr, long bytes);
/* Profiling hook: device buffer of 16 x uint64 per CTA (>= SM count * 16) receiving %globaltimer stamps of
 * each GEMM CTA's entry (slot 0) and exit (slot 7) and its SM clock at entry / exit (slots 12 / 13); NULL (default)
 * disables it. */
int idiff_set_gemm_trace(void* ptr);

/* ---------------------------------------------------------------------------------------------
 * idiff_attention: softmax(Q K^T * scale) V per (batch, head), flash-style online softmax with
 * S/O accumulators in registers.  Keys/values come from up to two segments: segment 0 = the visual
 * tokens (or the 77 text tokens), segment 1 = the 184 UniFusion object tokens of
 * GatedSelfAttentionDense (attention.py:304-309) -- queries exist only for the visual rows, which
 * is exactly the slice the reference keeps (:308).  Replaces F.scaled_dot_product_attention at
 * attention.py:134-144 (cross), :257-267 (self / gated-self).
 * Each operand is fp16 with row stride *_ld elements; head h occupies columns [h*d, (h+1)*d)
 * from the given pointer; batch b starts at row b*rows (rows = nq / n0 / n1).
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const void *q, *k0, *v0, *k1, *v1;
  void* out; /* fp16 [batch*nq, heads*head_dim] (out_ld) */
  int q_ld, k0_ld, v0_ld, k1_ld, v1_ld, out_ld;
  int batch, heads, head_dim; /* head_dim in {40, 80, 160} */
  int nq, n0, n1;             /* n1 may be 0 */
  int kv1_batch;              /* 1: segment 1 shared by all batch entries; else == batch */
  float scale;                /* head_dim^-0.5 (attention.py:102,164) */
  /* Instance-isolation mask of the gated self-attention at the 64x64 level (attention.py:187-255; live with
     efficient_attention=False, eval_local.py --use_masked_att): NULL, or uint32 words -- query i may attend key j
     iff (mask_q[b*nq + i] & mask_k[b*(n0+n1) + j]) != 0, or j is visual token i itself (the reference adds 1e-9
     on the diagonal).  idiff_attmask_words builds them from the (B, 30, 64, 64) att_masks. head_dim 40 only. */
  const void* mask_q;
  const void* mask_k;
} idiff_attn_args;
int idiff_attention(const idiff_attn_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Normalisation (HBM-bound passes)
 *   idiff_groupnorm: GroupNorm32 (util.py:223-225, eps 1e-5) / Normalize (attention.py:75-76,
 *   eps 1e-6) over NHWC fp16, statistics in fp32, optional fused SiLU (openaimodel.py:184,208).
 *   stats_ws: idiff_groupnorm_ws_floats(batch, groups) floats of scratch (per-chunk partial
 *   sums, reduced in a fixed order: results are bit-reproducible and batch-invariant).
 *   idiff_layernorm: nn.LayerNorm(C) (attention.py:294-295,320-322), rows held in registers.
 * ------------------------------------------------------------------------------------------- */
long idiff_groupnorm_ws_floats(int batch, int groups);
int idiff_groupnorm(const void* x, void* y, const float* gamma, const float* beta, float* stats_ws,
                    int batch, int hw, int channels, int groups, float eps, int fuse_silu,
                    void* stream);
int idiff_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows,
                    int channels, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * idiff_scaleu_concat: ScaleU skip-connection rescale (openaimodel.py:519-539):
 *   out[..., :C1]      = h * (tanh(b_c) + 1)
 *   out[..., C1:C1+C2] = Fourier_filter(skip, threshold=1, scale=s) = skip + (s-1) * P_low(skip)
 * with P_low the real part of the inverse DFT restricted to bins {-1,0}x{-1,0} (7 real
 * reductions per (b,c) plane; closed form of openaimodel.py:25-48).
 * coef_ws: idiff_scaleu_ws_floats(batch, c2) floats of scratch.
 * b1: per-channel factor tanh(b)+1 (C1 floats, device); s: tanh(scaleu_s)+1 (host scalar).
 * ------------------------------------------------------------------------------------------- */
long idiff_scaleu_ws_floats(int batch, int c2);
int idiff_scaleu_concat(const void* h, const void* skip, void* out, const float* b1, float s,
                        float* coef_ws, int batch, int height, int width, int c1, int c2,
                        void* stream);

/* ---------------------------------------------------------------------------------------------
 * Layout / resampling helpers
 * ------------------------------------------------------------------------------------------- */
/* fp32 NCHW (B,C,H,W) -> fp16 NHWC with channels zero-padded to c_pad */
int idiff_nchw_f32_to_nhwc_f16(const float* x, void* y, int batch, int c, int hw, int c_pad,
                               void* stream);
/* fp16 NHWC -> fp32 NCHW */
int idiff_nhwc_f16_to_nchw_f32(const void* x, float* y, int batch, int c, int hw, void* stream);
/* F.interpolate(scale_factor=2, mode="nearest") on NHWC fp16 (openaimodel.py:107) */
int idiff_upsample_nearest2x(const void* x, void* y, int batch, int h, int w, int c, void* stream);
/* im2col for the stride-2 padding-1 3x3 Downsample conv (openaimodel.py:130-134):
   out [B*(H/2)*(W/2), 9*C], k = (ky*3+kx)*C + c */
int idiff_im2col_s2(const void* x, void* y, int batch, int h, int w, int c, void* stream);
/* same layout for the first-stage encoder's Downsample (diffusionmodules/model.py:70-74): F.pad (0,1,0,1)
   then conv3x3 stride 2 padding 0, i.e. taps at (2*oy + ky, 2*ox + kx) with zero fill past the far edges */
int idiff_im2col_s2_pad01(const void* x, void* y, int batch, int h, int w, int c, void* stream);

/* ---------------------------------------------------------------------------------------------
 * idiff_fourier_embed: UniFusion instance-token builder front end
 * (text_grounding_net.py:216-225,248-276 + util.py:12-26): for every (b, slot) row writes
 *   out[row, :text_dim]            = text*m + (1-m)*null_text            (if text != NULL)
 *   out[row, text_dim + k*2D + j]     = sin(f_k * x_j)*m' + (1-m')*null_pos[...]
 *   out[row, text_dim + k*2D + D + j] = cos(f_k * x_j)*m' + (1-m')*null_pos[...]
 * f_k = 100^(k/16), k < 16.  m = masks[row]; m' = 0 if dropped, else masks[row] (mask_mode 0)
 * or ((sum_j x_j + masks[row]) > 0) (mask_mode 1: scribbles / polygons, :267,272).
 * ------------------------------------------------------------------------------------------- */
int idiff_fourier_embed(const float* coords, const float* masks, const float* text,
                        const float* null_text, const float* null_pos, void* out, int rows,
                        int coord_dim, int text_dim, int out_ld, int mask_mode, int dropped,
                        void* stream);

/* ---------------------------------------------------------------------------------------------
 * idiff_plms_update: fused sampler epilogue (plms.py:121-165 / plms_instance.py:166-210):
 *   e   = e_u + gs*(e_c - e_u)            (CFG; e_u may be NULL -> e = e_c)
 *   e'  = c0*e + c1*old1 + c2*old2 + c3*old3   (Adams-Bashforth weights chosen by the host;
 *         for the first-step Euler predictor pass c0=1; for the corrector e' = (e_prev + e)/2
 *         is expressed with old1)
 *   x_prev = sqrt(a_prev)*(x - sqrt(1-a_t)*e')/sqrt(a_t) + sqrt(1-a_prev)*e'
 * All fp32, n elements.  e_out receives the post-CFG e (history), x_out the new latent.
 * ------------------------------------------------------------------------------------------- */
int idiff_plms_update(const float* x, const float* e_c, const float* e_u, float gs,
                      const float* old1, const float* old2, const float* old3, float c0, float c1,
                      float c2, float c3, float a_t, float a_prev, float sqrt_one_minus_at,
                      float* e_out, float* x_out, long n, void* stream);
/* ---------------------------------------------------------------------------------------------
 * idiff_ddim_update: fused DDIM step (ddim.py:116-131), all fp32, n elements:
 *   e      = e_u + gs*(e_c - e_u)         (CFG; e_u may be NULL -> e = e_c)
 *   pred0  = (x - sqrt(1-a_t)*e) / sqrt(a_t)
 *   x_out  = sqrt(a_prev)*pred0 + sqrt(max(1-a_prev-sigma^2, 0))*e + sigma*z_i
 * z_i (drawn only for sigma > 0) is a standard normal that depends on (seed, index, i) alone: Philox4x32-10 with key
 * (seed & 0xffffffff, seed >> 32) and counter (c & 0xffffffff, c >> 32, index, 0), c = i/4, whose four words v0..v3
 * give elements 4c..4c+3 by Box-Muller on (v0, v1) and (v2, v3): u = (v + 0.5)*2^-32, r = sqrt(-2 ln u_a),
 * z = r cos(2 pi u_b), then r sin(2 pi u_b).  With x = 0, e_c = 0, e_u = NULL and sigma = 1, x_out is z.
 * e_out (may be NULL) receives the post-CFG e.
 * ------------------------------------------------------------------------------------------- */
int idiff_ddim_update(const float* x, const float* e_c, const float* e_u, float gs, float a_t, float a_prev,
                      float sigma, unsigned long long seed, int index, float* e_out, float* x_out, long n,
                      void* stream);
/* out = mean over `count` latents given as an array of device pointers (plms_instance.py:135) */
int idiff_latent_mean(const float* const* xs_dev, int count, float* out, long n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * idiff_conv_in_select: the UNet's input conv (3x3, padding 1, 4 -> cout channels) with one of two
 * weight sets per image: the model's own or the SD1.5 conv that openaimodel.py:469-480 swaps in.
 *   out[b, y, x, n] = bias_s[n] + sum_{ky,kx,c} w_s[(ky*3 + kx)*4 + c][n] * x16[b, c, y+ky-1, x+kx-1]
 * s = flags[b] (0: w0/b0, else w1/b1; int32 in device memory), x16 = x rounded to the storage type
 * (zero outside the image), fp32 accumulation.  x fp32 NCHW (B, 4, H, W); w 16-bit [36, cout]
 * (tap-major, then input channel); b fp32 [cout]; out 16-bit NHWC [B*H*W, cout].  cout even, <= 1024.
 * ------------------------------------------------------------------------------------------- */
int idiff_conv_in_select(const float* x, const void* w0, const float* b0, const void* w1, const float* b1,
                         const int* flags, void* out, int batch, int h, int w, int cout, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Instance-isolation attention mask, host prep on the GPU
 * ------------------------------------------------------------------------------------------- */
/* utils/input.py:34-37,79 (get_attmask_w_box): att_masks[b, k, x1:x2, y1:y2] = 1 for every instance k < counts[b]
   with x1 = rint(box[0] * size) ... (numpy round-half-even, in double); boxes fp32 (B, max_objs, 4) xyxy in [0,1],
   att_masks fp32 (B, max_objs, size, size) fully written (zeros elsewhere).  Note the reference indexes the FIRST
   spatial axis with x: kept as is. */
int idiff_boxes_to_attmask(const float* boxes, const int* counts, float* att_masks, int batch, int max_objs, int size,
                           void* stream);
/* attention.py:203-247 as bit words: att_masks fp32 (B, n_objs <= 30, P) with P = size*size visual tokens ->
   mask_q uint32 [B][P]       = (bits k: att_masks[b,k,p] > 0) | bit 31
   mask_k uint32 [B][P + 4*n_objs + tail]: visual p: the same bits without bit 31; object tokens in the order
   [box | point | scribble | mask] (text_grounding_net.py:291-300): box / mask token k -> bit k, point / scribble
   tokens and the `tail` trailing tokens -> bit 31 (attend / attended by everything).
   A batch entry with active[b] == 0 (all-zero masks or drop_box_mask: attention.py:201) gets all-ones words. */
int idiff_attmask_words(const float* att_masks, const int* active, void* mask_q, void* mask_k, int batch, int n_objs,
                        int pixels, int tail, void* stream);

/* timestep_embedding (util.py:160-180): out fp16 [B, dim] = [cos(t*f) | sin(t*f)],
   f_k = exp(-ln(1e4)*k/(dim/2)) */
int idiff_timestep_embedding(const float* t, void* out, int batch, int dim, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ConvNeXt mask encoder of UniFusion (mask conditioning; runs once per sample).  The pointwise and
 * strided convolutions are idiff_gemm calls (IDIFF_EPI_GELU for pwconv1); these are the other pieces.
 * ------------------------------------------------------------------------------------------- */
/* text_grounding_net.py:227-228: y = Conv2d(cin,3,3,1,1)(F.interpolate(segs, out_size, "nearest")) as
   NHWC fp16 (B, out_size, out_size, 3); seg_sum[b] = sum of the resized masks (the `> 0` test of :279).
   segs: fp32 (B, cin, in_size, in_size) with element strides `strides[4]` (host array; expanded / zero
   strides allowed); w: fp32 [3][cin][3][3]; bias fp32 [3]. */
int idiff_segs_inconv(const float* segs, const long* strides, const float* w, const float* bias, void* y,
                      float* seg_sum, int batch, int cin, int in_size, int out_size, void* stream);
/* NHWC fp16 (B,H,W,C) -> rows [B*(H/p)*(W/p), p*p*C], column (ky*p+kx)*C + c: the operand of the kernel-p,
   stride-p convolutions (convnext.py:71-81) run as GEMMs */
int idiff_patchify(const void* x, void* y, int batch, int h, int w, int c, int p, void* stream);
/* depthwise 7x7, padding 3 (convnext.py:28) on NHWC fp16; w fp32 [49][C] (tap-major), bias fp32 [C] */
int idiff_dwconv7x7(const void* x, const float* w, const float* bias, void* y, int batch, int h, int w_, int c,
                    void* stream);
/* text_grounding_net.py:229-230,277-285: out[b*T+t, r] = seg_sum[b] > 0 ? feat_nchw_flat[b][r*T+t] + pos[t,r]
   : null_pos[t,r], feat given as NHWC fp16 [B, P, C]; F = C*P/T features per token */
int idiff_seg_tokens(const void* feat, const void* null_pos, const float* pos, const float* seg_sum, void* out,
                     int batch, int pixels, int channels, int tokens, void* stream);

/* y = x * sigmoid(x) on fp16 (the nn.SiLU in front of ResBlock.emb_layers, openaimodel.py:200, when
   a ResBlock is driven through its module-level forward; the UNet path fuses it into a GEMM epilogue) */
int idiff_silu_f16(const void* x, void* y, long n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * First-stage decoder (AutoencoderKL.decode, ldm/models/autoencoder.py:33-37; Decoder, model.py:462-569):
 * convolutions / 1x1 projections are idiff_gemm calls, GroupNorm+swish idiff_groupnorm; these are the rest.
 * ------------------------------------------------------------------------------------------- */
/* autoencoder.py:34-35: y = post_quant_conv(z * inv_scale) (1x1, channels -> channels; w fp32 [C][C], bias [C])
   from fp32 NCHW (B, C, HW) to fp16 NHWC [B*HW, 64] (channels >= C zero: the conv3x3 operand granularity) */
int idiff_vae_latent_in(const float* z, const float* w, const float* bias, float inv_scale, void* out,
                        int batch, int channels, int hw, void* stream);
/* in-place softmax over the n columns of each of `rows` fp16 rows (row stride ld elements), fp32 arithmetic:
   the attention weights of AttnBlock (model.py:185-187); the 1/sqrt(c) scale is folded into the q projection */
int idiff_softmax_rows(void* x, int rows, int n, long ld, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CLIP text encoder (host prep, SURVEY.md section 8f-3): the per-phrase pooled feature of
 * utils/model.py:130-152 (get_clip_feature -> text_model pooler_output) and the prompt context of
 * ldm/modules/encoders/modules.py:144-172 (FrozenCLIPEmbedder -> last_hidden_state); both are Hugging Face
 * CLIPTextModel (transformers 4.27, requirements.txt:247).  Its linear layers are idiff_gemm calls (QuickGELU =
 * SiLU epilogue on weights pre-scaled by 1.702), its LayerNorms idiff_layernorm; these are the rest.
 * ------------------------------------------------------------------------------------------- */
/* out[r] = tok_table[ids[r]] + pos_table[r % tokens_per_seq]; ids int64 [rows] (clamped to the table), tables and
   out in the 16-bit storage type, [*, channels] row-major, channels % 8 == 0 */
int idiff_embed_tokens(const long long* ids, const void* tok_table, const void* pos_table, void* out, int rows,
                       int tokens_per_seq, int vocab, int channels, void* stream);
/* out = softmax(q k^T scale + causal mask) v per (sequence, head) for sequences of <= 128 tokens, head_dim 64.
   q / k / v: 16-bit [batch*tokens, >= heads*head_dim] with the common row stride ld_qkv (the fused QKV GEMM output);
   out [batch*tokens, heads*head_dim], row stride ld_out.  key_len (optional, int32 [batch]): keys at positions
   >= key_len[b] are padding and masked in addition to the causal mask. */
int idiff_causal_attention_small(const void* q, const void* k, const void* v, void* out, const int* key_len,
                                 int ld_qkv, int ld_out, int batch, int tokens, int heads, int head_dim, float scale,
                                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* IDIFF_B200_H */
