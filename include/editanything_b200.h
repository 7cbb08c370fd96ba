/* editanything_b200.h — C ABI of libea_b200.so (H100 / sm_90a only).
 *
 * The reference (sail-sg/EditAnything @ 8d2db4ae) is pure Python and has no FFI, plugin or
 * operator-registration interface (SURVEY.md §2, §8b): its hot path bottoms out in torch.nn
 * modules.  This header is therefore the boundary a maintainer would bind INSTEAD of those
 * torch.nn calls: one entry point per fused operator of the per-step network
 * (ControlNet(s) -> UNet -> CFG -> DDIM) and of the SAM ViT-H image encoder.  Each entry point
 * cites the reference function whose arithmetic it replaces (paths relative to the reference
 * root).  INTEGRATION.md shows the ctypes binding and where each call slots into the reference.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary
 *   - all tensor pointers are DEVICE pointers owned by the caller
 *   - activations are channels-last: images are NHWC [B, H, W, C], token matrices are [M, C]
 *   - "half" means the library storage type reported by ea_dtype_name(): "float16" (default
 *     build) or "bfloat16" (-DEA_USE_BF16); accumulation is always fp32
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*), never
 *     synchronises, never allocates, never throws; returns 0 or a negative ea_status
 *   - not re-entrant per stream; one process per GPU
 */
#ifndef EDITANYTHING_B200_H
#define EDITANYTHING_B200_H

#ifdef __cplusplus
extern "C" {
#endif

enum ea_status {
  EA_OK = 0,
  EA_ERR_ARG = -1,    /* null pointer / bad enum */
  EA_ERR_SHAPE = -2,  /* unsupported shape or alignment */
  EA_ERR_TMAP = -3,   /* cuTensorMapEncodeTiled failed */
  EA_ERR_CUDA = -4,   /* launch / runtime error */
  EA_ERR_NODRIVER = -5
};

enum ea_gemm_mode { EA_GEMM_LINEAR = 0, EA_GEMM_CONV_S1 = 1, EA_GEMM_CONV_S2 = 2, EA_GEMM_CONV_S2A = 3 };
enum ea_act { EA_ACT_NONE = 0, EA_ACT_SILU = 1, EA_ACT_GELU = 2, EA_ACT_GEGLU = 3 };

/* ---- library ---------------------------------------------------------------------------- */
int ea_version(void);
const char* ea_dtype_name(void);      /* "float16" | "bfloat16" */
const char* ea_strerror(int status);
/* The CUDA error (name, message, call site) behind the most recent EA_ERR_CUDA status of ea_gemm; "" if none. */
const char* ea_last_error(void);
int ea_init(void);                    /* resolves cuTensorMapEncodeTiled; 0 on success */
long long ea_launch_count(void);      /* kernels launched by this library since reset */
void ea_set_pdl(int on);              /* programmatic dependent launch between consecutive kernels
                                         (default on; env EA_PDL=0 disables) */
void ea_reset_launch_count(void);

/* ---- ea_gemm: wgmma GEMM / implicit-GEMM convolution --------------------------------------
 * out[M,N] = epilogue( A[M,K] * W[N,K]^T )
 * Replaces: nn.Linear / 1x1 nn.Conv2d / 3x3 nn.Conv2d (stride 1 and 2, pad 1) of
 *   ResBlock._forward            ldm/modules/diffusionmodules/openaimodel.py:254-274
 *   Downsample.forward           ldm/modules/diffusionmodules/openaimodel.py:133-159
 *   Upsample.forward (conv part) ldm/modules/diffusionmodules/openaimodel.py:90-118
 *   CrossAttention to_q/k/v/out  ldm/modules/attention.py:154-161,166-194
 *   GEGLU / FeedForward          ldm/modules/attention.py:49-76
 *   SpatialTransformer proj_in/out  ldm/modules/attention.py:296-318
 *   ControlNet zero convs        cldm/cldm.py:281-282,293-303
 *   SAM ViT-H qkv / proj / MLP / neck (segment_anything image_encoder, SURVEY.md App. C)
 * mode LINEAR : A is [M, lda] half.
 * mode CONV_S1: A is NHWC [Bsz, H, W, Cin] (pixel stride lda elements, default Cin), M = Bsz*H*W,
 *               W is [N, 9*Cin (+Cin_extra)] with K index = (kh*3+kw)*Cin + c.
 *               a_extra (optional): NHWC [Bsz,H,W,Cin_extra] raw block input whose 1x1
 *               skip-connection conv is folded in as extra K columns (openaimodel.py:233-240).
 * mode CONV_S2: A is NHWC [Bsz, 2H, 2W, Cin]; H, W are the OUTPUT size.
 * mode CONV_S2A: as CONV_S2 but padded (0,1,0,1) instead of 1 all round - the VAE encoder's Downsample
 *   (ldm/modules/diffusionmodules/model.py:79-86: F.pad(x, (0,1,0,1)) then a stride-2 pad-0 conv).
 * Epilogue order: +bias[n] -> +rowvec[batch(m), n] -> act -> *out_scale -> +residual[m,n]
 *                 -> (+= out[m,n] if accumulate) -> store out (and out2).
 * act GEGLU: W rows must be pre-interleaved per 128-row block as [64 value rows | 64 gate rows];
 *            output has N/2 columns: value * gelu(gate)   (attention.py:54-56).  Its epilogue applies the bias
 *            and the LayerNorm fold only: rowvec, residual, out2, out_f32, accumulate, row_scale and
 *            out_scale != 1 are rejected (EA_ERR_ARG).
 * Split-K: when the output has fewer tiles than the GPU has SMs, K is split across CTAs; each
 *            split CTA publishes its fp32 partial tile to `workspace`, waits for its siblings
 *            (all resident by construction) and finishes a 1/splits share of the tile with the
 *            full fused epilogue — deterministic summation order, no extra launch.  A split grid larger than
 *            the GPU's SMs (forced test configurations) is EA_ERR_SHAPE, before any launch.
 * Constraints: N % 8 == 0, K % 8 == 0, Cin % 64 == 0, all leading dims % 8 == 0,
 *              pointers 16-byte aligned.  Leading dims cover a whole row: LINEAR lda >= K; CONV lda (if set)
 *              >= Cin and ld_extra (if set) >= Cin_extra; ldw (if set) >= total K; ldo, ldo2 and ldr >= the
 *              output width (N, N/2 for GEGLU).  Anything else is EA_ERR_SHAPE, before any launch.
 */
#define EA_GEMM_MAX_PREFETCH 3
typedef struct ea_gemm_args {
  int mode;
  int M, N, K;               /* K used by LINEAR only */
  const void* a;             /* half */
  long long lda;             /* LINEAR: row stride; CONV: pixel stride (0 -> Cin) */
  const void* w;             /* half [N, ldw] */
  long long ldw;             /* 0 -> total K */
  int Bsz, H, W, Cin;        /* CONV: output spatial size, input channels */
  const void* a_extra;       /* CONV_S1 only, optional */
  int Cin_extra;
  long long ld_extra;
  const float* bias;         /* [N] fp32 or NULL */
  const float* rowvec;       /* [batches, rowvec_ld] fp32 or NULL (time-embedding add) */
  int rowvec_ld;
  int rows_per_batch;        /* LINEAR: rows per batch element for rowvec (0 -> batch 0) */
  const void* residual;      /* half [M, ldr] or NULL */
  long long ldr;
  void* out;                 /* half [M, ldo] */
  long long ldo;
  void* out2;                /* optional second destination (skip-concat slot) */
  long long ldo2;
  float* out_f32;            /* if non-NULL, write fp32 [M, ldo] here instead of out */
  int act;
  float out_scale;           /* set 1.0f when unused */
  int accumulate;
  int force_bn;              /* 0 = auto; else 32/64/128 (testing); any other width is EA_ERR_SHAPE */
  int force_splits;          /* 0 = auto; 1 = never split K; n = split K n ways (testing) */
  int force_2cta;            /* row tiles per CTA: 1 = two vertically adjacent 128-row tiles sharing each W stage,
                                -1 = one, 0 = the planner's choice (testing) */
  int force_persistent;      /* > 0: one CTA per SM walks the tile list (no split-K); 0 / -1 = one tile per CTA */
  /* LayerNorm folded into the GEMMs around it (BasicTransformerBlock norm1/2/3, ldm/modules/attention.py:
   * 263-275): LN(x) W^T = rstd[m] * (x (W*gamma)^T - mean[m] * g) + (W beta + b), g[n] = sum_k (W*gamma)[n,k].
   * The GEMM that PRODUCES x (proj_in / to_out + residual) also writes per-row partial statistics of the
   * values it stores (after rounding to the storage type), one pair per 32-column chunk j: (s_j = sum, M2_j = sum of
   * (x - s_j / 32)^2), rowstats_out fp32 [N/32][M][2] (deterministic: no atomics).  The GEMM that CONSUMES x
   * (to_q/k/v, GEGLU proj) takes W*gamma as `w`, W beta + b as `bias`, and ln_stats (= the producer's
   * rowstats_out, ln_parts = K/32 chunks), ln_g, ln_eps: it merges the partials in chunk order, about the first
   * chunk's mean, and its epilogue applies rstd / mean per output row.  LINEAR mode, no rowvec / rows_per_batch /
   * out_f32 / accumulate / row_scale, N % 32 == 0 and no GEGLU for the producer; K is never split for either.
   * No LayerNorm launch and no normalised tensor exists. */
  float* rowstats_out;
  const float* ln_stats;
  const float* ln_g;         /* fp32 [N] */
  int ln_parts;
  float ln_eps;
  const float* row_scale;    /* optional fp32 [M]: out row m is multiplied by row_scale[m] after act / out_scale and
                                before residual / accumulate - the spatial `conditioning_scale` map of
                                ControlNetModel2.forward (utils/stable_diffusion_controlnet.py:789-802), resized to
                                the residual's resolution, as a factor of the zero-conv accumulation */
  const void* prefetch[3];     /* optional L2 prefetch hints: up to EA_GEMM_MAX_PREFETCH ranges of device memory that a LATER */
  long long prefetch_bytes[3]; /* launch will read (its weights) - the first CTAs of this launch issue
                                  cp.async.bulk.prefetch.L2 over them while they work, so HBM streams the next layer's
                                  weights into the 50 MB L2 behind this layer's math.  Never changes results.
                                  NULL / 0 = unused slot. */
  void* workspace;           /* optional device scratch for split-K (small-M, weight-bound layers): */
  long long workspace_bytes; /* first 64 KB = int counters that MUST be zero before the first use
                                (the kernel re-zeroes them), rest = fp32 partial tiles.  NULL => K
                                is never split.  One workspace may serve every call on a stream. */
} ea_gemm_args;
int ea_gemm(const ea_gemm_args* args, void* stream);
/* ea_gemm_grouped: n_groups (1..3) problems of the SAME shape, epilogue flags and force_* fields - only the
 * pointers (and leading dimensions, out_scale) differ - as ONE launch: the UNet encoder and the ControlNets are the
 * same network with different weights applied to the same latent (cldm/cldm.py:22-45 vs 284-305), so every layer of
 * the three runs as one grid three times as large instead of three latency-bound launches.  The launch plan is
 * chosen once for all groups; args[0].workspace serves every group.  ea_gemm(a, s) == ea_gemm_grouped(a, 1, s).
 * Not re-entrant: one caller per process at a time (host-side staging of the parameter block is static). */
int ea_gemm_grouped(const ea_gemm_args* args, int n_groups, void* stream);
/* Diagnostic (no GPU needed): the launch plan ea_gemm would choose for m_tiles x N with k_blocks
 * 64-wide K-blocks: out5 = {BN, stages, splits, k_blocks_per_split, CTAs_per_SM}. */
int ea_gemm_plan(int m_tiles, int N, int k_blocks, int act, long long workspace_bytes, int n_sm,
                 int* out5);

/* ---- ea_attention: fused softmax(Q K^T * scale [+ rel-pos bias]) V -------------------------
 * Replaces CrossAttention.forward core  ldm/modules/attention.py:170-193 (QK^T in fp32,
 * softmax, PV) and SAM Attention.forward (decomposed rel-pos, SURVEY.md App. C).
 * q: [B, Nq, heads, d] with strides (q_bs, q_ns, d) elements; k, v likewise with Nkv rows;
 * out: [B, Nq, heads*d] contiguous rows of stride o_ns.  d % 8 == 0, d <= 512 (EA_ERR_SHAPE above, before any
 * launch); d <= 192 runs 128-row query tiles, 192 < d <= 512 (the VAE AttnBlock's one head of 512) a kernel of
 * 64-row query tiles and 32-key K / V tiles.  scale > 0 (finite).
 * rel_h / rel_w (optional, fp32 [B*heads, Nq, rel_s]): bias[q, kk] = rel_h[q, kk / rel_s] +
 * rel_w[q, kk % rel_s] added to the scaled logits (SAM add_decomposed_rel_pos).  With them, Nkv <= rel_s * rel_s
 * (else EA_ERR_SHAPE), and 128 rows of rel_w must fit in shared memory next to the K / V tiles; d > 192 with them
 * is EA_ERR_SHAPE.
 */
typedef struct ea_attn_args {
  const void* q; const void* k; const void* v; void* out;
  int B, heads, Nq, Nkv, d;
  long long q_bs, q_ns, k_bs, k_ns, v_bs, v_ns, o_bs, o_ns;  /* batch / row strides (elements) */
  float scale;
  const float* rel_h; const float* rel_w; int rel_s;
} ea_attn_args;
int ea_attention(const ea_attn_args* args, void* stream);

/* ---- normalisation ------------------------------------------------------------------------
 * ea_groupnorm: GroupNorm32 (fp32 statistics) + optional SiLU on NHWC half.
 *   Replaces normalization()+SiLU  openaimodel.py:196-200,216-219 ; util.py:217-219 ;
 *   Normalize (eps 1e-6)  attention.py:88-89.
 *   x may be a channel-concatenation of two tensors x[.., 0:C1] ++ x2[.., 0:C-C1]
 *   (skip-concat, cldm/cldm.py:39-41); pass x2 = NULL for a single source.
 *   One launch: the CTAs of an image publish partial sums and wait for each other (all resident: B <= SMs, at most
 *   SMs / B CTAs per image) before normalising.
 * ea_layernorm: nn.LayerNorm over the last dim of [M, C]  (attention.py:263-265).
 */
#define EA_GN_WS_FLOATS(B, groups) (2 * (B) + 2 * (groups) * 256)
typedef struct ea_gn_args {
  const void* x; long long ldx; int C1;
  const void* x2; long long ldx2;
  const float* gamma; const float* beta;
  void* out; long long ldo;
  int B, HW, C, groups;
  float eps; int silu;
  float* workspace;          /* >= 2*B + 2*groups*256 floats (EA_GN_WS_FLOATS), ZERO before the first call (the
                                kernel leaves its counters zero); one workspace may serve every call on a stream.
                                Layout: [B][2] int arrival counters, then one slot of 2*groups partial sums per
                                (image, CTA) - no floating-point atomics: results are bit-reproducible */
  int n_nets;                /* 0 / 1: one gamma / beta for all B images.  2 / 3: the images are n_nets stacked
                                batches of B / n_nets (the same layer of the UNet encoder and the ControlNets,
                                see ea_gemm_grouped); batch g > 0 uses gamma_more[g-1] / beta_more[g-1] */
  const float* gamma_more[2];
  const float* beta_more[2];
} ea_gn_args;
int ea_groupnorm(const ea_gn_args* args, void* stream);
int ea_layernorm(const void* x, long long ldx, const float* gamma, const float* beta, void* out,
                 long long ldo, int M, int C, float eps, void* stream);
/* LayerNorm2d over channels of NHWC == ea_layernorm on [B*H*W, C]. */

/* ---- small / memory-bound operators -------------------------------------------------------
 * ea_conv_direct: generic small 3x3 / 1x1 conv on CUDA cores (NHWC half, fp32 weights
 *   [kh, kw, Cin, Cout]), pad = ksize/2, stride 1 or 2, optional SiLU, optional dense half `add`
 *   tensor (ControlNet: h = conv_in(x) + guided_hint, cldm/cldm.py:293-297), output pixel stride
 *   ldo (0 -> Cout).  Used for the ControlNet hint stack (cldm/cldm.py:147-163) and conv_in
 *   4->320 (openaimodel.py:533-539).
 * ea_upsample2x: nearest x2 on NHWC (openaimodel.py:110-116).
 * ea_small_linear: y[M<=16, N] = act_out( W[N,K] * act_in(x[M,K]) + b ), fp32 in/out, half
 *   weights; time_embed and ResBlock.emb_layers (openaimodel.py:526-531,204-210).
 * ea_timestep_embedding: util.py:154-174 (cos | sin, max_period 10000).
 */
int ea_conv_direct(const void* x, const float* w, const float* bias, void* out, int B, int Hin,
                   int Win, int Cin, int Cout, int ksize, int stride, int silu,
                   const void* add, long long ldo, void* stream);
/* ea_conv_in: 3x3 stride-1 pad-1 conv with Cin in {4, 8} (UNet / ControlNet conv_in 4->320,
 *   openaimodel.py:533-539): x NHWC half [B,H,W,Cin], w fp32 [3,3,Cin,Cout], out NHWC half with pixel
 *   stride ldo (0 -> Cout); out2 (optional) receives the same values (UNet skip-concat slot); add
 *   (optional) dense half [B,H,W,Cout] added before the store (ControlNet guided hint, cldm/cldm.py:293-297). */
int ea_conv_in(const void* x, const float* w, const float* bias, void* out, long long ldo,
               void* out2, long long ldo2, const void* add, int B, int H, int W, int Cin, int Cout,
               void* stream);
int ea_upsample2x(const void* x, void* out, int B, int H, int W, int C, void* stream);
int ea_small_linear(const float* x, const void* w, const float* bias, float* y, int M, int N,
                    int K, int silu_in, int silu_out, void* stream);
int ea_timestep_embedding(const float* t, float* out, int B, int dim, void* stream);

/* ---- ea_out_cfg_ddim: final conv + classifier-free guidance + DDIM update ------------------
 * Replaces UNetModel.out conv (openaimodel.py:726-730) on the already GroupNorm+SiLU'd input,
 * the CFG combine (cldm/ddim_hacked.py:192; utils/stable_diffusion_controlnet_inpaint.py:1627-1631),
 * the DDIM eta=0 update (cldm/ddim_hacked.py:203-231) and the inpaint latent blend
 * (utils/stable_diffusion_controlnet_inpaint.py:1647-1656) in one launch.
 * xn: NHWC half [2*Nimg, H, W, C] (first Nimg = unconditional, last Nimg = conditional);
 * w: fp32 [4, 3, 3, C]; bias fp32 [4]; latents fp32 NHWC [Nimg, H, W, 4] updated in place;
 * eps_out (optional) fp32 [2*Nimg, H, W, 4] raw network output;
 * coef: device fp32 [16] = {sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev), k_init, k_noise, blend_on, mode,
 *   kx, kl, k1, k2, k0, px, p0, p1}.  mode 0: the DDIM update above.  mode 1 (with `hist`): a linear multistep
 *   predictor-corrector step - UniPCMultistepScheduler, the scheduler the reference installs on every pipeline
 *   (editany_lora.py:383,418): x0 = (x - coef[1] eps) / coef[0]; xc = kx x + kl last + k1 m1 + k2 m2 + k0 x0;
 *   x' = px xc + p0 x0 + p1 m1; then m2 <- m1, m1 <- x0, last <- xc, with hist = fp32 [3][Nimg,H,W,4] = {m1, m2, last}
 *   (the x0 predictions of the two previous steps and the previous corrected sample).  The coefficients depend on
 *   the timestep table only (editanything_b200/schedulers.py:coefficient_rows).
 * blend (optional): known fp32 NHWC [Nimg,H,W,4], mask fp32 [Nimg,H,W] (1 = keep known).  With `noise`
 *   (optional, fp32 like known) the kept region is add_noise(known, noise, t_next) = k_init * known +
 *   k_noise * noise (utils/stable_diffusion_controlnet_inpaint.py:1650-1656) and blend_on (0 / 1) gates the
 *   blend per step (the alignment_ratio window, :1648) - all per-step state is in `coef`.
 * lat_half_out (optional): half NHWC [2*Nimg,H,W,4] = updated latents duplicated for next step.
 * step_counter (optional): device int incremented by one (the captured-loop step index, see ea_step_gather).
 */
int ea_out_cfg_ddim(const void* xn, const float* w, const float* bias, float* latents,
                    float* eps_out, const float* coef, float guidance, const float* known,
                    const float* noise, const float* mask, void* lat_half_out, int* step_counter,
                    float* hist, int Nimg, int H, int W, int C, void* stream);
/* ea_out_ddim: ea_out_cfg_ddim without classifier-free guidance - the sampler's single network evaluation when
 * the guidance scale is <= 1 (utils/stable_diffusion_controlnet_inpaint.py:1329,1541-1544,1627-1631 skipped;
 * cldm/ddim_hacked.py:187-188): the update reads eps itself.  Same coef modes, history, blend and step counter as
 * ea_out_cfg_ddim, but every buffer holds the Nimg images once: xn NHWC half [Nimg, H, W, C], eps_out (optional)
 * fp32 [Nimg, H, W, 4], lat_half_out (optional) half [Nimg, H, W, 4]; latents / known / noise / mask / hist as above.
 * Nimg may be any count >= 1 (with latents == NULL: the eps of any batch). */
int ea_out_ddim(const void* xn, const float* w, const float* bias, float* latents, float* eps_out,
                const float* coef, const float* known, const float* noise, const float* mask,
                void* lat_half_out, int* step_counter, float* hist, int Nimg, int H, int W, int C, void* stream);
/* ea_out_cfg_vpred / ea_out_vpred: ea_out_cfg_ddim / ea_out_ddim for a v-prediction base model (the network predicts
 * v = sqrt(a_t) eps - sqrt(1-a_t) x0, e.g. stabilityai/stable-diffusion-2-1 at 768x768; cldm/ddim_hacked.py:194-217,
 * ldm/models/diffusion/ddpm.py:290-302).  Same arguments and buffers.  m = the network output after the guidance
 * combine (guided: applied to v, :190-192), then x0 = coef[0] x - coef[1] m and eps = coef[0] m + coef[1] x;
 * mode 0: x' = coef[2] x0 + coef[3] eps; mode 1: x0 enters the multistep recurrence above unchanged.  Blend,
 * history, lat_half_out and the step counter are as above; eps_out (optional) is the raw network output (v). */
int ea_out_cfg_vpred(const void* xn, const float* w, const float* bias, float* latents,
                     float* eps_out, const float* coef, float guidance, const float* known,
                     const float* noise, const float* mask, void* lat_half_out, int* step_counter,
                     float* hist, int Nimg, int H, int W, int C, void* stream);
int ea_out_vpred(const void* xn, const float* w, const float* bias, float* latents, float* eps_out,
                 const float* coef, const float* known, const float* noise, const float* mask,
                 void* lat_half_out, int* step_counter, float* hist, int Nimg, int H, int W, int C, void* stream);

/* ---- ea_latent_mix: alpha-mixing of the latents with the re-noised source -------------------------
 * The per-step mix of the alpha-mixing inpaint pipeline (utils/stable_diffusion_controlnet_inpaint.py:2039-2051),
 * launched after ea_out_* (run with its own blend off) in the same step.  Row r = *step_counter - 1 of the tables is
 * the step that epilogue just finished (it advanced the counter); with r outside [0, n_rows) nothing is touched.
 * latents fp32 NHWC [Nimg, H, W, 4], updated in place; known fp32 [Nimg, H, W, 4] (the source image latents);
 * mask fp32 [Nimg, H, W] (1 = keep the source); noise fp32 [n_rows][Nimg, H, W, 4] (row r read only when row r
 * of mix is active); mix fp32 [n_rows][4] = {k_init, k_noise, in_window, active}.  For an active row:
 *   p = k_init * known + k_noise * noise[r]          (add_noise(init, noise, t_{r+1}))
 *   x = m * (in_window != 0 ? p : x) + (1 - m) * ((1 - alpha) x + alpha p)
 * lat_half_out (optional): half [copies * Nimg, H, W, 4], the updated latents written `copies` (1 or 2) times, the
 * next step's network input.  latents / known / noise 16-byte aligned and lat_half_out 8-byte aligned, else
 * EA_ERR_SHAPE; a NULL operand or copies not 1 or 2 is EA_ERR_ARG; both before any launch. */
int ea_latent_mix(float* latents, const float* known, const float* mask, const float* noise, const float* mix,
                  float alpha, const int* step_counter, int n_rows, void* lat_half_out, int copies, int Nimg,
                  int H, int W, void* stream);

/* ---- ea_step_gather: first kernel of a captured denoising step ---------------------------------
 * The loop of utils/stable_diffusion_controlnet_inpaint.py:1540-1656 changes only scalars from step to step
 * (scheduler coefficients, the timestep behind every ResBlock's emb_layers projection, openaimodel.py:204-210).
 * They live in device tables with one row per step; this launch copies row min(*step_counter, n_rows-1) of
 * each of the n_tables (<= EA_STEP_MAX_TABLES) fp32 tables src[k] (row_elems[k] floats per row) into dst[k],
 * the fixed buffers the rest of the step reads.  Host work per step: one CUDA-graph launch. */
#define EA_STEP_MAX_TABLES 8
int ea_step_gather(const int* step_counter, int n_rows, int n_tables, const float* const* src,
                   float* const* dst, const long long* row_elems, void* stream);

/* ---- SAM helpers ---------------------------------------------------------------------------
 * ea_sam_relpos: rel_h[bh, q, kh] = sum_c q[bh, q, c] * Rh[qh(q), kh, c] (and rel_w), the
 *   decomposed relative position terms of SAM attention (SURVEY.md App. C; HF modeling_sam.py
 *   :789-801).  q: [B, S*S, heads, d] (strides q_bs, q_ns); Rh, Rw: fp32 [S, S, d] (already
 *   gathered by get_rel_pos); outputs fp32 [B*heads, S*S, S].
 * ea_window_partition / ea_window_unpartition: [B,H,W,C] <-> [B*nW, ws, ws, C] with zero pad
 *   (modeling_sam.py:900-952).
 */
int ea_sam_relpos(const void* q, long long q_bs, long long q_ns, const float* Rh, const float* Rw,
                  float* rel_h, float* rel_w, int B, int heads, int S, int d, void* stream);
int ea_window_partition(const void* x, void* out, int B, int H, int W, int C, int ws,
                        void* stream);
int ea_window_unpartition(const void* xw, const void* residual, void* out, int B, int H, int W,
                          int C, int ws, void* stream);
/* ea_sam_patchify: im2col of PatchEmbed's Conv2d(3, C, kernel = stride = ps) (segment_anything
 *   image_encoder PatchEmbed; HF modeling_sam.py:97-129): fp32 NCHW [B,Cin,H,W] ->
 *   half [B*(H/ps)*(W/ps), Cin*ps*ps], K index = (c*ps + kh)*ps + kw (flattened conv weight).
 * ea_nhwc_to_nchw_f32: half NHWC [B,HW,C] -> fp32 NCHW [B,C,HW] (image-embedding layout handed
 *   to the mask decoder). */
int ea_sam_patchify(const float* img, void* out, int B, int Cin, int H, int W, int ps,
                    void* stream);
int ea_nhwc_to_nchw_f32(const void* x, float* out, int B, int HW, int C, void* stream);

/* ---- VAE decoder helpers (SURVEY.md 8f row N1; reference ldm/modules/diffusionmodules/model.py) ----
 * ea_softmax_rows: p[r, :] = softmax(s[r, :]) for fp32 logits [rows, cols] (row stride lds) -> half
 *   [rows, cols] (row stride ldp); cols % 4 == 0.  (The VAE AttnBlock now runs on ea_attention.)
 * ea_image_out: half NHWC rows of width ldx (first C channels used) -> fp32 NCHW [B, C, HW],
 *   out = clamp(x * scale + shift, lo, hi): decode_latents' (image / 2 + 0.5).clamp(0, 1)
 *   (utils/stable_diffusion_controlnet_inpaint.py:718-724) fused with the layout change. */
int ea_softmax_rows(const float* s, long long lds, void* p, long long ldp, int rows, int cols,
                    void* stream);
int ea_image_out(const void* x, long long ldx, float* out, int B, long long HW, int C, float scale,
                 float shift, float lo, float hi, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EDITANYTHING_B200_H */
