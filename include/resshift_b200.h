/* resshift_b200 — C ABI of the H100-native (sm_90a) ResShift denoising hot path.
 *
 * The reference (zsyOAOA/ResShift) is pure Python/PyTorch and has no FFI; its plugin mechanism is
 * `instantiate_from_config` on yaml `target:` strings (reference utils/util_common.py:19-29, used at
 * sampler.py:87-88).  The entry points below are what a binding for the hot path needs; each cites the
 * reference interface it stands in for.  Conventions:
 *   - every function returns 0 on success, a negative code on failure; rs_last_error() gives the
 *     message (thread-local).  Nothing throws or exits across the boundary.
 *   - the CALLER owns all device memory (weight arena, workspace, inputs, outputs).  The library never
 *     allocates or frees device memory and never synchronises the device implicitly; all work is
 *     enqueued on the stream passed in (a cudaStream_t cast to void*), and is graph-capturable.
 *   - pointers are raw device pointers unless the name says `host`.  Tensors at the boundary are
 *     contiguous fp32 NCHW, exactly what the reference module receives/returns.
 *   - one host thread per engine (the reference is one single-threaded process per GPU, sampler.py:66-77).
 *     Different engines may be driven from different host threads at the same time, on the same or on different
 *     devices (one-time per-device setup is thread-safe).
 *   - devices: an engine belongs to the CUDA device that is current at rs_unet_set_arena (device memory of another
 *     device is refused as its arena), and a plan to the device
 *     that is current at rs_plan_bind, which must be its engine's.  A plan runs on the device it was bound on: every
 *     entry point that enqueues work on a plan or its sampler (rs_plan_forward / _profile / _profile_ops / _probe,
 *     rs_sampler_run / _run_host, rs_vq_encode / _decode / _decode_code, rs_kl_encode / _decode, their _begin / _end
 *     halves, rs_vq_profile_ops)
 *     returns an error when another device is current, and the stream passed in must belong to that device.
 */
#ifndef RESSHIFT_B200_H
#define RESSHIFT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RS_MAX_LEVELS 8

/* Keyword arguments of UNetModelSwin.__init__ (reference models/unet.py:632-657) that shipped yaml
 * files vary.  The constructor options the shipped files leave at one value are in rs_unet_options.
 * Covered: dims = 2 (the struct has no field for it), cond_lq = True (the reference cannot run
 * cond_lq = False), any dropout (identity at inference), cond_mask with or without an LQ feature
 * extractor, window_size 8 or 16, head dims (swin_embed_dim / swin_heads) of 32 or 64.  Refused by
 * rs_unet_create / rs_unet_create_ex: any other window_size or head dim (the window-attention
 * kernels are instantiated for those four combinations). */
typedef struct rs_unet_config {
  int32_t image_size;
  int32_t in_channels;
  int32_t model_channels;
  int32_t out_channels;
  int32_t n_levels;
  int32_t channel_mult[RS_MAX_LEVELS];
  int32_t num_res_blocks[RS_MAX_LEVELS];
  int32_t n_attn;
  int32_t attention_resolutions[RS_MAX_LEVELS];
  int32_t swin_depth;
  int32_t swin_embed_dim;
  int32_t swin_heads;        /* swin_embed_dim / num_head_channels, or num_heads */
  int32_t window_size;
  float mlp_ratio;
  int32_t cond_mask;
  int32_t lq_size;
} rs_unet_config;

/* The remaining UNetModelSwin.__init__ options, each 0 or 1.  rs_unet_create uses the values of every
 * shipped yaml: {use_scale_shift_norm 1, resblock_updown 0, conv_resample 1, patch_norm 0}. */
typedef struct rs_unet_options {
  int32_t use_scale_shift_norm;   /* 0: ResBlock adds emb_layers(emb) to h before out_layers (unet.py:202-205) */
  int32_t resblock_updown;        /* 1: ResBlocks with down / up = True resample (unet.py:187-193)            */
  int32_t conv_resample;          /* 0: Downsample = 2x2 average pool, Upsample = nearest 2x, no conv         */
  int32_t patch_norm;             /* 1: GroupNorm32 after patch_embed.proj and patch_unembed.proj              */
} rs_unet_options;

/* Keyword arguments of UNetModel.__init__ (reference models/unet.py:373-393), the global-attention UNet.  x has
 * out_channels channels; the LQ image (3 channels) is concatenated to it, so in_channels - out_channels is 3 (lq at
 * the latent size) or 12 (lq at twice the latent size, through F.pixel_unshuffle(lq, 2), :569-573).  num_heads /
 * num_head_channels as in the reference (num_head_channels -1: num_heads heads; output blocks then have ONE head, since
 * the reference builds them without num_heads, :517-523).  Refused by rs_unetmodel_create, with the reason in the
 * message: head dims other than 32, 64 or 128, channel counts GroupNorm32 cannot split, any other in_channels. */
typedef struct rs_unetmodel_config {
  int32_t image_size;
  int32_t in_channels;
  int32_t model_channels;
  int32_t out_channels;
  int32_t n_levels;
  int32_t channel_mult[RS_MAX_LEVELS];
  int32_t num_res_blocks[RS_MAX_LEVELS];
  int32_t n_attn;
  int32_t attention_resolutions[RS_MAX_LEVELS];
  int32_t num_heads;
  int32_t num_head_channels;
  int32_t use_new_attention_order;
} rs_unetmodel_config;

/* Keyword arguments of UNetModelConv.__init__ (reference models/unet.py:1026-1040), the attention- and GroupNorm-free
 * UNet of ResBlockConv blocks (:914-1004).  As for UNetModel, x has out_channels channels and in_channels - out_channels
 * is 3 (lq at the latent size) or 12 (lq at twice it, pixel_unshuffle).  Refused by rs_unetconv_create, with the reason
 * in the message: dims != 2, cond_lq == 0, any other in_channels, channel counts the conv kernels cannot take
 * (model_channels * channel_mult not a multiple of 8).  Latent H and W must be multiples of 2^(n_levels - 1)
 * (rs_plan_create). */
typedef struct rs_unetconv_config {
  int32_t in_channels;
  int32_t model_channels;
  int32_t out_channels;
  int32_t n_levels;
  int32_t channel_mult[RS_MAX_LEVELS];
  int32_t num_res_blocks[RS_MAX_LEVELS];
  int32_t cond_lq;
  int32_t dims;
} rs_unetconv_config;

/* ``autoencoder.params`` of the shipped yaml files: VQModelTorch(ddconfig, n_embed, embed_dim)
 * (reference ldm/models/autoencoder.py:12-26; ddconfig -> ldm/modules/diffusionmodules/model.py:452-470,563-581).
 * The ddconfig keys that place attention blocks or change the resampling and the output are in rs_vq_options;
 * dropout is identity at inference. */
typedef struct rs_vq_config {
  int32_t embed_dim;
  int32_t n_embed;
  int32_t z_channels;
  int32_t in_channels;
  int32_t out_ch;
  int32_t ch;
  int32_t n_levels;
  int32_t ch_mult[RS_MAX_LEVELS];
  int32_t num_res_blocks[RS_MAX_LEVELS];
} rs_vq_config;

/* The remaining Encoder / Decoder options of ddconfig (reference ldm/modules/diffusionmodules/model.py:452-660), each
 * 0 or 1.  rs_vq_create / rs_kl_create use the values of every shipped config: no level attention, the mid-block
 * attention, conv resampling, no tanh.  Every attention block is AttnBlock (model.py:152-203; attn_type "vanilla" or
 * "vanilla-xformers", the same math and parameters) and runs in the GEMM + row-softmax form up to 8192 positions, in
 * the fused form above (128, 256 or 512 channels, H and W multiples of 8; rs_vq_plan_create refuses other levels). */
typedef struct rs_vq_options {
  int32_t enc_attn[RS_MAX_LEVELS];   /* 1: an AttnBlock after every ResnetBlock of encoder level i: the level's curr_res
                                        (resolution halved i times) is in attn_resolutions (model.py:491-498,543-546) */
  int32_t dec_attn[RS_MAX_LEVELS];   /* 1: the same after every ResnetBlock of decoder level i: curr_res =
                                        (resolution // 2^(L-1)) * 2^(L-1-i) is in attn_resolutions (model.py:596-616,643-646) */
  int32_t mid_attn;                  /* 0: attn_type "none", mid.attn_1 is nn.Identity (model.py:280-298)             */
  int32_t resamp_with_conv;          /* 0: Downsample = 2x2 average pool, Upsample = nearest 2x, no conv (model.py:51-88) */
  int32_t tanh_out;                  /* 1: the decoder's image is tanh(conv_out(h)) (model.py:658-659)                 */
} rs_vq_options;

typedef struct rs_engine rs_engine;     /* architecture + packed weights      */
typedef struct rs_plan rs_plan;         /* engine bound to (batch, H, W)      */
typedef struct rs_sampler rs_sampler;   /* plan + diffusion schedule (T steps) */

int rs_version(void);
const char* rs_last_error(void);

/* ---- denoiser: models.unet.UNetModelSwin (reference models/unet.py:603-912) ------------------ */
int rs_unet_create(const rs_unet_config* cfg, rs_engine** out);
int rs_unet_create_ex(const rs_unet_config* cfg, const rs_unet_options* opts, rs_engine** out);
/* models.unet.UNetModel (reference models/unet.py:346-601).  opts: use_scale_shift_norm, resblock_updown and
 * conv_resample as for UNetModelSwin; patch_norm must be 0.  The engine works with every entry point below
 * (parameters, plans, forward / profile / probe, samplers); rs_plan_forward's lq is [B, 3, H, W] or [B, 3, 2H, 2W]
 * as in_channels says, and mask must be NULL.  Its AttentionBlocks run unet_attn (rs_op_unet_attention). */
int rs_unetmodel_create(const rs_unetmodel_config* cfg, const rs_unet_options* opts, rs_engine** out);
/* models.unet.UNetModelConv (reference models/unet.py:1006-1181).  opts as for rs_unetmodel_create (patch_norm must be
 * 0); every entry point below works with it, with rs_plan_forward's lq and mask as for UNetModel.  Its ResBlockConv
 * blocks read every tensor raw and through SiLU: the producing conv / resample writes both (rs_conv_args.silu_out). */
int rs_unetconv_create(const rs_unetconv_config* cfg, const rs_unet_options* opts, rs_engine** out);
void rs_unet_destroy(rs_engine* e);
/* state_dict inventory (reference key names / shapes; utils/util_net.py:86-98 relies on them) */
int rs_unet_param_count(const rs_engine* e);
int rs_unet_param_info(const rs_engine* e, int index, char* name, size_t name_cap, int32_t shape[4],
                       int32_t* ndim, int32_t* is_buffer);
/* packed (kernel-native, fp16/fp32) weight arena */
size_t rs_unet_arena_bytes(const rs_engine* e);
int rs_unet_set_arena(rs_engine* e, void* arena_dev);
/* repack one fp32 parameter (device pointer, reference layout: OIHW / [O, I] / [C]) into the arena */
int rs_unet_load_param(rs_engine* e, const char* name, const float* src_dev, void* stream);

/* ---- plan: the forward pass for a fixed (batch, latent H, latent W) -------------------------- */
int rs_plan_create(rs_engine* e, int batch, int height, int width, rs_plan** out);
void rs_plan_destroy(rs_plan* p);
size_t rs_plan_workspace_bytes(const rs_plan* p);
int rs_plan_bind(rs_plan* p, void* workspace_dev);   /* builds TMA descriptors; cheap, host only */
int rs_plan_num_launches(const rs_plan* p);          /* kernels per forward                       */
/* UNetModelSwin.forward(x, timesteps, lq=None, mask=None) (reference models/unet.py:865-895).
 * x [B, in_ch, H, W]; timesteps [B] (fp32); lq [B, 3, lq_h, lq_w]; mask [B, 1, lq_h, lq_w] or NULL;
 * out [B, out_ch, H, W].  All fp32 device pointers. */
int rs_plan_forward(rs_plan* p, const float* x, const float* timesteps, const float* lq, const float* mask,
                    float* out, void* stream);
/* measurement aid: one forward with CUDA events around every operator.  ms_by_kind[4] = conv/linear GEMM,
 * GroupNorm, window attention, upsample; conv_flops = algorithmic 2*MACs executed by the GEMM kernel. */
int rs_plan_profile(rs_plan* p, const float* x, const float* timesteps, const float* lq, const float* mask,
                    double* ms_by_kind, double* conv_flops, int32_t* n_conv_launches, void* stream);
/* per-operator variant: ms[i] and desc[i*desc_stride] for the first `cap` operators of the forward program */
int rs_plan_profile_ops(rs_plan* p, const float* x, const float* timesteps, const float* lq, const float* mask,
                        double* ms, char* desc, int desc_stride, int cap, int32_t* n_ops, void* stream);
/* debugging aid: copy an intermediate block output ("input_blocks.3", "middle_block", "output_blocks.11"; in
 * first-stage plans each attention block's "<prefix>.in", ".norm", ".q", ".k", ".attn" and "<prefix>" itself, e.g.
 * "encoder.mid.attn_1.q", the decoder's "quantize" and "quantize.padded", the same with the zero channels that pad it to
 * a multiple of 8) as fp32 NCHW into dst (device); returns channel count through
 * *channels.  Valid right after a forward or pass only for blocks whose buffer is still live (all of them under
 * RS_NO_REUSE=1); used by the parity tests. */
int rs_plan_probe(rs_plan* p, const char* block, float* dst, int32_t* channels, int32_t* h, int32_t* w,
                  void* stream);

/* ---- sampler: SpacedDiffusion.p_sample_loop_progressive (reference models/gaussian_diffusion.py:421-472,
 *      p_sample :332-365, _scale_input :598-603, prior_sample :517-529; models/respace.py:43-63) ------ */
int rs_sampler_create(rs_plan* p, int steps, const double* sqrt_etas_host, double kappa,
                      const int32_t* timestep_map_host, rs_sampler** out);
/* What the denoiser predicts (create_gaussian_diffusion's predict_type, reference models/script_util.py:35-44) and
 * how its input is scaled (_scale_input, models/gaussian_diffusion.py:598-609).  The step turns the model output into
 * x0 (p_mean_variance :277-292): xstart x0 = out; residual x0 = z_y - out; epsilon x0 = (x_t - sqrt_eta kappa out -
 * eta z_y) / (1 - eta); epsilon_scale x0 = (x_t - out - eta z_y) / (1 - eta). */
typedef enum rs_mean_type {
  RS_MEAN_XSTART = 0, RS_MEAN_EPSILON = 1, RS_MEAN_EPSILON_SCALE = 2, RS_MEAN_RESIDUAL = 3
} rs_mean_type;
typedef struct rs_sampler_options {
  int32_t mean_type;          /* rs_mean_type */
  int32_t normalize_input;    /* 0: the denoiser sees x_t unscaled */
  int32_t latent_flag;        /* 1: x_t / sqrt(eta kappa^2 + 1); 0: x_t / (sqrt_eta kappa 3 + 1) */
} rs_sampler_options;
/* rs_sampler_create is rs_sampler_create_ex with {RS_MEAN_XSTART, 1, 1}.  Unknown mean types and flags other than 0 / 1
 * are refused. */
int rs_sampler_create_ex(rs_plan* p, int steps, const double* sqrt_etas_host, double kappa,
                         const int32_t* timestep_map_host, const rs_sampler_options* options, rs_sampler** out);
void rs_sampler_destroy(rs_sampler* s);
/* z_y [B, C, H, W] fp32 (x_start for a DDIM inversion sampler); noises [(T+1), B, C, H, W] fp32 in the reference's
 * draw order (prior first; a DDIM inversion sampler does not read it, and it may be NULL there);
 * lq/mask as in rs_plan_forward; out_latent [B, C, H, W] fp32 (the loop's final `sample`).
 * use_graph != 0 replays a CUDA graph captured on first use (same pointers required on later calls). */
int rs_sampler_run(rs_sampler* s, const float* z_y, const float* noises, const float* lq, const float* mask,
                   float* out_latent, int use_graph, void* stream);
/* Same call with HOST buffers (pinned or pageable): copies in, runs, copies the latent back, and
 * synchronises the stream.  This is the end-to-end entry the benchmark's `e2e` figure times. */
int rs_sampler_run_host(rs_sampler* s, const float* z_y_host, const float* noises_host, const float* lq_host,
                        const float* mask_host, float* out_latent_host, void* staging_dev, size_t staging_bytes,
                        int use_graph, void* stream);
size_t rs_sampler_staging_bytes(const rs_sampler* s);
/* optional taps for parity tests: per-step pred_xstart (the converted x0 whatever the mean type) / sample,
 * [T, B, C, H, W] fp32 device buffers or NULL */
int rs_sampler_set_taps(rs_sampler* s, float* pred_xstart_steps, float* sample_steps);

/* ---- DDPM / DDIM sampler: SpacedDiffusionDDPM.p_sample_loop / ddim_sample_loop (reference
 *      models/gaussian_diffusion.py:742-1147, models/respace.py:65-99) on the same plan and entry points -------------
 * x_T = noises[0] (no shift), then T x (denoiser forward on x_t unscaled + one step kernel).  The schedule comes in as
 * the process's float64 tables, rows of `steps` values in the order of rs_ddpm_table_row; the library rounds each to
 * fp32 (_extract_into_tensor) and keeps the log variance of options->var_type.  rs_sampler_run / _run_host / _set_taps /
 * _destroy work unchanged; z_y is not read and may be NULL.  rs_sampler_tables refuses these samplers. */
typedef enum rs_ddpm_kind { RS_DDPM_ANCESTRAL = 0, RS_DDPM_DDIM = 1 } rs_ddpm_kind;
/* The learned types (learn_sigma=True, reference models/script_util.py:87-88) take the log variance from the model's
 * second C output channels: LEARNED log_var = v; LEARNED_RANGE log_var = frac log(betas)[t] + (1 - frac)
 * posterior_log_variance_clipped[t] with frac = (v + 1) / 2 (models/gaussian_diffusion.py:772-786).  Value 2 is left
 * unassigned: it was refused as unknown before the learned types existed, and stays so. */
typedef enum rs_ddpm_var_type {
  RS_VAR_FIXED_LARGE = 0, RS_VAR_FIXED_SMALL = 1, RS_VAR_LEARNED_RANGE = 3, RS_VAR_LEARNED = 4
} rs_ddpm_var_type;
typedef enum rs_ddpm_table_row {
  RS_DDPM_SQRT_RECIP_ACP = 0,       /* sqrt(1 / alphas_cumprod)                                               */
  RS_DDPM_SQRT_RECIPM1_ACP = 1,     /* sqrt(1 / alphas_cumprod - 1)                                           */
  RS_DDPM_COEF1 = 2,                /* posterior_mean_coef1 (multiplies x0)                                   */
  RS_DDPM_COEF2 = 3,                /* posterior_mean_coef2 (multiplies x_t)                                  */
  RS_DDPM_LOGVAR_LARGE = 4,         /* log(append(posterior_variance[1], betas[1:]))  (FIXED_LARGE)           */
  RS_DDPM_LOGVAR_SMALL = 5,         /* posterior_log_variance_clipped                  (FIXED_SMALL)          */
  RS_DDPM_ACP = 6,                  /* alphas_cumprod                                                         */
  RS_DDPM_ACP_PREV = 7,             /* alphas_cumprod_prev                                                    */
  RS_DDPM_TABLE_ROWS = 8,
  RS_DDPM_ACP_NEXT = 8,             /* alphas_cumprod_next (0 at T - 1): read by rs_ddim_reverse_sampler_create only */
  RS_DDPM_LOG_BETAS = 8             /* log(betas): LEARNED_RANGE's max_log, read by rs_ddpm_sampler_create with that
                                       var_type only (its min_log is RS_DDPM_LOGVAR_SMALL)                         */
} rs_ddpm_table_row;
typedef struct rs_ddpm_options {
  int32_t kind;               /* RS_DDPM_ANCESTRAL or RS_DDPM_DDIM                                         */
  int32_t mean_type;          /* RS_MEAN_EPSILON or RS_MEAN_XSTART                                         */
  int32_t var_type;           /* rs_ddpm_var_type: the ancestral step's noise; DDIM ignores it but for the
                                 model output's width                                                      */
  int32_t clip;               /* 1: clamp x0 to [-1, 1] (clip_denoised)                                    */
  double eta;                 /* DDIM's eta >= 0 (the ancestral step ignores it)                           */
} rs_ddpm_options;
/* tables_host [RS_DDPM_TABLE_ROWS][steps] float64 ([RS_DDPM_TABLE_ROWS + 1][steps], the last row RS_DDPM_LOG_BETAS,
 * with RS_VAR_LEARNED_RANGE); timestep_map_host [steps] (the model's timesteps; NULL = 0 .. T-1).  A fixed var_type
 * needs a plan whose model outputs as many channels as x has, a learned one twice as many (the mean half, then the
 * variance half).  Refused, each with its reason: NULL tables or options, an unknown kind / var_type, a mean type other
 * than eps or x0, clip other than 0 / 1, a negative or non-finite eta, steps outside [2, the plan's FiLM rows], a model
 * output width that does not match var_type. */
int rs_ddpm_sampler_create(rs_plan* p, int steps, const double* tables_host, const int32_t* timestep_map_host,
                           const rs_ddpm_options* options, rs_sampler** out);

/* ---- DDIM inversion: SpacedDiffusionDDPM.ddim_reverse_sample (reference models/gaussian_diffusion.py:1030-1066) in
 *      a t = 0 .. T-1 loop, on the same plan and entry points --------------------------------------------------------
 * x = x_start, then for t = 0 .. T-1: denoiser forward on x (unscaled, FiLM row t) + one reverse step
 * x <- x0 sqrt(acp_next[t]) + sqrt(1 - acp_next[t]) eps'; out_latent receives x_T.  rs_sampler_run / _run_host read
 * x_start from z_y (required) and draw nothing: noises is not read and may be NULL.  _set_taps / _destroy work
 * unchanged; rs_sampler_tables refuses these samplers. */
typedef struct rs_ddim_reverse_options {
  int32_t mean_type;          /* RS_MEAN_EPSILON or RS_MEAN_XSTART                                         */
  int32_t clip;               /* 1: clamp x0 to [-1, 1] (clip_denoised)                                    */
} rs_ddim_reverse_options;
/* tables_host [RS_DDPM_TABLE_ROWS + 1][steps] float64: the rows of rs_ddpm_sampler_create, then RS_DDPM_ACP_NEXT;
 * timestep_map_host as there.  The plan's model may output C or 2C channels (a learned variance): the step reads the
 * first C only.  Refused, each with its reason: NULL tables or options, a mean type other than eps or x0, clip other
 * than 0 / 1, steps outside [2, the plan's FiLM rows], any other model output width. */
int rs_ddim_reverse_sampler_create(rs_plan* p, int steps, const double* tables_host, const int32_t* timestep_map_host,
                                   const rs_ddim_reverse_options* options, rs_sampler** out);

/* ---- VQ-GAN first stage: ldm.models.autoencoder.VQModelTorch (reference ldm/models/autoencoder.py:12-47) -------
 * The engine handle is the same opaque type as the denoiser's: rs_unet_param_count / _param_info / _arena_bytes /
 * _set_arena / _load_param work on it unchanged (state_dict names and shapes of the reference's VQModelTorch, so
 * autoencoder_vq_f4.pth / ffhq512_vq_f8_dim8_face.pth load as they are). */
int rs_vq_create(const rs_vq_config* cfg, rs_engine** out);
/* rs_vq_create is rs_vq_create_ex with the shipped options {0..., 0..., 1, 1, 0}.  Option flags other than 0 / 1 and an
 * attention level whose channels are not a multiple of 64 are refused. */
int rs_vq_create_ex(const rs_vq_config* cfg, const rs_vq_options* opts, rs_engine** out);
/* plan for a fixed (batch, image H, image W); which = 0: encode (image -> latent), 1: decode (latent -> image).
 * Uses rs_plan_workspace_bytes / rs_plan_bind / rs_plan_destroy like a denoiser plan. */
int rs_vq_plan_create(rs_engine* e, int batch, int image_h, int image_w, int which, rs_plan** out);
/* VQModelTorch.encode (autoencoder.py:28-31): x [B, 3, H, W] fp32 -> h [B, embed_dim, H/f, W/f] fp32 (f = 2^(levels-1)) */
int rs_vq_encode(rs_plan* p, const float* x, float* h_out, void* stream);
/* VQModelTorch.decode (autoencoder.py:33-40): h [B, embed_dim, H/f, W/f] -> quantize (VectorQuantizer2,
 * ldm/modules/vqvae/quantize.py:271-284; skipped when force_not_quantize) -> post_quant_conv -> Decoder -> [B, 3, H, W] fp32.
 * idx_out: optional [B, H/f, W/f] int32 code indices. */
int rs_vq_decode(rs_plan* p, const float* h, float* out, int32_t* idx_out, int force_not_quantize, void* stream);
/* Each pass split at its fused attentions (attention blocks over more than 8192 positions, in pass order 0 .. n-1), so
 * that the query rows of each can be computed by several devices and exchanged in between.  _begin runs the input stage
 * and every op up to and including fused attention 0 (the whole op list on plans without one); rs_vq_run_between(p, a)
 * runs the ops after fused attention a-1 up to and including fused attention a, 1 <= a < n; _end runs the rest and the
 * output stage (quant_conv / the copy of the image).  rs_vq_encode = rs_vq_encode_begin + rs_vq_run_between(1 .. n-1) +
 * rs_vq_encode_end, and so for the decode and KL passes: the same launches in the same order.  On a plan with two or
 * more fused attentions, rs_vq_run_between and _end refuse calls out of that order. */
int rs_vq_encode_begin(rs_plan* p, const float* x, void* stream);
int rs_vq_encode_end(rs_plan* p, float* h_out, void* stream);
int rs_vq_decode_begin(rs_plan* p, const float* h, int32_t* idx_out, int force_not_quantize, void* stream);
int rs_vq_decode_end(rs_plan* p, float* out, void* stream);
int rs_vq_run_between(rs_plan* p, int a, void* stream);       /* VQ-GAN and KL plans */
/* n = the number of fused attentions of the plan's pass (0 when every attention has 8192 positions or fewer) */
int rs_vq_attention_count(rs_plan* p, int32_t* n);
/* Query rows [row_begin, row_end) of every image that fused attention a computes (default [0, T), T = its H*W);
 * multiples of 64 inside [0, T].  An empty range skips the attention launch.  Rows outside the range keep whatever the
 * attention output view held (the caller writes them before the next segment of the pass runs). */
int rs_vq_set_attention_rows_at(rs_plan* p, int a, int row_begin, int row_end);
/* fused attention a's output as its proj_out reads it (bound plans): fp16, element (n, t, c) at
 * ptr + n * image_stride + t * row_stride + c (strides in elements), n < batch, t < T, c < C.  It holds the attention
 * result from the end of the segment that computes it until the next segment reads it; nothing else in the plan writes
 * it in between. */
int rs_vq_attention_output_at(rs_plan* p, int a, void** ptr, long long* row_stride, long long* image_stride, int32_t* T,
                              int32_t* C);
/* rs_vq_set_attention_rows_at / rs_vq_attention_output_at with a = 0 */
int rs_vq_set_attention_rows(rs_plan* p, int row_begin, int row_end);
int rs_vq_attention_output(rs_plan* p, void** ptr, long long* row_stride, long long* image_stride, int32_t* T, int32_t* C);
/* diagnostics: per-launch times (ms) and descriptions of the plan's op list on the inputs of the last encode/decode
 * call (counterpart of rs_plan_profile_ops for the first-stage plans); VQ-GAN and KL plans */
int rs_vq_profile_ops(rs_plan* p, double* ms, char* desc, int desc_stride, int cap, int32_t* n_ops, void* stream);
/* VQModelTorch.decode_code (autoencoder.py:42-45) on a decode plan: idx [B, H/f, W/f] int32 code indices -> the codebook
 * rows (quantize.embed_code) -> post_quant_conv -> Decoder -> out [B, 3, H, W] fp32; bit-identical to rs_vq_decode of
 * those rows with force_not_quantize.  An index outside [0, n_embed) gives NaN at its position (nothing is read out of
 * bounds). */
int rs_vq_decode_code(rs_plan* p, const int32_t* idx, float* out, void* stream);

/* ---- KL first stage: ldm.models.autoencoder.AutoencoderKLTorch (reference ldm/models/autoencoder.py:52-86) ----------
 * The same Encoder / Decoder as the VQ-GAN with double_z: encoder.conv_out has 2 z_channels, quant_conv is
 * [2 embed_dim, 2 z_channels, 1, 1], post_quant_conv [z_channels, embed_dim, 1, 1], no codebook (cfg->n_embed is
 * ignored).  Parameters, arena, plans (rs_vq_plan_create with which = 0 / 1), rs_vq_set_attention_rows,
 * rs_vq_attention_output and rs_vq_profile_ops work as for the VQ-GAN; the rs_vq_encode / _decode calls refuse KL
 * plans and the rs_kl_* calls refuse VQ-GAN plans. */
int rs_kl_create(const rs_vq_config* cfg, rs_engine** out);
/* rs_kl_create with rs_vq_options, as rs_vq_create_ex */
int rs_kl_create_ex(const rs_vq_config* cfg, const rs_vq_options* opts, rs_engine** out);
/* AutoencoderKLTorch.encode (autoencoder.py:65-76) with DiagonalGaussianDistribution
 * (ldm/modules/distributions/distributions.py:24-37,61-62): x [B, 3, H, W] fp32 -> moments = quant_conv(Encoder(x))
 * [B, 2 embed_dim, H/f, W/f]; mean, logvar = moments[:, :e], clamp(moments[:, e:], -30, 20);
 * z_out [B, embed_dim, H/f, W/f] = mean + exp(0.5 logvar) * noise (sample()), or mean when noise is NULL (mode()).
 * noise: [B, embed_dim, H/f, W/f] fp32 or NULL; moments_out: [B, 2 embed_dim, H/f, W/f] fp32 or NULL. */
int rs_kl_encode(rs_plan* p, const float* x, const float* noise_or_null, float* z_out, float* moments_out_or_null,
                 void* stream);
/* AutoencoderKLTorch.decode (autoencoder.py:78-81): z [B, embed_dim, H/f, W/f] -> post_quant_conv -> Decoder ->
 * out [B, 3, H, W] fp32 */
int rs_kl_decode(rs_plan* p, const float* z, float* out, void* stream);
/* each pass split at its fused attentions as the rs_vq_*_begin / rs_vq_run_between / _end calls are */
int rs_kl_encode_begin(rs_plan* p, const float* x, void* stream);
int rs_kl_encode_end(rs_plan* p, const float* noise_or_null, float* z_out, float* moments_out_or_null, void* stream);
int rs_kl_decode_begin(rs_plan* p, const float* z, void* stream);
int rs_kl_decode_end(rs_plan* p, float* out, void* stream);

/* ---- image edges of the sampler (reference sampler.py:176-223,286; utils/util_image.py:216-273,889-979) --------- */
/* F.interpolate(x, scale_factor=sf, mode='bicubic') on fp32 NCHW (models/gaussian_diffusion.py:503-504) */
int rs_op_bicubic_upsample(const float* x, int N, int C, int H, int W, int sf, float* y, void* stream);
/* uint8 HWC image(s) -> fp32 NCHW in [-1, 1]: (v / 255 - 0.5) / 0.5 */
int rs_op_ingest_u8(const void* src_u8_nhwc, int N, int H, int W, int C, float* dst_nchw, void* stream);
/* fp32 NCHW in [-1, 1] -> clamp, * 0.5 + 0.5, optional mask-back blend with lq (mask = 1 keeps the model output),
 * round(v * 255) -> uint8 HWC in RGB (bgr = 0) or BGR (bgr = 1) order (util_image.tensor2img) */
int rs_op_emit_u8(const float* sr_nchw, const float* lq_nchw_or_null, const float* mask_or_null, int N, int H, int W,
                  int bgr, void* dst_u8_nhwc, void* stream);
/* overlap-average of tiled results (ImageSpliterTh.update / gather): tiles [nty*ntx, N, C, th, tw] fp32 at output
 * origins ys[nty] / xs[ntx] (device int32 arrays) -> out [N, C, H, W] */
int rs_op_tile_gather(const float* tiles, int N, int C, int H, int W, int th, int tw, int nty, int ntx, const int32_t* ys,
                      const int32_t* xs, float* out, void* stream);

/* ---- single operators (unit tests / reuse) --------------------------------------------------- */
/* p_sample update (reference models/gaussian_diffusion.py:361-364 with :218-221) */
int rs_p_sample(const float* x_t, const float* x0_pred, const float* noise, float* x_next, float coef1,
                float coef2, float std, int t_is_zero, long long numel, void* stream);
/* The step the sampler's loop launches: x_next = coef1[t] x_t + coef2[t] x0 + [t != 0] std[t] noise, all [N, C, HW]
 * fp32, with the coefficients read from T-entry device tables at t.  With next_in (t > 0 only) it also writes
 * fp16(x_next * in_scale[t - 1]) into channels [0, C) of the next denoiser input [N*HW][next_cpad] and leaves every other
 * channel as it was; counters[0, n_counters) are zeroed (the next forward's GroupNorm arrival counters).  t outside
 * [0, T), next_cpad < C and more counters than launched threads are refused. */
typedef struct rs_p_sample_args {
  const float* x_t; const float* x0; const float* noise; float* x_next;
  const float* coef1; const float* coef2; const float* stdv; const float* in_scale;   /* [T] fp32 device tables */
  int32_t T, t, N, C, HW;
  void* next_in; int32_t next_cpad;             /* optional fp16 [N*HW][next_cpad]                                     */
  uint32_t* counters; int32_t n_counters;       /* optional                                                             */
} rs_p_sample_args;
int rs_op_p_sample_ex(const rs_p_sample_args* a, void* stream);
/* The same step from the raw model output of a mean type (rs_sampler_options): x0 is converted in registers in the
 * reference's operation order, every operation rounded in fp32 (eps_coef = fp32(sqrt_eta) * kappa, eta, one_minus_eta
 * = fp32(1 - eta): rs_schedule_tables_ex's rows), then stepped as rs_op_p_sample_ex does (no counters).  x0_out
 * (optional) receives x0.  Refused: an unknown mean type, y or a conversion table missing for a type that reads it, t
 * outside [0, T), next_cpad < C. */
typedef struct rs_p_sample_pred_args {
  const float* out; const float* x_t; const float* y; const float* noise; float* x_next;   /* [N, C, HW] fp32       */
  const float* coef1; const float* coef2; const float* stdv; const float* in_scale;          /* [T] fp32 device tables */
  const float* eps_coef; const float* eta; const float* one_minus_eta;                       /* [T] fp32 device tables */
  int32_t T, t, N, C, HW;
  int32_t mean_type;
  void* next_in; int32_t next_cpad;             /* optional fp16 [N*HW][next_cpad]                                     */
  float* x0_out;                                /* optional [N, C, HW] fp32                                            */
} rs_p_sample_pred_args;
int rs_op_p_sample_pred(const rs_p_sample_pred_args* a, void* stream);
/* The DDPM sampler's step kernel (rs_ddpm_sampler_create) on its own: x0 from the model output (eps or x0, clamped
 * with clip), then the ancestral or DDIM update, with the grid the loop launches.  Tables are [T] fp32 device arrays:
 * the ancestral step reads coef1, coef2 and log_var, DDIM acp and acp_prev, eps prediction (and DDIM) sqrt_recip_acp
 * and sqrt_recipm1_acp.  next_in (t > 0 only) receives fp16(x_next) in channels [0, C); counters as in
 * rs_op_p_sample_ex; x0_out (optional) receives x0.  Refused: a table the step reads missing, an unknown kind or mean
 * type, clip other than 0 / 1, a negative eta, t outside [0, T), next_cpad < C, more counters than launched threads.
 * The trailing fields describe a learned-variance output; zero / NULL is a [N, C, HW] output with log_var's variance.
 * out_sN (> 0) is out's image stride in elements: C * HW, or at least 2C * HW for a learned var_type, whose variance
 * half starts C * HW after the mean half.  var_type (ancestral only; DDIM reads the stride alone) is an
 * rs_ddpm_var_type: 0 / 1 read log_var, RS_VAR_LEARNED the variance half, RS_VAR_LEARNED_RANGE the variance half with
 * log_var as min_log and log_betas as max_log.  Refused as well: an unknown var_type, a learned one with a stride below
 * 2C * HW or a missing table, a fixed ancestral step at a stride other than C * HW, a DDIM stride below C * HW. */
typedef struct rs_ddpm_step_args {
  const float* out; const float* x_t; const float* noise; float* x_next;                     /* [N, C, HW] fp32       */
  const float* sqrt_recip_acp; const float* sqrt_recipm1_acp;                                /* [T] fp32 device tables */
  const float* coef1; const float* coef2; const float* log_var; const float* acp; const float* acp_prev;
  int32_t T, t, N, C, HW;
  int32_t kind, mean_type, clip;
  float eta;
  void* next_in; int32_t next_cpad;
  uint32_t* counters; int32_t n_counters;
  float* x0_out;
  int64_t out_sN;               /* 0: C * HW                                                                     */
  int32_t var_type;             /* rs_ddpm_var_type; 0 (FIXED_LARGE) and 1 both read log_var                      */
  const float* log_betas;       /* [T] fp32 device table: RS_VAR_LEARNED_RANGE only                              */
} rs_ddpm_step_args;
int rs_op_ddpm_step(const rs_ddpm_step_args* a, void* stream);
/* The DDIM inversion step (rs_ddim_reverse_sampler_create) on its own, with the grid the loop launches: x0 from the
 * model output (eps or x0, clamped with clip), eps' = (sqrt_recip_acp[t] x_t - x0) / sqrt_recipm1_acp[t], then
 * x_next = x0 sqrt(acp_next[t]) + sqrt(1 - acp_next[t]) eps'.  Tables are [T] fp32 device arrays.  next_in (t < T - 1
 * only) receives fp16(x_next) in channels [0, C); counters as in rs_op_p_sample_ex; x0_out (optional) receives x0.
 * Refused: a NULL table, an unknown mean type, clip other than 0 / 1, t outside [0, T), next_cpad < C, more counters
 * than launched threads.  out_sN (trailing; 0 = C * HW) is out's image stride in elements, at least C * HW: a
 * learned-variance model's [N, 2C, HW] output is read at 2C * HW, its variance half never. */
typedef struct rs_ddim_reverse_step_args {
  const float* out; const float* x_t; float* x_next;                                          /* [N, C, HW] fp32       */
  const float* sqrt_recip_acp; const float* sqrt_recipm1_acp; const float* acp_next;          /* [T] fp32 device tables */
  int32_t T, t, N, C, HW;
  int32_t mean_type, clip;
  void* next_in; int32_t next_cpad;
  uint32_t* counters; int32_t n_counters;
  float* x0_out;
  int64_t out_sN;
} rs_ddim_reverse_step_args;
int rs_op_ddim_reverse_step(const rs_ddim_reverse_step_args* a, void* stream);
/* The denoiser's input packing: out[N*HW][Cpad] fp16 = cat([fp16(x * scale_tab[scale_idx]), lq, mask], channels) + zero
 * padding (scale 1 without scale_tab).  lq is one of: lq_nchw [N, Cl, HW] fp32 (optionally followed by mask_nchw
 * [N, 1, HW]); lq_nchw [N, Cl / 4, 2H, 2W] packed as pixel_unshuffle(lq, 2) (lq_unshuffle, W = the latent width); the
 * feature extractor's fp16 output lq_nhwc [N*HW][lq_ld]; or none.  Refused: Cpad below the channels written, Cl % 4 != 0
 * with unshuffle, a mask with unshuffle or lq_nhwc or without lq_nchw, lq_ld < Cl, scale_idx outside [0, scale_n), both
 * LQ forms at once, and more counters than launched threads. */
typedef struct rs_pack_input_args {
  const float* x; int32_t Cx;                   /* [N, Cx, HW] fp32                                                    */
  const float* scale_tab; int32_t scale_n, scale_idx;
  const float* lq_nchw; int32_t Cl;
  const float* mask_nchw;
  const void* lq_nhwc; int32_t lq_ld;
  void* out; int32_t Cpad;
  int32_t N, HW;
  int32_t lq_unshuffle, W;
  uint32_t* counters; int32_t n_counters;
} rs_pack_input_args;
int rs_op_pack_input(const rs_pack_input_args* a, void* stream);
/* The feature extractor's (and first stage's) input packing: out[N*HW][Cpad] fp16 = cat([a [N, Ca, HW], b [N, Cb, HW]])
 * + zero padding; b may be NULL with Cb = 0. */
int rs_op_pack_image(const float* a, int Ca, const float* b, int Cb, void* out, int Cpad, int N, int HW, void* stream);
/* The timestep path of a bound denoiser plan for `rows` (1 .. max(batch, 64)) device fp32 timesteps: the sinusoid
 * [rows, model_channels], time_embed.0 after SiLU [rows, 4 model_channels], time_embed.2 [rows, 4 model_channels] and the
 * FiLM rows of every ResBlock [rows, film_rows] (the emb_layers.1 of all ResBlocks in parameter order), copied to
 * whichever outputs are not NULL.  A sampler re-derives its FiLM table on its next run. */
int rs_plan_embedding(rs_plan* p, const float* tsteps, int rows, float* sin_out, float* mid_out, float* vec_out,
                      float* film_out, void* stream);
/* host only: dst[5 T + 1] = the sampler's fp32 tables coef1, coef2, std, in_scale, timesteps (T each), then the prior
 * coefficient kappa * sqrt_eta[T - 1] */
int rs_sampler_tables(const rs_sampler* s, float* dst);
/* host only: the same tables for a schedule without a plan (rs_sampler_create's arguments); what the per-step generic
 * path of gaussian_diffusion.p_sample takes its coefficients from */
int rs_schedule_tables(int steps, const double* sqrt_etas_host, double kappa, const int32_t* timestep_map_host, float* dst);
/* host only: dst[8 T + 1] = rs_schedule_tables' 5 T + 1 values for a sampler built with `options` (in_scale follows its
 * input scaling), then the conversion rows eps_coef, eta, one_minus_eta (T each) */
int rs_schedule_tables_ex(int steps, const double* sqrt_etas_host, double kappa, const int32_t* timestep_map_host,
                          const rs_sampler_options* options, float* dst);
/* quant_conv of the VQ-GAN encoder: y[n, co, hw] = b[co] + sum_ci w[co * w_ld + ci] x[n, ci, hw] (fp32 NCHW, fp16 w,
 * fp32 accumulation); Cin <= 8 (pointwise_conv_f32_kernel), or Cin a multiple of 8 from 16 to 64 with Cout <= 64
 * (pointwise_conv_wide_kernel: w 16-byte aligned, w_ld a multiple of 8) */
int rs_op_pointwise_conv(const float* x, const void* w_f16, int w_ld, const float* b, int Cin, int Cout, int N, int HW,
                         float* y, void* stream);
/* quant_conv + posterior sample of the KL first stage (rs_kl_encode's last launch) on h [N, Cin, HW]: moments
 * [N, 2E, HW], z [N, E, HW] = mean + exp(0.5 clamp(logvar, -30, 20)) * noise, or mean without noise.  Cin <= 16 and
 * 2E <= 16 (kl_posterior_kernel); otherwise Cin <= 16 or a multiple of 8 up to 128, and E <= 8 or a multiple of 8 from
 * 16 to 64 (kl_posterior_wide_kernel: w 16-byte aligned, w_ld a multiple of 8).  Both compute the same: fmaf from the
 * bias in ascending input order, mean + std * noise rounded as two operations. */
int rs_op_kl_posterior(const float* h, const void* w_f16, int w_ld, const float* b, int Cin, int E, const float* noise,
                       float* z, float* moments, int N, int HW, void* stream);

/* conv / linear on NHWC fp16 views (reference nn.Conv2d / nn.Linear call sites, see csrc/conv_gemm.cuh).
 * x [N,H,W,C] with row stride ld; w_packed fp16 [Cout][k*k][Ipad] from rs_op_pack_conv_weight; optional
 * residual / fp16 output views (row strides res_ld / out_ld) and fp32 NCHW output; act 0 none, 1 GELU(erf),
 * 2 SiLU; bn = 0 lets the library choose the channel tile. */
int rs_op_pack_conv_weight(const float* src_oihw, void* dst_f16, int O, int I, int KH, int KW, int Ipad, void* stream);
int rs_op_conv2d(const void* x, int N, int H, int W, int C, int ld, const void* w_packed, int Ipad, const float* bias,
                 int Cout, int ksize, int stride, const void* residual, int res_ld, void* out, int out_ld,
                 float* out_f32_nchw, int act, int bn, void* stream);
/* conv2d + GroupNorm statistics of its output: part[N][slots][cstride][2] = (mean, M2) of the stored values per image /
 * 128-pixel tile slot / channel at channel offset coff; with gstat, a finalisation kernel after the conv also writes
 * gstat[N][32][2] = (group mean, group rstd) of all cstride channels of part (cstride % 32 == 0).  counter is accepted
 * for compatibility and not read; expected_channels must be 0 or cstride, anything else returns an error.
 * reference: the GroupNorm32 that follows every conv (models/basic_ops.py:15-17) */
int rs_op_conv2d_stats(const void* x, int N, int H, int W, int C, int ld, const void* w_packed, int Ipad, const float* bias,
                       int Cout, int ksize, int stride, const void* residual, int res_ld, void* out, int out_ld, int act,
                       int bn, float* part, int cstride, int coff, int32_t* slots_out, float* gstat, void* counter,
                       int expected_channels, void* stream);
/* conv2d that may split its K loop over several CTAs (layers with few output tiles); scratch: 8*N*Ho*Wo*Cout floats;
 * part / gstat as rs_op_conv2d_stats, counter not read */
int rs_op_conv2d_splitk(const void* x, int N, int H, int W, int C, int ld, const void* w_packed, int Ipad, const float* bias,
                        int Cout, int ksize, int stride, const void* residual, int res_ld, void* out, int out_ld, int act,
                        float* part, int cstride, int coff, float* scratch, int32_t* splits_out, float* gstat, void* counter,
                        void* stream);
/* Every option of the conv launcher.  The three entries above are rs_op_conv2d_ex with some fields left at their
 * neutral values (NULL / 0, pad_lo = 1). */
typedef struct rs_conv_args {
  const void* x; int32_t N, H, W, C, ld;        /* NHWC fp16 input view, row stride ld                              */
  const void* w_packed; int32_t ipad;           /* fp16 [Cout][k*k][ipad] from rs_op_pack_conv_weight                */
  const float* bias; int32_t bias_sN;           /* [Cout] fp32 or NULL; bias_sN > 0: one row per image at
                                                   bias + n * bias_sN (one sub-tile)                                  */
  int32_t cout, ksize, stride;
  int32_t pad_lo;                               /* stride 2 only: 1 = padding 1 on every side, 0 = pad (0, 1, 0, 1)  */
  const void* residual; int32_t res_ld;         /* optional fp16 view on the output grid                             */
  void* out; int32_t out_ld;                    /* fp16 output view, or NULL with out_f32_nchw                       */
  float* out_f32_nchw;                          /* optional fp32 NCHW output [N, Cout, Ho, Wo]                       */
  int32_t act;                                  /* 0 none, 1 GELU(erf), 2 SiLU                                       */
  int32_t bn;                                   /* channel-tile width; 0 lets the library choose                     */
  int32_t msub;                                 /* 128-pixel sub-tiles per CTA: 0 lets the library choose (RS_CONV_MSUB=2
                                                   asks for two where the layer can take them); 1 or 2 is required   */
  float* part[2];                               /* GroupNorm statistics sinks part[i][N][slots][cstride[i]][2] or NULL */
  int32_t cstride[2], coff[2];
  float* gstat;                                 /* optional [N][32][2] group (mean, rstd) of all channels of sink 0  */
  float* splitk_scratch;                        /* non-NULL allows split-K: 8 * N * Ho * Wo * Cout floats            */
  void* silu_out; int32_t silu_ld;              /* optional second fp16 output view: SiLU of every fp16 value stored to
                                                   out (needs out), row stride silu_ld                               */
  const float* film; int32_t film_sN;           /* optional FiLM after the activation: with v = fp16(act(acc + bias)),
                                                   out = fp16(v * (1 + film[n film_sN + c]) + film[n film_sN + cout + c]);
                                                   film_sN 0 shares one row; no residual or statistics sinks, one
                                                   sub-tile, cout % 8 == 0 (silu_out too)                            */
} rs_conv_args;
/* info[12] (optional) = the configuration launched: grid, BN, msub, stages, CTAs per tile group, split-K factor,
 * persistent (0 / 1), staging block width of the TMA epilogue (0: direct epilogue), pixel box bw / bh / bn, statistics
 * slots per image.  A configuration that cannot be launched as required (bn without a compiled instance, msub = 2 with a
 * bn that has no two-sub-tile instance, or on a layer that cannot take two sub-tiles) returns an error. */
int rs_op_conv2d_ex(const rs_conv_args* a, int32_t* info, void* stream);
/* profiling aid: `iters` launches of the same conv; per-CTA timeline of the last one in dbg (8 x u64 per CTA);
 * info[7] = grid, BN, stages, shared memory bytes, CTAs per tile group, split-K factor, persistent kernel (0 / 1) */
int rs_op_conv2d_timeline(const void* x, int N, int H, int W, int C, int ld, const void* w_packed, int Ipad, const float* bias,
                          int Cout, int ksize, int stride, void* out, int out_ld, int bn, int iters, void* dbg,
                          int32_t* info, float* splitk_scratch_or_null, void* stream);
/* GroupNorm32 (+ FiLM scale/shift, + SiLU) (reference models/basic_ops.py:15-17, models/unet.py:198-202) */
int rs_op_groupnorm(const void* x, int N, int H, int W, int C, int ld, const float* gamma, const float* beta,
                    const float* film, long long film_sN, int silu, void* y, int y_ld, float* sums_scratch,
                    void* stream);
long long rs_op_groupnorm_scratch_floats(int N, int H, int W, int C);
/* the apply half alone, on gstat[N][32][2] = (group mean, group rstd) delivered by a producer (rs_op_conv2d_stats) */
int rs_op_groupnorm_apply(const void* x, int N, int H, int W, int C, int ld, const float* gamma, const float* beta,
                          const float* film, long long film_sN, int silu, void* y, int y_ld, const float* gstat,
                          void* stream);
/* ... or on the producers' raw (mean, M2) pairs part[N][slots][C][2]: the consumer combines them itself */
int rs_op_groupnorm_apply_pairs(const void* x, int N, int H, int W, int C, int ld, const float* gamma, const float* beta,
                                const float* film, long long film_sN, int silu, void* y, int y_ld, const float* part,
                                int slots, void* stream);
/* group statistics gstat[N][32][2] = (mean, rstd) from (mean, M2) pairs part[N][slots][C][2] (rows_per_slot values each)
 * as a kernel of its own — what the first-stage plans run in front of a GroupNorm whose producer has hundreds of tiles */
int rs_op_groupnorm_finalize(const float* part, int N, int slots, int C, int rows_per_slot, float eps, float* gstat, void* stream);
/* GroupNorm statistics routes of rs_op_groupnorm_ex: where the (mean, M2) pairs part[N][slots][C][2] come from and who
 * reduces them to the group statistics.  A plan picks one per GroupNorm by shape (rs_plan_profile_ops names it). */
#define RS_GN_GSTAT 0         /* the caller's gstat[N][32][2] = (group mean, group rstd): apply only                    */
#define RS_GN_CONV_PAIRS 1    /* the caller's pairs in equal slots (a conv / MLP epilogue: one per 128-pixel tile),
                                 combined by every apply CTA                                                            */
#define RS_GN_WINDOW_PAIRS 2  /* the same from the fused Swin attention: slots = (H/8)(W/8) windows of 64 pixels        */
#define RS_GN_FINALIZE 3      /* the caller's pairs reduced into the caller's gstat by a finalisation kernel, then apply */
#define RS_GN_STATS_PAIRS 4   /* a statistics kernel writes part (slots 0: the library's chunking), apply combines      */
#define RS_GN_STATS_GSTAT 5   /* ... and its last CTA per image reduces into gstat (arrival counters[N], zeroed here)    */
/* Every option of the GroupNorm launcher.  rs_op_groupnorm, _apply and _apply_pairs are rs_op_groupnorm_ex with
 * routes RS_GN_STATS_GSTAT, RS_GN_GSTAT and RS_GN_CONV_PAIRS. */
typedef struct rs_gn_args {
  const void* x; int32_t x_ld;                  /* NHWC fp16 input view [N][H][W][C], row stride x_ld >= C            */
  void* y; int32_t y_ld;                        /* output view; channels outside [0, C) of each row are not written    */
  int32_t N, H, W, C;                           /* C a multiple of 32, at most 2048                                    */
  const float* gamma; const float* beta;        /* [C]                                                                 */
  const float* film; long long film_sN;         /* optional FiLM rows: scale film[n sN + c], shift film[n sN + C + c];
                                                   film_sN = 0 shares one row between all images                       */
  int32_t silu;                                 /* 1: SiLU after the affine                                            */
  float eps;                                    /* > 0 (GroupNorm32: 1e-5 in the UNet, 1e-6 in the VQ-GAN / KL)        */
  int32_t route;                                /* RS_GN_*                                                             */
  float* part; int32_t slots;                   /* pairs [N][slots][C][2]: given (pairs / finalize routes) or written   */
  float* gstat;                                 /* [N][32][2] (mean, rstd): given (RS_GN_GSTAT) or written              */
  uint32_t* counter;                            /* [N] arrival counters of RS_GN_STATS_GSTAT                           */
} rs_gn_args;
/* info[8] (optional) = route, slots, rows per slot, statistics-kernel CTAs per image (0: none), finalisation kernel
 * ran (0 / 1), apply CTAs per image and channel slice, rows per apply CTA, channel slices.  The route is launched as
 * asked or refused with a message, never replaced by another. */
int rs_op_groupnorm_ex(const rs_gn_args* a, int32_t* info, void* stream);
/* single-head attention over all T positions of each image, out = softmax(q k^T C^-1/2) v (reference
 * ldm/modules/diffusionmodules/model.py:180-199, AttnBlock.forward between the q/k/v convs and proj_out; the VQ-GAN
 * plans run it for bottlenecks with H*W > 8192).  q, k, v fp16 [N][T][C] with row stride ld; out fp16 [N][T][C] dense.
 * C in {128, 256, 512}, T % 64 == 0; O(T*C) memory, deterministic, one launch. */
int rs_op_vq_attention(const void* q, const void* k, const void* v, int N, int T, int C, int ld, void* out, void* stream);
/* the same for the query rows [row_begin, row_end) of every image only (multiples of 64, non-empty, row_end <= T; keys
 * and values are still all T positions).  Those rows of out are bit-identical to rs_op_vq_attention's; no other row of
 * out is written, so ranges computed on different devices and copied together equal one full call. */
int rs_op_vq_attention_rows(const void* q, const void* k, const void* v, int N, int T, int C, int ld, int row_begin,
                            int row_end, void* out, void* stream);
/* multi-head attention over all T positions of each image, out = softmax(q k^T head_dim^-1/2) v per head (reference
 * models/unet.py:265-344, QKVAttentionLegacy / QKVAttention between the qkv conv and proj_out).  qkv fp16 [N][T][3C]
 * dense, C = heads * head_dim, split legacy-order (per head: q, k, v) or, with new_order, qkv-first (q | k | v, each
 * [heads][head_dim]); out fp16 [N][T][C] dense.  head_dim 32, 64 or 128, any T >= 1; deterministic, one launch. */
int rs_op_unet_attention(const void* qkv, int N, int T, int heads, int head_dim, int new_order, void* out, void* stream);
/* row softmax of the VQ-GAN attention above for H*W <= 8192, in place on the fp16 score matrix: s[r][0:cols] =
 * softmax(scale * s[r][0:cols]) for each of `rows` rows with row stride ld (elements); what lies beyond cols in a row is
 * not touched.  Needs rows >= 1, cols a multiple of 8 in [8, 8192], ld >= cols and a multiple of 8, s 16-byte aligned;
 * anything else returns an error. */
int rs_op_softmax_rows(void* s, int rows, int cols, long long ld, float scale, void* stream);
/* window attention core (reference models/swin_transformer.py:114-145,251-275); qkv [N,H,W,3*heads*32], 8x8 windows */
int rs_op_expand_relpos(const float* table_225xh, float* dense_hx64x64, int heads, void* stream);
int rs_op_window_attention(const void* qkv, int N, int H, int W, int heads, int shift, const float* bias_dense,
                           void* out, void* stream);
/* the same for window 8 or 16 and head_dim 32 or 64: table [(2 window - 1)^2, heads] -> dense
 * [heads][window^2][window^2]; qkv [N,H,W,3*heads*head_dim] -> out [N,H,W,heads*head_dim]; H and W multiples of window,
 * shift 0 or window / 2.  RS_ATTN_IMPL=simt runs the fp32 cross-check kernel instead of the tensor-core instance. */
int rs_op_expand_relpos_ex(const float* table, float* dense, int heads, int window, void* stream);
int rs_op_window_attention_ex(const void* qkv, int N, int H, int W, int heads, int window, int head_dim, int shift,
                              const float* bias_dense, void* out, void* stream);
/* the same with the launch given explicitly: hpc heads per CTA of the tensor-core instance (0: the launcher's rule, which
 * the plans use; otherwise a divisor of heads), simt != 0 for the fp32 cross-check (hpc 0 or 1).  A configuration is
 * launched as asked or refused with a message naming the argument.  info[5] (may be NULL): SIMT kernel (0 / 1), heads
 * per CTA, grid x (windows), grid y (head groups), dynamic shared memory in bytes. */
int rs_op_window_attention_cfg(const void* qkv, int N, int H, int W, int heads, int window, int head_dim, int shift,
                               const float* bias_dense, void* out, int hpc, int simt, int32_t* info, void* stream);
/* fused attention half of a Swin block: y = x + proj(window_attention(qkv(norm1(x)))) (reference
 * models/swin_transformer.py:246-275 with WindowAttention.forward :114-145); x NHWC fp16 [N,H,W,E] (in place when
 * y == x), norm1 statistics as the producers' (mean, M2) pairs gn_part[N][gn_slots][E][2] (gn_slots equal boxes of each
 * image), weights packed fp16; part_out (optional): pairs of y per 8x8 window of the shifted partition,
 * [N][(H/8)*(W/8)][E][2].  relbias_dense must be the output of rs_op_expand_relpos (relative_position_bias_table
 * gathered by relative_position_index, :82-97,130-133).  gstat_out_null and counters_null must be NULL: the group
 * statistics of y are the consuming GroupNorm's to combine from part_out. */
int rs_op_swin_attn(const void* x, int N, int H, int W, int E, int heads, int shift, const float* gn_part, int gn_slots,
                    const float* gamma, const float* beta, const void* wqkv_packed, const float* bqkv, const float* relbias_dense,
                    const void* wproj_packed, const float* bproj, void* y, float* part_out, float* gstat_out_null,
                    uint32_t* counters_null, void* stream);
/* the same on a persistent grid of `grid` CTAs (0: min(window pairs, SMs), what the plans run; otherwise at most the
 * number of window pairs), each walking a contiguous run of pairs.  info[3] (may be NULL): grid, window pairs per CTA
 * at most, windows per image. */
int rs_op_swin_attn_ex(const void* x, int N, int H, int W, int E, int heads, int shift, const float* gn_part, int gn_slots,
                       const float* gamma, const float* beta, const void* wqkv_packed, const float* bqkv,
                       const float* relbias_dense, const void* wproj_packed, const float* bproj, void* y, float* part_out,
                       int grid, int32_t* info, void* stream);
/* fused Swin MLP (reference models/swin_transformer.py:17-33,279): out = residual + fc2(GELU(fc1(x))) in one kernel,
 * E in {64, 128, 192, 256}, Hd % 64 == 0; dbg_timeline_or_null must be NULL */
int rs_op_mlp(const void* x, int N, int H, int W, int E, int Hd, const void* w1_packed, const float* b1,
              const void* w2_packed, const float* b2, const void* residual, void* out, void* dbg_timeline_or_null,
              void* stream);
/* the same with the output's GroupNorm statistics: part[i] (optional): (mean, M2) pairs of out,
 * part[i][N][slots][cstride[i]][2] at channel offset coff[i]; *slots_out = slots per image. */
int rs_op_mlp_ex(const void* x, int N, int H, int W, int E, int Hd, const void* w1_packed, const float* b1,
                 const void* w2_packed, const float* b2, const void* residual, void* out, float* const part[2],
                 const int32_t cstride[2], const int32_t coff[2], int32_t* slots_out, void* stream);
/* host-only: tile configuration the conv launcher picks: out[8] = BN, msub, stages, CTAs/SM, estimated cycles,
   CTAs per tile group (1 or 2), split-K factor, persistent kernel (0 / 1) */
int rs_debug_tile_config(int m_tiles, int cout, int num_kblocks, int32_t* out);
/* nearest x2 (reference models/unet.py:71-81) */
int rs_op_upsample2x(const void* x, int N, int H, int W, int C, void* y, void* stream);
/* the same with an optional second output silu_y (NULL: none) = SiLU of every fp16 value stored to y; dense NHWC, C % 8 == 0 */
int rs_op_upsample2x_ex(const void* x, int N, int H, int W, int C, void* y, void* silu_y, void* stream);
/* 2x2 average pool (Downsample without conv, reference models/unet.py:83-108): x [N,H,W,C] -> y [N,H/2,W/2,C] dense
 * NHWC fp16, H and W even, C % 8 == 0; silu_y as rs_op_upsample2x_ex */
int rs_op_avgpool2x2(const void* x, int N, int H, int W, int C, void* y, void* silu_y, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RESSHIFT_B200_H */
