/* libb200ad — C ABI of the H100-native audio-diffusion hot path.
 *
 * The reference (teticio/audio-diffusion) has no FFI: its boundary is Python duck-typing on the objects that
 * `AudioDiffusionPipeline.__call__` drives (audiodiffusion/pipeline_audio_diffusion.py:71-205) and on
 * `Mel` (audiodiffusion/mel.py:44-168).  Every entry point below names the reference call it replaces.
 *
 * Conventions: plain pointers and sizes; all tensor pointers are DEVICE pointers owned by the caller
 * (PyTorch); `stream` is a cudaStream_t passed as void*; kernels are enqueued and never synchronise;
 * return value 0 = ok, negative = error (message via b200ad_last_error()).  Handles are per device and
 * not thread-safe (the reference is single-threaded synchronous Python; one process per GPU).
 */
#ifndef B200AD_H
#define B200AD_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200AD_MAX_BLOCKS 8

const char* b200ad_last_error(void);
int b200ad_version(void);

/* ---- U-Net: replaces diffusers.UNet2DModel as constructed at scripts/train_unet.py:115-137 ------------ */
typedef struct {
  int in_channels, out_channels;      /* 1 / 1 (or vqvae latent_channels), train_unet.py:117-118        */
  int layers_per_block;               /* 2                                                               */
  int num_blocks;                     /* len(block_out_channels)                                         */
  int block_out_channels[B200AD_MAX_BLOCKS];
  int down_attn[B200AD_MAX_BLOCKS];   /* 1 where down_block_types[i] == "AttnDownBlock2D"                */
  int up_attn[B200AD_MAX_BLOCKS];     /* 1 where up_block_types[i] == "AttnUpBlock2D"                    */
  int norm_num_groups;                /* 32                                                              */
  float norm_eps;                     /* 1e-5                                                            */
  int attention_head_dim;             /* UNet2DModel: 8 (only 8 is implemented).  Conditional model: diffusers uses
                                         this number as the HEAD COUNT (8): head_dim = channels / 8            */
  /* UNet2DConditionModel as built at scripts/train_unet.py:139-159 (all zero for UNet2DModel):              */
  int cross_attention_dim;            /* width of the audio encoding (100); 0 = unconditional UNet2DModel   */
  int down_cross[B200AD_MAX_BLOCKS];  /* 1 where down_block_types[i] == "CrossAttnDownBlock2D"               */
  int up_cross[B200AD_MAX_BLOCKS];    /* 1 where up_block_types[i] == "CrossAttnUpBlock2D"                   */
} b200ad_unet_config;

typedef struct b200ad_unet b200ad_unet;

int b200ad_unet_create(const b200ad_unet_config* cfg, b200ad_unet** out);
void b200ad_unet_destroy(b200ad_unet* h);

/* Parameter table in diffusers state-dict naming (SURVEY §8b), so hub checkpoints bind unchanged. */
int b200ad_unet_num_params(const b200ad_unet* h);
const char* b200ad_unet_param_name(const b200ad_unet* h, int i);
/* writes up to 4 dims, returns ndim */
int b200ad_unet_param_shape(const b200ad_unet* h, int i, int64_t* dims);

/* Device bytes for the bf16-packed weights, and for activations at a given batch / resolution. */
size_t b200ad_unet_packed_bytes(const b200ad_unet* h);
size_t b200ad_unet_workspace_bytes(const b200ad_unet* h, int N, int H, int W);

/* Bind fp32 parameters (device pointers, in table order) and pack them for the tensor-core kernels into
 * `packed` (caller-owned device buffer of b200ad_unet_packed_bytes()).  Call again after weights change. */
int b200ad_unet_set_params(b200ad_unet* h, const float* const* params, void* packed, size_t packed_bytes, void* stream);

/* Bind (and zero) the activation workspace for batch N at H x W and build the launch plan. */
int b200ad_unet_bind_workspace(b200ad_unet* h, void* workspace, size_t bytes, int N, int H, int W, void* stream);

/* model_output = unet(sample, timestep)["sample"]   (pipeline_audio_diffusion.py:163, :237).
 * x, eps_out: fp32 NCHW [N, in/out_channels, H, W]; t: float[N] timesteps (device). */
int b200ad_unet_forward(b200ad_unet* h, const float* x, const float* t, float* eps_out, void* stream);

/* Conditional model only: encoder_hidden_states of the next forward (pipeline_audio_diffusion.py:160-161),
 * fp32 [N][S][cross_attention_dim] on the device; S = 1 (what audiodiffusion/audio_encoder.py produces) is implemented. */
int b200ad_unet_set_encoding(b200ad_unet* h, const float* enc, int S);

/* Scheduler-update coefficients (host scalars, computed exactly as DDPMScheduler.step / DDIMScheduler.step do,
 * pipeline_audio_diffusion.py:165-179):
 *   x0  = clamp((x - sqrt_1m_at * eps) * inv_sqrt_at, -clip, +clip)   (clamp only if do_clip)
 *   out = c_x0 * x0 + c_xt * x + c_eps * eps + c_z * z */
typedef struct {
  float sqrt_1m_at, inv_sqrt_at, clip, c_x0, c_xt, c_eps, c_z;
  int do_clip;
} b200ad_step_coef;

/* One denoising step with the scheduler update fused into the U-Net output kernel:
 * x_out = scheduler.step(unet(x, t), t, x)["prev_sample"].  z may be NULL (t == 0 / DDIM eta == 0);
 * eps_out may be NULL; x_out may alias x. */
int b200ad_unet_forward_step(b200ad_unet* h, const float* x, const float* t, const float* z,
                             const b200ad_step_coef* coef, float* x_out, float* eps_out, void* stream);

/* The same step with the coefficients in DEVICE memory (one b200ad_step_coef): nothing that changes from step to step is a
 * launch argument (x, t, z, coef_dev, x_out are fixed buffers the caller refreshes), so the launch sequence can be captured
 * into a CUDA graph once and replayed for every step of the loop (pipeline_audio_diffusion.py:159-185) — the batch-1 path
 * of the reference facade (audiodiffusion/__init__.py:59) is bound by host launch overhead otherwise.  z must be non-NULL
 * (steps without noise carry c_z = 0). */
int b200ad_unet_forward_step_dev(b200ad_unet* h, const float* x, const float* t, const float* z,
                                 const b200ad_step_coef* coef_dev, float* x_out, void* stream);
/* Writes one step's scalars to the device buffers the call above reads: *coef_dev = *coef, t_dev[0..n) = t.  The values
 * travel as kernel arguments, so the host may enqueue many steps ahead of the GPU. */
int b200ad_step_scalars_upload(const b200ad_step_coef* coef, float t, b200ad_step_coef* coef_dev, float* t_dev, int n,
                               void* stream);

/* Debug / parity: copy a named internal activation of the last forward to fp32 NCHW.
 * Names follow the oracle taps (e.g. "conv_in", "down_blocks.0.resnets.0", "mid_block.attentions.0").
 * Returns the number of channels, or negative. dst may be NULL to query (dims[0..2] = C, H, W). */
int b200ad_unet_debug_tensor(b200ad_unet* h, const char* name, float* dst, int* dims, void* stream);

/* Profiling: run one fused step with a CUDA-event pair around every launch of the plan; fills per-op device time
 * (ms), op kind (0 temb, 1 conv_in, 2 gn_finalize, 3 conv_tc, 4 unused, 5 parity_split, 6 attention, 7 conv_out, 15 gn_apply) and, for
 * conv_tc launches, the algorithmic FLOPs (2*N*H*W*cout*K). Synchronises the stream. Returns the number of ops. */
int b200ad_unet_profile_step(b200ad_unet* h, const float* x, const float* t, const float* z,
                             const b200ad_step_coef* coef, float* x_out, float* op_ms, int* op_kind,
                             double* op_flops, int max_ops, void* stream);

/* Number of kernel launches the last forward enqueued. */
int b200ad_unet_last_launch_count(const b200ad_unet* h);

/* ---- U-Net backward (scripts/train_unet.py:259 `accelerator.backward(loss)`) ----------------------------
 * Protocol: set_training(1) -> bind_workspace (every activation is kept) -> bind_backward -> per step: forward(x, t),
 * then backward(x, dL/d eps). Parameter gradients land in ONE flat fp32 buffer; parameter i of the
 * table lives at float offset b200ad_unet_grad_offset(h, i) — the Python mirror exposes them as `p.grad` views. */
int b200ad_unet_set_training(b200ad_unet* h, int on);
size_t b200ad_unet_grad_floats(b200ad_unet* h);
size_t b200ad_unet_grad_offset(b200ad_unet* h, int i);
/* Data-parallel training: overlap the gradient all-reduce with the rest of the backward pass (accelerate's DDP buckets,
 * scripts/train_unet.py:181).  Bucket k = floats [lo[k], lo[k+1]) of the flat gradient buffer (lo[0] = 0, lo[n] =
 * b200ad_unet_grad_floats, ascending, on parameter boundaries).  b200ad_unet_backward records bucket k's event on its stream
 * right after the last launch that adds into the bucket; b200ad_unet_grad_bucket_wait makes another stream (the one the
 * collective is issued on) wait for it.  Call after b200ad_unet_bind_backward; n = 0 removes the buckets. */
int b200ad_unet_set_grad_buckets(b200ad_unet* h, int n, const size_t* lo);
int b200ad_unet_grad_bucket_wait(b200ad_unet* h, int k, void* stream);
size_t b200ad_unet_backward_bytes(b200ad_unet* h);       /* arena for activation gradients, temporaries, transposed weights */
int b200ad_unet_bind_backward(b200ad_unet* h, void* arena, size_t bytes, float* grads, void* stream);
/* x: the forward input [N, 1, H, W]; g_eps: gradient of the loss w.r.t. the forward output, fp32 [N, 1, H, W].
 * accumulate = 0 zeroes the gradient buffer first; != 0 adds to it (gradient accumulation, `accelerator.accumulate`). */
int b200ad_unet_backward(b200ad_unet* h, const float* x, const float* g_eps, int accumulate, void* stream);
int b200ad_unet_backward_launch_count(const b200ad_unet* h);

/* ---- Latent autoencoder: replaces diffusers.AutoencoderKL as the pipeline drives it ---------------------
 * (audiodiffusion/pipeline_audio_diffusion.py:143-147 encode + sample, :187-190 decode; architecture
 * config/ldm_autoencoder_kl.yaml:18-28; state-dict keys as audiodiffusion/utils.py:156-303 produces them). */
typedef struct {
  int in_channels, out_channels;      /* 1 / 1                                                            */
  int latent_channels;                /* z_channels = 1 (1..4 supported)                                  */
  int layers_per_block;               /* num_res_blocks = 2                                               */
  int num_blocks;                     /* len(ch_mult) = 4  -> spatial factor 2^(num_blocks-1) = 8         */
  int block_out_channels[B200AD_MAX_BLOCKS]; /* ch * ch_mult = 128, 256, 512, 512                          */
  int norm_num_groups;                /* 32                                                               */
  float norm_eps;                     /* 1e-6                                                             */
} b200ad_vae_config;

typedef struct b200ad_vae b200ad_vae;

int b200ad_vae_create(const b200ad_vae_config* cfg, b200ad_vae** out);
void b200ad_vae_destroy(b200ad_vae* h);
int b200ad_vae_num_params(const b200ad_vae* h);
const char* b200ad_vae_param_name(const b200ad_vae* h, int i);
int b200ad_vae_param_shape(const b200ad_vae* h, int i, int64_t* dims);
size_t b200ad_vae_packed_bytes(const b200ad_vae* h);
size_t b200ad_vae_workspace_bytes(const b200ad_vae* h, int N, int H, int W);   /* H, W: image resolution */
int b200ad_vae_set_params(b200ad_vae* h, const float* const* params, void* packed, size_t packed_bytes, void* stream);
int b200ad_vae_bind_workspace(b200ad_vae* h, void* workspace, size_t bytes, int N, int H, int W, void* stream);

/* z = vqvae.encode(x).latent_dist.sample(): x fp32 [N, in, H, W]; noise fp32 [N, L, H/f, W/f] (the caller draws it with
 * its own generator, as DiagonalGaussianDistribution.sample does; NULL = posterior mean, i.e. .mode()); z fp32
 * [N, L, H/f, W/f] (NOT multiplied by scaling_factor); moments (optional) receives quant_conv's output [N, 2L, H/f, W/f]. */
int b200ad_vae_encode(b200ad_vae* h, const float* x, const float* noise, float* z, float* moments, void* stream);
/* x_out = vqvae.decode(z)["sample"]: z fp32 [N, L, H/f, W/f] -> fp32 [N, out, H, W]. */
int b200ad_vae_decode(b200ad_vae* h, const float* z, float* x_out, void* stream);
int b200ad_vae_debug_tensor(b200ad_vae* h, const char* name, float* dst, int* dims, void* stream);
int b200ad_vae_last_launch_count(const b200ad_vae* h);

/* ---- Training step, optimizer side: replaces F.mse_loss, clip_grad_norm_(1.0), torch.optim.AdamW.step and
 * EMAModel.step of scripts/train_unet.py:258-266 (the U-Net backward itself is not built yet — DESIGN.md §6). -- */
typedef struct {
  float lr;              /* this step's learning rate (the caller's LR schedule, train_unet.py:174-179, :264) */
  float beta1, beta2;    /* 0.95, 0.999                         train_unet.py:166-172 */
  float eps;             /* 1e-8 */
  float weight_decay;    /* 1e-6 (decoupled) */
  float max_grad_norm;   /* 1.0 (train_unet.py:262); <= 0 disables clipping */
  float ema_decay;       /* EMAModel's decay for this step (train_unet.py:185-190); < 0 disables the EMA update */
  int step;              /* 1-based optimizer step (bias correction) */
} b200ad_optim_hparams;
typedef struct b200ad_optim b200ad_optim;
/* Binds n_tensors fp32 device tensors (parameters, Adam moments, optional EMA shadows; sizes in elements). The handle owns
 * only its small device-side pointer / chunk tables. */
int b200ad_optim_create(int n_tensors, const int64_t* sizes, float* const* params, float* const* exp_avg,
                        float* const* exp_avg_sq, float* const* ema, b200ad_optim** out);
void b200ad_optim_destroy(b200ad_optim* h);
/* One fused step over all tensors. grads: HOST array of n_tensors device pointers. grad_norm_out (optional, device float)
 * receives the total gradient 2-norm before clipping. Two kernel launches. */
int b200ad_optim_step(b200ad_optim* h, const float* const* grads, const b200ad_optim_hparams* hp, float* grad_norm_out,
                      void* stream);
/* loss_out[0] = mean((pred - target)^2) (device float); grad_out (optional) = 2 (pred - target) / n. scratch: 1 double. */
int b200ad_mse_loss_grad(const float* pred, const float* target, size_t n, float* loss_out, float* grad_out,
                         double* scratch, void* stream);

/* ---- Op-level entry points (parity tests call the kernels in isolation) ------------------------------- */
/* conv2d (KHxKW in {1x1, 3x3}, stride 1 or 2, padding KH/2) on fp32 NCHW tensors through the wgmma
 * implicit-GEMM kernel; optional residual (fp32 NCHW, cout channels) and per-sample additive vector
 * temb [N][cout]; stats_out (optional) receives [N][cout/4][2] (sum, sumsq). scratch >= b200ad_conv2d_scratch_bytes. */
size_t b200ad_conv2d_scratch_bytes(int N, int cin, int cout, int H, int W, int K, int stride);
int b200ad_conv2d(const float* x, const float* w, const float* bias, const float* temb, const float* residual,
                  float* y, float* stats_out, int N, int cin, int cout, int H, int W, int K, int stride,
                  void* scratch, size_t scratch_bytes, void* stream);
/* conv2d(act(GroupNorm(x))) with the GroupNorm(+SiLU) apply fused into the conv kernel's operand staging — the form every
 * ResnetBlock2D conv takes in the U-Net plan. Stride 1; scratch >= b200ad_conv2d_scratch_bytes(..., stride 1). */
int b200ad_gn_conv2d(const float* x, const float* gamma, const float* beta, int groups, float eps, int silu,
                     const float* w, const float* bias, float* y, int N, int cin, int cout, int H, int W, int K,
                     void* scratch, size_t scratch_bytes, void* stream);
/* Data gradient of the stride-1 conv above (what autograd's conv2d backward returns for the input; first piece of the
 * U-Net backward, scripts/train_unet.py:259): gy [N, cout, H, W], w [cout, cin, K, K] -> gx [N, cin, H, W]. Runs on the
 * same wgmma kernel with transposed / mirrored weight packing. cin % 128 == 0, cout % 16 == 0;
 * scratch >= b200ad_conv2d_scratch_bytes(N, cout, cin, H, W, K, 1). */
int b200ad_conv2d_dgrad(const float* gy, const float* w, float* gx, int N, int cin, int cout, int H, int W, int K,
                        void* scratch, size_t scratch_bytes, void* stream);
/* Weight gradient of the same conv (autograd's conv2d backward for the weight): gy [N, cout, H, W], a [N, cin, H, W] (the
 * conv's input) -> dw fp32 [cout, cin, K, K] (overwritten). wgmma with pixels as the reduction dimension (both operands
 * MN-major); cout % 128 == 0, cin % 32 == 0. */
size_t b200ad_conv2d_wgrad_scratch_bytes(int N, int cin, int cout, int H, int W);
int b200ad_conv2d_wgrad(const float* gy, const float* a, float* dw, int N, int cin, int cout, int H, int W, int K,
                        void* scratch, size_t scratch_bytes, void* stream);
/* GroupNorm(groups, eps) [+ SiLU] on fp32 NCHW through the stats + apply kernels. */
int b200ad_group_norm(const float* x, const float* gamma, const float* beta, float* y, int N, int C, int H, int W,
                      int groups, float eps, int silu, void* scratch, size_t scratch_bytes, void* stream);

/* ---- Mel codec: replaces Mel.audio_slice_to_image / Mel.image_to_audio (audiodiffusion/mel.py:135-168) -- */
typedef struct {
  int x_res, y_res, sample_rate, n_fft, hop_length, top_db, n_iter;
} b200ad_mel_config;
size_t b200ad_mel_scratch_bytes(const b200ad_mel_config* cfg, int n);
/* audio [n][x_res*hop_length - 1] fp32 (device) -> uint8 images [n][y_res][x_res] (device). mel.py:145-149.
 * mel_basis_t: librosa.filters.mel(sr, n_fft, n_mels=y_res) transposed, fp32 [n_fft/2+1][y_res] (device; a
 * data-independent constant the caller builds once). */
int b200ad_mel_encode(const b200ad_mel_config* cfg, const float* mel_basis_t, const float* audio, uint8_t* images,
                      int n, void* scratch, size_t scratch_bytes, void* stream);
/* The same with `ref` of librosa.power_to_db chosen by the caller (mel.py:135 `ref` argument, default np.max):
 * ref_values (device, float[n], may be NULL = np.max) is the reference power per slice; mel_power_out (device,
 * float[n][y_res][x_res], may be NULL) receives the mel power spectrogram S a callable `ref(S)` is evaluated on;
 * images may be NULL when only S is wanted. */
int b200ad_mel_encode_ref(const b200ad_mel_config* cfg, const float* mel_basis_t, const float* audio, uint8_t* images,
                          int n, const float* ref_values, float* mel_power_out, void* scratch, size_t scratch_bytes,
                          void* stream);
/* uint8 images [n][y_res][x_res] -> audio [n][(x_res-1)*hop_length] fp32. mel.py:162-167.
 * mel_pinv: numpy.linalg.pinv(mel basis in fp64), fp64 [n_fft/2+1][y_res] (device constant).
 * phase_seed seeds the Griffin-Lim random phase (the reference leaves it unseeded). */
int b200ad_mel_decode(const b200ad_mel_config* cfg, const double* mel_pinv, const uint8_t* images, float* audio, int n,
                      uint64_t phase_seed, void* scratch, size_t scratch_bytes, void* stream);

/* float sample -> uint8 image, pipeline_audio_diffusion.py:192-194: round-half-even((x/2+.5).clamp(0,1)*255). */
int b200ad_sample_to_u8(const float* x, uint8_t* img, size_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200AD_H */
