/* sdxl_b200.h — C ABI of the H100-native (sm_90a) SDXL denoising engine (libsdxl_b200.so).
 *
 * This is the drop-in boundary for the diffusion sampling path of Gadersd/stable-diffusion-xl-burn:
 * the entry points a Rust `src/backend.rs` replacement would bind with `extern "C"` (see
 * INTEGRATION.md for the shim). Each function names the reference interface it replaces; citations
 * are file:line relative to the reference repository root.
 *
 * Conventions
 *  - Status: every function returns 0 on success, non-zero on error; `sdxl_last_error(ctx)` returns a
 *    human-readable message for the last failure on that context. No exception crosses the boundary
 *    (the reference panics on shape errors; here they are status codes).
 *  - Pointers are DEVICE pointers unless the parameter name ends in `_host` or the struct says so.
 *    Inputs are borrowed for the duration of the call; outputs are caller-allocated.
 *  - Tensors are contiguous. Public activations use the reference's layouts: NCHW for images/latents,
 *    [B,T,C] for token tensors, f16 (`uint16_t` bit pattern of IEEE binary16 == burn's `f16`) unless
 *    stated; NHWC/f32 is internal.
 *  - One sdxl_ctx per (device, stream). A ctx and the objects created from it are not thread-safe;
 *    independent ctxs are fully concurrent. All work is enqueued on the ctx stream; functions that
 *    return results to host memory synchronise that stream, all others are asynchronous.
 *  - There is NO CPU fallback: on a machine without an sm_90 GPU sdxl_ctx_create fails.
 */
#ifndef SDXL_B200_H_
#define SDXL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SDXL_API __attribute__((visibility("default")))
#else
#define SDXL_API
#endif

typedef uint16_t sdxl_half; /* IEEE binary16 bit pattern */
typedef struct sdxl_ctx sdxl_ctx;
typedef struct sdxl_unet sdxl_unet;

#define SDXL_MAX_LEVELS 8
#define SDXL_PROFILE_KINDS 24   /* entries of the per-kernel-kind arrays of the *_profile_plan entry points */

/* Mirrors DiffuserConfig (src/model/stablediffusion/mod.rs:269-278) + UNetConfig
 * (src/model/unet/mod.rs:59-69). Transformer blocks exist on levels 1 and 2 only
 * (unet/mod.rs:125,264); transformer_depths[level] is read for those levels, and
 * transformer_depths[n_levels-1] is the middle-block depth (unet/mod.rs:239). */
typedef struct sdxl_unet_cfg {
  int32_t adm_in_channels;                    /* 2816 base / 2560 refiner */
  int32_t in_channels;                        /* 4 */
  int32_t out_channels;                       /* 4 */
  int32_t model_channels;                     /* 320 base / 384 refiner */
  int32_t n_levels;                           /* len(channel_mults) */
  int32_t channel_mults[SDXL_MAX_LEVELS];     /* [1,2,4] base */
  int32_t n_head_channels;                    /* 64 (this build requires 64) */
  int32_t transformer_depths[SDXL_MAX_LEVELS];/* [_,2,10] base */
  int32_t context_dim;                        /* 2048 base / 1280 refiner */
  int32_t is_refiner;                         /* Diffuser.is_refiner: single forward, no CFG */
  int32_t n_steps;                            /* 1000 (stablediffusion/mod.rs:282) */
  int32_t edit_layout;                        /* 0; 1: the instruction-editing layout (sdxl_unet_set_edit_image, DESIGN.md §21) */
} sdxl_unet_cfg;

/* Mirrors Conditioning (src/model/stablediffusion/mod.rs:544-555); f16 like the reference's
 * Diffuser<LibTorch<f16>> after Conditioning::convert (src/bin/sample/main.rs:236-237).
 * n_batch images share the unconditional rows (the reference repeats them, mod.rs:535-536). */
typedef struct sdxl_conditioning {
  int32_t on_host;        /* 0: pointers are device memory, 1: host memory */
  int32_t n_batch;        /* context_full.dims()[0] */
  int32_t n_ctx;          /* 77 */
  const sdxl_half* context_full;                        /* [n_batch, n_ctx, 2048] */
  const sdxl_half* context_open_clip;                   /* [n_batch, n_ctx, 1280] */
  const sdxl_half* unconditional_context_full;          /* [n_ctx, 2048] */
  const sdxl_half* unconditional_context_open_clip;     /* [n_ctx, 1280] */
  const sdxl_half* channel_context;                     /* [n_batch, 2816] */
  const sdxl_half* channel_context_refiner;             /* [n_batch, 2560] */
  const sdxl_half* unconditional_channel_context;       /* [2816] */
  const sdxl_half* unconditional_channel_context_refiner; /* [2560] */
  int32_t resolution[2];  /* (height, width) in pixels; latent is /8 */
} sdxl_conditioning;

/* ---- context -------------------------------------------------------------------------------- */
/* Replaces the reference's fixed `LibTorchDevice::Cuda(0)` + libtorch default stream
 * (src/bin/sample/main.rs:131). cuda_stream may be NULL (the ctx creates its own). */
SDXL_API int sdxl_ctx_create(int device, void* cuda_stream, sdxl_ctx** out);
SDXL_API void sdxl_ctx_destroy(sdxl_ctx* ctx);
SDXL_API const char* sdxl_last_error(const sdxl_ctx* ctx);
SDXL_API int sdxl_ctx_synchronize(sdxl_ctx* ctx);
/* Number of this library's kernels launched on the ctx since creation (bench `gpu_launches`). */
SDXL_API uint64_t sdxl_ctx_launch_count(const sdxl_ctx* ctx);
/* The byte $SDXL_B200_FILL asks for, or -1 when it is unset or not a byte (0..255, decimal or 0x..). When it is set, every
 * device buffer the library allocates for itself is filled before first use: floating-point buffers with this byte,
 * integer and byte buffers with 0. A debugging aid: a read of memory nothing wrote then reaches the outputs. */
SDXL_API int sdxl_debug_fill(void);

/* ---- UNet / Diffuser ------------------------------------------------------------------------ */
/* Replaces load_diffuser_model (src/bin/sample/main.rs:35-41): builds the device-resident model from
 * a flat weight pack (format: DESIGN.md "weight pack"; tensor names = the reference's npy dump tree,
 * src/model/unet/load.rs, values f16 like the .mpk). The pack may live in host or device memory
 * (pack_on_device); the library keeps its own re-laid-out copy, the caller may free the pack. */
SDXL_API int sdxl_unet_load(sdxl_ctx* ctx, const sdxl_unet_cfg* cfg, const void* pack, size_t bytes,
                   int pack_on_device, sdxl_unet** out);
/* Multi-GPU load (SURVEY 8(b), 8(e)): prompt-sharded replicas, one process (or thread) per GPU. EVERY rank of `nccl_comm`
 * (an ncclComm_t the host application created, e.g. with ncclCommInitRank) calls this with the same cfg; only `root` passes a
 * pack (host or device), the other ranks pass pack = NULL, bytes = 0. One ncclBroadcast of the flat pack over NVLink on the
 * ctx stream (preceded by an 8-byte broadcast of its size), then the same local re-layout as sdxl_unet_load. No collective is
 * ever issued inside the sampling loop. libnccl.so.2 is resolved at first use (the copy already loaded in the process, else
 * $SDXL_B200_NCCL_LIB, else the loader path); without it the call fails with an error, the rest of the library works. */
SDXL_API int sdxl_unet_load_broadcast(sdxl_ctx* ctx, const sdxl_unet_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                      void* nccl_comm, int rank, int root, sdxl_unet** out);
SDXL_API void sdxl_unet_destroy(sdxl_unet* unet);
/* Step-invariant part of UNet::forward, hoisted: cross-attention K/V projections of `context`
 * (unet/mod.rs:1010-1011 for attn2) and the label-embedding MLP (unet/mod.rs:464-466).
 * context [B, n_ctx, context_dim] f16, y [B, adm_in_channels] f16. A call whose buffers for a new (B, n_ctx) cannot
 * be allocated returns non-zero and leaves the previous conditioning in effect. */
SDXL_API int sdxl_unet_set_conditioning(sdxl_unet* unet, int B, int n_ctx, const sdxl_half* context,
                               const sdxl_half* y);
/* == UNet::forward (src/model/unet/mod.rs:449-493) with the conditioning set above.
 * x [B,4,h,w] NCHW f16, t_host: the single timestep the reference passes as Int[1]
 * (stablediffusion/mod.rs:416), eps_out [B,4,h,w] NCHW f16 (caller-owned). */
SDXL_API int sdxl_unet_forward(sdxl_unet* unet, int B, int h, int w, const sdxl_half* x, int32_t t_host,
                      sdxl_half* eps_out);
/* Same, f32 NCHW in/out (no input/output rounding; used by the parity tests). */
SDXL_API int sdxl_unet_forward_f32(sdxl_unet* unet, int B, int h, int w, const float* x, int32_t t_host,
                          float* eps_out);

/* == Diffuser::sample_latent / sample_latent_with_inpainting / refine_latent
 * (src/model/stablediffusion/mod.rs:317-376) and the DDIM loops they call (:390-483), including
 * forward_diffuser's classifier-free guidance (:494-541; both branches are evaluated as one batched
 * forward, the combine keeps the reference's u + (c-u)*s form).
 *  step_start : 0 for sample_latent; refine_latent's step_start (e.g. 800) otherwise. When
 *               step_start > 0 `init_latent` is the latent to refine and is noised as mod.rs:363-367.
 *  init_latent: [n_batch,4,H/8,W/8] f32 NCHW. For step_start == 0 this is the initial noise
 *               (gen_noise, mod.rs:378-388); NULL => seeded Philox N(0,1) (stream seed, subsequence 0).
 *  noise      : optional injected per-call noise [n_noise,n_batch,4,H/8,W/8] f32 (refine entry noise
 *               and, for inpainting, one tensor per step in loop order); NULL => seeded Philox.
 *  inpaint_ref/inpaint_mask: both NULL, or reference latent f32 and mask bytes (1 = keep generated,
 *               mask_where semantics of mod.rs:465), each [n_batch,4,H/8,W/8].
 *  latent_out : [n_batch,4,H/8,W/8] f32 NCHW, device (or host if cond->on_host).
 * All pointer arguments live where cond->on_host says. */
SDXL_API int sdxl_sample_latent(sdxl_unet* unet, const sdxl_conditioning* cond, double guidance_scale,
                       int n_steps, int step_start, const float* init_latent, const float* noise,
                       int n_noise, uint64_t seed, const float* inpaint_ref,
                       const uint8_t* inpaint_mask, float* latent_out);

/* ---- samplers and noise schedules (DESIGN.md §16) --------------------------------------------------------------------
 * sigma_i = sqrt((1 - a_i) / a_i) over the model's alphas_cumprod; a fractional timestep t has log sigma(t) linear between
 * floor(t) and ceil(t). A schedule is n_steps pairs (t_k, sigma_k) and sigma_n = 0. The sampler state is xh = x / sqrt(a)
 * (k-diffusion's scaling), the UNet reads xh / sqrt(sigma_k^2 + 1), D = xh - sigma_k * eps with eps the guided prediction, and
 * step k is xh' = cx xh + cd D + ch D_prev + cn z with per-sampler coefficients computed on the host in double:
 *   EULER            xh + (sigma' - sigma) eps, the DDIM (eta 0) update in this scaling
 *   EULER_ANCESTRAL  k-diffusion sample_euler_ancestral (eta, s_noise)
 *   DPMPP_2M         k-diffusion sample_dpmpp_2m; first order on the first step of a call and on the step to sigma = 0
 *   LCM              diffusers' LCMScheduler.step (timestep scaling 10, sigma_data 0.5)
 * and (DESIGN.md §20; lambda = -log sigma, h = lambda' - lambda, D_j the denoised latent of step j; each step to sigma' = 0 returns
 * D exactly, with one evaluation):
 *   DPMPP_2M_SDE     k-diffusion sample_dpmpp_2m_sde, midpoint: with eta_h = eta h and phi = -expm1(-h - eta_h),
 *                    xh' = (sigma' / sigma) e^(-eta_h) xh + phi D [+ 0.5 phi (D - D_{k-1}) h / h_{k-1}] + s_noise sigma'
 *                    sqrt(-expm1(-2 eta_h)) z; the bracket once D_{k-1} exists in the call
 *   DPMPP_3M_SDE     k-diffusion sample_dpmpp_3m_sde: order 1, 2, 3 as D_{k-1}, D_{k-2} exist in the call; the same noise term
 *   UNIPC            diffusers' UniPCMultistepScheduler (solver_order 2, x0 prediction, bh2, corrector on, lower_order_final): UniC
 *                    corrects the current state from x_{k-1}, D_{k-1}, D_{k-2} and D_k (no extra evaluation, none on the first
 *                    step of a call), then UniP of order min(2, steps done in the call + 1, steps left) runs from it
 *   HEUN             k-diffusion sample_heun (s_churn 0): an Euler step to sigma', a second evaluation there, the trapezoid
 *   DPM_2            k-diffusion sample_dpm_2: an Euler step to sigma_mid = sqrt(sigma sigma'), a second evaluation there at the
 *                    fractional t of sigma_mid, then xh' = xh + (sigma' - sigma) d_mid
 * HEUN and DPM_2 evaluate the UNet twice per step (once on the step to sigma = 0); every attachment applies per evaluation, at its t.
 * Spacings over N training timesteps: REFERENCE t_k = N - 1 - k (N / n) (sdxl_sample_latent's, which runs the same n steps when n
 * divides N); LEADING (n - 1 - k)(N / n) + 1 (diffusers, steps_offset 1); TRAILING round(N - k N / n) - 1; LINSPACE
 * (N - 1)(1 - k / (n - 1)), fractional; KARRAS sigma_k = (smax^(1/rho) + k / (n - 1) (smin^(1/rho) - smax^(1/rho)))^rho with t_k from
 * the interpolation; LCM diffusers' LCMScheduler.set_timesteps with original_inference_steps = 50 (n <= 50). Any sampler goes with
 * any spacing. */
/* 4 is not assigned: sdxl_schedule_build refuses it, as it always has. */
enum { SDXL_SAMPLER_EULER = 0, SDXL_SAMPLER_EULER_ANCESTRAL = 1, SDXL_SAMPLER_DPMPP_2M = 2, SDXL_SAMPLER_LCM = 3,
       SDXL_SAMPLER_DPMPP_2M_SDE = 5, SDXL_SAMPLER_DPMPP_3M_SDE = 6, SDXL_SAMPLER_UNIPC = 7, SDXL_SAMPLER_HEUN = 8, SDXL_SAMPLER_DPM_2 = 9 };
enum { SDXL_SPACING_REFERENCE = 0, SDXL_SPACING_LEADING = 1, SDXL_SPACING_TRAILING = 2, SDXL_SPACING_LINSPACE = 3,
       SDXL_SPACING_KARRAS = 4, SDXL_SPACING_LCM = 5 };
typedef struct sdxl_schedule {
  int32_t sampler;      /* SDXL_SAMPLER_* */
  int32_t spacing;      /* SDXL_SPACING_* */
  int32_t n_steps;      /* length of the full schedule, 1 .. N */
  int32_t first_step;   /* 0, or k0 > 0: start from `init_latent` at sigma_k0 (img2img, refiner) */
  int32_t last_step;    /* 0 = n_steps, or stop early and return xh at sigma_last (the base half of base -> refiner) */
  int32_t renoise;      /* first_step > 0: 1 adds sigma_k0 * z to init_latent (img2img), 0 takes it as it is (ensemble hand-off) */
  int32_t no_cfg;       /* 1: one conditional forward per step, guidance ignored, the unconditional tensors may be NULL */
  float   karras_rho;   /* 0 = 7 */
  float   eta, s_noise; /* Euler-ancestral, DPM++ 2M SDE and 3M SDE; 0 = 1 */
} sdxl_schedule;
/* Pure host, needs no GPU: fills timesteps[0 .. n_steps) and sigmas[0 .. n_steps] (sigmas[n_steps] = 0) from an alphas_cumprod
 * table of n_train entries. Non-zero on an invalid schedule; sdxl_schedule_last_error() (per thread) names the field. */
SDXL_API int sdxl_schedule_build(const double* alphas_cumprod, int n_train, const sdxl_schedule* schedule, double* timesteps,
                                 double* sigmas);
SDXL_API const char* sdxl_schedule_last_error(void);
/* sdxl_sample_latent with a sampler and a schedule; every attachment of the UNet applies as it does there. Steps
 * [first_step, last_step) of the schedule run; latent_out is xh at sigma_last (the latent itself after the last step of the
 * schedule, where sigma = 0).
 *  init_latent: first_step == 0: the initial noise z (NULL => seeded), xh = sqrt(sigma_0^2 + 1) z so that the UNet's first
 *               input is z; first_step > 0: required, the latent to start from (xh at sigma_k0 when renoise == 0).
 *  noise / n_noise / seed: injected tensors are taken by index and the seeded Philox stream by subsequence, in this order
 *               and only those that exist: the initial noise when init_latent is NULL; the renoise tensor; then per step, in loop
 *               order, the inpainting blend's noise of each of the step's evaluations and then the sampler's (Euler-ancestral, LCM,
 *               DPM++ 2M SDE and 3M SDE, except on the step to sigma = 0). As in sdxl_sample_latent, the first tensor past the n_noise injected ones takes subsequence 0 of the seeded
 *               stream, not its index in the order: index and subsequence coincide only for a call with no injected tensor.
 *               Seeded noise is generated inside the step kernel and equals sdxl_randn(seed, subsequence).
 *  inpaint_ref / inpaint_mask: as in sdxl_sample_latent: before each forward, xh = mask ? xh : ref + sigma z at that forward's sigma.
 * With guidance the rows are [cond | uncond]; schedule->no_cfg runs [cond] alone (few-step distilled models), half the work.
 * The schedule is validated before any state changes; the error names the field. Multistep history does not cross calls. */
SDXL_API int sdxl_sample_latent_scheduled(sdxl_unet* unet, const sdxl_conditioning* cond, double guidance_scale,
                                          const sdxl_schedule* schedule, const float* init_latent, const float* noise, int n_noise,
                                          uint64_t seed, const float* inpaint_ref, const uint8_t* inpaint_mask, float* latent_out);
/* sdxl_unet_forward_f32 at a fractional timestep (the timestep embedding of t; T2I-Adapter windows compare lround(t)). For an
 * integer t the result is bit-identical to sdxl_unet_forward_f32's. t outside [0, n_steps - 1] is refused. */
SDXL_API int sdxl_unet_forward_f32_at(sdxl_unet* unet, int B, int h, int w, const float* x, double t, float* eps_out);

/* Step-wise control for benchmarking / external loops: */
/* prepare a sampler state for cond (uploads + hoists conditioning, allocates the latent). */
SDXL_API int sdxl_sampler_begin(sdxl_unet* unet, const sdxl_conditioning* cond, double guidance_scale);
/* == one iteration of the loop body at timestep t (alpha lookups + forward_diffuser + DDIM update)
 * on the internal latent; t_prev < 0 means alpha_prev = 1.0 (mod.rs:408-412). Asynchronous. */
SDXL_API int sdxl_sampler_step(sdxl_unet* unet, int t, int t_prev);
/* Same, but the latent comes from / goes to HOST memory inside the call (end-to-end timing):
 * latent_host [n_batch,4,h,w] f32 in, updated in place. Synchronises the stream. */
SDXL_API int sdxl_sampler_step_host(sdxl_unet* unet, int t, int t_prev, float* latent_host);
SDXL_API int sdxl_sampler_set_latent(sdxl_unet* unet, const float* latent, int on_host);
SDXL_API int sdxl_sampler_get_latent(sdxl_unet* unet, float* latent, int on_host);
/* alphas_cumprod[i] as the sampler sees it: the loaded table (f16-stored like the reference's .mpk, widened), or the one
 * sdxl_unet_set_prediction put in effect. */
SDXL_API double sdxl_unet_alpha(const sdxl_unet* unet, int i);
/* Algorithmic FLOPs (2*MAC over Linear/conv/attention, SURVEY 8(d) counting rule) and kernel-op count of
 * the launch plan currently built for this UNet (0 before the first forward). */
SDXL_API double sdxl_unet_plan_flops(const sdxl_unet* unet);
SDXL_API int sdxl_unet_plan_num_ops(const sdxl_unet* unet);
/* Number of launch plans built for this UNet so far: attachment changes that keep the plan (and its CUDA graph) leave it unchanged. */
SDXL_API uint64_t sdxl_unet_plan_builds(const sdxl_unet* unet);
/* FLOPs the plan's tensor-core launches actually issue: without the K/V projections hoisted to set_conditioning, with the
 * phase-decomposed upsample convolutions at their real cost and with channel / key padding (bench: `executed_flops`). */
SDXL_API double sdxl_unet_plan_flops_executed(const sdxl_unet* unet);
/* Device time of ONE execution of the current launch plan, summed per kernel kind and measured with CUDA
 * events on the ctx stream (eager launches). Kind index: 0 implicit-GEMM (wgmma), 1 attention, 2 GroupNorm,
 * 3 LayerNorm, 4 GEMV, 5 timestep-embedding, 6 first conv, 7 upsample copy, 8 phase-split copy, 9 f32->f16 cast,
 * 17 T2I-Adapter feature add, 18 PAG identity self-attention, 19 FreeU skip filter and backbone scale, 20 device-to-device copy
 * (DeepCache's feature where FreeU scales it in place).
 * All three arrays hold SDXL_PROFILE_KINDS entries (host). Used by bench.py for the per-kernel roofline. */
SDXL_API int sdxl_unet_profile_plan(sdxl_unet* unet, double* ms_by_kind_host, double* flops_by_kind_host,
                                    int* launches_by_kind_host);
/* Same measurement, one CSV row per launch (analysis aid; written to `path_host`). */
SDXL_API int sdxl_unet_profile_dump(sdxl_unet* unet, const char* path_host);
/* seeded N(0,1) exactly as the sampler generates it (device out). */
SDXL_API int sdxl_randn(sdxl_ctx* ctx, float* out, size_t n, uint64_t seed, uint64_t subsequence);

/* ---- operator level (== the burn ops / Backend hooks the hot path is built from) ------------ */
/* == Backend::qkv_attention (src/backend.rs:4-10, libtorch impl :32-79, generic :88-128).
 * q [B,T,C], k/v [B,S,C] f16, C = n_head*64, out [B,T,C] f16. mask: NULL (UNet, unet/mod.rs:1017: tensor-core
 * flash kernel) or an additive f16 [T,S] matrix such as attn_decoder_mask (text encoders, clip/mod.rs:88: short
 * sequences, CUDA-core kernel). The VAE's single-head d=512 call (autoencoder/mod.rs:572) is served inside
 * sdxl_vae_decode_latent, not here. */
SDXL_API int sdxl_qkv_attention(sdxl_ctx* ctx, const sdxl_half* q, const sdxl_half* k, const sdxl_half* v,
                       const sdxl_half* mask, int B, int T, int S, int C, int n_head, sdxl_half* out);
/* == nn::Linear::forward: x [M,K] f16, w [K,N] f16 ([in,out], python/save.py:20-25), bias [N] f16 or
 * NULL, residual [M,N] f32 or NULL; out f32 [M,N] (out_f16 = 0) or f16. geglu != 0 => N is the fused
 * 2*n_out projection and out is [M,N/2] f16 = h[:, :N/2] * gelu_erf(h[:, N/2:]) (unet/mod.rs:942-956). */
SDXL_API int sdxl_op_linear(sdxl_ctx* ctx, const sdxl_half* x, const sdxl_half* w, const sdxl_half* bias,
                   const float* residual, int M, int K, int N, int geglu, int out_f16, void* out);
/* == nn::conv::Conv2d::forward on NHWC data: x [B,H,W,Cin] f32, w OIHW f16 (python/save.py:56-72),
 * bias [Cout] f16 or NULL; ksize 1|3 (pad = ksize/2), stride 1|2 (Downsample, unet/mod.rs:760-774),
 * upsample != 0 => nearest-2x first (Upsample::forward, unet/mod.rs:742-751). out f32 NHWC. */
SDXL_API int sdxl_op_conv2d(sdxl_ctx* ctx, const float* x, const sdxl_half* w, const sdxl_half* bias, int B, int H,
                   int W, int Cin, int Cout, int ksize, int stride, int upsample, float* out);
/* == GroupNorm::forward (+ optional SILU::forward) on NHWC f32 [B,HW,C] (groupnorm/mod.rs:52-82,
 * silu.rs:14-16); x2 (nullable) is channel-concatenated after x1 (Tensor::cat, unet/mod.rs:484).
 * out f16 [B,HW,C1+C2]. */
SDXL_API int sdxl_op_group_norm(sdxl_ctx* ctx, const float* x1, int C1, const float* x2, int C2, int B, int HW,
                       int n_group, const float* gamma, const float* beta, float eps, int silu,
                       sdxl_half* out);
/* == LayerNorm::forward (layernorm/mod.rs:34-49): x [rows,C] f32 -> f16. */
SDXL_API int sdxl_op_layer_norm(sdxl_ctx* ctx, const float* x, const float* gamma, const float* beta, float eps,
                       int rows, int C, sdxl_half* out);
/* == timestep_embedding (unet/mod.rs:21-39): t_host[n] ints -> out [n,dim] f32 (cos half, sin half). */
SDXL_API int sdxl_op_timestep_embedding(sdxl_ctx* ctx, const int32_t* t_host, int n, int dim, int max_period,
                               float* out);

/* ------------------------------------------------------------------------------------------------
 * Latent decoder (SURVEY.md §8(f) rank 1): replaces LatentDecoder::{decode_latent, latent_to_image}
 * (reference src/model/stablediffusion/mod.rs:199-237, 263-266) over Autoencoder::decode_latent and Decoder::forward
 * (src/model/autoencoder/mod.rs:66-69, 193-216). The reference hard-codes the layer widths
 * (AutoencoderConfig::init, autoencoder/mod.rs:28-45); they are parameters here only so that tests can run a
 * small instance. Weight names follow the reference's loader (autoencoder/load.rs): post_quant_conv,
 * decoder/conv_in, decoder/mid/{block_1,attn,block_2}, decoder/blocks/<i>/{res1,res2,res3,upsampler},
 * decoder/norm_out, decoder/conv_out; conv weights OIHW f16, biases / norm affine f16.
 * ------------------------------------------------------------------------------------------------ */
typedef struct sdxl_vae sdxl_vae;
typedef struct sdxl_vae_cfg {
  int32_t latent_channels;              /* 4 */
  int32_t n_blocks;                     /* 4 */
  int32_t block_in[SDXL_MAX_LEVELS];    /* 512, 512, 512, 256  (DecoderConfig channels, autoencoder/mod.rs:33) */
  int32_t block_out[SDXL_MAX_LEVELS];   /* 512, 512, 256, 128 */
  int32_t n_group;                      /* 32 */
  double scale_factor;                  /* 0.13025 for SDXL (stablediffusion/load.rs:78) */
  /* encoder half (EncoderConfig, autoencoder/mod.rs:30-31); n_enc_blocks = 0: decoder only, encoder tensors not read */
  int32_t n_enc_blocks;                 /* 4 */
  int32_t enc_in[SDXL_MAX_LEVELS];      /* 128, 128, 256, 512 */
  int32_t enc_out[SDXL_MAX_LEVELS];     /* 128, 256, 512, 512 */
  int32_t enc_z_channels;               /* 8 (mean + logvar); the first latent_channels are kept (autoencoder/mod.rs:62) */
} sdxl_vae_cfg;

/* replaces load_latent_decoder (stablediffusion/load.rs:70-84): same flat pack container as sdxl_unet_load. */
SDXL_API int sdxl_vae_load(sdxl_ctx* ctx, const sdxl_vae_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                           sdxl_vae** out);
SDXL_API void sdxl_vae_destroy(sdxl_vae* vae);
/* == LatentDecoder::decode_latent (stablediffusion/mod.rs:263-266): latent f32 [B,C,h,w] NCHW -> image f32
 * [B,3,8h,8w] NCHW (nominally in [-1,1]). `on_host` != 0: both pointers are host memory. h*w must be a multiple of 64. */
SDXL_API int sdxl_vae_decode_latent(sdxl_vae* vae, int B, int h, int w, const float* latent, int on_host, float* image_out);
/* == LatentDecoder::latent_to_image (stablediffusion/mod.rs:200-237): RawImages buffer, u8 [B, 8h, 8w, 3],
 * value = trunc(clamp(((x + 1) / 2) * 255, 0, 255)); a NaN pixel channel becomes 0. */
SDXL_API int sdxl_vae_latent_to_image(sdxl_vae* vae, int B, int h, int w, const float* latent, int on_host, uint8_t* rgb_out);
/* == LatentDecoder::encode_image (stablediffusion/mod.rs:258-261) over Autoencoder::encode_image (autoencoder/mod.rs:58-64):
 * image f32 [B,3,H,W] NCHW in [-1,1] -> latent f32 [B,latent_channels,H/8,W/8] (mean channels of quant_conv, times
 * scale_factor; no sampling, like the reference). Encoder weights: encoder/conv_in, encoder/blocks/<i>/{res1,res2,
 * downsampler/conv}, encoder/mid/{block_1,attn,block_2}, encoder/norm_out, encoder/conv_out, quant_conv
 * (autoencoder/load.rs:82-116). (H/8)*(W/8) must be a multiple of 64. */
SDXL_API int sdxl_vae_encode_image(sdxl_vae* vae, int B, int H, int W, const float* image, int on_host, float* latent_out);
/* == LatentDecoder::image_to_latent (stablediffusion/mod.rs:239-256): RawImages u8 [B,H,W,3] -> latent. */
SDXL_API int sdxl_vae_image_to_latent(sdxl_vae* vae, int B, int H, int W, const uint8_t* rgb, int on_host, float* latent_out);
SDXL_API double sdxl_vae_encode_plan_flops(const sdxl_vae* vae);
/* algorithmic FLOPs (2*MAC over conv / linear / QK^T / PV) of the current decode plan; per-kind CUDA-event profile and
 * per-op CSV as for the UNet plan. */
SDXL_API double sdxl_vae_plan_flops(const sdxl_vae* vae);
SDXL_API int sdxl_vae_profile_plan(sdxl_vae* vae, double* ms_by_kind, double* flops_by_kind, int* launches_by_kind);
SDXL_API int sdxl_vae_profile_dump(sdxl_vae* vae, const char* path);

/* ------------------------------------------------------------------------------------------------
 * BPE tokenizers of the Embedder (SURVEY.md §8(f) rank 2). CPU host code, no device work, no sdxl_ctx.
 * Replaces ClipTokenizer (reference src/token/clip.rs:80-230), OpenClipTokenizer (src/token/open_clip.rs:71-221) and
 * tokenize_text (src/model/stablediffusion/mod.rs:778-793). The vocabulary files are the reference's own
 * (tokenizer/clip/bpe_simple_vocab_16e6.txt; tokenizer/open_clip/{merges,vocab}.txt), passed by path. Token ids are
 * bit-exact with the reference (known-answer vector src/token/clip.rs:232-249). Errors: non-zero status,
 * text in sdxl_tokenizer_last_error() (thread-local); where the reference would panic (piece not in the vocabulary)
 * an error is returned instead.
 * ------------------------------------------------------------------------------------------------ */
typedef struct sdxl_tokenizer sdxl_tokenizer;
SDXL_API const char* sdxl_tokenizer_last_error(void);
/* == ClipTokenizer::new (clip.rs:91-122); pads with <|endoftext|> (49407) */
SDXL_API int sdxl_tokenizer_create_clip(const char* merges_path, sdxl_tokenizer** out);
/* == OpenClipTokenizer::new (open_clip.rs:82-113); pads with 0 */
SDXL_API int sdxl_tokenizer_create_open_clip(const char* merges_path, const char* vocab_path, sdxl_tokenizer** out);
SDXL_API void sdxl_tokenizer_destroy(sdxl_tokenizer* tok);
/* == Tokenizer::encode(text, add_sot, add_eot) (clip.rs:181-205). ids_out may be NULL to query *n_out. */
SDXL_API int sdxl_tokenizer_encode(const sdxl_tokenizer* tok, const char* text_utf8, int add_sot, int add_eot,
                                   uint32_t* ids_out, int capacity, int* n_out);
/* == Tokenizer::decode (clip.rs:207-213); NUL-terminated UTF-8, *n_out = length without the NUL. */
SDXL_API int sdxl_tokenizer_decode(const sdxl_tokenizer* tok, const uint32_t* ids, int n, char* out, int capacity, int* n_out);
/* == tokenize_text (stablediffusion/mod.rs:778-793): encode(text, true, true) resized to seq_len with the padding token. */
SDXL_API int sdxl_tokenize_text(const sdxl_tokenizer* tok, const char* text_utf8, int seq_len, int32_t* tokens_out);
/* start_of_text_token / end_of_text_token / padding_token (clip.rs:215-229) */
SDXL_API int sdxl_tokenizer_special(const sdxl_tokenizer* tok, uint32_t* sot, uint32_t* eot, uint32_t* pad);

/* ------------------------------------------------------------------------------------------------
 * Text encoders of the Embedder (SURVEY.md §8(f) rank 2): replaces CLIP::{forward_hidden, forward_hidden_pooled}
 * (reference src/model/clip/mod.rs:82-147) for both CLIP-L and OpenCLIP-bigG. Weight names follow
 * load_clip_text_transformer (src/model/clip/load.rs:79-115): token_embedding/weight [n_vocab,n_state],
 * position_embedding/weight [n_ctx,n_state], blocks/<i>/{attn_ln,mlp_ln}/{weight,bias},
 * blocks/<i>/attn/{query,key,value,out}/{weight [in,out],bias}, blocks/<i>/mlp/{fc1,fc2}/{weight,bias},
 * layer_norm/{weight,bias}, text_projection [n_state,embed_dim] (optional); all f16 in the pack.
 * ------------------------------------------------------------------------------------------------ */
typedef struct sdxl_clip sdxl_clip;
typedef struct sdxl_clip_cfg {          /* == CLIPConfig (clip/mod.rs:18-26) */
  int32_t n_vocab;                      /* 49408 */
  int32_t n_state;                      /* 768 CLIP-L, 1280 OpenCLIP-bigG */
  int32_t embed_dim;                    /* 768 / 1280 */
  int32_t n_head;                       /* 12 / 20 (head dim 64) */
  int32_t n_ctx;                        /* 77 */
  int32_t n_layer;                      /* 12 / 32 */
  int32_t quick_gelu;                   /* 1 CLIP-L (QuickGELU), 0 OpenCLIP (erf GELU) */
} sdxl_clip_cfg;
SDXL_API int sdxl_clip_load(sdxl_ctx* ctx, const sdxl_clip_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                            sdxl_clip** out);
SDXL_API void sdxl_clip_destroy(sdxl_clip* clip);
/* == CLIP::forward_hidden(tokens [B,n_ctx], hidden_idx): the stream after blocks[0..hidden_idx], f32 [B,n_ctx,n_state].
 * tokens are host int32 (tokenize_text output); the causal mask is applied as attn_decoder_mask does (backend.rs:21). */
SDXL_API int sdxl_clip_forward_hidden(sdxl_clip* clip, int B, const int32_t* tokens_host, int hidden_idx, float* hidden_out,
                                      int out_on_host);
/* == CLIP::forward_hidden_pooled: hidden as above plus pooled [B,embed_dim] = layer_norm(x_final)[b, argmax(tokens[b])] @ text_projection */
SDXL_API int sdxl_clip_forward_hidden_pooled(sdxl_clip* clip, int B, const int32_t* tokens_host, int hidden_idx,
                                             float* hidden_out, float* pooled_out, int out_on_host);
SDXL_API double sdxl_clip_plan_flops(const sdxl_clip* clip);

/* ---- LoRA adapters ----------------------------------------------------------------------------------
 * Low-rank weight deltas merged into the device-resident weights (DESIGN.md §7). An adapter is an SDXLPK01 pack (the container
 * of sdxl_unet_load) whose tensors are keyed by the reference's layer path (e.g.
 * `input_blocks/4/transformer/transformer_0/attn1/query`, `output_blocks/2/upsample/conv`, `blocks/7/mlp/fc1`):
 *   <path>/lora_down  f16 [r, in] (Linear) or [r, I, kh, kw] (conv)
 *   <path>/lora_up    f16 [out, r] (Linear) or [O, r, 1, 1] (conv)
 *   <path>/alpha      optional, one element (f16 or f32); missing => alpha = r
 * With adapters a = 1..n of scales s_a active, every touched weight W (as loaded, never a previous merge) becomes
 *   W' = f16( f32(W) + sum_a (s_a * alpha_a / r_a) * sum_r up_a[:, r] * down_a[r, :] )
 * computed in f32 in a fixed order (adapters in array order, then rank index ascending), deterministically. In the reference's
 * [in,out] Linear layout the delta is (up . down)^T. Exception: the 3x3 conv after a nearest-2x upsample is stored as four
 * phase kernels whose 3x3 source is not retained; its delta is summed into the phase kernels in f32 and added to the loaded
 * phase weights, one f16 rounding away from loading a merged pack.
 * The call REPLACES the active set: n = 0 restores the loaded weights bit for bit and frees the backups; a new set is derived
 * from the loaded weights again (layers no longer touched are restored). Every tensor of every adapter is validated (known
 * layer, dtype, shapes, equal rank of down and up) before any weight is written: on failure the call returns non-zero, names the
 * tensor in sdxl_last_error and the model is unchanged. The first touch of a layer copies it to a device backup held until
 * n = 0 or destroy. The launch plan and its CUDA graph stay valid; for the UNet the hoisted conditioning (cross-attention K/V,
 * label MLP) is recomputed when conditioning is set. At most SDXL_MAX_ADAPTERS adapters per call. Queued on the ctx stream.
 * Other families (DESIGN.md §19). Per layer an adapter holds exactly one delta family and optional modifiers; logical shapes are
 * [N, Kd], Kd = I*kh*kw in PyTorch order (i, kh, kw):
 *   LoRA   lora_down, lora_up (above)                                  P = up @ down                     c = alpha / r
 *   LoHa   hada_w1_a [N, r], hada_w1_b [r, Kd] or [r, I, kh, kw],      P = (w1_a @ w1_b) * (w2_a @ w2_b)  c = alpha / r
 *          hada_w2_a [N, r'], hada_w2_b [r', Kd] or [r', I, kh, kw]                                         (r: rows of hada_w1_b)
 *   LoKr   lokr_w1 [a, b] or lokr_w1_a [a, r] + lokr_w1_b [r, b];      P[i*c+j, (p*d+q)*taps+t] = w1[i,p] * w2[j, q*taps+t],
 *          lokr_w2 [c, d(,kh,kw)] or lokr_w2_a [c, r] + lokr_w2_b      a*c = N, b*d = I;  c = alpha / r if a factor is a
 *          [r, d(,kh,kw)] or [r, d*kh*kw]                              product (r its rank), else 1 (alpha ignored)
 *   full   diff [N, I(,kh,kw)] or [N, Kd]                              P = diff                          c = 1
 * all f16. Modifiers: alpha (one element; missing => alpha = r) and dora_scale m (f32; LoRA, LoHa, LoKr): [N], [N,1] or [N,1,1,1]
 * takes the norm n per output row over Kd; [1,I] or [1,I,1,1] per input channel over N and the taps. With scale s_a:
 *   C_a = s_a * c_a * P_a                              (no dora_scale: the LoRA term above; a negative alpha is used as given)
 *   C_a = s_a * (m_a * V_a / n_a - W), V_a = W + c_a * P_a   (dora_scale; 0 where n_a = 0; no epsilon)
 *   W'  = f16(f32(W) + sum C), non-DoRA terms in call order, then DoRA terms in call order; a zero sum keeps W's bits.
 * Norms and DoRA terms are computed in double in a fixed order. Refused, with nothing changed and the layer and tensor named:
 * 4615 two families on one layer, 4616 an incomplete family, 4617 a factor of the wrong shape, 4618 ranks that do not agree
 * (within a factor pair, or the two LoKr factors when both are given as products: alpha / r needs one r),
 * 4619 LoKr factors whose Kronecker product is not [N, I], 4620 a dora_scale of another shape, 4621 a dora_scale on a layer
 * without a delta, 4622 a dora_scale on an upsample conv (its 3x3 weight is not retained, so n cannot be taken), 4623 a
 * dora_scale that is not f32, 4624 scratch that cannot be allocated. Factors other than f16 are refused with 4607. */
#define SDXL_MAX_ADAPTERS 16
typedef struct sdxl_adapter {
  const void* pack;        /* SDXLPK01 pack, host or device memory (pack_on_device); borrowed for the call */
  size_t bytes;
  int32_t pack_on_device;
  float scale;             /* s_a */
} sdxl_adapter;
SDXL_API int sdxl_unet_set_adapters(sdxl_unet* unet, int n, const sdxl_adapter* adapters);
SDXL_API int sdxl_clip_set_adapters(sdxl_clip* clip, int n, const sdxl_adapter* adapters);

/* ---- ControlNet --------------------------------------------------------------------------------------
 * Spatial conditioning (DESIGN.md §8), the published SDXL ControlNet architecture (diffusers ControlNetModel, SGM cldm.ControlNet):
 * a copy of the UNet's time / label MLPs, first conv, input blocks and middle block, a hint encoder and one 1x1 "zero conv" per
 * skip tensor. Pack (SDXLPK01): the UNet's names for the encoder half (lin{1,2}_time_embed, lin{1,2}_label_embed, input_blocks/...,
 * middle_block/...) plus input_hint_block/{0,2,...,14}/{weight,bias} (SGM indices), zero_convs/<i>/{weight,bias} [C,C,1,1] and
 * middle_block_out/{weight,bias}. A net is built on one ctx and may be attached to any UNet of that ctx whose cfg matches. */
typedef struct sdxl_controlnet sdxl_controlnet;
typedef struct sdxl_controlnet_cfg {
  sdxl_unet_cfg unet;                           /* encoder half; channels, levels, depths, context_dim, adm must equal the UNet's */
  int32_t hint_in_channels;                     /* 3 */
  int32_t n_hint_blocks;                        /* 4: total downscale 2^(n-1) must be 8 */
  int32_t hint_block_channels[SDXL_MAX_LEVELS]; /* 16, 32, 96, 256 (multiples of 8) */
} sdxl_controlnet_cfg;
SDXL_API int sdxl_controlnet_load(sdxl_ctx* ctx, const sdxl_controlnet_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                  sdxl_controlnet** out);
/* Destroying a net that is still attached to a UNet (sdxl_unet_set_controls) is a caller error: detach first. */
SDXL_API void sdxl_controlnet_destroy(sdxl_controlnet* net);
#define SDXL_MAX_CONTROLS 4
typedef struct sdxl_control {
  const sdxl_controlnet* net;
  const float* hint;        /* f32 NCHW [n_hint, hint_in_channels, height, width] in [0, 1]; host if hint_on_host; borrowed for the call */
  int32_t hint_on_host;
  int32_t n_hint;           /* UNet row b uses hint b % n_hint (CFG rows [cond | uncond] share the image's hint) */
  int32_t height, width;    /* pixels; the latent must be height/8 x width/8 */
  float scale;              /* residual scale s: skip_i += s * zero_conv_i(h_i) */
} sdxl_control;
/* Replaces the UNet's set of attached controls (n = 0 detaches all). After the UNet's middle block each control runs its own encoder
 * on the same x, t, context and label (h0 = conv_in(x) + hint_emb) and adds s * zero_conv_i(h_i) to skip i and
 * s * middle_block_out(mid) to the middle output, controls in array order. Everything is validated before anything changes (cfg
 * fields, ctx, n_hint >= 1, n <= SDXL_MAX_CONTROLS): on failure the previous set stays attached. The hints are encoded during the
 * call. A call that keeps the nets, n_hint and sizes and changes only scales or hint values rewrites buffers in place (no new
 * launch plan); any other change rebuilds the plan at the next forward. A runtime failure after validation (device allocation or
 * launch error) during such an in-place rewrite can leave controls 0..k-1 updated and k..n-1 not: call again, or detach. A forward or sampler_begin whose latent is not
 * height/8 x width/8, or whose batch is not a multiple of n_hint, fails. */
SDXL_API int sdxl_unet_set_controls(sdxl_unet* unet, int n, const sdxl_control* controls);
/* Test aid: the hint encoder's output hint_emb f32 NCHW [n, model_channels, H/8, W/8] of hint f32 NCHW [n, 3, H, W]; both
 * pointers are host memory if on_host. */
SDXL_API int sdxl_controlnet_embed_hint(sdxl_controlnet* net, int n, int H, int W, const float* hint, int on_host, float* out);

/* ---- CLIP vision encoder (the image encoder of IP-Adapter) -------------------------------------------------
 * HF CLIPVisionModelWithProjection (DESIGN.md §9): x = pre_layernorm([class_embedding ; patch_conv(pixels)] + position_embedding),
 * n_layer pre-LN blocks without a mask, image_embeds = post_layernorm(x[:, 0]) @ visual_projection. Pack (SDXLPK01), Linear weights
 * [in, out]: patch_embedding/weight [n_state, 3, p, p], class_embedding [n_state], position_embedding/weight [T, n_state],
 * pre_layernorm/{weight,bias}, blocks/<i>/{attn_ln, mlp_ln, attn/{query,key,value,out}, mlp/{fc1,fc2}} (the text encoder's names),
 * post_layernorm/{weight,bias}, visual_projection [n_state, proj_dim] (no bias). T = (image_size / patch_size)^2 + 1. */
typedef struct sdxl_clip_vision sdxl_clip_vision;
typedef struct sdxl_clip_vision_cfg {
  int32_t n_state, n_head, n_layer;   /* head dim n_state / n_head: a multiple of 8 up to 128 (ViT-H/14: 1280/16, bigG/14: 1664/16) */
  int32_t mlp_dim;                    /* 5120 (ViT-H), 8192 (ViT-bigG) */
  int32_t image_size, patch_size;     /* 224, 14 */
  int32_t proj_dim;                   /* 1024 (ViT-H), 1280 (ViT-bigG) */
  int32_t quick_gelu;                 /* 0: exact-erf GELU */
} sdxl_clip_vision_cfg;
SDXL_API int sdxl_clip_vision_load(sdxl_ctx* ctx, const sdxl_clip_vision_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                   sdxl_clip_vision** out);
SDXL_API void sdxl_clip_vision_destroy(sdxl_clip_vision* v);
/* image_embeds_out f32 [N, proj_dim] of pixels f32 NCHW [N, 3, image_size, image_size] as CLIPImageProcessor produces them (resized,
 * centre-cropped, normalised); both host memory if on_host. */
SDXL_API int sdxl_clip_vision_encode(sdxl_clip_vision* v, int N, const float* pixels, int on_host, float* image_embeds_out);
/* hidden_out f32 [N, T, n_state] = HF hidden_states[hidden_idx] of the same pixels, hidden_idx in [0, n_layer]: the pre_layrnorm
 * output for 0, else the residual stream after blocks 0..hidden_idx-1 (no post_layernorm; the convention of
 * sdxl_clip_forward_hidden). Only hidden_idx blocks run. IP-Adapter Plus reads hidden_states[-2], i.e. hidden_idx = n_layer - 1. */
SDXL_API int sdxl_clip_vision_encode_hidden(sdxl_clip_vision* v, int N, const float* pixels, int on_host, int hidden_idx,
                                            float* hidden_out);

/* ---- IP-Adapter (image prompts) -----------------------------------------------------------------------
 * The published IP-Adapter for SDXL, base variant (DESIGN.md §9; diffusers IPAdapterAttnProcessor2_0 + ImageProjection): an
 * image embedding e [D] (CLIP vision image_embeds) becomes tokens_per_image tokens
 *   tokens = LayerNorm(e @ proj + b).reshape(tokens_per_image, context_dim)           (LayerNorm eps 1e-5)
 * and every UNet cross-attention (attn2) becomes decoupled cross-attention:
 *   h = softmax(q K_txt^T / 8) V_txt + s_blk * softmax(q K_ip^T / 8) V_ip,   K_ip = tokens @ ip_key, V_ip = tokens @ ip_value
 * before the out projection. Pack (SDXLPK01), Linear weights [in, out]:
 *   image_proj/proj/{weight [D, T*context_dim], bias}, image_proj/norm/{weight, bias} [context_dim],
 *   <transformer block path>/attn2/ip_key/weight and .../ip_value/weight [context_dim, C] for every UNet transformer block, e.g.
 *   input_blocks/4/transformer/transformer_0/attn2/ip_key/weight.
 * An adapter is built on one ctx and may be attached to any UNet of that ctx whose cfg equals its `unet`. The refiner is not
 * supported.
 *
 * IP-Adapter Plus (resampler_depth > 0; h94 `ip-adapter-plus*_sdxl_vit-h`, diffusers IPAdapterPlusImageProjection): the image input
 * is the vision encoder's penultimate hidden states h [L, D] (sdxl_clip_vision_encode_hidden, hidden_idx = n_layer - 1) and a
 * perceiver Resampler of width W = 64 * resampler_heads turns them into Q = tokens_per_image tokens (every LayerNorm eps 1e-5):
 *   x = h @ proj_in + b_in;  lat = latents
 *   per layer i: kv = [LN1_i(x) ; LN2_i(lat)] (L + Q rows), q = LN2_i(lat) @ to_q, [k | v] = kv @ to_kv,
 *                lat += (softmax(q k^T / 8) v per 64-wide head) @ to_out,  lat += gelu_erf(LNff_i(lat) @ fc1) @ fc2
 *   tokens = LayerNorm(lat @ proj_out + b_out)                                        [Q, context_dim]
 * Its pack holds, instead of image_proj/{proj,norm}, Linear weights [in, out] without biases unless named:
 *   image_proj/latents [Q, W], image_proj/proj_in/{weight [D, W], bias}, image_proj/layers/<i>/attn/{norm1,norm2}/{weight,bias},
 *   image_proj/layers/<i>/attn/{to_q [W, W], to_kv [W, 2W] (K columns, then V), to_out [W, W]}/weight,
 *   image_proj/layers/<i>/ff/norm/{weight,bias}, image_proj/layers/<i>/ff/{fc1 [W, 4W], fc2 [4W, W]}/weight,
 *   image_proj/proj_out/{weight [W, context_dim], bias}, image_proj/norm_out/{weight,bias}, and the same ip_key / ip_value. */
typedef struct sdxl_ip_adapter sdxl_ip_adapter;
typedef struct sdxl_ip_adapter_cfg {
  sdxl_unet_cfg unet;            /* must equal the cfg of the UNet it is attached to; context_dim a multiple of 8 */
  int32_t image_embed_dim;       /* D: 1024 (ViT-H/14 encoder), 1280 (ViT-bigG/14 encoder); Plus: the hidden width, 1280 for ViT-H/14 */
  int32_t tokens_per_image;      /* 4; Plus: Q = 16 */
  int32_t resampler_depth;       /* 0: the base adapter; Plus: the number of perceiver layers (4) */
  int32_t resampler_heads;       /* Plus: the Resampler's heads of width 64 (20); ignored when resampler_depth = 0 */
} sdxl_ip_adapter_cfg;
SDXL_API int sdxl_ip_adapter_load(sdxl_ctx* ctx, const sdxl_ip_adapter_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                  sdxl_ip_adapter** out);
/* Destroying an adapter that is still attached to a UNet (sdxl_unet_set_image_prompt) is a caller error: detach first. */
SDXL_API void sdxl_ip_adapter_destroy(sdxl_ip_adapter* adapter);
typedef struct sdxl_image_prompt {
  const sdxl_ip_adapter* adapter;
  const float* embeds;             /* f32 [n_batch * n_images, D]: image i of prompt b at row b * n_images + i;
                                      Plus: f32 [n_batch * n_images, seq_len, D] hidden states in the same order */
  const float* negative_embeds;    /* same shape, or NULL: the unconditional rows use the projection of zero embeddings. Plus: required
                                      (h94 / diffusers use the hidden states of an all-zero pixel tensor, which the library cannot
                                      compute from the prompt); NULL is refused */
  int32_t on_host;                 /* both pointers are host memory; borrowed for the call */
  int32_t n_batch, n_images;       /* S_ip = n_images * tokens_per_image tokens per row, images concatenated in order */
  float scale;                     /* s_blk of every block, unless block_scales_host is given */
  const float* block_scales_host;  /* NULL or s_blk of each UNet transformer block in execution order (input blocks, middle, output) */
  int32_t seq_len;                 /* Plus: L, the hidden-state rows per image (257 for ViT-H/14), in [1, 4096]; ignored otherwise */
} sdxl_image_prompt;
/* Attaches an image prompt to the UNet (NULL detaches). Row rule: in the sampler's CFG batch [cond | uncond] of n images, cond row
 * b uses embeds prompt b % n_batch and uncond row b negative prompt b % n_batch; with PAG attached the batch is [cond | uncond | ptb]
 * and perturbed row b, a conditional row, uses embeds prompt b % n_batch; a direct sdxl_unet_forward of B rows uses prompt
 * r % n_batch for row r. Everything is validated before anything changes (ctx, cfg, n_batch >= 1, n_images >= 1, finite scales, the
 * current conditioning batch a multiple of n_batch; Plus: negative_embeds given, seq_len in range): on failure the previous state stays. A call with the same adapter, n_batch and
 * n_images rewrites tokens, K/V and scales in place (same launch plan and CUDA graph); any other change rebuilds the plan at the
 * next forward. The image K/V are recomputed whenever the conditioning is set. An attached ControlNet's attentions see text only. */
SDXL_API int sdxl_unet_set_image_prompt(sdxl_unet* unet, const sdxl_image_prompt* prompt);
/* Image-prompt sets (DESIGN.md §13): up to SDXL_MAX_IMAGE_PROMPTS prompts at once, each optionally limited to a region per image.
 * Every UNet cross-attention computes, for query t of the T = h_l * w_l queries of its level (raster order),
 *   h = softmax(q K_txt^T / 8) V_txt
 *   for each prompt p in array order:
 *     unmasked: h += s_p,blk * softmax(q K_p^T / 8) V_p                            (all its images' tokens in one softmax)
 *     masked:   h += sum over images i of s_p,blk * m_p,i,l[t] * softmax(q K_p,i^T / 8) V_p,i   (one softmax per image)
 * where m_p,i,l is mask plane i resized to the level as diffusers' IPAdapterMaskProcessor.downsample does: ratio = width / height,
 * mh = int(sqrt(T / ratio)), mh += (T % mh != 0), mw = T / mh (both kept >= 1), bicubic resize (torch's, A = -0.75, align_corners
 * false, no clamping) to (mh, mw), flattened row-major and zero-padded or cut to T. The masks are used as given: diffusers binarises
 * them at 0.5 first. A source is one unmasked prompt or one image of a masked prompt; at most SDXL_MAX_IP_SOURCES per set. */
#define SDXL_MAX_IMAGE_PROMPTS 4
#define SDXL_MAX_IP_SOURCES 8
typedef struct sdxl_ip_mask {
  const float* mask;               /* f32 [n_images, height, width] of its prompt, shared by every batch row and both CFG halves;
                                      NULL: the prompt is unmasked */
  int32_t on_host;                 /* mask is host memory; borrowed for the call */
  int32_t height, width;           /* pixels: positive multiples of 8; the latent must be height/8 x width/8 */
} sdxl_ip_mask;
/* Attaches n image prompts (n = 0 detaches); masks is NULL or n entries. Each prompt follows sdxl_unet_set_image_prompt's rules (its
 * own adapter, n_batch, n_images, scales and negatives; row rule per prompt). Everything is validated before anything changes (each
 * prompt as sdxl_unet_set_image_prompt does, n <= SDXL_MAX_IMAGE_PROMPTS, at most SDXL_MAX_IP_SOURCES sources, finite mask values,
 * mask height and width positive multiples of 8): on failure the previous set stays. A call with the same adapters, n_batch, n_images,
 * mask presence and mask sizes rewrites tokens, K/V, scales and masks in place (same launch plan and CUDA graph); any other call
 * rebuilds the plan at the next forward. A forward or sampler_begin on a latent other than a masked prompt's height/8 x width/8 is
 * refused. sdxl_unet_set_image_prompt(u, p) is sdxl_unet_set_image_prompts(u, p ? 1 : 0, p, NULL). */
SDXL_API int sdxl_unet_set_image_prompts(sdxl_unet* unet, int n, const sdxl_image_prompt* prompts, const sdxl_ip_mask* masks);
/* Test aid: tokens f16 [n * tokens_per_image, context_dim] of embeds f32 [n, D]; both host memory if on_host. A Plus adapter is
 * refused (use sdxl_ip_adapter_resample). */
SDXL_API int sdxl_ip_adapter_project(sdxl_ip_adapter* adapter, int n, const float* embeds, int on_host, sdxl_half* tokens_out);
/* Test aid (Plus adapters only): tokens f16 [n * tokens_per_image, context_dim] = Resampler(hidden) of hidden states f32
 * [n, seq_len, D]; both host memory if on_host. */
SDXL_API int sdxl_ip_adapter_resample(sdxl_ip_adapter* adapter, int n, int seq_len, const float* hidden, int on_host,
                                      sdxl_half* tokens_out);
/* Test aid: out = softmax(q k^T / 8) v + scale * softmax(q k_ip^T / 8) v_ip per head (head dim 64); q/out [B,T,C], k/v [B,S,C],
 * k_ip/v_ip [B,S_ip,C] f16 device memory. */
SDXL_API int sdxl_op_ip_attention(sdxl_ctx* ctx, const sdxl_half* q, const sdxl_half* k, const sdxl_half* v, const sdxl_half* k_ip,
                                  const sdxl_half* v_ip, int B, int T, int S, int S_ip, int C, int n_head, float scale, sdxl_half* out);

/* ---- T2I-Adapter --------------------------------------------------------------------------------------
 * Spatial conditioning that runs once per image (DESIGN.md §11): diffusers T2IAdapter with adapter_type "full_adapter_xl"
 * (TencentARC t2i-adapter-*-sdxl-1.0). For a hint c f32 NCHW [n, in_channels, H, W] in [0, 1] (H, W multiples of 32) and the widths
 * ch = (mc*m0, mc*m1, mc*m2, mc*m2) of the UNet cfg:
 *   x = conv_in(pixel_unshuffle(c, 16))                              3x3 pad 1, in_channels*256 -> ch0
 *   level k = 0..3: x = avg_pool2(x) if k == 2;  x = in_conv_k(x) if k in (1, 2) (1x1);
 *                   n_res_blocks times x = x + block2(relu(block1(x))) (block1 3x3 pad 1, block2 1x1);  F_k = x
 * F_0, F_1 are [n, ch, H/16, W/16], F_2, F_3 [n, ch, H/32, W/32]. Pack (SDXLPK01), conv weights OIHW f16, biases f16:
 *   conv_in/{weight,bias}, body/{1,2}/in_conv/{weight,bias}, body/{k}/resnets/{j}/block{1,2}/{weight,bias}.
 * Only SDXL-base-shaped UNet cfgs qualify: not the refiner, n_levels = 3, no transformer on level 0, and three distinct widths.
 * An adapter is built on one ctx and may be attached to any UNet of that ctx whose cfg equals its `unet`. */
typedef struct sdxl_t2i_adapter sdxl_t2i_adapter;
typedef struct sdxl_t2i_adapter_cfg {
  sdxl_unet_cfg unet;            /* must equal the cfg of the UNet it is attached to */
  int32_t in_channels;           /* hint channels: 3 (1 allowed) */
  int32_t n_res_blocks;          /* 2 */
} sdxl_t2i_adapter_cfg;
SDXL_API int sdxl_t2i_adapter_load(sdxl_ctx* ctx, const sdxl_t2i_adapter_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                   sdxl_t2i_adapter** out);
/* The UNet keeps only the features computed at attach time, so an attached adapter may be destroyed. */
SDXL_API void sdxl_t2i_adapter_destroy(sdxl_t2i_adapter* adapter);
#define SDXL_MAX_T2I_ADAPTERS 4
typedef struct sdxl_t2i_control {
  const sdxl_t2i_adapter* adapter;
  const float* hint;        /* f32 NCHW [n_hint, in_channels, height, width] in [0, 1]; host if hint_on_host; borrowed for the call */
  int32_t hint_on_host;
  int32_t n_hint;           /* UNet row b uses feature set b % n_hint (CFG rows [cond | uncond] share the image's) */
  int32_t height, width;    /* pixels, multiples of 32; the latent must be height/8 x width/8 */
  float scale;              /* s_a */
} sdxl_t2i_control;
/* Replaces the UNet's attached T2I-Adapter set (n = 0 detaches). The features F_k = sum_a s_a * F_{a,k} (f32, adapters in array order,
 * diffusers MultiAdapter with adapter_weights) are computed during the call and added in place, in the UNet's own encoder, to the
 * output of the last input block of each level (for a level without transformers that is its Downsample: input_blocks/3, 5, 8 for
 * SDXL base) and to the middle block's output, before any ControlNet residual; the skip saved for a block carries the feature too
 * (diffusers down_intrablock_additional_residuals). A ControlNet's encoder does not see them. They are added only at forwards whose
 * timestep t >= t_min (diffusers adapter_conditioning_factor; 0: always), read on the device, so the sampler and the CUDA graph honour
 * it. Everything is validated before anything changes (ctx, cfg, n <= SDXL_MAX_T2I_ADAPTERS, n_hint >= 1, equal n_hint, height and
 * width across items, sizes multiples of 32, finite scales): on failure the previous set stays attached. A call with the same n_hint
 * and size as the attached set rewrites the features and t_min in place (same launch plan and CUDA graph); any other change rebuilds
 * the plan at the next forward. A forward or sampler_begin whose latent is not height/8 x width/8, or whose batch is not a multiple
 * of n_hint, fails. */
SDXL_API int sdxl_unet_set_t2i_adapters(sdxl_unet* unet, int n, const sdxl_t2i_control* controls, int32_t t_min);
/* Test aid: the four F_k of one adapter at scale 1, f32 NCHW, concatenated in k order, of hint f32 NCHW [n, in_channels, H, W]; both
 * pointers are host memory if on_host. */
SDXL_API int sdxl_t2i_adapter_features(sdxl_t2i_adapter* adapter, int n, int H, int W, const float* hint, int on_host, float* out);

/* ---- inpainting UNet -----------------------------------------------------------------------------------
 * A UNet cfg with in_channels = 2 * out_channels + 1 > 8 (9 for SDXL: diffusers' stable-diffusion-xl-1.0-inpainting-0.1) has the
 * inpainting layout (DESIGN.md §12): its first conv reads the latent (out_channels), the mask (1) and the masked image's latent
 * (out_channels), concatenated in that order. The latent the forward entry points, the sampler and sdxl_sample_latent take and return
 * has out_channels channels; the other in_channels - out_channels come from the condition attached here, the same at every step. */
typedef struct sdxl_inpaint_condition {
  const float* cond;       /* f32 NCHW [n, in_channels - out_channels, height/8, width/8]: the mask (1 = repaint), then the
                              masked image's latent (scaled like sdxl_vae_encode_image); borrowed for the call */
  int32_t on_host;
  int32_t n;               /* UNet row b uses row b % n */
  int32_t height, width;   /* pixels; the latent must be height/8 x width/8 */
} sdxl_inpaint_condition;
/* Copies the condition into a buffer the UNet owns (NULL detaches). Everything is validated before anything changes (the UNet has the
 * inpainting layout, cond non-null, n >= 1, height and width positive multiples of 8): on failure the previous condition stays
 * attached. A call with the same n and size rewrites the buffer in place (same launch plan and CUDA graph); any other change rebuilds
 * the plan at the next forward. A forward or sampler_begin on an inpainting UNet fails when no condition is attached, when the latent
 * is not height/8 x width/8, or when the batch (the images, for the sampler: the CFG rows [cond | uncond] of image b both read row
 * b % n) is not a multiple of n. */
SDXL_API int sdxl_unet_set_inpaint_condition(sdxl_unet* unet, const sdxl_inpaint_condition* c);

/* ---- instruction-based editing (InstructPix2Pix) ------------------------------------------------------------
 * diffusers' StableDiffusionXLInstructPix2PixPipeline (DESIGN.md §21; diffusers/sdxl-instructpix2pix-768). A cfg with edit_layout = 1
 * has in_channels = 2 * out_channels: its first conv reads the latent (out_channels) and the source image's latent L (out_channels),
 * concatenated in that order. The latent the forward entry points and the samplers take and return has out_channels channels; L is
 * attached here, unscaled by the sampler's input scaling. Refused at load: edit_layout other than 0 or 1 (5700), in_channels other than
 * 2 * out_channels (5701), with is_refiner (5702); a ControlNet cfg with the edit layout (5703).
 * Rows. A direct forward of B rows: row r reads image r % n. The sampling loops with CFG run three row groups of the n_batch images,
 * [cond | img | uncond], with context and pooled/time ids [c | n | n] (the negative prompt twice) and first-conv condition
 * [L | L | 0]; the guided output (diffusers' order of terms, f32 in that order) is
 *   g = (u + s * (c - i)) + s_img * (i - u)          s = guidance_scale, s_img = image_guidance
 * and guidance rescale, v-prediction and every sampler take this g (sdxl_unet_set_prediction). no_cfg runs [c] with L alone.
 * Refused at a forward or sampler_begin on an edit UNet, each leaving every state as it was: nothing attached (5720), an image of another
 * size (5721), a batch that is not a multiple of n (5722), PAG attached (5723; it would need a fourth group), ControlNets (5724),
 * T2I-Adapters (5725) or image prompts (5726) attached; and the latent-blend arguments inpaint_ref / inpaint_mask of the sampling calls
 * (5727). */
typedef struct sdxl_edit_image {
  const float* latent;     /* f32 NCHW [n, out_channels, height/8, width/8]: the source image's VAE latent (posterior mean, not scaled by
                              the VAE scaling factor); borrowed for the call */
  int32_t on_host;
  int32_t n;               /* row rule above */
  int32_t height, width;   /* pixels; the latent must be height/8 x width/8 */
  float image_guidance;    /* s_img, finite */
} sdxl_edit_image;
/* Copies the source latent into a buffer the UNet owns (NULL detaches). Everything is validated before anything changes (the UNet has
 * the edit layout 5710, latent non-null 5711, n >= 1 5712, height and width positive multiples of 8 5713, image_guidance finite 5714;
 * 5715: the buffer cannot be allocated): on failure the previous image stays attached. A call with the same n and size rewrites the
 * image and s_img in place (same launch plan and CUDA graph); any other change rebuilds the plan at the next forward. */
SDXL_API int sdxl_unet_set_edit_image(sdxl_unet* unet, const sdxl_edit_image* e);

/* ---- perturbed-attention guidance (PAG) ------------------------------------------------------------------
 * Ahn et al. 2024, as diffusers' StableDiffusionXL*PAGPipeline runs it (DESIGN.md §14). The sampler adds a third row group to its
 * batch: [cond | uncond | ptb] (the refiner, without CFG: [cond | ptb]). The perturbed rows repeat the conditional rows' context, pooled
 * and time ids, image-prompt tokens and hints, but in every selected self-attention (attn1 of a transformer block) they compute
 * to_out(to_v(x)): softmax(q k^T) is replaced by the identity. The other rows, every cross-attention and every ControlNet are unchanged.
 * The guided noise of a step at timestep t is
 *   e = (u + (c - u) * guidance) + p_t * (c - ptb)      resp.   e = c + p_t * (c - ptb) without CFG,
 *   p_t = max(scale - adaptive_scale * (n_steps - t), 0)    (diffusers' pag_adaptive_scale; 0: p_t = scale),
 * and the DDIM update is the one of sdxl_sample_latent. */
typedef struct sdxl_pag {
  float scale;                     /* pag_scale, finite and > 0 */
  float adaptive_scale;            /* pag_adaptive_scale, finite and >= 0 */
  int32_t n_layers;                /* == sdxl_unet_num_self_attentions(unet) */
  const uint8_t* layers_host;      /* [n_layers]: 1 = identity self-attention on the perturbed rows; one per transformer block in
                                      execution order (down blocks, middle block, up blocks); at least one set */
  int32_t forward_perturbed_rows;  /* direct sdxl_unet_forward*: the last this-many rows of the batch are perturbed (0: none; fewer
                                      than the batch); the sampler ignores it */
} sdxl_pag;
/* Self-attentions of the UNet, one per transformer block (70 for SDXL base, 44 for the refiner). */
SDXL_API int sdxl_unet_num_self_attentions(const sdxl_unet* unet);
/* Attaches PAG to the UNet (NULL detaches). Everything is validated before anything changes: on failure the previous attachment stays.
 * A call that changes only scale, adaptive_scale or forward_perturbed_rows keeps the launch plan (a new perturbed row count rebuilds
 * it at the next direct forward that uses it); a new layer set, attaching and detaching rebuild it at the next forward. Attaching or
 * detaching between sdxl_sampler_begin and sdxl_sampler_step requires a new sdxl_sampler_begin. */
SDXL_API int sdxl_unet_set_pag(sdxl_unet* unet, const sdxl_pag* pag);

/* ---- FreeU ------------------------------------------------------------------------------------------------
 * Si et al. 2023, as diffusers' enable_freeu(s1, s2, b1, b2) runs it (DESIGN.md §15). At every skip concatenation cat([x, r]) of the
 * output blocks of the two deepest levels (diffusers' up_blocks[0] and [1]; output_blocks/0..5) the first half of x's channels is
 * multiplied by b and the skip r (after any ControlNet residual) becomes fourier_filter(r, threshold 1, s): the four lowest
 * frequencies of each channel, {0, -1} x {0, -1} after fftshift's centring, are scaled by s. (s, b) is (s1, b1) at the deepest level,
 * (s2, b2) at the one above. Every row of the batch (conditional, unconditional, perturbed) is filtered; ControlNets are not.
 * The FreeU authors recommend s1 = 0.9, s2 = 0.2, b1 = 1.3, b2 = 1.4 for SDXL. */
typedef struct sdxl_freeu {
  float s1, s2, b1, b2;
} sdxl_freeu;
/* Attaches FreeU to the UNet. NULL detaches, and so does any value equal to 0 (diffusers enables FreeU only when all four are
 * nonzero). A non-finite value is refused and leaves the previous state. A call that changes only the values keeps the launch plan
 * and its CUDA graph; attaching and detaching rebuild it at the next forward. Attaching or detaching between sdxl_sampler_begin and
 * sdxl_sampler_step requires a new sdxl_sampler_begin. */
SDXL_API int sdxl_unet_set_freeu(sdxl_unet* unet, const sdxl_freeu* freeu);

/* ---- DeepCache ---------------------------------------------------------------------------------------------
 * Ma et al., CVPR 2024, uniform schedule (DESIGN.md §17). The UNet has 3 * n_levels input and 3 * n_levels output blocks (9 and 9
 * for SDXL base, 12 and 12 for the refiner); output block j pops the skip of input block 3 * n_levels - 1 - j. For the branch b and
 * e = 3 * n_levels - 1 - b:
 *   full forward    the whole UNet, unchanged. The tensor entering output block e as its backbone input x (the output of output block
 *                   e - 1, or of the middle block when e = 0, after any ControlNet or T2I-Adapter addition) is kept as the feature,
 *                   before FreeU scales it.
 *   cached forward  the time and label MLPs at the current t, the first conv and input blocks 1..b (with the T2I-Adapter features
 *                   that fall in them), then output blocks e..3 * n_levels - 1 with x = feature at block e (FreeU there if it
 *                   applies), then the head. The skips are the fresh outputs of input blocks b..0. Each attached ControlNet runs its
 *                   time and label MLPs, hint, first conv and input blocks 1..b and adds its zero-conv residuals to skips 0..b; its
 *                   middle residual belongs to the part that is skipped. Image prompts, PAG rows and the inpainting condition act
 *                   wherever their layers fall in the blocks that run.
 * Sampling (sdxl_sample_latent, sdxl_sample_latent_scheduled, sdxl_sampler_step and sdxl_sampler_step_host): UNet evaluation j since
 * the last sdxl_sampler_begin (j = 0, 1, ...) is full when j % interval == 0 and cached otherwise, for every row of the batch. Every
 * sampling entry point calls sdxl_sampler_begin, so each call's first step is full. Evaluations, not steps, are counted: with a
 * two-evaluation sampler (SDXL_SAMPLER_HEUN, SDXL_SAMPLER_DPM_2) at interval 2, each step runs one full and one cached evaluation.
 * The feature is what the last full forward computed from its inputs: a full forward after a change of the conditioning or of an
 * attachment's values is what refreshes it. */
typedef struct sdxl_deepcache {
  int32_t interval;        /* >= 1: a full forward every interval-th sampler step, cached ones in between; 1 = every step full */
  int32_t branch;          /* b in [0, 3 * n_levels - 1]: the shallow branch (0 = input_blocks/0 with the last output block) */
  int32_t forward_cached;  /* direct sdxl_unet_forward*: 1 runs the cached forward on the feature the last full forward kept;
                              0 runs the full forward, which keeps it; the samplers ignore it */
} sdxl_deepcache;
/* Attaches DeepCache to the UNet (NULL detaches). Everything is validated before anything changes: on failure the previous state stays
 * and the error names the field. A call that changes only interval or forward_cached keeps the launch plan and its CUDA graphs; a new
 * branch, attaching and detaching rebuild it at the next forward. Attaching or detaching between sdxl_sampler_begin and
 * sdxl_sampler_step requires a new sdxl_sampler_begin. A cached direct forward is refused when no full forward has kept a feature
 * since the plan was last built (a new branch, batch or latent size, or any attachment change rebuilds it). */
SDXL_API int sdxl_unet_set_deepcache(sdxl_unet* unet, const sdxl_deepcache* dc);

/* ---- prediction type, guidance rescale and the noise table ------------------------------------------------------------
 * DESIGN.md §18. What the sampling loops (sdxl_sample_latent, sdxl_sample_latent_scheduled, sdxl_sampler_step and
 * sdxl_sampler_step_host) read the UNet's output as. With the rows [cond | uncond | ptb], m the output of a row, the guided output is
 * g = u + (c - u) * s, plus p_t * (c - ptb) with PAG (an edit UNet's rows [cond | img | uncond]: sdxl_unet_set_edit_image's g), and then:
 *   guidance rescale (phi > 0, calls with CFG rows only; diffusers' rescale_noise_cfg, Lin et al. 2023): for each image b,
 *                    g <- phi * g * std(c_b) / std(g_b) + (1 - phi) * g, both std unbiased over the C * H * W elements of the image,
 *                    the ratio read as 1 when std(g_b) = 0. It acts on the model output, v for a v model. no_cfg calls and the refiner,
 *                    which run without CFG, ignore phi.
 *   epsilon          g is the noise: the DDIM loop x' = sqrt(a') * (x - sqrt(1 - a) * g) / sqrt(a) + sqrt(1 - a') * g, the
 *                    scheduled samplers D = xh - sigma * g.
 *   v                g is v (Salimans & Ho 2022): the DDIM loop x0 = sqrt(a) * x - sqrt(1 - a) * g, eps = sqrt(a) * g + sqrt(1 - a) * x,
 *                    x' = sqrt(a') * x0 + sqrt(1 - a') * eps; the scheduled samplers D = xh / (sigma^2 + 1) - sigma / sqrt(sigma^2 + 1) * g.
 * The table: every loop, sdxl_unet_alpha and so every sdxl_schedule_build on it use the one in effect. A zero-terminal-SNR table
 * (Lin et al. 2023, Algorithm 1) is computed by the caller, as diffusers does it in float32 with the last entry set to 2^-24
 * (sdxl_b200.schedulers.alphas_cumprod); the loaded table is f16-rounded and is not rescaled here. */
enum { SDXL_PREDICTION_EPSILON = 0, SDXL_PREDICTION_V = 1 };
typedef struct sdxl_prediction {
  int32_t type;                       /* SDXL_PREDICTION_* */
  float   guidance_rescale;           /* phi in [0, 1]; 0 = off */
  int32_t n_alphas;                   /* 0: keep the loaded alphas_cumprod; else cfg.n_steps */
  const double* alphas_cumprod_host;  /* n_alphas entries, strictly decreasing inside (0, 1) */
} sdxl_prediction;
/* Sets the UNet's prediction type, guidance rescale and noise table. NULL restores epsilon, phi 0 and the loaded table, bit for bit.
 * Everything is validated before anything changes: a refusal (5600..5604) names the field and leaves the previous state. Nothing here
 * rebuilds the launch plan, and a change between sdxl_sampler_begin and sdxl_sampler_step applies from the next step. */
SDXL_API int sdxl_unet_set_prediction(sdxl_unet* unet, const sdxl_prediction* p);

/* ---- `sample` front-end helpers --------------------------------------------------------------------- */
/* Inpainting mask from a crop window in pixels (src/bin/sample/main.rs:144-190): latent coordinates = pixel / (img_h / lat_h),
 * ones inside the window, zero outside, inverted by crop_out; mask = 1 keeps the generated latent. Negative bound = not given
 * (0 / image extent). Output: host uint8 [n_channels, lat_h, lat_w] (the [1,4,h,w] Bool tensor of the reference). */
SDXL_API int sdxl_make_inpaint_mask(int img_w, int img_h, int lat_w, int lat_h, int crop_left, int crop_right, int crop_top,
                                    int crop_bottom, int crop_out, int n_channels, uint8_t* mask_out_host);

/* ---- burn record (.mpk) helper ----------------------------------------------------------------------- */
/* The reference ships weights as burn 0.13 NamedMpkFileRecorder<HalfPrecisionSettings> records (src/bin/convert/main.rs:65-70,
 * loaded at src/bin/sample/main.rs:28-51): MessagePack, tensors as {"value": [f16 bit patterns as msgpack uints], "shape": [..]}.
 * sdxl_b200/burn_record.py walks the tree; these decode / encode the value arrays (host memory, no CUDA). */
SDXL_API int sdxl_mpk_decode_u16(const uint8_t* buf, size_t len, size_t count, uint16_t* out, size_t* consumed);
SDXL_API size_t sdxl_mpk_encode_u16(const uint16_t* in, size_t count, uint8_t* out);

#ifdef __cplusplus
}
#endif
#endif /* SDXL_B200_H_ */
