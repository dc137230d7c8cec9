// Host-side launch API of the sm_90a kernels (internal to libsdxl_b200.so; the public boundary is
// include/sdxl_b200.h). All pointers are device pointers. All launchers return cudaError_t-style
// int (0 = ok) and never synchronise.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace sdxl {

// Launch helper: cudaLaunchKernelEx with optional programmatic dependent launch (PDL). Kernels launched
// with pdl=true MUST execute griddep_wait() (common.cuh) before touching global memory written by the
// preceding kernel. SDXL_B200_NO_PDL=1 disables the attribute globally.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline int launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                         Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (pdl && pdl_enabled()) ? 1 : 0;
  return (int)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline int launch_kernel_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                                 int cluster_size, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_size > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_size;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl && pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return (int)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Opt-in to more than 48 KB of dynamic shared memory for `kernel`. The attribute is per DEVICE (one process may drive several
// devices through several contexts), so call sites keep one flag per device: `static bool done[64]`.
template <typename K>
inline int smem_optin(K kernel, int bytes, bool (&done)[64]) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return (int)e;
  if (dev < 0 || dev >= 64) return 2001;
  if (!done[dev]) {
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return (int)e;
    done[dev] = true;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Implicit GEMM on wgmma (igemm.cu): out[pixel, n] = epilogue( sum_seg sum_c A_seg[pixel+tap, c] *
// Wt[n, k(seg,c)] ). Linear layers are the 1-segment / 1x1 case of the same kernel.
// ------------------------------------------------------------------------------------------------
constexpr int IGEMM_MAX_SEG = 20;
struct IgemmSeg {
  int16_t map;   // 0 -> tmA0, 1 -> tmA1
  int16_t dw, dh;  // tap offset added to the tile's (w0,h0)
  int16_t db;    // offset added to the tile's batch coordinate (stride-2 phase images)
  int32_t nkb;   // number of 64-channel K blocks in this segment
};
enum IgemmMode : int { IGEMM_LINEAR = 0, IGEMM_GEGLU = 1 };
struct alignas(64) IgemmParams {
  CUtensorMap tmA0, tmA1, tmB;
  IgemmSeg seg[IGEMM_MAX_SEG];
  int nseg;
  int Wt, Ht, Bt;             // A box in pixels, Wt*Ht*Bt == 128
  int W, H, Bn;               // output extents
  int tilesW, tilesH, tilesB, tilesN;
  int N;                      // valid output columns (GEGLU: columns of the fused [value|gate] GEMM)
  int BN;                     // N tile: 64, 128, 160 or 256
  int nstages;
  int mode;                   // IgemmMode
  void* out;                  // f16 or f32 [pixels, ldo]
  int out_f32;
  int ldo;
  const float* bias;          // nullable; index b*bias_bstride + n
  int bias_bstride;
  const float* res;           // nullable f32 residual [pixels, ldr]
  int ldr;
  // output pixel of tile pixel (b, h, w): (b*H + h) * opix_row + w * opix_w + opix_off (defaults W, 1, 0). The nearest-2x
  // upsample + 3x3 conv is run as four 2x2 convolutions on the original image, each writing one (row, column) parity of the
  // upsampled output: opix_row = 4W, opix_w = 2, opix_off = a*2W + b.
  int opix_row, opix_w, opix_off;
};
// A operand view: NHWC f16 tensor [Bn, H, W, C] with channel pitch `pitch` (elements, multiple of 8).
int make_tmap_act(CUtensorMap* tm, const __half* base, int Bn, int H, int W, int C, int pitch, int Wt,
                  int Ht, int Bt);
// B operand view: K-major weights [N, K] f16 with row pitch K (multiple of 8); box (64, BN).
int make_tmap_wgt(CUtensorMap* tm, const __half* base, int N, int K, int BN);
// Picks Wt/Ht/Bt (product 128) for an output image of W x H.
void igemm_pick_box(int W, int H, int* Wt, int* Ht, int* Bt);
// Operand views for igemm_configure: NHWC f16 activations (channel pitch in elements) and K-major weights.
struct IgemmOperands {
  const __half* a0; int a0Bn, a0H, a0W, a0C, a0pitch;
  const __half* a1; int a1Bn, a1H, a1W, a1C, a1pitch;   // nullable second source (segments with map == 1)
  const __half* w; int N, Ktot;
};
// Chooses the pixel box, N tile and pipeline depth, and builds the TMA descriptors. The caller
// fills seg[]/nseg and the epilogue fields (out, out_f32, ldo, bias, bias_bstride, res, ldr).
int igemm_configure(IgemmParams& p, const IgemmOperands& o, int outW, int outH, int outB, int mode, int geglu_bn);
int igemm_launch(cudaStream_t st, IgemmParams& p);
// Chooses an N tile for (M pixels, N columns) minimising wave-quantisation loss on `num_sms` SMs.
int igemm_pick_bn(int m_tiles, int N, int num_sms, bool geglu);

// ------------------------------------------------------------------------------------------------
// Attention (attention.cu): out[b, t, h*64:(h+1)*64] = softmax(q k^T / 8) v, head dim 64 (+ optional image sources).
// q/k/v are column windows of row-major f16 matrices (fused QKV / KV GEMM outputs).
// ------------------------------------------------------------------------------------------------
constexpr int ATTN_MAX_SRC = 8;   // image sources per attention (SDXL_MAX_IP_SOURCES)
struct AttnIpSource {
  CUtensorMap tm;              // 3D map (64 cols, S rows, batch); K and V are column windows of it
  int S, k_col0, v_col0;
  const float* scale;          // device scalar
  const float* mask;           // device [T] per-query weights, or nullptr
};
struct AttnParams {
  CUtensorMap tmQ, tmK, tmV;  // 3D maps (64 cols, rows, batch)
  int T, S, n_head, B;
  int q_col0, k_col0, v_col0;  // column of head 0 inside each matrix
  __half* out;                 // [B*T, ldo]
  int ldo;
  float scale_log2e;           // (1/sqrt(d)) * log2(e)
  // Second key/value source (IP-Adapter's decoupled cross-attention), used when S_ip > 0:
  //   out = softmax(q k^T) v + (*ip_scale) * softmax(q k_ip^T) v_ip      (two separate softmaxes, same scale)
  CUtensorMap tmKip, tmVip;    // 3D maps (64 cols, S_ip rows, batch)
  int S_ip;
  int k_ip_col0, v_ip_col0;
  const float* ip_scale;       // device scalar
  // Several image sources (DESIGN.md §13): the fields above are source 0, ip_src[k - 1] is source k < n_src. Each source adds
  //   (*scale) * mask[t] * softmax(q k_src^T) v_src          (its own softmax; mask == nullptr: 1)
  // in source order to the text attention of query row t of every batch row.
  int n_src;                   // 1 .. ATTN_MAX_SRC when S_ip > 0
  const float* ip_mask;        // source 0's per-query weights [T] (device), or nullptr
  AttnIpSource ip_src[ATTN_MAX_SRC - 1];
};
int make_tmap_rows(CUtensorMap* tm, const __half* base, int rows_per_batch, int nbatch, int cols, int pitch);
int attention_launch(cudaStream_t st, const AttnParams& p);
// An image-prompt mask plane f32 [H, W] resized to one level's queries: out[T] = bicubic resize to (mh, mw) (torch's
// F.interpolate(mode="bicubic", align_corners=False)) flattened row-major, zero-padded or cut to T.
int ip_mask_resize_launch(cudaStream_t st, const float* mask, int H, int W, int mh, int mw, int T, float* out);

// ------------------------------------------------------------------------------------------------
// Norms (norm.cu)
// ------------------------------------------------------------------------------------------------
// GroupNorm over NHWC f32 input (optionally the channel-concatenation of two tensors), n_group groups (a multiple of 4 up
// to 64; the UNet and VAE use 32), biased variance, eps inside the sqrt (reference groupnorm/mod.rs:52-82). Writes f16.
struct GnParams {
  const float* x1; int C1;    // [B, HW, C1]
  const float* x2; int C2;    // nullable, [B, HW, C2]  (cat([x1, x2], channel))
  int B, HW, n_group;
  const float* gamma; const float* beta;  // [C1+C2]
  float eps;
  int silu;                   // apply x*sigmoid(x) after the affine
  __half* y;                  // [B, HW, C1+C2] normalised (+SiLU) output
  __half* raw;                // nullable: un-normalised f16 copy of cat([x1,x2]) (skip-conv operand)
  float* partial;             // scratch of gn_scratch_floats(B', n_group') floats (B' >= B, n_group' >= n_group), initialised once
                              // with gn_scratch_init and then shared by any number of GroupNorms
  int nchunk;                 // filled by gn_launch
  __half* y_lo;               // nullable: f16(t - float(y)), the rounding residue of y (hi/lo split operand of the UNet's last conv)
};
size_t gn_scratch_floats(int B, int n_group);
// zeroes the arrival counters of a freshly allocated scratch (once; the kernels leave them at zero)
int gn_scratch_init(cudaStream_t st, float* scratch, int B, int n_group);
int gn_launch(cudaStream_t st, GnParams& p);
// LayerNorm over the last dim of f32 [rows, C] -> f16 [rows, C] (reference layernorm/mod.rs:34-49).
int layernorm_launch(cudaStream_t st, const float* x, const float* gamma, const float* beta, float eps,
                     int rows, int C, __half* y);

// ------------------------------------------------------------------------------------------------
// Small / elementwise kernels (elementwise.cu)
// ------------------------------------------------------------------------------------------------
// out[b,n] = act( dot(in[b,:], W[n,:]) + bias[n] + add[b*add_bstride + n] ); W f16 [N,ldw] K-major (row pitch ldw >= K).
// in_silu: apply SiLU to the input on load. out_silu: SiLU on the output.
int gemv_launch(cudaStream_t st, const float* in, int in_bstride, int Bv, int K, const __half* W, int ldw,
                const float* bias, const float* add, int add_bstride, int N, int in_silu, int out_silu,
                float* out, int out_bstride);
// timestep_embedding (reference unet/mod.rs:21-39): out[b, :] = [cos(t*f_i), sin(t*f_i)], dim even.
int timestep_embedding_launch(cudaStream_t st, const int* t_dev, int nt, int dim, float max_period,
                              float* out);
// the same of float timesteps; bit-identical to the int form at integer values
int timestep_embedding_f32_launch(cudaStream_t st, const float* t_dev, int nt, int dim, float max_period, float* out);
// First conv: x NCHW f16 [B,Cin,H,W] (Cin<=8) -> NHWC f32 [B,H,W,Cout], 3x3 pad 1. w: [Cout][3][3][Cin] f32.
int conv_in_launch(cudaStream_t st, const __half* x, int B, int Cin, int H, int W, const float* w,
                   const float* bias, int Cout, float* y);
// general form: x f16 or f32 NCHW with Bx images; output batch b reads image b % Bx. add (nullable): f32 NHWC [n_add,H,W,Cout]
// added to the output at batch b % n_add (a ControlNet's hint embedding).
int conv_in_launch_t(cudaStream_t st, const void* x, int x_f32, int Bx, int B, int Cin, int H, int W,
                     const float* w, const float* bias, int Cout, float* y, const float* add = nullptr, int n_add = 1);
// two-source form (the inpainting UNet): input channels [0, C1) from x as above, [C1, C1 + C2) from x2 f32 NCHW [n2, C2, H, W]
// at batch b % n2; C1 + C2 <= 9. w: [Cout][3][3][C1 + C2].
int conv_in_cat_launch(cudaStream_t st, const void* x, int x_f32, int Bx, int B, int C1, const float* x2, int n2, int C2, int H, int W,
                       const float* w, const float* bias, int Cout, float* y, const float* add = nullptr, int n_add = 1);
// y = f16(silu(x)) of NHWC f32 [B,H,W,C]; phase != 0: written as the stride-2 phase split of phase_split_launch.
int silu_f16_launch(cudaStream_t st, const float* x, int B, int H, int W, int C, int phase, __half* y);
// wo[i] = f16(s * w[i]) (i < nw), bo[i] = s * b[i] (i < nb)
int scale_weights_launch(cudaStream_t st, const __half* w, size_t nw, const float* b, int nb, float s, __half* wo, float* bo);
// Nearest-2x upsample of NHWC: f32 [B,H,W,C] -> f16 [B,2H,2W,C] (reference unet/mod.rs:742-751).
int upsample2x_launch(cudaStream_t st, const float* x, int B, int H, int W, int C, __half* y);
// Stride-2 phase split: f32 [B,H,W,C] -> f16 [4(phase=ph*2+pw), B, H/2, W/2, C]; phase image
// P[ph][pw][i][j] = x[2i+ph][2j+pw].
int phase_split_launch(cudaStream_t st, const float* x, int B, int H, int W, int C, __half* y);
int cast_f32_to_f16_launch(cudaStream_t st, const float* x, size_t n, __half* y);
int cast_f16_to_f32_launch(cudaStream_t st, const __half* x, size_t n, float* y);
// eps NHWC f32 [B,HW,ldx] (first C valid) -> NCHW [B,C,HW], f16 or f32 output
int nhwc_to_nchw_f16_launch(cudaStream_t st, const float* x, int B, int HW, int C, int ldx, __half* y);
int nhwc_to_nchw_f32_launch(cudaStream_t st, const float* x, int B, int HW, int C, int ldx, float* y);
// Sampler elementwise (reference stablediffusion/mod.rs:407-428, 463-465, 539-540).
// eps layout: NHWC f32 [nfwd*Bimg, HW, ld]; cond rows first, then uncond (if cfg).
// x: NCHW f32 master latent [Bimg,C,HW], updated in place. use_pag (DESIGN.md §14): a last group of Bimg perturbed rows follows,
// eps rows [cond | uncond | ptb] (use_cfg) or [cond | ptb], and e = (u + (c - u) * guidance) + p_t * (c - ptb), resp. c + p_t * (c - ptb).
// What the guided model output g of the two step kernels is (DESIGN.md §18). The default is the epsilon prediction without
// guidance rescale, the kernels' first instantiation.
//   v       g is the v prediction: cfg_ddim takes x0 = sqrt_a * x - sqrt_1ma * g and eps = sqrt_a * g + sqrt_1ma * x, the guided
//           step D = dx * xh - de * g (schedule.h: d_scale)
//   factor  per-image guidance-rescale factors [Bimg] on the device (guidance_stats_launch): g = g * factor[b] before its use
struct Prediction {
  int v = 0;
  const float* factor = nullptr;
  float dx = 0.f, de = 0.f;
};
// use_img (image guidance, DESIGN.md §21): the eps rows are [cond | img | uncond] and e = (u + (c - i) * guidance) + img_guidance * (i - u)
// in that order; use_cfg and use_pag are then not read. The step kernels and guidance_stats_launch take it the same way.
int cfg_ddim_launch(cudaStream_t st, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag, float guidance,
                    float p_t, float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map, float* x, const Prediction& pr = {},
                    int use_img = 0, float img_guidance = 0.f);
// Guidance rescale (diffusers' rescale_noise_cfg, Lin et al. 2023): for each image b of the rows [cond | uncond] or
// [cond | uncond | ptb], with c_b its conditional output and g_b its guided output as the step kernels compute them,
//   factor[b] = phi * std(c_b) / std(g_b) + (1 - phi)   (unbiased std over C * HW; std(c_b) / std(g_b) read as 1 when std(g_b) = 0)
// One launch: per-block (n, mean, M2) partials in double, merged in block order by the last block of each image (an arrival
// counter orders the blocks; no value goes through an atomic). scratch: guidance_stats_scratch_bytes(Bimg) bytes, initialised once
// with guidance_stats_scratch_init.
size_t guidance_stats_scratch_bytes(int Bimg);
int guidance_stats_scratch_init(cudaStream_t st, void* scratch, int Bimg);
int guidance_stats_launch(cudaStream_t st, const float* eps, int ld, int Bimg, int C, int HW, int use_pag, float guidance, float p_t,
                          float phi, void* scratch, float* factor, int use_img = 0, float img_guidance = 0.f);
// PAG's identity self-attention on `rows` token rows: out[r, 0:C] = qkv[r, 2C:3C] (qkv row pitch 3C, out row pitch C); C % 8 == 0,
// both pointers 16-byte aligned.
int pag_identity_launch(cudaStream_t st, const __half* qkv, int C, long rows, __half* out);
// x = mask ? x : ref*sqrt_a + noise*sqrt_1ma over n_per_img_batch elements.
int inpaint_blend_launch(cudaStream_t st, float* x, const float* ref, const float* noise, const uint8_t* mask,
                         size_t n_per_img_batch, float sqrt_a, float sqrt_1ma);
// x = x*sa + noise*sb  (refine_latent entry, reference stablediffusion/mod.rs:363-367)
int axpby_launch(cudaStream_t st, float* x, const float* noise, size_t n, float sa, float sb);
// Standard normal noise, Philox4x32-10 + Box-Muller, element i of stream (seed, subseq).
int randn_launch(cudaStream_t st, float* out, size_t n, uint64_t seed, uint64_t subseq);
// One step of a scheduled sampler (DESIGN.md §16) on the k-diffusion-scaled state xh, f32 NCHW [Bimg, C, HW], in one launch:
//   e   = guided eps of the NHWC rows [cond], [cond | uncond], [cond | ptb] or [cond | uncond | ptb] (cfg_ddim's combines)
//   D   = xh - sigma * e                          (eps == nullptr: no model output, D = xh: the entry of a call; v: Prediction)
//   xh' = cx * xh + cd * D + ch * hist + cn * z   (hist read when ch != 0, then D written to it when write_hist)
//   xh' = mask ? xh' : ref + sigma_blend * zb     (mask != nullptr: the latent blend before the next forward)
//   x_in = c_in * xh'                             (the next forward's input)
// z and zb are read from memory when non-null, else generated in the kernel as randn_launch(seed, z_subseq / zb_subseq) would.
struct GuidedStepParams {
  const float* eps;
  int ld, Bimg, C, HW, use_cfg, use_pag;
  float guidance, p_t, sigma;
  float cx, cd, ch, cn, c_in;
  float* xh;
  float* x_in;
  float* hist;
  int write_hist;
  const float* z;
  const float* zb;
  uint64_t seed, z_subseq, zb_subseq;
  const uint8_t* mask;
  const float* ref;
  float sigma_blend;
};
// The two-row form of the step (DESIGN.md §20), for samplers that keep a saved state xs and a second history slot h2 (each f32 NCHW
// like xh). With it, from the values before the launch:
//   xh' = cx xh + cs xs + cd D + ch hist + ch2 h2 + cn z                    (then the blend and x_in as above)
//   xs' = sx xh + ss xs + sd D + sh hist + sh2 h2                           (write_xs)
//   h2' = hist (shift), hist' = D (write_hist)
// xs is read when cs or ss is non-zero, hist when ch or sh is or shift is asked, h2 when ch2 or sh2 is.
struct StepRows {
  float* xs = nullptr;
  float* h2 = nullptr;
  float cs = 0.f, ch2 = 0.f;
  float sx = 0.f, ss = 0.f, sd = 0.f, sh = 0.f, sh2 = 0.f;
  int write_xs = 0, shift = 0;
};
// rows == nullptr: the one-row form above. use_img: cfg_ddim_launch's image-guidance combine of the rows [cond | img | uncond].
int guided_step_launch(cudaStream_t st, const GuidedStepParams& p, const Prediction& pr = {}, const StepRows* rows = nullptr,
                       int use_img = 0, float img_guidance = 0.f);

// Latent-decoder kernels (vae_kernels.cu)
// P[r,:] = softmax(scale * S[r,:]); S f32 [rows, lds] -> P f16 [rows, ldp]; cols % 4 == 0.
int softmax_rows_launch(cudaStream_t st, const float* S, size_t lds, int rows, int cols, float scale, __half* P,
                        size_t ldp);
// y[c, r] = x[r, c]; x f16 [rows, ldx], y f16 [cols, ldy].
int transpose_f16_launch(cudaStream_t st, const __half* x, size_t ldx, int rows, int cols, __half* y, size_t ldy);
// 1x1 conv on the rescaled latent: y = W (x * inv_scale) + b; NCHW f32 [B, C<=8, HW]; W f32 [C, C].
int post_quant_launch(cudaStream_t st, const float* x, int B, int C, int HW, const float* w, const float* bias,
                      float inv_scale, float* y);
// u8[b,p,c] = trunc(clamp(((x+1)/2)*255, 0, 255)), c < 3, from NHWC f32 [npix, ldx]; NaN -> 0.
int image_u8_launch(cudaStream_t st, const float* x, long npix, int ldx, uint8_t* out);

// u8 [B,HW,3] -> f32 NCHW [B,3,HW], ((v/255)*2)-1.
int image_from_u8_launch(cudaStream_t st, const uint8_t* in, int B, long HW, float* out);
// quant_conv on the first Cout output channels, times scale: x NHWC f32 [B,HW,Cz] -> y NCHW f32 [B,Cout,HW]; w f32 [Cz,Cz].
int quant_out_launch(cudaStream_t st, const float* x, int B, int Cz, int Cout, long HW, const float* w, const float* bias,
                     float scale, float* y);

// Text-encoder kernels (clip_kernels.cu)
// x[b*T+t,:] = tok_emb[tokens[b,t],:] + pos_emb[t,:] (f16 tables -> f32); *err is set to 1 on an id outside [0, n_vocab).
int embed_tokens_launch(cudaStream_t st, const int* tokens, int rows, int T, int C, int n_vocab, const __half* tok_emb,
                        const __half* pos_emb, float* x, int* err);
// Masked attention for short sequences, scale 1/sqrt(head_dim): additive f16 mask [T,S] (nullable) and/or causal (key <= query).
// head_dim: 64 (the text encoders' kernel) or another multiple of 8 up to 128.
int attention_small_launch(cudaStream_t st, const __half* q, int q_pitch, int q_col0, const __half* k, const __half* v,
                           int kv_pitch, int k_col0, int v_col0, int B, int T, int S, int n_head, const __half* mask,
                           int causal, __half* out, int ldo, int head_dim = 64);
// CLIP vision embedding: pixels f32 NCHW [N,3,S,S] -> f16 patch rows [N*(S/p)^2, Kpad], columns in OIHW (c, kh, kw) order.
int patchify_launch(cudaStream_t st, const float* pixels, int N, int S, int p, int Kpad, __half* y);
// x f32 [N*T, C] = LayerNorm([class ; patches[n]] + position) (T = patches per image + 1).
int vision_embed_ln_launch(cudaStream_t st, const float* patches, const __half* cls, const __half* pos, int N, int T, int C,
                           const float* gamma, const float* beta, float eps, float* x);
// y = gelu_erf(x) (quick = 0) or x * sigmoid(1.702 x) (quick = 1); f32 -> f16, n % 4 == 0.
int mlp_act_launch(cudaStream_t st, const float* x, size_t n, int quick, __half* y);
// y[b,:] = LayerNorm(x[b*T + idx[b], :]) in f32.
int ln_gather_f32_launch(cudaStream_t st, const float* x, const int* idx, int B, int T, int C, const float* gamma,
                         const float* beta, float eps, float* y);
// The LayerNorms of one IP-Adapter Plus perceiver-attention layer: x f32 [n*L, C] (LN1: g1, b1) and lat f32 [n*Q, C] (LN2: g2, b2)
// -> kv f16 [n, L+Q, C] (per image: the L rows of LN1(x), then the Q rows of LN2(lat)) and q f16 [n*Q, C] (the LN2 rows again).
int perceiver_ln_launch(cudaStream_t st, const float* x, const float* lat, int n, int L, int Q, int C, const float* g1,
                        const float* b1, const float* g2, const float* b2, float eps, __half* kv, __half* q);

// T2I-Adapter kernels (t2i_kernels.cu)
// PixelUnshuffle(16): hint f32 NCHW [n, C, H, W] -> f16 NHWC [n, H/16, W/16, C*256], channel ci*256 + i*16 + j <- hint[ci, 16y+i, 16x+j].
int pixel_unshuffle_launch(cudaStream_t st, const float* x, int n, int C, int H, int W, __half* y);
// y = f16(relu(x)), n % 4 == 0.
int relu_f16_launch(cudaStream_t st, const float* x, size_t n, __half* y);
// 2x2 stride-2 average pool: f32 NHWC [n, H, W, C] -> f16 NHWC [n, H/2, W/2, C], C % 4 == 0.
int avg_pool2_f16_launch(cudaStream_t st, const float* x, int n, int H, int W, int C, __half* y);
// x[b] += F[b % n_hint] (f32, per_img floats per image, a multiple of 4) when *t >= *t_min; t and t_min are device ints. PDL plan op.
int t2i_add_launch(cudaStream_t st, float* x, const float* F, long per_img, int B, int n_hint, const int* t, const int* t_min);

// FreeU at one decoder skip concatenation (freeu.cu, DESIGN.md §15), in place on f32 NHWC tensors of B rows at H x W: the skip
// r [B, H, W, C] becomes diffusers' fourier_filter(r, threshold 1, scale *s) and the channels [0, Cx / 2) of x [B, H, W, Cx] are
// multiplied by *b. tw: freeu_twiddles(H, W) on the device; s, b: device floats. PDL plan op, one launch.
int freeu_launch(cudaStream_t st, float* r, int C, float* x, int Cx, int B, int H, int W, const float* tw, const float* s,
                 const float* b);
// Host: the twiddle table of an H x W skip, 2 * (H + W) floats [cos 2 pi h / H | sin 2 pi h / H | cos 2 pi w / W | sin 2 pi w / W],
// computed in double precision.
void freeu_twiddles(int H, int W, float* out);

// Weight re-layout at load time (elementwise.cu)
// Linear [K(in), N(out)] row-major f16 -> K-major [N, Kpad] f16 (zero padded), dst row pitch Kpad;
// rows written at dst_row0 + perm(n) where perm handles the GEGLU value/gate interleave (geglu_bn>0).
int transpose_linear_launch(cudaStream_t st, const __half* src, int K, int N, __half* dst, int Kpad,
                            int dst_row0, int geglu_bn);
// Conv OIHW f16 -> [O, (kh,kw,I padded to Ipad)] f16 at column offset col0 of a [O, Ktot] matrix.
int repack_conv_launch(cudaStream_t st, const __half* src, int O, int I, int KH, int KW, __half* dst,
                       int Ktot, int col0, int Ipad);
// 3x3 conv that follows a nearest-2x upsample -> four 2x2 phase kernels on the original image (sums of the 3x3 taps that
// read the same source pixel, added in f32, rounded once): dst [4 (a*2+b)][O][4 (th*2+tw) * Ipad].
int repack_upconv_launch(cudaStream_t st, const __half* src, int O, int I, __half* dst, int Ipad);
int vec_add_f32_launch(cudaStream_t st, float* dst, const float* src, int n);  // dst += src
// bias f16 [N] -> f32, optional GEGLU permutation, optional accumulate (dst += src).
int bias_to_f32_launch(cudaStream_t st, const __half* src, int N, float* dst, int geglu_bn, int accumulate);

// LoRA merge (elementwise.cu). The delta of one weight slot is the [N, Kd] matrix
//   delta = sum_t coef_t * (up_t [N, r_t] @ down_t [r_t, Kd])      (f32; terms in order, rank index ascending)
// Kd = I * taps: column k of the delta is input channel i = k / taps, tap = k % taps (down's natural [r, I, kh, kw] order).
// Element (n, k) is stored at dst[(row0 + geglu_perm(n)) * ld + col0 + tap * Ipad + i] as f16(src + delta), with src the
// backed-up weight at the same offset (f32 storage: float(f16(src + delta))). With `delta_out` set the kernel writes the f32
// delta [N, Kd] there instead (upsample convs, DoRA layers and LoKr factors; see lora_upconv_merge_launch, dora_*_launch).
// A term's product P (the `up @ down` above) depends on its kind (DESIGN.md §19):
//   LORA_LORA   P = up [N, r] @ down [r, Kd]
//   LORA_LOHA   P = (up @ down) * (up2 [N, r2] @ down2 [r2, Kd])            (both pairs staged like LORA, then multiplied)
//   LORA_LOKR   P[i*c + j, (p*d + q)*taps + t] = w1[i, p] * w2[j, q*taps + t]  (w1 f32 [N/c, I/d], w2 f32 [c, d*taps])
//   LORA_FULL   P = down as f16 [N, Kd]
//   LORA_F32    P = w1 as f32 [N, Kd] (a delta staged by an earlier launch; with coef 1 the kernel just applies it)
// A set of LORA_LORA terms only runs the kernel's original instantiation.
#define LORA_MAX_TERMS 16
enum { LORA_LORA = 0, LORA_LOHA = 1, LORA_LOKR = 2, LORA_FULL = 3, LORA_F32 = 4 };
struct LoraTerm {
  const __half* up; const __half* down; int r; float coef;
  int kind;
  const __half* up2; const __half* down2; int r2;   // LORA_LOHA
  const float* w1; const float* w2; int c, d;       // LORA_LOKR (w2 rows c, w2 input channels d); LORA_F32: w1
};
struct LoraMergeParams {
  int N, Kd, taps;
  int nterm;
  LoraTerm term[LORA_MAX_TERMS];
  const void* src; void* dst; int f32;
  size_t ld; int row0, col0, Ipad, geglu_bn;
  float* delta_out;
};
int lora_merge_launch(cudaStream_t st, const LoraMergeParams& p);
// Upsample conv: the 3x3 f32 delta [O, I*9] is summed into the four 2x2 phase kernels with the tap sets of
// repack_upconv_kernel and added to the backed-up phase weights src (layout of repack_upconv_launch's dst).
int lora_upconv_merge_launch(cudaStream_t st, const __half* src, const float* delta, int O, int I, __half* dst, int Ipad);
// DoRA (DESIGN.md §19). `slot` gives the weight W through its slot map (src, f32, ld, row0, col0, Ipad, geglu_bn, N, Kd, taps;
// its terms are not read); dw is the adapter's f32 delta [N, Kd] (coef included, scale not). axis 0: one norm per output row n
// over all Kd; axis 1: one norm per input channel i over N and the taps.
//   dora_norm:  norm[j] = sqrt(sum (W + dw)^2) in double, one CTA per row or input channel, fixed order and tree reduction.
//               No atomics.
//   dora_accum: acc[n, k] += f32(s * (m[j] * (W + dw) / norm[j] - W)) computed in double; 0 where norm[j] == 0.
int dora_norm_launch(cudaStream_t st, const LoraMergeParams& slot, const float* dw, int axis, double* norm);
int dora_accum_launch(cudaStream_t st, const LoraMergeParams& slot, const float* dw, const float* m, const double* norm, int axis,
                      float s, float* acc);

}  // namespace sdxl
