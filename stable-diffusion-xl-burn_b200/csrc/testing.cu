// Test-only C entry points to the internal launchers of kernels.h (linked into libsdxl_b200_testing.so, never into the
// product library). Each wrapper takes plain arguments, fills the launcher's parameter struct exactly as the UNet's launch
// plan does (engine_core.h: PlanBuilder) and launches on `stream`, so tests can pin the fused layouts the plan uses —
// second K sources, per-batch bias rows, scattered upsample outputs, column windows of fused QKV / KV matrices — kernel by
// kernel against a float64 reference. The VAE, text / vision encoder, T2I-Adapter and sampler kernels are reached the same
// way. All pointers are device pointers; every function returns the launcher's status.
#include "kernels.h"
#include "schedule.h"

#define SDXL_TEST_API extern "C" __attribute__((visibility("default")))

using namespace sdxl;

// segs: nseg rows of (map, dw, dh, db, nkb). opix_row == 0 keeps igemm_configure's dense output map.
SDXL_TEST_API int sdxl_test_igemm(void* stream, const void* a0, int a0Bn, int a0H, int a0W, int a0C, int a0pitch, const void* a1,
                                  int a1Bn, int a1H, int a1W, int a1C, int a1pitch, const void* w, int N, int Ktot, int outW,
                                  int outH, int outB, int mode, int geglu_bn, const int* segs, int nseg, void* out, int out_f32,
                                  int ldo, const float* bias, int bias_bstride, const float* res, int ldr, int opix_row,
                                  int opix_w, int opix_off) {
  if (nseg < 1 || nseg > IGEMM_MAX_SEG) return 5002;
  IgemmParams p{};
  p.nseg = nseg;
  for (int i = 0; i < nseg; ++i)
    p.seg[i] = {(int16_t)segs[5 * i], (int16_t)segs[5 * i + 1], (int16_t)segs[5 * i + 2], (int16_t)segs[5 * i + 3], segs[5 * i + 4]};
  p.out = out; p.out_f32 = out_f32; p.ldo = ldo;
  p.bias = bias; p.bias_bstride = bias_bstride;
  p.res = res; p.ldr = ldr;
  const IgemmOperands o{(const __half*)a0, a0Bn, a0H, a0W, a0C, a0pitch, (const __half*)a1, a1Bn, a1H, a1W, a1C, a1pitch,
                        (const __half*)w, N, Ktot};
  if (int r = igemm_configure(p, o, outW, outH, outB, mode, geglu_bn)) return r;
  if (opix_row) { p.opix_row = opix_row; p.opix_w = opix_w; p.opix_off = opix_off; }
  return igemm_launch((cudaStream_t)stream, p);
}

// Flash attention as PlanBuilder::attn / attn_ip set it up: q, k, v are column windows of row-major matrices (one tensor map
// per matrix, K and V share theirs); kip == nullptr: no image-prompt source.
SDXL_TEST_API int sdxl_test_attention(void* stream, const void* q, int q_pitch, int q_col0, const void* kv, int kv_pitch, int k_col0,
                                      int v_col0, int B, int T, int S, int n_head, void* out, int ldo, const void* kip,
                                      int kip_pitch, int k_ip_col0, int v_ip_col0, int S_ip, const float* ip_scale) {
  AttnParams p{};
  p.T = T; p.S = S; p.n_head = n_head; p.B = B;
  p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
  p.out = (__half*)out; p.ldo = ldo;
  p.scale_log2e = (float)(1.4426950408889634 / 8.0);
  int r = make_tmap_rows(&p.tmQ, (const __half*)q, T, B, q_pitch, q_pitch);
  if (!r) r = make_tmap_rows(&p.tmK, (const __half*)kv, S, B, kv_pitch, kv_pitch);
  if (r) return r;
  p.tmV = p.tmK;
  if (kip) {
    p.S_ip = S_ip; p.k_ip_col0 = k_ip_col0; p.v_ip_col0 = v_ip_col0; p.ip_scale = ip_scale; p.n_src = 1;
    if ((r = make_tmap_rows(&p.tmKip, (const __half*)kip, S_ip, B, kip_pitch, kip_pitch))) return r;
    p.tmVip = p.tmKip;
  }
  return attention_launch((cudaStream_t)stream, p);
}

// The same with n_src image sources as PlanBuilder::attn_ip sets them up: source k reads K / V as column windows src_info[4k + 1]
// / src_info[4k + 2] of src_kv[k] [B * src_info[4k + 3], src_info[4k]] and adds *scales[k] * masks[k][t] (masks[k] nullable) times
// its own softmax. The pointer and info arrays are host memory.
SDXL_TEST_API int sdxl_test_attention_multi(void* stream, const void* q, int q_pitch, int q_col0, const void* kv, int kv_pitch, int k_col0,
                                            int v_col0, int B, int T, int S, int n_head, void* out, int ldo, int n_src,
                                            const void* const* src_kv, const int* src_info, const float* const* scales,
                                            const float* const* masks) {
  if (n_src < 1 || n_src > ATTN_MAX_SRC) return 5003;
  AttnParams p{};
  p.T = T; p.S = S; p.n_head = n_head; p.B = B;
  p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
  p.out = (__half*)out; p.ldo = ldo;
  p.scale_log2e = (float)(1.4426950408889634 / 8.0);
  int r = make_tmap_rows(&p.tmQ, (const __half*)q, T, B, q_pitch, q_pitch);
  if (!r) r = make_tmap_rows(&p.tmK, (const __half*)kv, S, B, kv_pitch, kv_pitch);
  if (r) return r;
  p.tmV = p.tmK;
  p.n_src = n_src;
  for (int k = 0; k < n_src; ++k) {
    const int* f = src_info + 4 * k;
    CUtensorMap tm;
    if ((r = make_tmap_rows(&tm, (const __half*)src_kv[k], f[3], B, f[0], f[0]))) return r;
    if (k == 0) {
      p.tmKip = p.tmVip = tm;
      p.S_ip = f[3]; p.k_ip_col0 = f[1]; p.v_ip_col0 = f[2]; p.ip_scale = scales[0]; p.ip_mask = masks[0];
    } else {
      p.ip_src[k - 1] = {tm, f[3], f[1], f[2], scales[k], masks[k]};
    }
  }
  return attention_launch((cudaStream_t)stream, p);
}

// The image-prompt mask resize run when masks are attached (engine.cu: ip_stage).
SDXL_TEST_API int sdxl_test_ip_mask_resize(void* stream, const float* mask, int H, int W, int mh, int mw, int T, float* out) {
  return ip_mask_resize_launch((cudaStream_t)stream, mask, H, W, mh, mw, T, out);
}

SDXL_TEST_API int sdxl_test_attention_small(void* stream, const void* q, int q_pitch, int q_col0, const void* k, const void* v,
                                            int kv_pitch, int k_col0, int v_col0, int B, int T, int S, int n_head, const void* mask,
                                            int causal, void* out, int ldo, int head_dim) {
  return attention_small_launch((cudaStream_t)stream, (const __half*)q, q_pitch, q_col0, (const __half*)k, (const __half*)v, kv_pitch,
                                k_col0, v_col0, B, T, S, n_head, (const __half*)mask, causal, (__half*)out, ldo, head_dim);
}

// The IP-Adapter Plus Resampler's per-layer LayerNorms (engine.cu: ip_resample).
SDXL_TEST_API int sdxl_test_perceiver_ln(void* stream, const float* x, const float* lat, int n, int L, int Q, int C, const float* g1,
                                         const float* b1, const float* g2, const float* b2, float eps, void* kv, void* q) {
  return perceiver_ln_launch((cudaStream_t)stream, x, lat, n, L, Q, C, g1, b1, g2, b2, eps, (__half*)kv, (__half*)q);
}

SDXL_TEST_API size_t sdxl_test_gn_scratch_floats(int B, int n_group) { return gn_scratch_floats(B, n_group); }
SDXL_TEST_API int sdxl_test_gn_scratch_init(void* stream, float* scratch, int B, int n_group) {
  return gn_scratch_init((cudaStream_t)stream, scratch, B, n_group);
}
// GroupNorm on a caller-owned scratch (initialised once with sdxl_test_gn_scratch_init, as the plan does); raw / y_lo nullable.
SDXL_TEST_API int sdxl_test_gn(void* stream, const float* x1, int C1, const float* x2, int C2, int B, int HW, int n_group,
                               const float* gamma, const float* beta, float eps, int silu, void* y, void* raw, void* y_lo,
                               float* scratch) {
  GnParams p{x1, C1, x2, C2, B, HW, n_group, gamma, beta, eps, silu, (__half*)y, (__half*)raw, scratch, 0, (__half*)y_lo};
  return gn_launch((cudaStream_t)stream, p);
}

SDXL_TEST_API int sdxl_test_gemv(void* stream, const float* in, int in_bstride, int Bv, int K, const void* W, int ldw,
                                 const float* bias, const float* add, int add_bstride, int N, int in_silu, int out_silu, float* out,
                                 int out_bstride) {
  return gemv_launch((cudaStream_t)stream, in, in_bstride, Bv, K, (const __half*)W, ldw, bias, add, add_bstride, N, in_silu, out_silu,
                     out, out_bstride);
}

SDXL_TEST_API int sdxl_test_conv_in(void* stream, const void* x, int x_f32, int Bx, int B, int Cin, int H, int W, const float* w,
                                    const float* bias, int Cout, float* y, const float* add, int n_add) {
  return conv_in_launch_t((cudaStream_t)stream, x, x_f32, Bx, B, Cin, H, W, w, bias, Cout, y, add, n_add);
}
// The inpainting UNet's first conv: channels [0, C1) from x (image b % Bx), [C1, C1 + C2) from x2 f32 (image b % n2).
SDXL_TEST_API int sdxl_test_conv_in_cat(void* stream, const void* x, int x_f32, int Bx, int B, int C1, const float* x2, int n2, int C2,
                                        int H, int W, const float* w, const float* bias, int Cout, float* y) {
  return conv_in_cat_launch((cudaStream_t)stream, x, x_f32, Bx, B, C1, x2, n2, C2, H, W, w, bias, Cout, y);
}

// PAG's identity self-attention on `rows` rows of a fused QKV matrix (pitch 3C) into out (pitch C), as the plan's OP_PAG_IDENTITY.
SDXL_TEST_API int sdxl_test_pag_identity(void* stream, const void* qkv, int C, long rows, void* out) {
  return pag_identity_launch((cudaStream_t)stream, (const __half*)qkv, C, rows, (__half*)out);
}

// FreeU at one skip concatenation, as the plan's OP_FREEU: the twiddle table (host, 2 * (H + W) floats) and the in-place launch.
SDXL_TEST_API void sdxl_test_freeu_twiddles(int H, int W, float* out_host) { freeu_twiddles(H, W, out_host); }
SDXL_TEST_API int sdxl_test_freeu(void* stream, float* r, int C, float* x, int Cx, int B, int H, int W, const float* tw, const float* s,
                                  const float* b) {
  return freeu_launch((cudaStream_t)stream, r, C, x, Cx, B, H, W, tw, s, b);
}

SDXL_TEST_API int sdxl_test_repack_upconv(void* stream, const void* src, int O, int I, void* dst, int Ipad) {
  return repack_upconv_launch((cudaStream_t)stream, (const __half*)src, O, I, (__half*)dst, Ipad);
}
SDXL_TEST_API int sdxl_test_repack_conv(void* stream, const void* src, int O, int I, int KH, int KW, void* dst, int Ktot, int col0,
                                        int Ipad) {
  return repack_conv_launch((cudaStream_t)stream, (const __half*)src, O, I, KH, KW, (__half*)dst, Ktot, col0, Ipad);
}
SDXL_TEST_API int sdxl_test_transpose_linear(void* stream, const void* src, int K, int N, void* dst, int Kpad, int dst_row0,
                                             int geglu_bn) {
  return transpose_linear_launch((cudaStream_t)stream, (const __half*)src, K, N, (__half*)dst, Kpad, dst_row0, geglu_bn);
}
SDXL_TEST_API int sdxl_test_bias_to_f32(void* stream, const void* src, int N, float* dst, int geglu_bn, int accumulate) {
  return bias_to_f32_launch((cudaStream_t)stream, (const __half*)src, N, dst, geglu_bn, accumulate);
}

// nterm LoRA terms: up[t] [N, r[t]] f16, down[t] [r[t], Kd] f16, coef[t].
SDXL_TEST_API int sdxl_test_lora_merge(void* stream, int N, int Kd, int taps, int nterm, const void* const* up, const void* const* down,
                                       const int* r, const float* coef, const void* src, void* dst, int f32, size_t ld, int row0,
                                       int col0, int Ipad, int geglu_bn, float* delta_out) {
  if (nterm < 1 || nterm > LORA_MAX_TERMS) return 1;
  LoraMergeParams p{};
  p.N = N; p.Kd = Kd; p.taps = taps; p.nterm = nterm;
  for (int i = 0; i < nterm; ++i) p.term[i] = {(const __half*)up[i], (const __half*)down[i], r[i], coef[i]};
  p.src = src; p.dst = dst; p.f32 = f32;
  p.ld = ld; p.row0 = row0; p.col0 = col0; p.Ipad = Ipad; p.geglu_bn = geglu_bn;
  p.delta_out = delta_out;
  return lora_merge_launch((cudaStream_t)stream, p);
}
// nterm terms of any kind (kernels.h: LORA_*): per term ints[5 t ..] = kind, r, r2, c, d and ptrs[6 t ..] = up, down, up2,
// down2, w1, w2.
SDXL_TEST_API int sdxl_test_lora_merge_kinds(void* stream, int N, int Kd, int taps, int nterm, const int* ints, const void* const* ptrs,
                                             const float* coef, const void* src, void* dst, int f32, size_t ld, int row0, int col0,
                                             int Ipad, int geglu_bn, float* delta_out) {
  if (nterm < 1 || nterm > LORA_MAX_TERMS) return 1;
  LoraMergeParams p{};
  p.N = N; p.Kd = Kd; p.taps = taps; p.nterm = nterm;
  for (int i = 0; i < nterm; ++i) {
    LoraTerm& T = p.term[i];
    const int* v = ints + 5 * i;
    const void* const* q = ptrs + 6 * i;
    T.kind = v[0]; T.r = v[1]; T.r2 = v[2]; T.c = v[3]; T.d = v[4]; T.coef = coef[i];
    T.up = (const __half*)q[0]; T.down = (const __half*)q[1]; T.up2 = (const __half*)q[2]; T.down2 = (const __half*)q[3];
    T.w1 = (const float*)q[4]; T.w2 = (const float*)q[5];
  }
  p.src = src; p.dst = dst; p.f32 = f32;
  p.ld = ld; p.row0 = row0; p.col0 = col0; p.Ipad = Ipad; p.geglu_bn = geglu_bn;
  p.delta_out = delta_out;
  return lora_merge_launch((cudaStream_t)stream, p);
}
static LoraMergeParams dora_slot(int N, int Kd, int taps, const void* src, int f32, size_t ld, int row0, int col0, int Ipad, int geglu_bn) {
  LoraMergeParams p{};
  p.N = N; p.Kd = Kd; p.taps = taps; p.src = src; p.f32 = f32;
  p.ld = ld; p.row0 = row0; p.col0 = col0; p.Ipad = Ipad; p.geglu_bn = geglu_bn;
  return p;
}
SDXL_TEST_API int sdxl_test_dora_norm(void* stream, int N, int Kd, int taps, const void* src, int f32, size_t ld, int row0, int col0,
                                      int Ipad, int geglu_bn, const float* dw, int axis, double* norm) {
  return dora_norm_launch((cudaStream_t)stream, dora_slot(N, Kd, taps, src, f32, ld, row0, col0, Ipad, geglu_bn), dw, axis, norm);
}
SDXL_TEST_API int sdxl_test_dora_accum(void* stream, int N, int Kd, int taps, const void* src, int f32, size_t ld, int row0, int col0,
                                       int Ipad, int geglu_bn, const float* dw, const float* m, const double* norm, int axis, float s,
                                       float* acc) {
  return dora_accum_launch((cudaStream_t)stream, dora_slot(N, Kd, taps, src, f32, ld, row0, col0, Ipad, geglu_bn), dw, m, norm, axis,
                           s, acc);
}
SDXL_TEST_API int sdxl_test_lora_upconv_merge(void* stream, const void* src, const float* delta, int O, int I, void* dst, int Ipad) {
  return lora_upconv_merge_launch((cudaStream_t)stream, (const __half*)src, delta, O, I, (__half*)dst, Ipad);
}

// The latent decoder's and encoder's small kernels (vae_kernels.cu).
SDXL_TEST_API int sdxl_test_softmax_rows(void* stream, const float* S, size_t lds, int rows, int cols, float scale, void* P,
                                         size_t ldp) {
  return softmax_rows_launch((cudaStream_t)stream, S, lds, rows, cols, scale, (__half*)P, ldp);
}
SDXL_TEST_API int sdxl_test_transpose_f16(void* stream, const void* x, size_t ldx, int rows, int cols, void* y, size_t ldy) {
  return transpose_f16_launch((cudaStream_t)stream, (const __half*)x, ldx, rows, cols, (__half*)y, ldy);
}
SDXL_TEST_API int sdxl_test_post_quant(void* stream, const float* x, int B, int C, int HW, const float* w, const float* bias,
                                       float inv_scale, float* y) {
  return post_quant_launch((cudaStream_t)stream, x, B, C, HW, w, bias, inv_scale, y);
}
SDXL_TEST_API int sdxl_test_quant_out(void* stream, const float* x, int B, int Cz, int Cout, long HW, const float* w, const float* bias,
                                      float scale, float* y) {
  return quant_out_launch((cudaStream_t)stream, x, B, Cz, Cout, HW, w, bias, scale, y);
}
SDXL_TEST_API int sdxl_test_image_u8(void* stream, const float* x, long npix, int ldx, uint8_t* out) {
  return image_u8_launch((cudaStream_t)stream, x, npix, ldx, out);
}
SDXL_TEST_API int sdxl_test_image_from_u8(void* stream, const uint8_t* in, int B, long HW, float* out) {
  return image_from_u8_launch((cudaStream_t)stream, in, B, HW, out);
}

// The CLIP text and vision towers' small kernels (clip_kernels.cu).
SDXL_TEST_API int sdxl_test_embed_tokens(void* stream, const int* tokens, int rows, int T, int C, int n_vocab, const void* tok_emb,
                                         const void* pos_emb, float* x, int* err) {
  return embed_tokens_launch((cudaStream_t)stream, tokens, rows, T, C, n_vocab, (const __half*)tok_emb, (const __half*)pos_emb, x, err);
}
SDXL_TEST_API int sdxl_test_patchify(void* stream, const float* pixels, int N, int S, int p, int Kpad, void* y) {
  return patchify_launch((cudaStream_t)stream, pixels, N, S, p, Kpad, (__half*)y);
}
SDXL_TEST_API int sdxl_test_vision_embed_ln(void* stream, const float* patches, const void* cls, const void* pos, int N, int T, int C,
                                            const float* gamma, const float* beta, float eps, float* x) {
  return vision_embed_ln_launch((cudaStream_t)stream, patches, (const __half*)cls, (const __half*)pos, N, T, C, gamma, beta, eps, x);
}
SDXL_TEST_API int sdxl_test_mlp_act(void* stream, const float* x, size_t n, int quick, void* y) {
  return mlp_act_launch((cudaStream_t)stream, x, n, quick, (__half*)y);
}
SDXL_TEST_API int sdxl_test_ln_gather_f32(void* stream, const float* x, const int* idx, int B, int T, int C, const float* gamma,
                                          const float* beta, float eps, float* y) {
  return ln_gather_f32_launch((cudaStream_t)stream, x, idx, B, T, C, gamma, beta, eps, y);
}

// The T2I-Adapter's kernels (t2i_kernels.cu); t and t_min are device ints.
SDXL_TEST_API int sdxl_test_pixel_unshuffle(void* stream, const float* x, int n, int C, int H, int W, void* y) {
  return pixel_unshuffle_launch((cudaStream_t)stream, x, n, C, H, W, (__half*)y);
}
SDXL_TEST_API int sdxl_test_relu_f16(void* stream, const float* x, size_t n, void* y) {
  return relu_f16_launch((cudaStream_t)stream, x, n, (__half*)y);
}
SDXL_TEST_API int sdxl_test_avg_pool2_f16(void* stream, const float* x, int n, int H, int W, int C, void* y) {
  return avg_pool2_f16_launch((cudaStream_t)stream, x, n, H, W, C, (__half*)y);
}
SDXL_TEST_API int sdxl_test_t2i_add(void* stream, float* x, const float* F, long per_img, int B, int n_hint, const int* t,
                                    const int* t_min) {
  return t2i_add_launch((cudaStream_t)stream, x, F, per_img, B, n_hint, t, t_min);
}

// The sampler's elementwise kernels and the UNet's resampling copies and casts (elementwise.cu).
// The sampler's guided DDIM update, with or without PAG (engine.cu: sampler_step).
SDXL_TEST_API int sdxl_test_cfg_ddim(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag,
                                     float guidance, float p_t, float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map, float* x) {
  return cfg_ddim_launch((cudaStream_t)stream, eps, ld, Bimg, C, HW, use_cfg, use_pag, guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap,
                         sqrt_1map, x);
}
// The same with the v prediction (v != 0) and the per-image guidance-rescale factors (factor nullable), kernels.h: Prediction.
SDXL_TEST_API int sdxl_test_cfg_ddim_pred(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag,
                                          float guidance, float p_t, float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map,
                                          float* x, int v, const float* factor) {
  Prediction pr;
  pr.v = v;
  pr.factor = factor;
  return cfg_ddim_launch((cudaStream_t)stream, eps, ld, Bimg, C, HW, use_cfg, use_pag, guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap,
                         sqrt_1map, x, pr);
}
// Guidance rescale's statistics kernel (engine.cu: step_prediction) on a scratch initialised once, as the sampler's; factor [Bimg] out.
SDXL_TEST_API size_t sdxl_test_guidance_stats_scratch_bytes(int Bimg) { return guidance_stats_scratch_bytes(Bimg); }
SDXL_TEST_API int sdxl_test_guidance_stats_scratch_init(void* stream, void* scratch, int Bimg) {
  return guidance_stats_scratch_init((cudaStream_t)stream, scratch, Bimg);
}
SDXL_TEST_API int sdxl_test_guidance_stats(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_pag, float guidance,
                                           float p_t, float phi, void* scratch, float* factor) {
  return guidance_stats_launch((cudaStream_t)stream, eps, ld, Bimg, C, HW, use_pag, guidance, p_t, phi, scratch, factor);
}
// Image guidance (DESIGN.md §21): the v / rescale forms above with the combine of the rows [cond | img | uncond] at scale s_img.
SDXL_TEST_API int sdxl_test_cfg_ddim_img(void* stream, const float* eps, int ld, int Bimg, int C, int HW, float guidance, float s_img,
                                         float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map, float* x, int v, const float* factor) {
  Prediction pr;
  pr.v = v;
  pr.factor = factor;
  return cfg_ddim_launch((cudaStream_t)stream, eps, ld, Bimg, C, HW, 1, 0, guidance, 0.f, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, x, pr, 1,
                         s_img);
}
SDXL_TEST_API int sdxl_test_guidance_stats_img(void* stream, const float* eps, int ld, int Bimg, int C, int HW, float guidance, float s_img,
                                               float phi, void* scratch, float* factor) {
  return guidance_stats_launch((cudaStream_t)stream, eps, ld, Bimg, C, HW, 0, guidance, 0.f, phi, scratch, factor, 1, s_img);
}
SDXL_TEST_API int sdxl_test_inpaint_blend(void* stream, float* x, const float* ref, const float* noise, const uint8_t* mask, size_t n,
                                          float sqrt_a, float sqrt_1ma) {
  return inpaint_blend_launch((cudaStream_t)stream, x, ref, noise, mask, n, sqrt_a, sqrt_1ma);
}
SDXL_TEST_API int sdxl_test_axpby(void* stream, float* x, const float* noise, size_t n, float sa, float sb) {
  return axpby_launch((cudaStream_t)stream, x, noise, n, sa, sb);
}
SDXL_TEST_API int sdxl_test_cast_f32_to_f16(void* stream, const float* x, size_t n, void* y) {
  return cast_f32_to_f16_launch((cudaStream_t)stream, x, n, (__half*)y);
}
SDXL_TEST_API int sdxl_test_cast_f16_to_f32(void* stream, const void* x, size_t n, float* y) {
  return cast_f16_to_f32_launch((cudaStream_t)stream, (const __half*)x, n, y);
}
SDXL_TEST_API int sdxl_test_upsample2x(void* stream, const float* x, int B, int H, int W, int C, void* y) {
  return upsample2x_launch((cudaStream_t)stream, x, B, H, W, C, (__half*)y);
}
SDXL_TEST_API int sdxl_test_phase_split(void* stream, const float* x, int B, int H, int W, int C, void* y) {
  return phase_split_launch((cudaStream_t)stream, x, B, H, W, C, (__half*)y);
}
SDXL_TEST_API int sdxl_test_silu_f16(void* stream, const float* x, int B, int H, int W, int C, int phase, void* y) {
  return silu_f16_launch((cudaStream_t)stream, x, B, H, W, C, phase, (__half*)y);
}
SDXL_TEST_API int sdxl_test_nhwc_to_nchw_f16(void* stream, const float* x, int B, int HW, int C, int ldx, void* y) {
  return nhwc_to_nchw_f16_launch((cudaStream_t)stream, x, B, HW, C, ldx, (__half*)y);
}
SDXL_TEST_API int sdxl_test_nhwc_to_nchw_f32(void* stream, const float* x, int B, int HW, int C, int ldx, float* y) {
  return nhwc_to_nchw_f32_launch((cudaStream_t)stream, x, B, HW, C, ldx, y);
}
SDXL_TEST_API int sdxl_test_scale_weights(void* stream, const void* w, size_t nw, const float* b, int nb, float s, void* wo, float* bo) {
  return scale_weights_launch((cudaStream_t)stream, (const __half*)w, nw, b, nb, s, (__half*)wo, bo);
}
SDXL_TEST_API int sdxl_test_vec_add_f32(void* stream, float* dst, const float* src, int n) {
  return vec_add_f32_launch((cudaStream_t)stream, dst, src, n);
}

// The scheduled samplers (schedule.h, elementwise.cu): the host coefficient function, out = (cx, cd, ch, cn, c_in), the step kernel
// with GuidedStepParams filled as sdxl_sample_latent_scheduled fills it, and the float timestep embedding of the UNet plan.
SDXL_TEST_API void sdxl_test_step_coef(const sdxl_schedule* s, int k, const double* timesteps, const double* sigmas, int has_prev,
                                       float* out) {
  const Stage q = step_stages(nullptr, *s, k, timesteps, sigmas, has_prev ? 1 : 0).st[0];
  out[0] = q.cx; out[1] = q.cd; out[2] = q.ch; out[3] = q.cn; out[4] = q.c_in;
}
// Every stage of step k with n_hist history slots filled (schedule.h: step_stages) over an alphas_cumprod table of n_train
// entries; returns the number of stages. out[2][17] per stage: t, sigma, sigma_next, cx, cs, cd, ch, ch2, cn, sx, ss, sd, sh, sh2,
// c_in, write_xs, write_hist + 2 * shift.
SDXL_TEST_API int sdxl_test_step_stages(const double* alphas, int n_train, const sdxl_schedule* s, int k, const double* timesteps,
                                        const double* sigmas, int n_hist, double* out) {
  const SigmaTable T(alphas, n_train);
  const StepStages ss = step_stages(&T, *s, k, timesteps, sigmas, n_hist);
  for (int i = 0; i < ss.n; ++i) {
    const Stage& q = ss.st[i];
    const double v[17] = {q.t, q.sigma, q.sigma_next, q.cx, q.cs, q.cd, q.ch, q.ch2, q.cn, q.sx, q.ss, q.sd, q.sh, q.sh2, q.c_in,
                          (double)q.write_xs, (double)q.write_hist + 2.0 * q.shift};
    for (int j = 0; j < 17; ++j) out[17 * i + j] = v[j];
  }
  return ss.n;
}
// The same with the prediction type (SDXL_PREDICTION_*: v takes schedule.h's d_scale at sigma, as the engine does) and the per-image
// guidance-rescale factors (factor nullable); with rows, the two-row form (kernels.h: StepRows).
static int guided_step_test(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag, float guidance,
                            float p_t, float sigma, float cx, float cd, float ch, float cn, float c_in, float* xh, float* x_in, float* hist,
                            int write_hist, const float* z, const float* zb, uint64_t seed, uint64_t z_subseq, uint64_t zb_subseq,
                            const uint8_t* mask, const float* ref, float sigma_blend, int prediction, const float* factor,
                            const StepRows* rows, int use_img = 0, float s_img = 0.f) {
  GuidedStepParams p{};
  p.eps = eps; p.ld = ld; p.Bimg = Bimg; p.C = C; p.HW = HW; p.use_cfg = use_cfg; p.use_pag = use_pag;
  p.guidance = guidance; p.p_t = p_t; p.sigma = sigma;
  p.cx = cx; p.cd = cd; p.ch = ch; p.cn = cn; p.c_in = c_in;
  p.xh = xh; p.x_in = x_in; p.hist = hist; p.write_hist = write_hist;
  p.z = z; p.zb = zb; p.seed = seed; p.z_subseq = z_subseq; p.zb_subseq = zb_subseq;
  p.mask = mask; p.ref = ref; p.sigma_blend = sigma_blend;
  Prediction pr;
  pr.factor = factor;
  if (prediction == SDXL_PREDICTION_V) {
    const DScale q = d_scale(prediction, sigma);
    pr.v = 1; pr.dx = q.dx; pr.de = q.de;
  }
  return guided_step_launch((cudaStream_t)stream, p, pr, rows, use_img, s_img);
}
SDXL_TEST_API int sdxl_test_guided_step_pred(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag,
                                             float guidance, float p_t, float sigma, float cx, float cd, float ch, float cn, float c_in,
                                             float* xh, float* x_in, float* hist, int write_hist, const float* z, const float* zb,
                                             uint64_t seed, uint64_t z_subseq, uint64_t zb_subseq, const uint8_t* mask, const float* ref,
                                             float sigma_blend, int prediction, const float* factor) {
  return guided_step_test(stream, eps, ld, Bimg, C, HW, use_cfg, use_pag, guidance, p_t, sigma, cx, cd, ch, cn, c_in, xh, x_in, hist,
                          write_hist, z, zb, seed, z_subseq, zb_subseq, mask, ref, sigma_blend, prediction, factor, nullptr);
}
// sdxl_test_guided_step_pred's arguments, then the saved state xs, the second history slot h2, rc = (cs, ch2),
// sr = (sx, ss, sd, sh, sh2) and the write_xs and shift flags.
SDXL_TEST_API int sdxl_test_guided_step_rows(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag,
                                             float guidance, float p_t, float sigma, float cx, float cd, float ch, float cn, float c_in,
                                             float* xh, float* x_in, float* hist, int write_hist, const float* z, const float* zb,
                                             uint64_t seed, uint64_t z_subseq, uint64_t zb_subseq, const uint8_t* mask, const float* ref,
                                             float sigma_blend, int prediction, const float* factor, float* xs, float* h2,
                                             const float* rc, const float* sr, int write_xs, int shift) {
  StepRows r;
  r.xs = xs; r.h2 = h2;
  r.cs = rc[0]; r.ch2 = rc[1];
  r.sx = sr[0]; r.ss = sr[1]; r.sd = sr[2]; r.sh = sr[3]; r.sh2 = sr[4];
  r.write_xs = write_xs; r.shift = shift;
  return guided_step_test(stream, eps, ld, Bimg, C, HW, use_cfg, use_pag, guidance, p_t, sigma, cx, cd, ch, cn, c_in, xh, x_in, hist,
                          write_hist, z, zb, seed, z_subseq, zb_subseq, mask, ref, sigma_blend, prediction, factor, &r);
}
// sdxl_test_guided_step_rows's arguments (use_cfg = 1, no PAG) with the image-guidance combine at s_img; use_rows = 0: the one-row
// form, xs, h2, rc, sr, write_xs and shift unread.
SDXL_TEST_API int sdxl_test_guided_step_img(void* stream, const float* eps, int ld, int Bimg, int C, int HW, float guidance, float s_img,
                                            float sigma, float cx, float cd, float ch, float cn, float c_in, float* xh, float* x_in,
                                            float* hist, int write_hist, const float* z, uint64_t seed, uint64_t z_subseq, int prediction,
                                            const float* factor, int use_rows, float* xs, float* h2, const float* rc, const float* sr,
                                            int write_xs, int shift) {
  StepRows r;
  if (use_rows) {
    r.xs = xs; r.h2 = h2;
    r.cs = rc[0]; r.ch2 = rc[1];
    r.sx = sr[0]; r.ss = sr[1]; r.sd = sr[2]; r.sh = sr[3]; r.sh2 = sr[4];
    r.write_xs = write_xs; r.shift = shift;
  }
  return guided_step_test(stream, eps, ld, Bimg, C, HW, 1, 0, guidance, 0.f, sigma, cx, cd, ch, cn, c_in, xh, x_in, hist, write_hist, z,
                          nullptr, seed, z_subseq, 0, nullptr, nullptr, 0.f, prediction, factor, use_rows ? &r : nullptr, 1, s_img);
}
SDXL_TEST_API int sdxl_test_guided_step(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag,
                                        float guidance, float p_t, float sigma, float cx, float cd, float ch, float cn, float c_in,
                                        float* xh, float* x_in, float* hist, int write_hist, const float* z, const float* zb,
                                        uint64_t seed, uint64_t z_subseq, uint64_t zb_subseq, const uint8_t* mask, const float* ref,
                                        float sigma_blend) {
  return sdxl_test_guided_step_pred(stream, eps, ld, Bimg, C, HW, use_cfg, use_pag, guidance, p_t, sigma, cx, cd, ch, cn, c_in, xh, x_in,
                                    hist, write_hist, z, zb, seed, z_subseq, zb_subseq, mask, ref, sigma_blend, SDXL_PREDICTION_EPSILON,
                                    nullptr);
}
SDXL_TEST_API int sdxl_test_timestep_embedding_f32(void* stream, const float* t, int nt, int dim, float max_period, float* out) {
  return timestep_embedding_f32_launch((cudaStream_t)stream, t, nt, dim, max_period, out);
}
