// Test-only C entry points to the internal launchers of kernels.h (linked into libsdxl_b200_testing.so, never into the
// product library). Each wrapper takes plain arguments, fills the launcher's parameter struct exactly as the UNet's launch
// plan does (engine_core.h: PlanBuilder) and launches on `stream`, so tests can pin the fused layouts the plan uses —
// second K sources, per-batch bias rows, scattered upsample outputs, column windows of fused QKV / KV matrices — kernel by
// kernel against a float64 reference. All pointers are device pointers; every function returns the launcher's status.
#include "kernels.h"

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
// The sampler's guided DDIM update with PAG (engine.cu: sampler_step).
SDXL_TEST_API int sdxl_test_cfg_pag_ddim(void* stream, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, float guidance,
                                         float p_t, float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map, float* x) {
  return cfg_pag_ddim_launch((cudaStream_t)stream, eps, ld, Bimg, C, HW, use_cfg, guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, x);
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
SDXL_TEST_API int sdxl_test_lora_upconv_merge(void* stream, const void* src, const float* delta, int O, int I, void* dst, int Ipad) {
  return lora_upconv_merge_launch((cudaStream_t)stream, (const __half*)src, delta, O, I, (__half*)dst, Ipad);
}
