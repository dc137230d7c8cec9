// Kernels that only the CLIP towers need: the text encoders (Embedder: CLIP-L / OpenCLIP-bigG, reference src/model/clip/mod.rs)
// and the vision encoders of IP-Adapter (HF CLIPVisionModelWithProjection). The
// sequences are 77 tokens, so these are small CUDA-core kernels; the Linear layers run on the wgmma GEMM (igemm.cu).
#include "common.cuh"
#include "kernels.h"

namespace sdxl {

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------------
// x[b*T + t, :] = token_embedding[tokens[b, t], :] + position_embedding[t, :]     (clip/mod.rs:89-97)
// tables f16, output f32 residual stream. An id outside the table is reported through *err (the reference panics).
// ------------------------------------------------------------------------------------------------
__global__ void embed_tokens_kernel(const int* __restrict__ tokens, int rows, int T, int C, int n_vocab,
                                    const __half* __restrict__ tok_emb, const __half* __restrict__ pos_emb,
                                    float* __restrict__ x, int* __restrict__ err) {
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.x;
  if (row >= rows) return;
  int id = tokens[row];
  if (id < 0 || id >= n_vocab) {
    if (threadIdx.x == 0) atomicExch(err, 1);
    id = 0;
  }
  const __half2* te = reinterpret_cast<const __half2*>(tok_emb + (size_t)id * C);
  const __half2* pe = reinterpret_cast<const __half2*>(pos_emb + (size_t)(row % T) * C);
  float2* o = reinterpret_cast<float2*>(x + (size_t)row * C);
  for (int i = threadIdx.x; i < (C >> 1); i += blockDim.x) {
    const float2 a = __half22float2(te[i]), b = __half22float2(pe[i]);
    o[i] = make_float2(a.x + b.x, a.y + b.y);
  }
}
int embed_tokens_launch(cudaStream_t st, const int* tokens, int rows, int T, int C, int n_vocab, const __half* tok_emb,
                        const __half* pos_emb, float* x, int* err) {
  if (C & 1) return 7101;
  return launch_kernel(embed_tokens_kernel, dim3(rows), dim3(128), (size_t)0, st, true, tokens, rows, T, C, n_vocab, tok_emb,
                       pos_emb, x, err);
}

// ------------------------------------------------------------------------------------------------
// Masked multi-head attention for short sequences, head dim 64 (Backend::qkv_attention with a mask,
// reference src/backend.rs:32-79 / 88-128): out = softmax(q k^T / 8 + mask) v. One warp per (batch, head, query).
// q/k/v are column windows of row-major f16 matrices; mask is an additive f16 [T, S] matrix (nullable) and/or the
// causal rule key <= query (attn_decoder_mask: -inf strictly above the diagonal). Online softmax over 32-key chunks,
// f32 math. A query whose keys are all masked produces zeros (the reference's softmax would give NaN).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) attention_small_kernel(const __half* __restrict__ q, int q_pitch, int q_col0,
                                                              const __half* __restrict__ k, const __half* __restrict__ v,
                                                              int kv_pitch, int k_col0, int v_col0, int B, int T, int S, int n_head,
                                                              const __half* __restrict__ mask, int causal, float scale,
                                                              __half* __restrict__ out, int ldo) {
  __shared__ float qs[4][64];
  griddep_wait();
  griddep_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long item = (long)blockIdx.x * 4 + warp;
  const long total = (long)B * n_head * T;
  const bool active = item < total;
  int t = 0, h = 0, b = 0;
  if (active) {
    t = (int)(item % T);
    h = (int)((item / T) % n_head);
    b = (int)(item / ((long)T * n_head));
    const __half2 qq = *reinterpret_cast<const __half2*>(q + ((size_t)b * T + t) * q_pitch + q_col0 + h * 64 + 2 * lane);
    qs[warp][2 * lane] = __low2float(qq) * scale;
    qs[warp][2 * lane + 1] = __high2float(qq) * scale;
  }
  __syncwarp();
  if (!active) return;
  float m = -INFINITY, l = 0.f, ax = 0.f, ay = 0.f;
  const __half* kb = k + (size_t)b * S * kv_pitch + k_col0 + h * 64;
  const __half* vb = v + (size_t)b * S * kv_pitch + v_col0 + h * 64;
  const int s_end = causal ? min(S, t + 1) : S;
  for (int j0 = 0; j0 < s_end; j0 += 32) {
    const int j = j0 + lane;
    float s = -INFINITY;
    if (j < s_end) {
      const uint4* kr = reinterpret_cast<const uint4*>(kb + (size_t)j * kv_pitch);
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 u = kr[c];
        const __half2* hp = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(hp[e]);
          acc = fmaf(qs[warp][c * 8 + 2 * e], f.x, acc);
          acc = fmaf(qs[warp][c * 8 + 2 * e + 1], f.y, acc);
        }
      }
      s = acc;
      if (mask) s += __half2float(mask[(size_t)t * S + j]);
    }
    float cm = s;
#pragma unroll
    for (int o = 16; o; o >>= 1) cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, o));
    const float m_new = fmaxf(m, cm);
    if (m_new == -INFINITY) continue;  // everything so far is masked
    const float corr = (m == -INFINITY) ? 0.f : __expf(m - m_new);
    const float p = (s == -INFINITY) ? 0.f : __expf(s - m_new);
    float ps = p;
#pragma unroll
    for (int o = 16; o; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
    l = l * corr + ps;
    ax *= corr;
    ay *= corr;
    const int nj = min(32, s_end - j0);
    for (int jj = 0; jj < nj; ++jj) {
      const float pj = __shfl_sync(0xffffffffu, p, jj);
      const float2 vv = __half22float2(*reinterpret_cast<const __half2*>(vb + (size_t)(j0 + jj) * kv_pitch + 2 * lane));
      ax = fmaf(pj, vv.x, ax);
      ay = fmaf(pj, vv.y, ay);
    }
    m = m_new;
  }
  const float inv = l > 0.f ? 1.f / l : 0.f;
  *reinterpret_cast<__half2*>(out + ((size_t)b * T + t) * ldo + h * 64 + 2 * lane) = __floats2half2_rn(ax * inv, ay * inv);
}
// The same attention for head dims D other than 64 (multiples of 8 up to 128: the CLIP vision towers use 80 and 104), scale
// 1/sqrt(D). Kept beside the d = 64 kernel so that the text encoders' kernel is unchanged. Lane l accumulates the output columns
// 2 (l + 32 i), i < NP.
template <int D>
__global__ void attention_small_hd_kernel(const __half* __restrict__ q, int q_pitch, int q_col0,
                                                                 const __half* __restrict__ k, const __half* __restrict__ v,
                                                                 int kv_pitch, int k_col0, int v_col0, int B, int T, int S, int n_head,
                                                                 const __half* __restrict__ mask, int causal, float scale,
                                                                 __half* __restrict__ out, int ldo) {
  constexpr int NP = (D / 2 + 31) / 32;
  __shared__ float qs[4][D];
  griddep_wait();
  griddep_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long item = (long)blockIdx.x * 4 + warp;
  const long total = (long)B * n_head * T;
  const bool active = item < total;
  int t = 0, h = 0, b = 0;
  if (active) {
    t = (int)(item % T);
    h = (int)((item / T) % n_head);
    b = (int)(item / ((long)T * n_head));
    for (int c = lane; c < D / 2; c += 32) {
      const __half2 qq = *reinterpret_cast<const __half2*>(q + ((size_t)b * T + t) * q_pitch + q_col0 + h * D + 2 * c);
      qs[warp][2 * c] = __low2float(qq) * scale;
      qs[warp][2 * c + 1] = __high2float(qq) * scale;
    }
  }
  __syncwarp();
  if (!active) return;
  float m = -INFINITY, l = 0.f, ax[NP], ay[NP];
#pragma unroll
  for (int i = 0; i < NP; ++i) ax[i] = ay[i] = 0.f;
  const __half* kb = k + (size_t)b * S * kv_pitch + k_col0 + h * D;
  const __half* vb = v + (size_t)b * S * kv_pitch + v_col0 + h * D;
  const int s_end = causal ? min(S, t + 1) : S;
  for (int j0 = 0; j0 < s_end; j0 += 32) {
    const int j = j0 + lane;
    float s = -INFINITY;
    if (j < s_end) {
      const uint4* kr = reinterpret_cast<const uint4*>(kb + (size_t)j * kv_pitch);
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < D / 8; ++c) {
        const uint4 u = kr[c];
        const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          __half2_raw r;
          r.x = (unsigned short)(w4[e] & 0xffffu);
          r.y = (unsigned short)(w4[e] >> 16);
          const float2 f = __half22float2(__half2(r));
          acc = fmaf(qs[warp][c * 8 + 2 * e], f.x, acc);
          acc = fmaf(qs[warp][c * 8 + 2 * e + 1], f.y, acc);
        }
      }
      s = acc;
      if (mask) s += __half2float(mask[(size_t)t * S + j]);
    }
    float cm = s;
#pragma unroll
    for (int o = 16; o; o >>= 1) cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, o));
    const float m_new = fmaxf(m, cm);
    if (m_new == -INFINITY) continue;  // everything so far is masked
    const float corr = (m == -INFINITY) ? 0.f : __expf(m - m_new);
    const float p = (s == -INFINITY) ? 0.f : __expf(s - m_new);
    float ps = p;
#pragma unroll
    for (int o = 16; o; o >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
    l = l * corr + ps;
#pragma unroll
    for (int i = 0; i < NP; ++i) { ax[i] *= corr; ay[i] *= corr; }
    const int nj = min(32, s_end - j0);
    for (int jj = 0; jj < nj; ++jj) {
      const float pj = __shfl_sync(0xffffffffu, p, jj);
      const __half* vr = vb + (size_t)(j0 + jj) * kv_pitch;
#pragma unroll
      for (int i = 0; i < NP; ++i) {   // lanes past D / 2 re-read the last column and are not stored
        const int c = min(lane + 32 * i, D / 2 - 1);
        const float2 vv = __half22float2(*reinterpret_cast<const __half2*>(vr + 2 * c));
        ax[i] = fmaf(pj, vv.x, ax[i]);
        ay[i] = fmaf(pj, vv.y, ay[i]);
      }
    }
    m = m_new;
  }
  const float inv = l > 0.f ? 1.f / l : 0.f;
#pragma unroll
  for (int i = 0; i < NP; ++i) {
    const int c = lane + 32 * i;
    if (c < D / 2)
      *reinterpret_cast<__half2*>(out + ((size_t)b * T + t) * ldo + h * D + 2 * c) = __floats2half2_rn(ax[i] * inv, ay[i] * inv);
  }
}

int attention_small_launch(cudaStream_t st, const __half* q, int q_pitch, int q_col0, const __half* k, const __half* v,
                           int kv_pitch, int k_col0, int v_col0, int B, int T, int S, int n_head, const __half* mask, int causal,
                           __half* out, int ldo, int head_dim) {
  if ((q_pitch & 7) || (kv_pitch & 7) || (q_col0 & 7) || (k_col0 & 7) || (v_col0 & 7) || (ldo & 1)) return 7102;
  const long total = (long)B * n_head * T;
  const dim3 grid(cdiv(total, 4)), block(128);
  const float scale = 1.f / sqrtf((float)head_dim);
  switch (head_dim) {
#define SDXL_ATTN_SMALL_HD(D) \
    case D: return launch_kernel(attention_small_hd_kernel<D>, grid, block, (size_t)0, st, true, q, q_pitch, q_col0, k, v, kv_pitch, \
                                 k_col0, v_col0, B, T, S, n_head, mask, causal, scale, out, ldo);
    SDXL_ATTN_SMALL_HD(8) SDXL_ATTN_SMALL_HD(16) SDXL_ATTN_SMALL_HD(24) SDXL_ATTN_SMALL_HD(32) SDXL_ATTN_SMALL_HD(40)
    SDXL_ATTN_SMALL_HD(48) SDXL_ATTN_SMALL_HD(56) SDXL_ATTN_SMALL_HD(72) SDXL_ATTN_SMALL_HD(80) SDXL_ATTN_SMALL_HD(88)
    SDXL_ATTN_SMALL_HD(96) SDXL_ATTN_SMALL_HD(104) SDXL_ATTN_SMALL_HD(112) SDXL_ATTN_SMALL_HD(120) SDXL_ATTN_SMALL_HD(128)
#undef SDXL_ATTN_SMALL_HD
    case 64:
      return launch_kernel(attention_small_kernel, grid, block, (size_t)0, st, true, q, q_pitch, q_col0, k, v, kv_pitch,
                           k_col0, v_col0, B, T, S, n_head, mask, causal, scale, out, ldo);
    default: return 7104;
  }
}

// ------------------------------------------------------------------------------------------------
// CLIP vision embedding (HF CLIPVisionEmbeddings).
// patchify: pixels f32 NCHW [N, 3, S, S] -> f16 [N * G * G, Kpad], row n * G * G + py * G + px, column (c, kh, kw) = the OIHW
// flatten of the p x p stride-p patch conv, zero padded to Kpad (the patch conv is then one GEMM on igemm).
// ------------------------------------------------------------------------------------------------
__global__ void patchify_kernel(const float* __restrict__ px, int S, int p, int G, int Kpad, __half* __restrict__ y) {
  griddep_wait();
  griddep_launch_dependents();
  const long row = blockIdx.x;
  const int n = (int)(row / (G * G)), pi = (int)(row % (G * G)), py = pi / G, pxi = pi % G;
  const int K = 3 * p * p;
  for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
    float v = 0.f;
    if (k < K) {
      const int c = k / (p * p), kh = (k / p) % p, kw = k % p;
      v = px[(((size_t)n * 3 + c) * S + py * p + kh) * S + pxi * p + kw];
    }
    y[row * Kpad + k] = __float2half_rn(v);
  }
}
int patchify_launch(cudaStream_t st, const float* pixels, int N, int S, int p, int Kpad, __half* y) {
  if (p < 1 || S % p || Kpad < 3 * p * p) return 7105;
  const int G = S / p;
  return launch_kernel(patchify_kernel, dim3((unsigned)(N * G * G)), dim3(128), (size_t)0, st, true, pixels, S, p, G, Kpad, y);
}

// x[n*T + t, :] = pre_layrnorm((t == 0 ? class_embedding : patches[n*(T-1) + t-1, :]) + position_embedding[t, :]), the f32 residual
// stream. One block per row; exact two-pass statistics like the other LayerNorms.
__global__ void vision_embed_ln_kernel(const float* __restrict__ patches, const __half* __restrict__ cls, const __half* __restrict__ pos,
                                       int T, int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                       float* __restrict__ x) {
  __shared__ float red[32];
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.x, t = row % T, n = row / T;
  float* xr = x + (size_t)row * C;
  const float* pr = t ? patches + ((size_t)n * (T - 1) + t - 1) * C : nullptr;
  auto block_sum = [&](float s) {
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    __syncthreads();
    return tot;
  };
  float s = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float v = (t ? pr[i] : __half2float(cls[i])) + __half2float(pos[(size_t)t * C + i]);
    xr[i] = v;
    s += v;
  }
  const float mean = block_sum(s) / C;
  float q = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) { const float d = xr[i] - mean; q = fmaf(d, d, q); }
  const float rstd = 1.f / sqrtf(block_sum(q) / C + eps);
  for (int i = threadIdx.x; i < C; i += blockDim.x) xr[i] = (xr[i] - mean) * rstd * gamma[i] + beta[i];
}
int vision_embed_ln_launch(cudaStream_t st, const float* patches, const __half* cls, const __half* pos, int N, int T, int C,
                           const float* gamma, const float* beta, float eps, float* x) {
  return launch_kernel(vision_embed_ln_kernel, dim3((unsigned)(N * T)), dim3(256), (size_t)0, st, true, patches, cls, pos, T, C, gamma,
                       beta, eps, x);
}

// ------------------------------------------------------------------------------------------------
// MLP activation between fc1 and fc2 (clip/mod.rs:296-304): mode 0 = nn::Gelu (exact erf), 1 = QuickGELU
// x * sigmoid(1.702 x) (clip/mod.rs:316-318). f32 in (fc1 accumulators), f16 out (fc2 operand).
// ------------------------------------------------------------------------------------------------
__global__ void mlp_act_kernel(const float* __restrict__ x, size_t n4, int quick, __half* __restrict__ y) {
  griddep_wait();
  griddep_launch_dependents();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(x)[i];
    if (quick) {
      v.x = v.x / (1.f + __expf(-1.702f * v.x));
      v.y = v.y / (1.f + __expf(-1.702f * v.y));
      v.z = v.z / (1.f + __expf(-1.702f * v.z));
      v.w = v.w / (1.f + __expf(-1.702f * v.w));
    } else {
      v.x = gelu_erf_f(v.x); v.y = gelu_erf_f(v.y); v.z = gelu_erf_f(v.z); v.w = gelu_erf_f(v.w);
    }
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    uint2 pk;
    pk.x = *reinterpret_cast<const uint32_t*>(&a);
    pk.y = *reinterpret_cast<const uint32_t*>(&b);
    reinterpret_cast<uint2*>(y)[i] = pk;
  }
}
int mlp_act_launch(cudaStream_t st, const float* x, size_t n, int quick, __half* y) {
  if (n & 3) return 7103;
  int grid = cdiv((long)(n >> 2), 256);
  if (grid > 132 * 8) grid = 132 * 8;
  return launch_kernel(mlp_act_kernel, dim3(grid), dim3(256), (size_t)0, st, true, x, n >> 2, quick, y);
}

// ------------------------------------------------------------------------------------------------
// y[b, :] = LayerNorm(x[b*T + idx[b], :]) in f32 (the pooled end-of-text feature, clip/mod.rs:131-134). One warp per row,
// exact two-pass statistics like layernorm/mod.rs:42-49.
// ------------------------------------------------------------------------------------------------
__global__ void ln_gather_f32_kernel(const float* __restrict__ x, const int* __restrict__ idx, int T, int C,
                                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                     float* __restrict__ y) {
  griddep_wait();
  griddep_launch_dependents();
  const int b = blockIdx.x, lane = threadIdx.x;
  const float* r = x + ((size_t)b * T + idx[b]) * C;
  float s = 0.f;
  for (int i = lane; i < C; i += 32) s += r[i];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
  for (int i = lane; i < C; i += 32) { const float d = r[i] - mean; q = fmaf(d, d, q); }
#pragma unroll
  for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = 1.f / sqrtf(q / C + eps);
  for (int i = lane; i < C; i += 32) y[(size_t)b * C + i] = (r[i] - mean) * rstd * gamma[i] + beta[i];
}
int ln_gather_f32_launch(cudaStream_t st, const float* x, const int* idx, int B, int T, int C, const float* gamma,
                         const float* beta, float eps, float* y) {
  return launch_kernel(ln_gather_f32_kernel, dim3(B), dim3(32), (size_t)0, st, true, x, idx, T, C, gamma, beta, eps, y);
}

// ------------------------------------------------------------------------------------------------
// The two LayerNorms of one IP-Adapter Plus perceiver-attention layer (h94 resampler.py PerceiverAttention), in one launch.
// Row r of the per-image concatenation [n, L + Q, C]: j = r % (L + Q) < L is LN1 of x[img * L + j], otherwise LN2 of
// lat[img * Q + j - L]. Every row goes to kv (the operand of to_kv and the attention's keys / values); the LN2 rows also go to
// q[img * Q + j - L] (the operand of to_q). One block per row, exact two-pass statistics like the other LayerNorms.
// ------------------------------------------------------------------------------------------------
__global__ void perceiver_ln_kernel(const float* __restrict__ x, const float* __restrict__ lat, int L, int Q, int C,
                                    const float* __restrict__ g1, const float* __restrict__ b1, const float* __restrict__ g2,
                                    const float* __restrict__ b2, float eps, __half* __restrict__ kv, __half* __restrict__ q) {
  __shared__ float red[32];
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.x, S = L + Q, img = row / S, j = row % S;
  const bool is_lat = j >= L;
  const float* src = is_lat ? lat + ((size_t)img * Q + (j - L)) * C : x + ((size_t)img * L + j) * C;
  const float* gamma = is_lat ? g2 : g1;
  const float* beta = is_lat ? b2 : b1;
  __half* qr = is_lat ? q + ((size_t)img * Q + (j - L)) * C : nullptr;
  __half* kr = kv + (size_t)row * C;
  auto block_sum = [&](float s) {
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    float tot = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
    __syncthreads();
    return tot;
  };
  float s = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) s += src[i];
  const float mean = block_sum(s) / C;
  float sq = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) { const float d = src[i] - mean; sq = fmaf(d, d, sq); }
  const float rstd = 1.f / sqrtf(block_sum(sq) / C + eps);
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const __half h = __float2half_rn((src[i] - mean) * rstd * gamma[i] + beta[i]);
    kr[i] = h;
    if (qr) qr[i] = h;
  }
}
int perceiver_ln_launch(cudaStream_t st, const float* x, const float* lat, int n, int L, int Q, int C, const float* g1,
                        const float* b1, const float* g2, const float* b2, float eps, __half* kv, __half* q) {
  if (n < 1 || L < 1 || Q < 1 || C < 1) return 7106;
  return launch_kernel(perceiver_ln_kernel, dim3((unsigned)(n * (L + Q))), dim3(256), (size_t)0, st, true, x, lat, L, Q, C, g1, b1, g2,
                       b2, eps, kv, q);
}

}  // namespace sdxl
