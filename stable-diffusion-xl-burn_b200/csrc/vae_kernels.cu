// Kernels that only the latent decoder needs (reference src/model/autoencoder/mod.rs, stablediffusion/mod.rs:199-266):
// the single-head d=512 attention's row softmax over a materialised score matrix, an f16 matrix transpose for the
// P·V GEMM's K-major V operand, the 1x1 post_quant_conv on the 4-channel latent, and the image converters.
// All are HBM-bound byte movers; the contractions of the decoder run on the wgmma implicit-GEMM kernel (igemm.cu).
#include "common.cuh"
#include "kernels.h"

namespace sdxl {

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------------
// P[r, :] = softmax(scale * S[r, :]) ; S f32 [rows, lds], P f16 [rows, ldp]. One CTA per row; the row is cached in
// shared memory when it fits so S is read from HBM once. Deterministic: fixed tree reductions, no atomics.
// ------------------------------------------------------------------------------------------------
constexpr int kSoftmaxThreads = 256;
constexpr int kSoftmaxRed = kSoftmaxThreads / 32;  // the kernel's static shared memory: one reduction slot per warp
__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();  // red reuse
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int i = 1; i < kSoftmaxThreads / 32; ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
  return r;
}
__global__ void __launch_bounds__(kSoftmaxThreads) softmax_rows_kernel(const float* __restrict__ S, size_t lds, int cols,
                                                                       float scale_log2e, __half* __restrict__ P,
                                                                       size_t ldp, int cache_row) {
  extern __shared__ float srow[];
  __shared__ float red[kSoftmaxRed];
  griddep_wait();
  griddep_launch_dependents();
  const float* g = S + (size_t)blockIdx.x * lds;
  __half* out = P + (size_t)blockIdx.x * ldp;
  const int nv = cols >> 2;  // cols % 4 == 0 (checked by the launcher)
  float m = -INFINITY;
  for (int i = threadIdx.x; i < nv; i += kSoftmaxThreads) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    if (cache_row) reinterpret_cast<float4*>(srow)[i] = v;
    m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  m = block_reduce(m, red, true);
  const float4* src = cache_row ? reinterpret_cast<const float4*>(srow) : reinterpret_cast<const float4*>(g);
  const float ms = m * scale_log2e;
  float sum = 0.f;
  for (int i = threadIdx.x; i < nv; i += kSoftmaxThreads) {
    float4 v = src[i];
    v.x = exp2f(fmaf(v.x, scale_log2e, -ms));
    v.y = exp2f(fmaf(v.y, scale_log2e, -ms));
    v.z = exp2f(fmaf(v.z, scale_log2e, -ms));
    v.w = exp2f(fmaf(v.w, scale_log2e, -ms));
    if (cache_row) reinterpret_cast<float4*>(srow)[i] = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  sum = block_reduce(sum, red, false);
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < nv; i += kSoftmaxThreads) {
    float4 v = src[i];
    if (!cache_row) {
      v.x = exp2f(fmaf(v.x, scale_log2e, -ms));
      v.y = exp2f(fmaf(v.y, scale_log2e, -ms));
      v.z = exp2f(fmaf(v.z, scale_log2e, -ms));
      v.w = exp2f(fmaf(v.w, scale_log2e, -ms));
    }
    const __half2 a = __floats2half2_rn(v.x * inv, v.y * inv), b = __floats2half2_rn(v.z * inv, v.w * inv);
    uint2 pk;
    pk.x = *reinterpret_cast<const uint32_t*>(&a);
    pk.y = *reinterpret_cast<const uint32_t*>(&b);
    reinterpret_cast<uint2*>(out)[i] = pk;
  }
}
int softmax_rows_launch(cudaStream_t st, const float* S, size_t lds, int rows, int cols, float scale, __half* P, size_t ldp) {
  if ((cols & 3) || (lds & 3) || (ldp & 3) || rows <= 0) return 6001;
  const size_t smem = (size_t)cols * sizeof(float);
  const int cache = smem <= 160 * 1024;
  // without the opt-in, static and dynamic shared memory together must fit in 48 KB: at cols = 12288 (a 96 x 128 latent) the
  // row alone is 48 KB and red[] does not fit beside it
  if (cache && smem + sizeof(float) * kSoftmaxRed > 48 * 1024) {
    static bool optin[64];
    if (int r = smem_optin(softmax_rows_kernel, 160 * 1024, optin)) return r;
  }
  const float sl2e = scale * 1.4426950408889634f;
  return launch_kernel(softmax_rows_kernel, dim3(rows), dim3(kSoftmaxThreads), cache ? smem : 0, st, true, S, lds, cols, sl2e,
                       P, ldp, cache);
}

// ------------------------------------------------------------------------------------------------
// y[c, r] = x[r, c] ; x f16 [rows, ldx] (first `cols` columns), y f16 [cols, ldy]. 64x64 tiles through shared memory.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) transpose_f16_kernel(const __half* __restrict__ x, size_t ldx, int rows, int cols,
                                                            __half* __restrict__ y, size_t ldy) {
  __shared__ __half tile[64][66];
  griddep_wait();
  griddep_launch_dependents();
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 64; i += 8) {
    const int r = r0 + i, c = c0 + 2 * tx;
    __half2 v = __floats2half2_rn(0.f, 0.f);
    if (r < rows && c + 1 < cols) v = *reinterpret_cast<const __half2*>(x + (size_t)r * ldx + c);
    else if (r < rows && c < cols) v = __halves2half2(x[(size_t)r * ldx + c], __float2half_rn(0.f));
    tile[i][2 * tx] = __low2half(v);
    tile[i][2 * tx + 1] = __high2half(v);
  }
  __syncthreads();
  for (int i = ty; i < 64; i += 8) {
    const int c = c0 + i, r = r0 + 2 * tx;
    if (c >= cols) continue;
    if (r + 1 < rows) *reinterpret_cast<__half2*>(y + (size_t)c * ldy + r) = __halves2half2(tile[2 * tx][i], tile[2 * tx + 1][i]);
    else if (r < rows) y[(size_t)c * ldy + r] = tile[2 * tx][i];
  }
}
int transpose_f16_launch(cudaStream_t st, const __half* x, size_t ldx, int rows, int cols, __half* y, size_t ldy) {
  if ((ldx & 1) || (ldy & 1) || rows <= 0 || cols <= 0) return 6002;
  return launch_kernel(transpose_f16_kernel, dim3(cdiv(cols, 64), cdiv(rows, 64)), dim3(256), 0, st, true, x, ldx, rows, cols,
                       y, ldy);
}

// ------------------------------------------------------------------------------------------------
// post_quant_conv on the rescaled latent (reference autoencoder/mod.rs:66-69, stablediffusion/mod.rs:263-266):
// y[b,o,p] = bias[o] + sum_i w[o,i] * (x[b,i,p] * inv_scale) ; NCHW f32 in and out, C <= 8. Exact f32 like the reference.
// ------------------------------------------------------------------------------------------------
__global__ void post_quant_kernel(const float* __restrict__ x, int B, int C, int HW, const float* __restrict__ w,
                                  const float* __restrict__ bias, float inv_scale, float* __restrict__ y) {
  const long total = (long)B * HW;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int p = (int)(i % HW);
    const int b = (int)(i / HW);
    float v[8];
    for (int c = 0; c < C; ++c) v[c] = x[((size_t)b * C + c) * HW + p] * inv_scale;
    for (int o = 0; o < C; ++o) {
      float acc = 0.f;
      for (int c = 0; c < C; ++c) acc = fmaf(w[o * C + c], v[c], acc);
      y[((size_t)b * C + o) * HW + p] = acc + bias[o];
    }
  }
}
int post_quant_launch(cudaStream_t st, const float* x, int B, int C, int HW, const float* w, const float* bias,
                      float inv_scale, float* y) {
  if (C > 8 || C < 1) return 6003;
  int grid = cdiv((long)B * HW, 256);
  if (grid > 132 * 8) grid = 132 * 8;
  post_quant_kernel<<<grid, 256, 0, st>>>(x, B, C, HW, w, bias, inv_scale, y);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// RawImages conversion (reference stablediffusion/mod.rs:211-229): u8[b, p, c] = trunc(clamp(((x + 1) / 2) * 255, 0, 255))
// from the decoder's NHWC f32 output [B, HW, ldx] (first 3 channels); NaN -> 0.
// ------------------------------------------------------------------------------------------------
__global__ void image_u8_kernel(const float* __restrict__ x, long npix, int ldx, uint8_t* __restrict__ out) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (long)gridDim.x * blockDim.x) {
    const float* px = x + (size_t)i * ldx;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = ((px[c] + 1.0f) / 2.0f) * 255.0f;
      // NaN -> 0 (the reference would panic on unwrap). fminf / fmaxf return the non-NaN operand, so the clamp alone would
      // turn NaN into 255: the comparison is false for NaN.
      v = v >= 0.0f ? fminf(v, 255.0f) : 0.0f;
      out[(size_t)i * 3 + c] = (uint8_t)v;
    }
  }
}
int image_u8_launch(cudaStream_t st, const float* x, long npix, int ldx, uint8_t* out) {
  int grid = cdiv(npix, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  image_u8_kernel<<<grid, 256, 0, st>>>(x, npix, ldx, out);
  return (int)cudaGetLastError();
}


// ------------------------------------------------------------------------------------------------
// image_to_latent front end (reference stablediffusion/mod.rs:239-256): u8 [B, HW, 3] -> f32 NCHW [B, 3, HW],
// ((v / 255) * 2) - 1 in f32, in that order.
// ------------------------------------------------------------------------------------------------
__global__ void image_from_u8_kernel(const uint8_t* __restrict__ in, int B, long HW, float* __restrict__ out) {
  const long total = (long)B * HW;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long b = i / HW, p = i % HW;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[((size_t)b * 3 + c) * HW + p] = ((float)in[(size_t)i * 3 + c] / 255.0f) * 2.0f - 1.0f;
  }
}
int image_from_u8_launch(cudaStream_t st, const uint8_t* in, int B, long HW, float* out) {
  int grid = cdiv((long)B * HW, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  image_from_u8_kernel<<<grid, 256, 0, st>>>(in, B, HW, out);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// quant_conv + slice + scale (reference autoencoder/mod.rs:58-64, stablediffusion/mod.rs:258-261):
// y[b, o, p] = (bias[o] + sum_i w[o, i] * x[b, p, i]) * scale for o < Cout (the first Cout of the Cz moments channels);
// x NHWC f32 [B, HW, Cz], y NCHW f32 [B, Cout, HW]. Exact f32.
// ------------------------------------------------------------------------------------------------
__global__ void quant_out_kernel(const float* __restrict__ x, int B, int Cz, int Cout, long HW, const float* __restrict__ w,
                                 const float* __restrict__ bias, float scale, float* __restrict__ y) {
  const long total = (long)B * HW;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long b = i / HW, p = i % HW;
    float v[16];
    for (int c = 0; c < Cz; ++c) v[c] = x[(size_t)i * Cz + c];
    for (int o = 0; o < Cout; ++o) {
      float acc = 0.f;
      for (int c = 0; c < Cz; ++c) acc = fmaf(w[o * Cz + c], v[c], acc);
      y[((size_t)b * Cout + o) * HW + p] = (acc + bias[o]) * scale;
    }
  }
}
int quant_out_launch(cudaStream_t st, const float* x, int B, int Cz, int Cout, long HW, const float* w, const float* bias,
                     float scale, float* y) {
  if (Cz > 16 || Cout > Cz || Cout < 1) return 6004;
  int grid = cdiv((long)B * HW, 256);
  if (grid > 132 * 8) grid = 132 * 8;
  quant_out_kernel<<<grid, 256, 0, st>>>(x, B, Cz, Cout, HW, w, bias, scale, y);
  return (int)cudaGetLastError();
}

}  // namespace sdxl
