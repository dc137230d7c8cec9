// Small HBM-bound kernels of the UNet step: embedding GEMVs, first conv, resampling copies, sampler
// elementwise math (CFG + DDIM, inpainting blend), Philox noise, and load-time weight re-layout.
// All are plain coalesced / 128-bit vectorised CUDA; none of them is GEMM-shaped.
#include "common.cuh"
#include "kernels.h"

#include <stdlib.h>

namespace sdxl {

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

bool pdl_enabled() {
  static const bool on = getenv("SDXL_B200_NO_PDL") == nullptr;
  return on;
}

// ------------------------------------------------------------------------------------------------
// GEMV: one warp per output column, up to 8 batch rows accumulated together.
// ------------------------------------------------------------------------------------------------
template <int MAXB>
__global__ void gemv_kernel(const float* __restrict__ in, int in_bstride, int Bv, int K,
                            const __half* __restrict__ W, int ldw, const float* __restrict__ bias,
                            const float* __restrict__ add, int add_bstride, int N, int in_silu, int out_silu,
                            float* __restrict__ out, int out_bstride) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float acc[MAXB];
#pragma unroll
  for (int b = 0; b < MAXB; ++b) acc[b] = 0.f;
  const __half* w = W + (size_t)n * ldw;
  if ((K & 7) == 0 && (ldw & 7) == 0 && (in_bstride & 3) == 0 && (reinterpret_cast<uintptr_t>(in) & 15) == 0) {
    // four 16-byte weight loads in flight per lane before the first FMA (a K = 1280 row is 5 loads per lane: one DRAM round
    // trip each if issued one per iteration), activations as float4 (L1 hits)
    for (int k0 = lane * 8; k0 < K; k0 += 1024) {
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        raw[u] = (k0 + u * 256 < K) ? __ldg(reinterpret_cast<const uint4*>(w + k0 + u * 256)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int kk = k0 + u * 256;
        if (kk < K) {
          const __half2* h2 = reinterpret_cast<const __half2*>(&raw[u]);
          float wf[8];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(h2[i]);
            wf[2 * i] = f.x;
            wf[2 * i + 1] = f.y;
          }
#pragma unroll
          for (int b = 0; b < MAXB; ++b) {
            if (b < Bv) {
              const float4* x4 = reinterpret_cast<const float4*>(in + (size_t)b * in_bstride + kk);
              const float4 xa = __ldg(x4), xb = __ldg(x4 + 1);
              float xv[8] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                float v = xv[i];
                if (in_silu) v = silu_f(v);
                acc[b] = fmaf(v, wf[i], acc[b]);
              }
            }
          }
        }
      }
    }
  } else {
    for (int k = lane; k < K; k += 32) {
      const float wv = __half2float(w[k]);
#pragma unroll
      for (int b = 0; b < MAXB; ++b) {
        if (b < Bv) {
          float v = in[(size_t)b * in_bstride + k];
          if (in_silu) v = silu_f(v);
          acc[b] = fmaf(v, wv, acc[b]);
        }
      }
    }
  }
#pragma unroll
  for (int b = 0; b < MAXB; ++b) {
    if (b < Bv) {
      float s = warp_sum(acc[b]);
      if (lane == 0) {
        if (bias) s += bias[n];
        if (add) s += add[(size_t)b * add_bstride + n];
        if (out_silu) s = silu_f(s);
        out[(size_t)b * out_bstride + n] = s;
      }
    }
  }
}
int gemv_launch(cudaStream_t st, const float* in, int in_bstride, int Bv, int K, const __half* W, int ldw, const float* bias,
                const float* add, int add_bstride, int N, int in_silu, int out_silu, float* out, int out_bstride) {
  if (Bv > 8) return 2001;
  const int warps = 8;
  if (Bv <= 2)
    gemv_kernel<2><<<cdiv(N, warps), warps * 32, 0, st>>>(in, in_bstride, Bv, K, W, ldw, bias, add, add_bstride, N, in_silu,
                                                           out_silu, out, out_bstride);
  else
    gemv_kernel<8><<<cdiv(N, warps), warps * 32, 0, st>>>(in, in_bstride, Bv, K, W, ldw, bias, add, add_bstride, N, in_silu,
                                                           out_silu, out, out_bstride);
  return (int)cudaGetLastError();
}

// timestep_embedding (reference unet/mod.rs:21-39): cos half first, then sin half.
__global__ void timestep_embedding_kernel(const int* __restrict__ t, int nt, int dim, float max_period,
                                          float* __restrict__ out) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nt * half) return;
  const int b = i / half, j = i % half;
  const float freq = expf((float)j * (-logf(max_period) / (float)half));
  const float arg = (float)t[b] * freq;
  out[(size_t)b * dim + j] = cosf(arg);
  out[(size_t)b * dim + half + j] = sinf(arg);
}
int timestep_embedding_launch(cudaStream_t st, const int* t_dev, int nt, int dim, float max_period, float* out) {
  const int n = nt * (dim / 2);
  timestep_embedding_kernel<<<cdiv(n, 128), 128, 0, st>>>(t_dev, nt, dim, max_period, out);
  return (int)cudaGetLastError();
}
// The same of a float timestep (the UNet plan's: schedules place timesteps between the training ones). For an integer-valued
// t the arithmetic is the int kernel's after its (float) conversion, so the embedding is bit-identical.
__global__ void timestep_embedding_f32_kernel(const float* __restrict__ t, int nt, int dim, float max_period,
                                              float* __restrict__ out) {
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nt * half) return;
  const int b = i / half, j = i % half;
  const float freq = expf((float)j * (-logf(max_period) / (float)half));
  const float arg = t[b] * freq;
  out[(size_t)b * dim + j] = cosf(arg);
  out[(size_t)b * dim + half + j] = sinf(arg);
}
int timestep_embedding_f32_launch(cudaStream_t st, const float* t_dev, int nt, int dim, float max_period, float* out) {
  const int n = nt * (dim / 2);
  timestep_embedding_f32_kernel<<<cdiv(n, 128), 128, 0, st>>>(t_dev, nt, dim, max_period, out);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// First conv (4 -> model_channels, 3x3 pad 1; reference unet/mod.rs:116-120). K = 36: CUDA cores.
// x: NCHW (f16 or f32) [Bx, Cin, H, W]; output batch b reads image (b % Bx). y: NHWC f32.
// ------------------------------------------------------------------------------------------------
// One thread = 4 output channels x 8 consecutive pixels of a row: every weight float4 read from shared memory feeds 32 FMAs
// (at one pixel per thread the kernel was bound by the LDS.128 per 4 FMAs: 158 us for the UNet's 2x128x128x320 output).
// kCat (the inpainting UNet): input channels [C1, Cin) come from a second source x2, f32 NCHW [n2, Cin - C1, H, W], output batch
// b reading image b % n2. Which source a (kh, c) pair reads is the same in every lane. kCat = false compiles to the one-source
// kernel: x2 / n2 / C1 are unused and the dead branch is removed.
constexpr int kConvInPix = 8;
template <typename TIn, bool kCat = false>
__global__ void __launch_bounds__(256) conv_in_kernel(const TIn* __restrict__ x, int Bx, int B, int Cin, int H, int W,
                                                      const float* __restrict__ w, const float* __restrict__ bias, int Cout,
                                                      float* __restrict__ y, const float* __restrict__ add, int n_add,
                                                      const float* __restrict__ x2, int n2, int C1) {
  extern __shared__ float sw[];  // [9*Cin][Cout]  (k-major: lanes = consecutive output channels, conflict-free)
  const int kk = 9 * Cin;
  for (int co = threadIdx.x; co < Cout; co += blockDim.x)          // lanes = consecutive rows of w: conflict-free smem writes,
    for (int k = 0; k < kk; ++k) sw[k * Cout + co] = w[co * kk + k];   // the rows' lines stay in L1 across the k loop
  __syncthreads();
  const int cvec = Cout / 4;
  const int nseg = (W + kConvInPix - 1) / kConvInPix;
  const long total = (long)B * H * nseg * cvec;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int cv = (int)(idx % cvec);
    const long seg = idx / cvec;
    const int w0 = (int)(seg % nseg) * kConvInPix;
    const int hh = (int)((seg / nseg) % H);
    const int b = (int)(seg / ((long)nseg * H));
    const TIn* xb = x + (size_t)(b % Bx) * (kCat ? C1 : Cin) * H * W;
    const float* x2b = kCat ? x2 + (size_t)(b % n2) * (Cin - C1) * H * W : nullptr;
    const float4 b4 = bias ? *reinterpret_cast<const float4*>(bias + cv * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 acc[kConvInPix];
#pragma unroll
    for (int i = 0; i < kConvInPix; ++i) acc[i] = b4;
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = hh + kh - 1;
      if (ih < 0 || ih >= H) continue;
      for (int c = 0; c < Cin; ++c) {
        float xv[kConvInPix + 2];                                  // the row segment with its halo; same address in all lanes
        if (kCat && c >= C1) {
          const float* xr = x2b + ((size_t)(c - C1) * H + ih) * W;
#pragma unroll
          for (int i = 0; i < kConvInPix + 2; ++i) {
            const int iw = w0 + i - 1;
            xv[i] = (iw >= 0 && iw < W) ? xr[iw] : 0.f;
          }
        } else {
          const TIn* xr = xb + ((size_t)c * H + ih) * W;
#pragma unroll
          for (int i = 0; i < kConvInPix + 2; ++i) {
            const int iw = w0 + i - 1;
            xv[i] = (iw >= 0 && iw < W) ? (float)xr[iw] : 0.f;
          }
        }
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const float4 wv = *reinterpret_cast<const float4*>(sw + ((kh * 3 + kw) * Cin + c) * Cout + cv * 4);
#pragma unroll
          for (int i = 0; i < kConvInPix; ++i) {
            const float v = xv[i + kw];
            acc[i].x = fmaf(v, wv.x, acc[i].x); acc[i].y = fmaf(v, wv.y, acc[i].y);
            acc[i].z = fmaf(v, wv.z, acc[i].z); acc[i].w = fmaf(v, wv.w, acc[i].w);
          }
        }
      }
    }
    float* yo = y + (((size_t)b * H + hh) * W + w0) * Cout + cv * 4;
    if (add) {   // ControlNet: h0 = conv_in(x) + hint_emb[b % n_add]
      const float* ao = add + (((size_t)(b % n_add) * H + hh) * W + w0) * Cout + cv * 4;
#pragma unroll
      for (int i = 0; i < kConvInPix; ++i)
        if (w0 + i < W) {
          const float4 a = *reinterpret_cast<const float4*>(ao + (size_t)i * Cout);
          acc[i].x += a.x; acc[i].y += a.y; acc[i].z += a.z; acc[i].w += a.w;
        }
    }
#pragma unroll
    for (int i = 0; i < kConvInPix; ++i)
      if (w0 + i < W) *reinterpret_cast<float4*>(yo + (size_t)i * Cout) = acc[i];
  }
}
int conv_in_launch_t(cudaStream_t st, const void* x, int x_f32, int Bx, int B, int Cin, int H, int W, const float* w,
                     const float* bias, int Cout, float* y, const float* add, int n_add) {
  if (Cin > 8 || (Cout & 3) || (add && n_add < 1)) return 2002;
  const size_t smem = (size_t)Cout * 9 * Cin * sizeof(float);
  static bool done_f[64], done_h[64];
  if (smem > 200 * 1024) return 2002;
  if (int r = smem_optin(conv_in_kernel<float>, 200 * 1024, done_f)) return r;
  if (int r = smem_optin(conv_in_kernel<__half>, 200 * 1024, done_h)) return r;
  const long total = (long)B * H * ((W + kConvInPix - 1) / kConvInPix) * (Cout / 4);
  int grid = cdiv(total, 256);
  if (grid > 132 * 4) grid = 132 * 4;
  if (x_f32)
    conv_in_kernel<float><<<grid, 256, smem, st>>>((const float*)x, Bx, B, Cin, H, W, w, bias, Cout, y, add, n_add, nullptr, 1, Cin);
  else
    conv_in_kernel<__half><<<grid, 256, smem, st>>>((const __half*)x, Bx, B, Cin, H, W, w, bias, Cout, y, add, n_add, nullptr, 1, Cin);
  return (int)cudaGetLastError();
}
int conv_in_cat_launch(cudaStream_t st, const void* x, int x_f32, int Bx, int B, int C1, const float* x2, int n2, int C2, int H, int W,
                       const float* w, const float* bias, int Cout, float* y, const float* add, int n_add) {
  const int Cin = C1 + C2;
  if (!x2 || C1 < 1 || C2 < 1 || Cin > 9 || n2 < 1 || (Cout & 3) || (add && n_add < 1)) return 2002;
  const size_t smem = (size_t)Cout * 9 * Cin * sizeof(float);   // 320 x 81 floats: 104 KB at SDXL's 9 channels
  static bool done_f[64], done_h[64];
  if (smem > 200 * 1024) return 2002;
  if (int r = smem_optin(conv_in_kernel<float, true>, 200 * 1024, done_f)) return r;
  if (int r = smem_optin(conv_in_kernel<__half, true>, 200 * 1024, done_h)) return r;
  const long total = (long)B * H * ((W + kConvInPix - 1) / kConvInPix) * (Cout / 4);
  int grid = cdiv(total, 256);
  if (grid > 132 * 4) grid = 132 * 4;
  if (x_f32)
    conv_in_kernel<float, true><<<grid, 256, smem, st>>>((const float*)x, Bx, B, Cin, H, W, w, bias, Cout, y, add, n_add, x2, n2, C1);
  else
    conv_in_kernel<__half, true><<<grid, 256, smem, st>>>((const __half*)x, Bx, B, Cin, H, W, w, bias, Cout, y, add, n_add, x2, n2, C1);
  return (int)cudaGetLastError();
}
int conv_in_launch(cudaStream_t st, const __half* x, int B, int Cin, int H, int W, const float* w, const float* bias,
                   int Cout, float* y) {
  return conv_in_launch_t(st, x, 0, B, B, Cin, H, W, w, bias, Cout, y);
}

// ------------------------------------------------------------------------------------------------
// resampling copies (NHWC, 4 channels per thread)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint2 pack4h(float4 v) {
  __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&a);
  r.y = *reinterpret_cast<uint32_t*>(&b);
  return r;
}
__global__ void upsample2x_kernel(const float* __restrict__ x, int B, int H, int W, int C, __half* __restrict__ y) {
  const int cv = C / 4;
  const long total = (long)B * (2 * H) * (2 * W) * cv;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv);
    const long pix = idx / cv;
    const int ow = (int)(pix % (2 * W));
    const int oh = (int)((pix / (2 * W)) % (2 * H));
    const int b = (int)(pix / ((long)4 * W * H));
    const float4 v = *reinterpret_cast<const float4*>(x + (((size_t)b * H + (oh >> 1)) * W + (ow >> 1)) * C + c * 4);
    *reinterpret_cast<uint2*>(y + pix * C + c * 4) = pack4h(v);
  }
}
int upsample2x_launch(cudaStream_t st, const float* x, int B, int H, int W, int C, __half* y) {
  if (C & 3) return 2003;
  const long total = (long)B * 4 * H * W * (C / 4);
  int grid = cdiv(total, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  upsample2x_kernel<<<grid, 256, 0, st>>>(x, B, H, W, C, y);
  return (int)cudaGetLastError();
}
__global__ void phase_split_kernel(const float* __restrict__ x, int B, int H, int W, int C, __half* __restrict__ y) {
  const int cv = C / 4;
  const int H2 = H / 2, W2 = W / 2;
  const long total = (long)B * H * W * cv;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv);
    const long pix = idx / cv;
    const int w = (int)(pix % W);
    const int h = (int)((pix / W) % H);
    const int b = (int)(pix / ((long)W * H));
    const float4 v = *reinterpret_cast<const float4*>(x + pix * C + c * 4);
    const int ph = (h & 1) * 2 + (w & 1);
    const size_t o = ((((size_t)ph * B + b) * H2 + (h >> 1)) * W2 + (w >> 1)) * C + c * 4;
    *reinterpret_cast<uint2*>(y + o) = pack4h(v);
  }
}
int phase_split_launch(cudaStream_t st, const float* x, int B, int H, int W, int C, __half* y) {
  if ((C & 3) || (H & 1) || (W & 1)) return 2004;
  const long total = (long)B * H * W * (C / 4);
  int grid = cdiv(total, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  phase_split_kernel<<<grid, 256, 0, st>>>(x, B, H, W, C, y);
  return (int)cudaGetLastError();
}

// ControlNet hint encoder, between two convs: y = f16(silu(x)), NHWC; with `phase` the output is the stride-2 phase split of
// phase_split_kernel (the next conv has stride 2), so no f32 copy and no separate split pass.
__global__ void silu_f16_kernel(const float* __restrict__ x, int B, int H, int W, int C, int phase, __half* __restrict__ y) {
  const int cv = C / 4;
  const long total = (long)B * H * W * cv;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv);
    const long pix = idx / cv;
    float4 v = *reinterpret_cast<const float4*>(x + pix * C + c * 4);
    v.x = silu_f(v.x); v.y = silu_f(v.y); v.z = silu_f(v.z); v.w = silu_f(v.w);
    size_t o = pix * C + c * 4;
    if (phase) {
      const int w = (int)(pix % W);
      const int h = (int)((pix / W) % H);
      const int b = (int)(pix / ((long)W * H));
      const int ph = (h & 1) * 2 + (w & 1);
      o = ((((size_t)ph * B + b) * (H / 2) + (h >> 1)) * (W / 2) + (w >> 1)) * C + c * 4;
    }
    *reinterpret_cast<uint2*>(y + o) = pack4h(v);
  }
}
int silu_f16_launch(cudaStream_t st, const float* x, int B, int H, int W, int C, int phase, __half* y) {
  if ((C & 3) || (phase && ((H & 1) || (W & 1)))) return 2005;
  const long total = (long)B * H * W * (C / 4);
  int grid = cdiv(total, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  if (grid < 1) grid = 1;
  silu_f16_kernel<<<grid, 256, 0, st>>>(x, B, H, W, C, phase, y);
  return (int)cudaGetLastError();
}

// ControlNet scale folded into a zero conv: wo = f16(s * w), bo = s * b (s = 1 keeps the bits).
__global__ void scale_weights_kernel(const __half* __restrict__ w, size_t nw, const float* __restrict__ b, int nb, float s,
                                     __half* __restrict__ wo, float* __restrict__ bo) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nw; i += (size_t)gridDim.x * blockDim.x)
    wo[i] = __float2half_rn(s * __half2float(w[i]));
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)nb; i += (size_t)gridDim.x * blockDim.x)
    bo[i] = s * b[i];
}
int scale_weights_launch(cudaStream_t st, const __half* w, size_t nw, const float* b, int nb, float s, __half* wo, float* bo) {
  int grid = cdiv((long)nw, 256);
  if (grid > 132 * 8) grid = 132 * 8;
  if (grid < 1) grid = 1;
  scale_weights_kernel<<<grid, 256, 0, st>>>(w, nw, b, nb, s, wo, bo);
  return (int)cudaGetLastError();
}

__global__ void cast_f32_f16_kernel(const float* __restrict__ x, size_t n, __half* __restrict__ y) {
  griddep_wait();
  griddep_launch_dependents();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = __float2half_rn(x[i]);
}
__global__ void cast_f16_f32_kernel(const __half* __restrict__ x, size_t n, float* __restrict__ y) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = __half2float(x[i]);
}
int cast_f32_to_f16_launch(cudaStream_t st, const float* x, size_t n, __half* y) {
  int grid = cdiv((long)n, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  if (grid < 1) grid = 1;
  return launch_kernel(cast_f32_f16_kernel, dim3(grid), dim3(256), (size_t)0, st, true, x, n, y);
}
int cast_f16_to_f32_launch(cudaStream_t st, const __half* x, size_t n, float* y) {
  int grid = cdiv((long)n, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  if (grid < 1) grid = 1;
  cast_f16_f32_kernel<<<grid, 256, 0, st>>>(x, n, y);
  return (int)cudaGetLastError();
}
__global__ void nhwc_to_nchw_f16_kernel(const float* __restrict__ x, int B, int HW, int C, int ldx,
                                        __half* __restrict__ y) {
  const long total = (long)B * C * HW;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int p = (int)(i % HW);
    const int c = (int)((i / HW) % C);
    const int b = (int)(i / ((long)HW * C));
    y[i] = __float2half_rn(x[((size_t)b * HW + p) * ldx + c]);
  }
}
__global__ void nhwc_to_nchw_f32_kernel(const float* __restrict__ x, int B, int HW, int C, int ldx,
                                        float* __restrict__ y) {
  const long total = (long)B * C * HW;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int p = (int)(i % HW);
    const int c = (int)((i / HW) % C);
    const int b = (int)(i / ((long)HW * C));
    y[i] = x[((size_t)b * HW + p) * ldx + c];
  }
}
int nhwc_to_nchw_f32_launch(cudaStream_t st, const float* x, int B, int HW, int C, int ldx, float* y) {
  const long total = (long)B * C * HW;
  nhwc_to_nchw_f32_kernel<<<cdiv(total, 256), 256, 0, st>>>(x, B, HW, C, ldx, y);
  return (int)cudaGetLastError();
}
int nhwc_to_nchw_f16_launch(cudaStream_t st, const float* x, int B, int HW, int C, int ldx, __half* y) {
  const long total = (long)B * C * HW;
  nhwc_to_nchw_f16_kernel<<<cdiv(total, 256), 256, 0, st>>>(x, B, HW, C, ldx, y);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// sampler elementwise math. All latents are f32 NCHW [Bimg, C, HW].
// ------------------------------------------------------------------------------------------------
// DDIM eta=0 on the guided eps of the NHWC rows [cond], [cond | uncond], [cond | ptb] or [cond | uncond | ptb]:
//   e = u + (c - u) * g (use_cfg) or c;  then, with perturbed-attention guidance, e = e + p_t * (c - ptb)
// kV, kRescale: kernels.h Prediction; <false, false> is the epsilon step and never reads `factor`. kImg: image guidance (DESIGN.md §21)
// on the rows [cond | img | uncond], e = (u + (c - i) * g) + s_img * (i - u); use_cfg and use_pag are not read.
template <bool kV, bool kRescale, bool kImg = false>
__global__ void cfg_ddim_kernel(const float* __restrict__ eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag,
                                float g, float p_t, float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map,
                                float* __restrict__ x, const float* __restrict__ factor, float s_img) {
  const long total = (long)Bimg * C * HW;
  const int ptb_row0 = (use_cfg ? 2 : 1) * Bimg;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int p = (int)(i % HW);
    const int c = (int)((i / HW) % C);
    const int b = (int)(i / ((long)HW * C));
    const float ec = eps[((size_t)b * HW + p) * ld + c];
    float e = ec;
    if constexpr (kImg) {
      const float ei = eps[((size_t)(Bimg + b) * HW + p) * ld + c];
      const float eu = eps[((size_t)(2 * Bimg + b) * HW + p) * ld + c];
      e = (eu + (ec - ei) * g) + s_img * (ei - eu);
    } else {
      if (use_cfg) {
        // u + (c - u) * s   (reference stablediffusion/mod.rs:539-540)
        const float eu = eps[((size_t)(Bimg + b) * HW + p) * ld + c];
        e = eu + (ec - eu) * g;
      }
      if (use_pag) {
        const float ep = eps[((size_t)(ptb_row0 + b) * HW + p) * ld + c];
        e = e + p_t * (ec - ep);
      }
    }
    if constexpr (kRescale) e *= factor[b];
    const float xv = x[i];
    if constexpr (kV) {   // x0 and eps of the v prediction, then the same DDIM step
      const float predx0 = sqrt_a * xv - sqrt_1ma * e;
      const float pred_eps = sqrt_a * e + sqrt_1ma * xv;
      x[i] = predx0 * sqrt_ap + pred_eps * sqrt_1map;
    } else {
      // DDIM eta=0 (reference stablediffusion/mod.rs:423-428)
      const float predx0 = (xv - e * sqrt_1ma) / sqrt_a;
      x[i] = predx0 * sqrt_ap + e * sqrt_1map;
    }
  }
}
int cfg_ddim_launch(cudaStream_t st, const float* eps, int ld, int Bimg, int C, int HW, int use_cfg, int use_pag, float guidance,
                    float p_t, float sqrt_a, float sqrt_1ma, float sqrt_ap, float sqrt_1map, float* x, const Prediction& pr, int use_img,
                    float img_guidance) {
  const long total = (long)Bimg * C * HW;
  auto kernel = pr.v ? (pr.factor ? cfg_ddim_kernel<true, true> : cfg_ddim_kernel<true, false>)
                     : (pr.factor ? cfg_ddim_kernel<false, true> : cfg_ddim_kernel<false, false>);
  if (use_img)
    kernel = pr.v ? (pr.factor ? cfg_ddim_kernel<true, true, true> : cfg_ddim_kernel<true, false, true>)
                  : (pr.factor ? cfg_ddim_kernel<false, true, true> : cfg_ddim_kernel<false, false, true>);
  kernel<<<cdiv(total, 256), 256, 0, st>>>(eps, ld, Bimg, C, HW, use_cfg, use_pag, guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map,
                                           x, pr.factor, img_guidance);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Guidance rescale statistics (kernels.h: guidance_stats_launch). Grid (blocks per image, Bimg); each thread runs Welford's update in
// double over a fixed set of elements of its image, then warps and blocks merge (n, mean, M2) with Chan et al.'s formula in a fixed
// order (the last block's warp 0 merges the block partials), so the result is the same on every run and stays exact when
// |mean| >> std. The guided value repeats the step kernels'
// expressions (cfg_ddim_kernel, guided_step_kernel) term for term, so it is the value the step then scales.
// ------------------------------------------------------------------------------------------------
static constexpr int kGsThreads = 256, kGsMaxBlocks = 128, kGsPerThread = 2;
struct Moments {
  double n, mean, m2;
};
__device__ __forceinline__ void welford(Moments& m, double x) {
  m.n += 1.0;
  const double d = x - m.mean;
  m.mean += d / m.n;
  m.m2 += d * (x - m.mean);
}
__device__ __forceinline__ Moments chan_merge(const Moments& a, const Moments& b) {
  const double n = a.n + b.n;
  if (n == 0.0) return a;
  const double d = b.mean - a.mean;
  return {n, a.mean + d * (b.n / n), a.m2 + b.m2 + d * d * (a.n * b.n / n)};
}
__device__ __forceinline__ Moments shfl_down(const Moments& m, int o) {
  return {__shfl_down_sync(0xffffffffu, m.n, o), __shfl_down_sync(0xffffffffu, m.mean, o), __shfl_down_sync(0xffffffffu, m.m2, o)};
}
// scratch layout: [Bimg] arrival counters (zero between launches), padded to 16 bytes | [Bimg][kGsMaxBlocks][2] block partials (c, g)
static inline size_t gs_counter_bytes(int Bimg) { return ((size_t)Bimg * sizeof(unsigned) + 15) & ~(size_t)15; }
size_t guidance_stats_scratch_bytes(int Bimg) { return gs_counter_bytes(Bimg) + (size_t)Bimg * kGsMaxBlocks * 2 * sizeof(Moments); }
int guidance_stats_scratch_init(cudaStream_t st, void* scratch, int Bimg) {
  return (int)cudaMemsetAsync(scratch, 0, gs_counter_bytes(Bimg), st);
}
// kImg: the image-guidance combine of cfg_ddim_kernel<.., .., true> on the rows [cond | img | uncond]; use_pag is not read.
template <bool kImg = false>
__global__ void __launch_bounds__(kGsThreads) guidance_stats_kernel(const float* __restrict__ eps, int ld, int Bimg, int C, int HW,
                                                                     int use_pag, float g, float p_t, float phi, unsigned* counters,
                                                                     Moments* partial, float* __restrict__ factor, float s_img) {
  const int b = blockIdx.y, nb = gridDim.x;
  const long n = (long)C * HW;
  const int ptb_row0 = 2 * Bimg;
  Moments mc{0, 0, 0}, mg{0, 0, 0};
  for (long i = (long)blockIdx.x * kGsThreads + threadIdx.x; i < n; i += (long)nb * kGsThreads) {   // NHWC order within the image
    const int p = (int)(i / C);
    const int c = (int)(i % C);
    const float ec = eps[((size_t)b * HW + p) * ld + c];
    float e;
    if constexpr (kImg) {
      const float ei = eps[((size_t)(Bimg + b) * HW + p) * ld + c];
      const float eu = eps[((size_t)(2 * Bimg + b) * HW + p) * ld + c];
      e = (eu + (ec - ei) * g) + s_img * (ei - eu);
    } else {
      const float eu = eps[((size_t)(Bimg + b) * HW + p) * ld + c];
      e = eu + (ec - eu) * g;
      if (use_pag) {
        const float ep = eps[((size_t)(ptb_row0 + b) * HW + p) * ld + c];
        e = e + p_t * (ec - ep);
      }
    }
    welford(mc, ec);
    welford(mg, e);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const Moments oc = shfl_down(mc, o), og = shfl_down(mg, o);
    mc = chan_merge(mc, oc);
    mg = chan_merge(mg, og);
  }
  __shared__ Moments s_warp[kGsThreads / 32][2];
  __shared__ unsigned s_ticket;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) {
    s_warp[warp][0] = mc;
    s_warp[warp][1] = mg;
  }
  __syncthreads();
  Moments* mine = partial + ((size_t)b * kGsMaxBlocks + blockIdx.x) * 2;
  if (threadIdx.x == 0) {
    for (int w = 1; w < kGsThreads / 32; ++w) {
      mc = chan_merge(mc, s_warp[w][0]);
      mg = chan_merge(mg, s_warp[w][1]);
    }
    mine[0] = mc;
    mine[1] = mg;
    __threadfence();   // this block's partials are visible device-wide before it takes its ticket
    s_ticket = atomicAdd(&counters[b], 1u);
  }
  __syncthreads();
  if (s_ticket != (unsigned)(nb - 1) || warp != 0) return;
  // the last block of image b: lane l merges block partials [l * per, (l + 1) * per) in order, then the lanes merge as above
  __threadfence();
  const Moments* all = partial + (size_t)b * kGsMaxBlocks * 2;
  const int per = (nb + 31) / 32;
  Moments c_all{0, 0, 0}, g_all{0, 0, 0};
  for (int k = lane * per; k < (lane + 1) * per && k < nb; ++k) {
    const Moments pc{__ldcg(&all[2 * k].n), __ldcg(&all[2 * k].mean), __ldcg(&all[2 * k].m2)};
    const Moments pg{__ldcg(&all[2 * k + 1].n), __ldcg(&all[2 * k + 1].mean), __ldcg(&all[2 * k + 1].m2)};
    c_all = chan_merge(c_all, pc);
    g_all = chan_merge(g_all, pg);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const Moments oc = shfl_down(c_all, o), og = shfl_down(g_all, o);
    c_all = chan_merge(c_all, oc);
    g_all = chan_merge(g_all, og);
  }
  if (lane != 0) return;
  double ratio = 1.0;
  if (n > 1 && g_all.m2 > 0.0) ratio = sqrt(c_all.m2 / g_all.m2);   // std(c) / std(g): the (n - 1) divisors cancel
  factor[b] = (float)((double)phi * ratio + (1.0 - (double)phi));
  counters[b] = 0u;   // ready for the next launch
}
int guidance_stats_launch(cudaStream_t st, const float* eps, int ld, int Bimg, int C, int HW, int use_pag, float guidance, float p_t,
                          float phi, void* scratch, float* factor, int use_img, float img_guidance) {
  const long n = (long)C * HW;
  if (Bimg < 1 || n < 1) return (int)cudaErrorInvalidValue;
  const int want = cdiv(n, (long)kGsThreads * kGsPerThread), nb = want < kGsMaxBlocks ? want : kGsMaxBlocks;
  auto kernel = use_img ? guidance_stats_kernel<true> : guidance_stats_kernel<false>;
  kernel<<<dim3(nb, Bimg), kGsThreads, 0, st>>>(eps, ld, Bimg, C, HW, use_pag, guidance, p_t, phi, (unsigned*)scratch,
                                                (Moments*)((uint8_t*)scratch + gs_counter_bytes(Bimg)), factor, img_guidance);
  return (int)cudaGetLastError();
}

// PAG's identity self-attention: out[r, 0:C] = qkv[r, 2C:3C] (the V window of the fused QKV rows), 16-byte vectors.
__global__ void pag_identity_kernel(const uint4* __restrict__ qkv, int C8, long n, uint4* __restrict__ out) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long r = i / C8;
    const int c = (int)(i - r * C8);
    out[i] = qkv[r * 3 * C8 + 2 * C8 + c];
  }
}
int pag_identity_launch(cudaStream_t st, const __half* qkv, int C, long rows, __half* out) {
  if (C % 8 || ((uintptr_t)qkv | (uintptr_t)out) % 16) return (int)cudaErrorInvalidValue;
  const long n = rows * (C / 8);
  if (n == 0) return 0;
  const long blocks = cdiv(n, 256);
  pag_identity_kernel<<<(unsigned)(blocks < 8192 ? blocks : 8192), 256, 0, st>>>((const uint4*)qkv, C / 8, n, (uint4*)out);
  return (int)cudaGetLastError();
}
// x = mask ? x : (ref*sqrt_a + noise*sqrt_1ma)   (reference stablediffusion/mod.rs:463-465)
__global__ void inpaint_blend_kernel(float* __restrict__ x, const float* __restrict__ ref,
                                     const float* __restrict__ noise, const uint8_t* __restrict__ mask, size_t n,
                                     float sqrt_a, float sqrt_1ma) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float nr = ref[i] * sqrt_a + noise[i] * sqrt_1ma;
    x[i] = mask[i] ? x[i] : nr;
  }
}
int inpaint_blend_launch(cudaStream_t st, float* x, const float* ref, const float* noise, const uint8_t* mask, size_t n,
                         float sqrt_a, float sqrt_1ma) {
  inpaint_blend_kernel<<<cdiv((long)n, 256), 256, 0, st>>>(x, ref, noise, mask, n, sqrt_a, sqrt_1ma);
  return (int)cudaGetLastError();
}
__global__ void axpby_kernel(float* __restrict__ x, const float* __restrict__ noise, size_t n, float sa, float sb) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    x[i] = x[i] * sa + noise[i] * sb;
}
int axpby_launch(cudaStream_t st, float* x, const float* noise, size_t n, float sa, float sb) {
  axpby_kernel<<<cdiv((long)n, 256), 256, 0, st>>>(x, noise, n, sa, sb);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG + Box-Muller. Element i of stream (seed, subseq): counter =
// (i/4 lo32, i/4 hi32, subseq lo32, subseq hi32), key = (seed lo32, seed hi32); lane i%4 of the
// 4 normals produced from the 4 output words. oracle/philox.py is the bit-identical restatement, and noise4() below (the
// scheduled samplers' in-kernel noise) repeats this arithmetic: change the three together (tests/test_schedulers_gpu.py compares
// the two kernels bit for bit).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}
__global__ void randn_kernel(float* __restrict__ out, size_t n, uint64_t seed, uint64_t subseq) {
  const size_t nblk = (n + 3) / 4;
  for (size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x; blk < nblk;
       blk += (size_t)gridDim.x * blockDim.x) {
    uint32_t c[4] = {(uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)subseq, (uint32_t)(subseq >> 32)};
    philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    float z[4];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float u1 = ((float)(c[2 * j] >> 8) + 0.5f) * (1.0f / 16777216.0f);
      const float u2 = ((float)(c[2 * j + 1] >> 8) + 0.5f) * (1.0f / 16777216.0f);
      const float rad = sqrtf(-2.0f * logf(u1));
      const float ang = 6.283185307179586f * u2;
      z[2 * j] = rad * cosf(ang);
      z[2 * j + 1] = rad * sinf(ang);
    }
    for (int j = 0; j < 4; ++j)
      if (blk * 4 + j < n) out[blk * 4 + j] = z[j];
  }
}
int randn_launch(cudaStream_t st, float* out, size_t n, uint64_t seed, uint64_t subseq) {
  randn_kernel<<<cdiv((long)((n + 3) / 4), 256), 256, 0, st>>>(out, n, seed, subseq);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// The scheduled samplers' step (DESIGN.md §16; kernels.h: GuidedStepParams). One thread per block of four consecutive
// elements of the NCHW state, which is the block one Philox counter produces: in-kernel noise repeats randn_kernel's
// arithmetic on the same counter, so it equals randn_launch(seed, subseq) bit for bit. The state, history, noise and reference
// go through 16-byte vectors when the block is whole and the pointers are aligned; the mask is read byte by byte. The eps rows
// are NHWC and are gathered element by element: each of a thread's four loads is a warp-wide gather with stride 4 * ld floats,
// none of them coalesced on its own (the four together cover one contiguous span, served from L1 / L2).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void noise4(const float* __restrict__ z, uint64_t seed, uint64_t subseq, size_t blk, size_t n, bool vec,
                                       float out[4]) {
  if (z) {
    if (vec) {
      const float4 v = *reinterpret_cast<const float4*>(z + blk * 4);
      out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
    } else {
      for (int j = 0; j < 4; ++j) out[j] = blk * 4 + j < n ? z[blk * 4 + j] : 0.f;
    }
    return;
  }
  uint32_t c[4] = {(uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)subseq, (uint32_t)(subseq >> 32)};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float u1 = ((float)(c[2 * j] >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float u2 = ((float)(c[2 * j + 1] >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float rad = sqrtf(-2.0f * logf(u1));
    const float ang = 6.283185307179586f * u2;
    out[2 * j] = rad * cosf(ang);
    out[2 * j + 1] = rad * sinf(ang);
  }
}
__device__ __forceinline__ void load4(const float* __restrict__ p, size_t blk, size_t n, bool vec, float out[4]) {
  if (vec) {
    const float4 v = *reinterpret_cast<const float4*>(p + blk * 4);
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
  } else {
    for (int j = 0; j < 4; ++j) out[j] = blk * 4 + j < n ? p[blk * 4 + j] : 0.f;
  }
}
__device__ __forceinline__ void store4(float* __restrict__ p, size_t blk, size_t n, bool vec, const float v[4]) {
  if (vec) {
    *reinterpret_cast<float4*>(p + blk * 4) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    for (int j = 0; j < 4; ++j)
      if (blk * 4 + j < n) p[blk * 4 + j] = v[j];
  }
}
// kV, kRescale: kernels.h Prediction; <false, false> is the epsilon step and never reads `pr`. kRows: kernels.h StepRows, the
// two-row form; without it `r` is never read. kImg: cfg_ddim_kernel's image-guidance combine with scale s_img (guided_step_img_kernel).
template <bool kV, bool kRescale, bool kRows, bool kImg>
__device__ __forceinline__ void guided_step(const GuidedStepParams& p, int aligned, const Prediction& pr, const StepRows& r, float s_img) {
  const size_t n = (size_t)p.Bimg * p.C * p.HW, nblk = (n + 3) / 4;
  const size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= nblk) return;
  const bool vec = aligned && blk * 4 + 4 <= n;
  float xh[4], D[4];
  load4(p.xh, blk, n, vec, xh);
  if (p.eps) {
    const int grp_u = p.Bimg, grp_p = (p.use_cfg ? 2 : 1) * p.Bimg;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t i = blk * 4 + j;
      D[j] = 0.f;
      if (i >= n) continue;
      const int px = (int)(i % p.HW);
      const int c = (int)((i / p.HW) % p.C);
      const int b = (int)(i / ((size_t)p.HW * p.C));
      const float ec = p.eps[((size_t)b * p.HW + px) * p.ld + c];
      float e = ec;
      if constexpr (kImg) {   // cfg_ddim_kernel's, rows [cond | img | uncond]
        const float ei = p.eps[((size_t)(p.Bimg + b) * p.HW + px) * p.ld + c];
        const float eu = p.eps[((size_t)(2 * p.Bimg + b) * p.HW + px) * p.ld + c];
        e = (eu + (ec - ei) * p.guidance) + s_img * (ei - eu);
      } else {
        if (p.use_cfg) {   // u + (c - u) * s, cfg_ddim_kernel's order
          const float eu = p.eps[((size_t)(grp_u + b) * p.HW + px) * p.ld + c];
          e = eu + (ec - eu) * p.guidance;
        }
        if (p.use_pag) {   // cfg_ddim_kernel's
          const float ep = p.eps[((size_t)(grp_p + b) * p.HW + px) * p.ld + c];
          e = e + p.p_t * (ec - ep);
        }
      }
      if constexpr (kRescale) e *= pr.factor[b];
      if constexpr (kV) D[j] = pr.dx * xh[j] - pr.de * e;
      else D[j] = xh[j] - p.sigma * e;
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) D[j] = xh[j];
  }
  float nx[4];
  if constexpr (kRows) {   // every operand is read before anything is written: both rows see the values before the launch
    float xs[4] = {0.f, 0.f, 0.f, 0.f}, h1[4] = {0.f, 0.f, 0.f, 0.f}, h2[4] = {0.f, 0.f, 0.f, 0.f};
    if (r.cs != 0.f || r.ss != 0.f) load4(r.xs, blk, n, vec, xs);
    if (p.ch != 0.f || r.sh != 0.f || r.shift) load4(p.hist, blk, n, vec, h1);
    if (r.ch2 != 0.f || r.sh2 != 0.f) load4(r.h2, blk, n, vec, h2);
#pragma unroll
    for (int j = 0; j < 4; ++j) nx[j] = p.cx * xh[j] + r.cs * xs[j] + p.cd * D[j] + p.ch * h1[j] + r.ch2 * h2[j];
    if (r.write_xs) {
      float s[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) s[j] = r.sx * xh[j] + r.ss * xs[j] + r.sd * D[j] + r.sh * h1[j] + r.sh2 * h2[j];
      store4(r.xs, blk, n, vec, s);
    }
    if (r.shift) store4(r.h2, blk, n, vec, h1);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) nx[j] = p.cx * xh[j] + p.cd * D[j];
    if (p.ch != 0.f) {
      float h[4];
      load4(p.hist, blk, n, vec, h);
#pragma unroll
      for (int j = 0; j < 4; ++j) nx[j] += p.ch * h[j];
    }
  }
  if (p.write_hist) store4(p.hist, blk, n, vec, D);
  if (p.cn != 0.f) {
    float z[4];
    noise4(p.z, p.seed, p.z_subseq, blk, n, vec, z);
#pragma unroll
    for (int j = 0; j < 4; ++j) nx[j] += p.cn * z[j];
  }
  if (p.mask) {   // the latent-blend inpainting of the NEXT forward: xh = mask ? xh : ref + sigma' * z
    float z[4], r[4];
    noise4(p.zb, p.seed, p.zb_subseq, blk, n, vec, z);
    load4(p.ref, blk, n, vec, r);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (blk * 4 + j < n && !p.mask[blk * 4 + j]) nx[j] = r[j] + p.sigma_blend * z[j];
  }
  store4(p.xh, blk, n, vec, nx);
#pragma unroll
  for (int j = 0; j < 4; ++j) nx[j] *= p.c_in;
  store4(p.x_in, blk, n, vec, nx);
}
template <bool kV, bool kRescale, bool kRows>
__global__ void __launch_bounds__(256) guided_step_kernel(const GuidedStepParams p, int aligned, const Prediction pr, const StepRows r) {
  guided_step<kV, kRescale, kRows, false>(p, aligned, pr, r, 0.f);
}
template <bool kV, bool kRescale, bool kRows>
__global__ void __launch_bounds__(256) guided_step_img_kernel(const GuidedStepParams p, int aligned, const Prediction pr, const StepRows r,
                                                              float s_img) {
  guided_step<kV, kRescale, kRows, true>(p, aligned, pr, r, s_img);
}
// The instantiation of (kV, kRescale) = (pr.v, pr.factor) at the given kRows, without and with image guidance.
template <bool kRows>
static auto guided_step_pick(const Prediction& pr) {
  return pr.v ? (pr.factor ? guided_step_kernel<true, true, kRows> : guided_step_kernel<true, false, kRows>)
              : (pr.factor ? guided_step_kernel<false, true, kRows> : guided_step_kernel<false, false, kRows>);
}
template <bool kRows>
static auto guided_step_img_pick(const Prediction& pr) {
  return pr.v ? (pr.factor ? guided_step_img_kernel<true, true, kRows> : guided_step_img_kernel<true, false, kRows>)
              : (pr.factor ? guided_step_img_kernel<false, true, kRows> : guided_step_img_kernel<false, false, kRows>);
}
int guided_step_launch(cudaStream_t st, const GuidedStepParams& p, const Prediction& pr, const StepRows* rows, int use_img,
                       float img_guidance) {
  const size_t n = (size_t)p.Bimg * p.C * p.HW;
  if (!n) return 0;
  if (!p.xh || !p.x_in || ((p.ch != 0.f || p.write_hist) && !p.hist) || (p.mask && !p.ref)) return (int)cudaErrorInvalidValue;
  uintptr_t a = (uintptr_t)p.xh | (uintptr_t)p.x_in | (uintptr_t)p.hist | (uintptr_t)p.z | (uintptr_t)p.zb | (uintptr_t)p.ref;
  const unsigned grid = cdiv((long)((n + 3) / 4), 256);
  const bool img = use_img && p.eps;
  if (rows) {
    const StepRows& r = *rows;
    if (((r.cs != 0.f || r.ss != 0.f || r.write_xs) && !r.xs) || ((r.sh != 0.f || r.shift) && !p.hist) ||
        ((r.ch2 != 0.f || r.sh2 != 0.f || r.shift) && !r.h2))
      return (int)cudaErrorInvalidValue;
    a |= (uintptr_t)r.xs | (uintptr_t)r.h2;
    if (img) guided_step_img_pick<true>(pr)<<<grid, 256, 0, st>>>(p, a % 16 == 0, pr, r, img_guidance);
    else guided_step_pick<true>(pr)<<<grid, 256, 0, st>>>(p, a % 16 == 0, pr, r);
    return (int)cudaGetLastError();
  }
  if (img) guided_step_img_pick<false>(pr)<<<grid, 256, 0, st>>>(p, a % 16 == 0, pr, StepRows{}, img_guidance);
  else guided_step_pick<false>(pr)<<<grid, 256, 0, st>>>(p, a % 16 == 0, pr, StepRows{});
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// load-time weight re-layout
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int geglu_perm(int n, int N, int bn) {
  if (bn <= 0) return n;
  const int half_n = N / 2, hb = bn / 2;
  const int g = n >= half_n;
  const int m = g ? n - half_n : n;
  return (m / hb) * bn + g * hb + (m % hb);
}
// src [K][N] row-major -> dst [N][Kpad] (tiled transpose through smem)
__global__ void transpose_linear_kernel(const __half* __restrict__ src, int K, int N, __half* __restrict__ dst,
                                        int Kpad, int dst_row0, int geglu_bn) {
  __shared__ __half tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? src[(size_t)k * N + n] : __float2half(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < Kpad) dst[(size_t)(dst_row0 + geglu_perm(n, N, geglu_bn)) * Kpad + k] = tile[threadIdx.x][i];
  }
}
int transpose_linear_launch(cudaStream_t st, const __half* src, int K, int N, __half* dst, int Kpad, int dst_row0,
                            int geglu_bn) {
  dim3 grid(cdiv(N, 32), cdiv(Kpad, 32));
  transpose_linear_kernel<<<grid, dim3(32, 8), 0, st>>>(src, K, N, dst, Kpad, dst_row0, geglu_bn);
  return (int)cudaGetLastError();
}
// OIHW -> dst[o][col0 + (kh*KW+kw)*Ipad + i]
__global__ void repack_conv_kernel(const __half* __restrict__ src, int O, int I, int KH, int KW,
                                   __half* __restrict__ dst, int Ktot, int col0, int Ipad) {
  const long total = (long)O * KH * KW * Ipad;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int i = (int)(idx % Ipad);
    const int tap = (int)((idx / Ipad) % (KH * KW));
    const int o = (int)(idx / ((long)Ipad * KH * KW));
    const __half v = i < I ? src[(((size_t)o * I + i) * KH + tap / KW) * KW + tap % KW] : __float2half(0.f);
    dst[(size_t)o * Ktot + col0 + (size_t)tap * Ipad + i] = v;
  }
}
int repack_conv_launch(cudaStream_t st, const __half* src, int O, int I, int KH, int KW, __half* dst, int Ktot,
                       int col0, int Ipad) {
  const long total = (long)O * KH * KW * Ipad;
  int grid = cdiv(total, 256);
  if (grid > 132 * 32) grid = 132 * 32;
  repack_conv_kernel<<<grid, 256, 0, st>>>(src, O, I, KH, KW, dst, Ktot, col0, Ipad);
  return (int)cudaGetLastError();
}
// Nearest-2x upsample followed by a 3x3 pad-1 conv (reference unet/mod.rs:742-751, autoencoder/mod.rs:311-319): output pixel
// (2i+a, 2j+b) reads upsampled rows 2i+a-1 .. 2i+a+1 = source rows {i-1, i, i} for a = 0 and {i, i, i+1} for a = 1 (same for
// columns), so each output parity (a, b) is a 2x2 convolution of the source image with summed taps:
//   a = 0: tap th=0 (dh=-1) = kh{0},   th=1 (dh=0)  = kh{1,2};     a = 1: th=0 (dh=0) = kh{0,1},   th=1 (dh=+1) = kh{2}
__global__ void repack_upconv_kernel(const __half* __restrict__ src, int O, int I, __half* __restrict__ dst, int Ipad) {
  const long total = (long)4 * O * 4 * Ipad;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int i = (int)(idx % Ipad);
    const int tap = (int)((idx / Ipad) % 4);
    const int o = (int)((idx / ((long)Ipad * 4)) % O);
    const int ph = (int)(idx / ((long)Ipad * 4 * O));
    const int a = ph >> 1, b = ph & 1, th = tap >> 1, tw = tap & 1;
    float acc = 0.f;
    if (i < I) {
      const int kh0 = a == 0 ? (th == 0 ? 0 : 1) : (th == 0 ? 0 : 2), kh1 = a == 0 ? (th == 0 ? 0 : 2) : (th == 0 ? 1 : 2);
      const int kw0 = b == 0 ? (tw == 0 ? 0 : 1) : (tw == 0 ? 0 : 2), kw1 = b == 0 ? (tw == 0 ? 0 : 2) : (tw == 0 ? 1 : 2);
      for (int kh = kh0; kh <= kh1; ++kh)
        for (int kw = kw0; kw <= kw1; ++kw) acc += __half2float(src[(((size_t)o * I + i) * 3 + kh) * 3 + kw]);
    }
    dst[idx] = __float2half_rn(acc);
  }
}
int repack_upconv_launch(cudaStream_t st, const __half* src, int O, int I, __half* dst, int Ipad) {
  const long total = (long)4 * O * 4 * Ipad;
  int grid = cdiv(total, 256);
  if (grid > 132 * 32) grid = 132 * 32;
  repack_upconv_kernel<<<grid, 256, 0, st>>>(src, O, I, dst, Ipad);
  return (int)cudaGetLastError();
}
__global__ void bias_to_f32_kernel(const __half* __restrict__ src, int N, float* __restrict__ dst, int geglu_bn,
                                   int accumulate) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const int d = geglu_perm(n, N, geglu_bn);
  const float v = __half2float(src[n]);
  dst[d] = accumulate ? dst[d] + v : v;
}
__global__ void vec_add_f32_kernel(float* __restrict__ dst, const float* __restrict__ src, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}
int vec_add_f32_launch(cudaStream_t st, float* dst, const float* src, int n) {
  vec_add_f32_kernel<<<cdiv(n, 256), 256, 0, st>>>(dst, src, n);
  return (int)cudaGetLastError();
}
int bias_to_f32_launch(cudaStream_t st, const __half* src, int N, float* dst, int geglu_bn, int accumulate) {
  bias_to_f32_kernel<<<cdiv(N, 256), 256, 0, st>>>(src, N, dst, geglu_bn, accumulate);
  return (int)cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// LoRA merge: one 64 x 64 tile of the delta per CTA, 256 threads, 4 x 4 outputs per thread (rows ty + 16i, columns tx + 16j).
// up / down are staged through shared memory as f32 in chunks of 32 ranks; every output is accumulated by one thread in a
// fixed order (terms in call order, rank index ascending): deterministic, no atomics. CUDA-core FMA (see DESIGN.md).
// ------------------------------------------------------------------------------------------------
constexpr int LORA_TILE = 64, LORA_RC = 32;
// acc[i][j] = sum_r up[n, r] * down[r, k] over the tile's outputs, rank index ascending
__device__ __forceinline__ void lora_rank_product(float (&acc)[4][4], float (*Us)[LORA_TILE + 1], float (*Ds)[LORA_TILE],
                                                  const __half* __restrict__ up, const __half* __restrict__ down, int R,
                                                  int N, int Kd, int n0, int k0) {
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int r0 = 0; r0 < R; r0 += LORA_RC) {
    const int rc = R - r0 < LORA_RC ? R - r0 : LORA_RC;
    __syncthreads();
    for (int e = tid; e < LORA_RC * LORA_TILE; e += 256) {
      {  // up [N, r] row-major: consecutive threads read consecutive ranks of one row
        const int x = e / LORA_RC, rr = e % LORA_RC, n = n0 + x;
        Us[rr][x] = (rr < rc && n < N) ? __half2float(up[(size_t)n * R + r0 + rr]) : 0.f;
      }
      {
        const int rr = e / LORA_TILE, x = e % LORA_TILE, k = k0 + x;
        Ds[rr][x] = (rr < rc && k < Kd) ? __half2float(down[(size_t)(r0 + rr) * Kd + k]) : 0.f;
      }
    }
    __syncthreads();
    for (int rr = 0; rr < rc; ++rr) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = Us[rr][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Ds[rr][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
  }
}
// kMixed = false: every term is LORA_LORA (the kind field is not read).
template <bool kMixed>
__global__ void __launch_bounds__(256) lora_merge_kernel(const LoraMergeParams p) {
  __shared__ float Us[LORA_RC][LORA_TILE + 1];   // +1: the staging stores walk rr at fixed x
  __shared__ float Ds[LORA_RC][LORA_TILE];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.y * LORA_TILE, k0 = blockIdx.x * LORA_TILE;
  float tot[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) tot[i][j] = 0.f;
  for (int t = 0; t < p.nterm; ++t) {
    const LoraTerm T = p.term[t];
    float acc[4][4];
    if (!kMixed || T.kind == LORA_LORA || T.kind == LORA_LOHA) {
      lora_rank_product(acc, Us, Ds, T.up, T.down, T.r, p.N, p.Kd, n0, k0);
      if (kMixed && T.kind == LORA_LOHA) {
        float acc2[4][4];
        lora_rank_product(acc2, Us, Ds, T.up2, T.down2, T.r2, p.N, p.Kd, n0, k0);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = __fmul_rn(acc[i][j], acc2[i][j]);
      }
    } else {
      const int b = p.Kd / p.taps / (T.d > 0 ? T.d : 1);   // LORA_LOKR: columns of w1
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = n0 + ty + 16 * i, k = k0 + tx + 16 * j;
          float v = 0.f;
          if (n < p.N && k < p.Kd) {
            if (T.kind == LORA_FULL) {
              v = __half2float(T.down[(size_t)n * p.Kd + k]);
            } else if (T.kind == LORA_F32) {
              v = T.w1[(size_t)n * p.Kd + k];
            } else {   // LORA_LOKR
              const int ich = k / p.taps, tap = k % p.taps;
              v = __fmul_rn(T.w1[(size_t)(n / T.c) * b + ich / T.d], T.w2[(size_t)(n % T.c) * T.d * p.taps + (ich % T.d) * p.taps + tap]);
            }
          }
          acc[i][j] = v;
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) tot[i][j] = __fadd_rn(tot[i][j], __fmul_rn(T.coef, acc[i][j]));
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = n0 + ty + 16 * i;
    if (n >= p.N) continue;
    const size_t row = (size_t)(p.row0 + geglu_perm(n, p.N, p.geglu_bn)) * p.ld;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx + 16 * j;
      if (k >= p.Kd) continue;
      const float d = tot[i][j];
      if (p.delta_out) { p.delta_out[(size_t)n * p.Kd + k] = d; continue; }
      const size_t off = row + p.col0 + (size_t)(k % p.taps) * p.Ipad + k / p.taps;
      // a zero delta leaves the weight's bits alone (f32(W) + 0 would turn -0 into +0)
      if (p.f32) {
        const float w = ((const float*)p.src)[off];
        ((float*)p.dst)[off] = d == 0.f ? w : __half2float(__float2half_rn(w + d));
      } else {
        const __half w = ((const __half*)p.src)[off];
        ((__half*)p.dst)[off] = d == 0.f ? w : __float2half_rn(__half2float(w) + d);
      }
    }
  }
}
int lora_merge_launch(cudaStream_t st, const LoraMergeParams& p) {
  if (p.nterm < 1 || p.nterm > LORA_MAX_TERMS || p.taps < 1) return 1;
  bool mixed = false;
  for (int t = 0; t < p.nterm; ++t) {
    const LoraTerm& T = p.term[t];
    if (T.kind < LORA_LORA || T.kind > LORA_F32) return 1;
    if (T.kind == LORA_LOKR && (T.c < 1 || T.d < 1 || p.N % T.c || (p.Kd / p.taps) % T.d)) return 1;
    mixed |= T.kind != LORA_LORA;
  }
  dim3 grid(cdiv(p.Kd, LORA_TILE), cdiv(p.N, LORA_TILE));
  if (mixed) lora_merge_kernel<true><<<grid, 256, 0, st>>>(p);
  else lora_merge_kernel<false><<<grid, 256, 0, st>>>(p);
  return (int)cudaGetLastError();
}

// W of element (n, k) of a slot's logical [N, Kd] matrix (the lora_merge_kernel map), read from p.src
__device__ __forceinline__ double dora_w(const LoraMergeParams& p, int n, int k) {
  const size_t off = (size_t)(p.row0 + geglu_perm(n, p.N, p.geglu_bn)) * p.ld + p.col0 + (size_t)(k % p.taps) * p.Ipad + k / p.taps;
  return p.f32 ? (double)((const float*)p.src)[off] : (double)__half2float(((const __half*)p.src)[off]);
}
constexpr int DORA_THREADS = 256;
// one CTA per norm: thread x sums (W + dw)^2 over the elements x, x + 256, ... of its row (axis 0: k ascending) or input
// channel (axis 1: e = n * taps + tap ascending) in double, then a fixed tree reduction. No atomics.
__global__ void __launch_bounds__(DORA_THREADS) dora_norm_kernel(const LoraMergeParams p, const float* __restrict__ dw, int axis,
                                                                   double* __restrict__ norm) {
  __shared__ double red[DORA_THREADS];
  const int j = blockIdx.x;
  const int len = axis == 0 ? p.Kd : p.N * p.taps;
  double s = 0.0;
  for (int e = threadIdx.x; e < len; e += DORA_THREADS) {
    const int n = axis == 0 ? j : e / p.taps, k = axis == 0 ? e : j * p.taps + e % p.taps;
    const double v = dora_w(p, n, k) + (double)dw[(size_t)n * p.Kd + k];
    s = fma(v, v, s);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = DORA_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) norm[j] = sqrt(red[0]);
}
int dora_norm_launch(cudaStream_t st, const LoraMergeParams& slot, const float* dw, int axis, double* norm) {
  if (slot.taps < 1 || slot.N < 1 || slot.Kd < 1) return 1;
  dora_norm_kernel<<<axis == 0 ? slot.N : slot.Kd / slot.taps, DORA_THREADS, 0, st>>>(slot, dw, axis, norm);
  return (int)cudaGetLastError();
}
__global__ void dora_accum_kernel(const LoraMergeParams p, const float* __restrict__ dw, const float* __restrict__ m,
                                  const double* __restrict__ norm, int axis, float s, float* __restrict__ acc) {
  const long total = (long)p.N * p.Kd;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
    const int n = (int)(e / p.Kd), k = (int)(e % p.Kd);
    const int j = axis == 0 ? n : k / p.taps;
    const double nj = norm[j];
    if (nj == 0.0) continue;
    const double w = dora_w(p, n, k);
    const double c = (double)s * ((double)m[j] * (w + (double)dw[e]) / nj - w);
    acc[e] = __fadd_rn(acc[e], (float)c);
  }
}
int dora_accum_launch(cudaStream_t st, const LoraMergeParams& slot, const float* dw, const float* m, const double* norm, int axis,
                      float s, float* acc) {
  if (slot.taps < 1) return 1;
  const long total = (long)slot.N * slot.Kd;
  if (total < 1) return 1;
  dora_accum_kernel<<<(unsigned)cdiv(total, 256), 256, 0, st>>>(slot, dw, m, norm, axis, s, acc);
  return (int)cudaGetLastError();
}
// same index map and tap sets as repack_upconv_kernel; padded input channels are not written
__global__ void lora_upconv_merge_kernel(const __half* __restrict__ src, const float* __restrict__ delta, int O, int I,
                                         __half* __restrict__ dst, int Ipad) {
  const long total = (long)4 * O * 4 * Ipad;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int i = (int)(idx % Ipad);
    if (i >= I) continue;
    const int tap = (int)((idx / Ipad) % 4);
    const int o = (int)((idx / ((long)Ipad * 4)) % O);
    const int ph = (int)(idx / ((long)Ipad * 4 * O));
    const int a = ph >> 1, b = ph & 1, th = tap >> 1, tw = tap & 1;
    const int kh0 = a == 0 ? (th == 0 ? 0 : 1) : (th == 0 ? 0 : 2), kh1 = a == 0 ? (th == 0 ? 0 : 2) : (th == 0 ? 1 : 2);
    const int kw0 = b == 0 ? (tw == 0 ? 0 : 1) : (tw == 0 ? 0 : 2), kw1 = b == 0 ? (tw == 0 ? 0 : 2) : (tw == 0 ? 1 : 2);
    float d = 0.f;
    for (int kh = kh0; kh <= kh1; ++kh)
      for (int kw = kw0; kw <= kw1; ++kw) d += delta[((size_t)o * I + i) * 9 + kh * 3 + kw];
    dst[idx] = d == 0.f ? src[idx] : __float2half_rn(__half2float(src[idx]) + d);
  }
}
int lora_upconv_merge_launch(cudaStream_t st, const __half* src, const float* delta, int O, int I, __half* dst, int Ipad) {
  const long total = (long)4 * O * 4 * Ipad;
  int grid = cdiv(total, 256);
  if (grid > 132 * 32) grid = 132 * 32;
  lora_upconv_merge_kernel<<<grid, 256, 0, st>>>(src, delta, O, I, dst, Ipad);
  return (int)cudaGetLastError();
}

}  // namespace sdxl
