// Kernels of the T2I-Adapter (DESIGN.md §11): the three small passes of the adapter forward that are not convolutions (those run
// on igemm.cu) and the per-step add of the features into the UNet's encoder.
#include "common.cuh"
#include "kernels.h"

namespace sdxl {

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

__device__ __forceinline__ uint2 t2i_pack4h(float4 v) {
  __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 r;
  r.x = *reinterpret_cast<uint32_t*>(&a);
  r.y = *reinterpret_cast<uint32_t*>(&b);
  return r;
}

// PixelUnshuffle(16) of an f32 NCHW hint [n, C, H, W] into the f16 NHWC operand of conv_in [n, H/16, W/16, C*256]:
// channel ci*256 + i*16 + j of pixel (y, x) is hint[ci, 16y + i, 16x + j]. One thread per (pixel, ci, i): 16 contiguous floats in,
// 16 contiguous halves out.
__global__ void pixel_unshuffle_kernel(const float* __restrict__ x, int n, int C, int H, int W, __half* __restrict__ y) {
  const int h = H / 16, w = W / 16;
  const long total = (long)n * h * w * C * 16;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int i = (int)(idx % 16);
    const int ci = (int)((idx / 16) % C);
    const long pix = idx / (16L * C);
    const int px = (int)(pix % w);
    const int py = (int)((pix / w) % h);
    const int b = (int)(pix / ((long)w * h));
    const float4* src = reinterpret_cast<const float4*>(x + (((size_t)b * C + ci) * H + 16 * py + i) * W + 16 * px);
    uint2 o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) o[q] = t2i_pack4h(src[q]);
    uint4* dst = reinterpret_cast<uint4*>(y + (size_t)pix * C * 256 + ci * 256 + i * 16);
    dst[0] = make_uint4(o[0].x, o[0].y, o[1].x, o[1].y);
    dst[1] = make_uint4(o[2].x, o[2].y, o[3].x, o[3].y);
  }
}
int pixel_unshuffle_launch(cudaStream_t st, const float* x, int n, int C, int H, int W, __half* y) {
  if (n < 1 || C < 1 || H < 16 || W < 16 || (H % 16) || (W % 16)) return 2101;
  int grid = cdiv((long)n * (H / 16) * (W / 16) * C * 16, 256);
  if (grid > 132 * 16) grid = 132 * 16;
  pixel_unshuffle_kernel<<<grid, 256, 0, st>>>(x, n, C, H, W, y);
  return (int)cudaGetLastError();
}

// y = f16(max(x, 0)), n % 4 == 0 (the ReLU between block1 and block2 of an adapter resnet).
__global__ void relu_f16_kernel(const float* __restrict__ x, size_t n4, __half* __restrict__ y) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(x)[i];
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    reinterpret_cast<uint2*>(y)[i] = t2i_pack4h(v);
  }
}
int relu_f16_launch(cudaStream_t st, const float* x, size_t n, __half* y) {
  if (n % 4) return 2102;
  int grid = cdiv((long)(n / 4), 256);
  if (grid > 132 * 16) grid = 132 * 16;
  if (grid < 1) grid = 1;
  relu_f16_kernel<<<grid, 256, 0, st>>>(x, n / 4, y);
  return (int)cudaGetLastError();
}

// 2x2 average pool, stride 2, of f32 NHWC [n, H, W, C] -> f16 NHWC [n, H/2, W/2, C]; the mean is formed in f32 and rounded once.
__global__ void avg_pool2_f16_kernel(const float* __restrict__ x, int n, int H, int W, int C, __half* __restrict__ y) {
  const int cv = C / 4, h = H / 2, w = W / 2;
  const long total = (long)n * h * w * cv;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % cv);
    const long pix = idx / cv;
    const int px = (int)(pix % w);
    const int py = (int)((pix / w) % h);
    const int b = (int)(pix / ((long)w * h));
    const float* p = x + (((size_t)b * H + 2 * py) * W + 2 * px) * C + c * 4;
    const float4 a = *reinterpret_cast<const float4*>(p), bb = *reinterpret_cast<const float4*>(p + C);
    const float4 cc = *reinterpret_cast<const float4*>(p + (size_t)W * C), d = *reinterpret_cast<const float4*>(p + (size_t)W * C + C);
    const float4 m = make_float4((a.x + bb.x + cc.x + d.x) * 0.25f, (a.y + bb.y + cc.y + d.y) * 0.25f, (a.z + bb.z + cc.z + d.z) * 0.25f,
                                 (a.w + bb.w + cc.w + d.w) * 0.25f);
    reinterpret_cast<uint2*>(y)[idx] = t2i_pack4h(m);
  }
}
int avg_pool2_f16_launch(cudaStream_t st, const float* x, int n, int H, int W, int C, __half* y) {
  if ((C % 4) || (H % 2) || (W % 2) || n < 1 || H < 2 || W < 2) return 2103;
  int grid = cdiv((long)n * (H / 2) * (W / 2) * (C / 4), 256);
  if (grid > 132 * 16) grid = 132 * 16;
  avg_pool2_f16_kernel<<<grid, 256, 0, st>>>(x, n, H, W, C, y);
  return (int)cudaGetLastError();
}

// x[b] += F[b % n_hint] over f32 NHWC images of per_img floats, unless *t < *t_min (the adapter's timestep window). A plan op:
// PDL contract of kernels.h, so nothing is read before griddep_wait().
__global__ void t2i_add_kernel(float* __restrict__ x, const float* __restrict__ F, long per_img4, int B, int n_hint,
                               const int* __restrict__ t, const int* __restrict__ t_min) {
  griddep_wait();
  griddep_launch_dependents();
  if (*t < *t_min) return;
  float4* x4 = reinterpret_cast<float4*>(x);
  const float4* F4 = reinterpret_cast<const float4*>(F);
  const long total = (long)B * per_img4;
  for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
    const long b = idx / per_img4;
    const float4 f = F4[(b % n_hint) * per_img4 + (idx - b * per_img4)];
    float4 v = x4[idx];
    v.x += f.x; v.y += f.y; v.z += f.z; v.w += f.w;
    x4[idx] = v;
  }
}
int t2i_add_launch(cudaStream_t st, float* x, const float* F, long per_img, int B, int n_hint, const int* t, const int* t_min) {
  if ((per_img % 4) || B < 1 || n_hint < 1 || (B % n_hint)) return 2104;
  int grid = cdiv((long)B * (per_img / 4), 256);
  if (grid > 132 * 8) grid = 132 * 8;
  if (grid < 1) grid = 1;
  return launch_kernel(t2i_add_kernel, dim3(grid), dim3(256), (size_t)0, st, true, x, F, per_img / 4, B, n_hint, t, t_min);
}

}  // namespace sdxl
