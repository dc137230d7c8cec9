// GroupNorm(+SiLU) and LayerNorm for the UNet step. HBM-bound: each input element is read twice
// (stats, apply) / once (LayerNorm, row held in registers) with 128-bit loads; reductions use
// warp shuffles + a small deterministic partial-sum table (no atomics).
//   reference: groupnorm/mod.rs:52-82 (reshape to [B,32,C/32*HW], biased variance, eps inside sqrt,
//   per-channel affine), layernorm/mod.rs:34-49, silu.rs:14-16.
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace sdxl {

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }
static constexpr int kGnMaxChunk = 512;

// scratch layout: [B + 16, padded to 4] arrival counters (zero between uses) | [B][kGnMaxChunk][G][2] chunk partials |
// [B][G][2] final (mean, rstd). The counters come first so that a scratch initialised for (B, G) serves every GroupNorm with
// B' <= B and G' <= G: they sit at the same place whatever the shape, and only they must be zero on entry.
static inline size_t gn_counter_floats(int B) { return ((size_t)B + 16 + 3) & ~(size_t)3; }
size_t gn_scratch_floats(int B, int n_group) { return gn_counter_floats(B) + (size_t)B * kGnMaxChunk * n_group * 2 + (size_t)B * n_group * 2; }
static inline float* gn_partials(float* scratch, int B) { return scratch + gn_counter_floats(B); }
static inline float* gn_final(float* scratch, int B, int n_group) { return gn_partials(scratch, B) + (size_t)B * kGnMaxChunk * n_group * 2; }
static inline unsigned* gn_counters(float* scratch) { return reinterpret_cast<unsigned*>(scratch); }
int gn_scratch_init(cudaStream_t st, float* scratch, int B, int n_group) {
  (void)n_group;
  return (int)cudaMemsetAsync(gn_counters(scratch), 0, gn_counter_floats(B) * sizeof(unsigned), st);
}

// Pivot of a (sample, group): the mean of four of its elements (first / middle channel at the first / middle pixel). Sums are
// taken of (x - pivot), so that var = E[(x-K)^2] - E[x-K]^2 has no cancellation when |mean| >> sigma (the reference centres
// first, groupnorm/mod.rs:75-82; real activations have groups with |mean| / sigma in the hundreds). Same value in every CTA.
__device__ __forceinline__ float gn_pivot(const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2, int b, int HW,
                                          int c0, int cpg) {
  float k = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int c = c0 + i * (cpg >> 1);
    const float* src = c < C1 ? x1 + (size_t)b * HW * C1 + c : x2 + (size_t)b * HW * C2 + (c - C1);
    const int Cs = c < C1 ? C1 : C2;
    k += __ldg(src) + __ldg(src + (size_t)(HW >> 1) * Cs);
  }
  return 0.25f * k;
}

// ---- stats: grid (nchunk, B); block = V*R threads, V = C/4 float4 columns, R pixel rows in flight.
// The last CTA of a sample to finish (arrival counter; control only, the arithmetic order is fixed) turns the chunk partials
// into the sample's (mean, rstd) per group, so the apply kernel does not repeat that in every CTA.
__global__ void gn_stats_kernel(const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2, int HW,
                                int n_group, int R, float eps, float* __restrict__ partial, float* __restrict__ final_stats,
                                unsigned* __restrict__ counters) {
  extern __shared__ float sm[];  // [R][C][2]
  __shared__ unsigned s_ticket;
  griddep_wait();
  griddep_launch_dependents();
  const int C = C1 + C2;
  const int V = C >> 2;
  const int v = threadIdx.x % V, rr = threadIdx.x / V;
  const int b = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int per = (HW + nchunk - 1) / nchunk;
  const int p0 = chunk * per;
  const int p1 = min(HW, p0 + per);
  const int c = v * 4;
  const float* src;
  int cc, Cs;
  if (c < C1) { src = x1; cc = c; Cs = C1; } else { src = x2; cc = c - C1; Cs = C2; }
  src += (size_t)b * HW * Cs + cc;
  const int cpg = C / n_group;
  // per-channel pivot = pivot of the channel's group (a float4 may straddle two groups)
  float4 K;
  {
    const int g0 = c / cpg, g3 = (c + 3) / cpg;
    const float k0 = gn_pivot(x1, C1, x2, C2, b, HW, g0 * cpg, cpg);
    const float k3 = g3 == g0 ? k0 : gn_pivot(x1, C1, x2, C2, b, HW, g3 * cpg, cpg);
    K.x = k0;
    K.y = (c + 1) / cpg == g0 ? k0 : k3;
    K.z = (c + 2) / cpg == g0 ? k0 : k3;
    K.w = k3;
  }
  float4 s = make_float4(0, 0, 0, 0), q = make_float4(0, 0, 0, 0);
  int p = p0 + rr;
  for (; p + 7 * R < p1; p += 8 * R) {  // eight independent 128-bit loads in flight per thread
    float4 a[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) a[u] = *reinterpret_cast<const float4*>(src + (size_t)(p + u * R) * Cs);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float dx = a[u].x - K.x, dy = a[u].y - K.y, dz = a[u].z - K.z, dw = a[u].w - K.w;
      s.x += dx; s.y += dy; s.z += dz; s.w += dw;
      q.x = fmaf(dx, dx, q.x); q.y = fmaf(dy, dy, q.y);
      q.z = fmaf(dz, dz, q.z); q.w = fmaf(dw, dw, q.w);
    }
  }
  for (; p < p1; p += R) {
    const float4 a = *reinterpret_cast<const float4*>(src + (size_t)p * Cs);
    const float dx = a.x - K.x, dy = a.y - K.y, dz = a.z - K.z, dw = a.w - K.w;
    s.x += dx; s.y += dy; s.z += dz; s.w += dw;
    q.x = fmaf(dx, dx, q.x); q.y = fmaf(dy, dy, q.y); q.z = fmaf(dz, dz, q.z); q.w = fmaf(dw, dw, q.w);
  }
  float* row = sm + ((size_t)rr * C + c) * 2;
  row[0] = s.x; row[1] = q.x; row[2] = s.y; row[3] = q.y; row[4] = s.z; row[5] = q.z; row[6] = s.w; row[7] = q.w;
  __syncthreads();
  if (threadIdx.x < n_group) {
    const int g = threadIdx.x;
    float S = 0.f, Q = 0.f;
    for (int r = 0; r < R; ++r)
      for (int j = 0; j < cpg; ++j) {
        const float* e = sm + ((size_t)r * C + g * cpg + j) * 2;
        S += e[0];
        Q += e[1];
      }
    float* o = partial + (((size_t)b * nchunk + chunk) * n_group + g) * 2;
    o[0] = S;
    o[1] = Q;
    __threadfence();  // this CTA's partials are visible device-wide before it takes its ticket
  }
  __syncthreads();
  if (threadIdx.x == 0) s_ticket = atomicAdd(&counters[b], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(nchunk - 1)) return;
  // last CTA of sample b: 8 lanes per group walk the chunk partials in chunk order (deterministic), in double precision.
  // Only whole warps take part (blockDim.x >= 32 but not always a multiple of it) and n_group % 4 == 0 (gn_launch), so every
  // warp either reduces four complete groups or skips the loop: the full-mask shuffles below always see all 32 lanes.
  __threadfence();
  const int nred = blockDim.x & ~31;
  for (int g = threadIdx.x >> 3; threadIdx.x < nred && g < n_group; g += nred >> 3) {
    const int sub = threadIdx.x & 7;
    double S = 0.0, Q = 0.0;
    for (int k0 = sub; k0 < nchunk; k0 += 64) {   // eight independent loads in flight, summed in chunk order
      float2 e[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = k0 + 8 * j;
        e[j] = k < nchunk ? __ldcg(reinterpret_cast<const float2*>(partial + (((size_t)b * nchunk + k) * n_group + g) * 2))
                          : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { S += (double)e[j].x; Q += (double)e[j].y; }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      S += __shfl_xor_sync(0xffffffffu, S, o);
      Q += __shfl_xor_sync(0xffffffffu, Q, o);
    }
    if (sub == 0) {
      const double n = (double)cpg * HW;
      const double m = S / n;               // mean of (x - pivot): O(sigma), so the subtraction below does not cancel
      double var = Q / n - m * m;
      if (var < 0.0) var = 0.0;
      final_stats[((size_t)b * n_group + g) * 2] = (float)((double)gn_pivot(x1, C1, x2, C2, b, HW, g * cpg, cpg) + m);
      final_stats[((size_t)b * n_group + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
  }
  if (threadIdx.x == 0) counters[b] = 0u;  // ready for the next GroupNorm that uses this scratch
}

// ---- apply: grid (ctas, B); block = V8*R threads: a thread owns 8 fixed channels (scale/shift in registers) and walks
// pixel rows, no index divisions in the loop
__global__ void gn_apply_kernel(const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2, int HW,
                                int n_group, const float* __restrict__ gamma, const float* __restrict__ beta, int silu,
                                const float* __restrict__ final_stats, int R, __half* __restrict__ y, __half* __restrict__ raw,
                                __half* __restrict__ y_lo) {
  griddep_wait();
  griddep_launch_dependents();
  const int C = C1 + C2;
  const int V8 = C >> 3;
  const int v = threadIdx.x % V8, rr = threadIdx.x / V8;
  if (rr >= R) return;
  const int b = blockIdx.y;
  const int cpg = C / n_group;
  const int c = v * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (c + i) / cpg;
    const float mean = final_stats[((size_t)b * n_group + g) * 2], rstd = final_stats[((size_t)b * n_group + g) * 2 + 1];
    sc[i] = rstd * gamma[c + i];
    sh[i] = fmaf(-mean, sc[i], beta[c + i]);   // y = x * sc + sh: the cancellation costs |mean| / sigma * 2^-24 absolute, far below f16
  }
  const float* src;
  int cc, Cs;
  if (c < C1) { src = x1; cc = c; Cs = C1; } else { src = x2; cc = c - C1; Cs = C2; }
  src += (size_t)b * HW * Cs + cc;
  __half* yo = y + (size_t)b * HW * C + c;
  __half* ro = raw ? raw + (size_t)b * HW * C + c : nullptr;
  __half* lo = y_lo ? y_lo + (size_t)b * HW * C + c : nullptr;
  const int step = gridDim.x * R;
  auto emit = [&](int p, const float4& a0, const float4& a1) {
    float f[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    uint32_t h[4];
    if (ro) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        __half2 t = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        h[i] = *reinterpret_cast<uint32_t*>(&t);
      }
      *reinterpret_cast<uint4*>(ro + (size_t)p * C) = make_uint4(h[0], h[1], h[2], h[3]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float t = fmaf(f[i], sc[i], sh[i]);
      if (silu) t = silu_f(t);
      f[i] = t;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 t = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      h[i] = *reinterpret_cast<uint32_t*>(&t);
      if (lo) {   // what the f16 rounding dropped (exact in f32), itself rounded to f16: y + y_lo carries ~22 bits of t
        const float2 back = __half22float2(t);
        f[2 * i] -= back.x;
        f[2 * i + 1] -= back.y;
      }
    }
    *reinterpret_cast<uint4*>(yo + (size_t)p * C) = make_uint4(h[0], h[1], h[2], h[3]);
    if (lo) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        __half2 t = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        h[i] = *reinterpret_cast<uint32_t*>(&t);
      }
      *reinterpret_cast<uint4*>(lo + (size_t)p * C) = make_uint4(h[0], h[1], h[2], h[3]);
    }
  };
  int p = blockIdx.x * R + rr;
  for (; p + 3 * step < HW; p += 4 * step) {  // four rows (eight 16-byte loads) in flight per thread
    float4 a[4][2];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float* s = src + (size_t)(p + u * step) * Cs;
      a[u][0] = *reinterpret_cast<const float4*>(s);
      a[u][1] = *reinterpret_cast<const float4*>(s + 4);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) emit(p + u * step, a[u][0], a[u][1]);
  }
  for (; p < HW; p += step) {
    const float* s = src + (size_t)p * Cs;
    emit(p, *reinterpret_cast<const float4*>(s), *reinterpret_cast<const float4*>(s + 4));
  }
}

int gn_launch(cudaStream_t st, GnParams& p) {
  const int C = p.C1 + p.C2;
  // n_group % 4 == 0: the stats kernel's final reduction gives each group 8 lanes of a full-mask warp shuffle
  if ((p.C1 & 7) || (p.C2 & 7) || p.n_group < 4 || (p.n_group & 3) || p.n_group > 64 || C % p.n_group) return 3001;
  const int V = C / 4;
  if (V > 1024) return 3002;
  int R = 512 / V;
  if (R < 1) R = 1;
  if (R > 16) R = 16;
  // chunking depends on HW only (never on the batch size): every sample's statistics are summed in the
  // same order whatever B is, which keeps the whole forward batch-invariant bit for bit.
  int nchunk = 132;   // one CTA per SM of an H100 SXM
  const int max_chunks = cdiv(p.HW, R);
  if (nchunk > max_chunks) nchunk = max_chunks;
  p.nchunk = nchunk;
  const size_t smem1 = (size_t)R * C * 2 * sizeof(float);
  static bool optin[64];
  if (int r = smem_optin(gn_stats_kernel, 160 * 1024, optin)) return r;
  float* fin = gn_final(p.partial, p.B, p.n_group);
  unsigned* cnt = gn_counters(p.partial);
  int e = launch_kernel(gn_stats_kernel, dim3(nchunk, p.B), dim3(V * R), smem1, st, true, p.x1, p.C1, p.x2, p.C2, p.HW,
                        p.n_group, R, p.eps, gn_partials(p.partial, p.B), fin, cnt);
  if (e) return e;
  const int V8 = C / 8;
  int R2 = 256 / V8;
  if (R2 < 1) R2 = 1;
  if (R2 > 32) R2 = 32;
  int ctas = cdiv(p.HW, R2 * 4);
  const int cap = (132 * 8) / (p.B > 0 ? p.B : 1);
  if (ctas > cap) ctas = cap;
  if (ctas < 1) ctas = 1;
  return launch_kernel(gn_apply_kernel, dim3(ctas, p.B), dim3(V8 * R2), (size_t)0, st, true, p.x1, p.C1, p.x2, p.C2, p.HW,
                       p.n_group, p.gamma, p.beta, p.silu, (const float*)fin, R2, p.y, p.raw, p.y_lo);
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row cached in registers (NV float4 per lane), exact two-pass
// (mean, then centred second moment) as the reference's layernorm() does.
// ------------------------------------------------------------------------------------------------
template <int NV>
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float eps, int rows, int C,
                                 __half* __restrict__ y) {
  griddep_wait();
  griddep_launch_dependents();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (size_t)row * C;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
      v[i] = *reinterpret_cast<const float4*>(xr + c);
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    } else {
      v[i] = make_float4(0, 0, 0, 0);
    }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      q += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + c));
      const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + c));
      __half2 a = __floats2half2_rn(v[i].x * rstd * g.x + bt.x, v[i].y * rstd * g.y + bt.y);
      __half2 b = __floats2half2_rn(v[i].z * rstd * g.z + bt.z, v[i].w * rstd * g.w + bt.w);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&a);
      o.y = *reinterpret_cast<uint32_t*>(&b);
      *reinterpret_cast<uint2*>(y + (size_t)row * C + c) = o;
    }
  }
}

int layernorm_launch(cudaStream_t st, const float* x, const float* gamma, const float* beta, float eps, int rows,
                     int C, __half* y) {
  if (C & 3) return 3003;
  const int nv = cdiv(C, 128);
  static const int warps_env = getenv("SDXL_B200_LN_WARPS") ? atoi(getenv("SDXL_B200_LN_WARPS")) : 0;
  const int warps = (warps_env >= 1 && warps_env <= 32) ? warps_env : 8;
  dim3 grid(cdiv(rows, warps));
  if (nv <= 1) return launch_kernel(layernorm_kernel<1>, grid, dim3(warps * 32), (size_t)0, st, true, x, gamma, beta, eps, rows, C, y);
  else if (nv <= 2) return launch_kernel(layernorm_kernel<2>, grid, dim3(warps * 32), (size_t)0, st, true, x, gamma, beta, eps, rows, C, y);
  else if (nv <= 5) return launch_kernel(layernorm_kernel<5>, grid, dim3(warps * 32), (size_t)0, st, true, x, gamma, beta, eps, rows, C, y);
  else if (nv <= 10) return launch_kernel(layernorm_kernel<10>, grid, dim3(warps * 32), (size_t)0, st, true, x, gamma, beta, eps, rows, C, y);
  else if (nv <= 16) return launch_kernel(layernorm_kernel<16>, grid, dim3(warps * 32), (size_t)0, st, true, x, gamma, beta, eps, rows, C, y);
  return 3004;
}

}  // namespace sdxl
