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

// Running statistics of one channel column of a thread: the count n (shared by the four channels of a float4), and per channel
// a centre K, the offset r of the running mean from K, and m2, the sum of squared deviations from the running mean K + r.
// merge() adds k <= N rows: it centres them on their own mean (two-pass, in registers), adds them by Chan's pairwise update and
// then moves K to the new mean, keeping in r what the move rounded away (exactly, by Fast2Sum, when |r| <= |K|; otherwise, for a
// mean near zero or a first row far from the rest, within one f32 rounding of the move). So the sums add deviations from the
// running mean, never |mean| itself, and no statistic depends on which row a thread happens to read first.
struct GnRun {
  float n = 0.f;
  float4 K, r = make_float4(0, 0, 0, 0), m2 = make_float4(0, 0, 0, 0);

  // a[0 .. k-1] are the rows (1 <= k <= N); the rest are ignored
  template <int N>
  __device__ __forceinline__ void merge(float4 (&a)[N], int k) {
    const float fk = (float)k, nn = n + fk, kinv = fk * __frcp_rn(nn), w = n * kinv, inv_k = k == N ? 1.f / (float)N : __frcp_rn(fk);
    merge1(a, k, &float4::x, kinv, w, inv_k);
    merge1(a, k, &float4::y, kinv, w, inv_k);
    merge1(a, k, &float4::z, kinv, w, inv_k);
    merge1(a, k, &float4::w, kinv, w, inv_k);
    n = nn;
  }
  // kinv = k / (n + k), w = n k / (n + k): Chan's weights (both 0 / 1 on the first merge, where n = 0)
  template <int N>
  __device__ __forceinline__ void merge1(float4 (&a)[N], int k, float float4::*f, float kinv, float w, float inv_k) {
    float& Kf = K.*f;
    float& rf = r.*f;
    float sb = 0.f;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      a[u].*f = u < k ? a[u].*f - Kf : 0.f;
      sb += a[u].*f;
    }
    const float mb = sb * inv_k;
    float m2b = 0.f;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      const float e = u < k ? a[u].*f - mb : 0.f;
      m2b = fmaf(e, e, m2b);
    }
    const float delta = mb - rf;                     // block mean - running mean
    m2.*f += fmaf(w * delta, delta, m2b);
    rf = fmaf(kinv, delta, rf);                      // new mean - K
    const float Kn = Kf + rf;                        // re-centre on the new mean
    rf -= Kn - Kf;
    Kf = Kn;
  }
  __device__ __forceinline__ float mean(float float4::*f) const { return K.*f + r.*f; }
};

// ---- stats: grid (nchunk, B); block = V*R threads, V = C/4 float4 columns, R pixel rows in flight.
// Each thread keeps a GnRun of its column over the rows p0 + rr, p0 + rr + R, ... of its chunk; the CTA folds its R * cpg
// (count, mean, m2) partials per group in double (sum of count * mean, then the centred second moment around that mean), and the
// last CTA of a sample to finish (arrival counter; control only, the arithmetic order is fixed) merges the chunks' (mean, m2)
// the same way in double and writes the sample's (mean, rstd) per group, so the apply kernel does not repeat that in every CTA.
// No statistic depends on which element a thread happens to read first (the reference centres first, groupnorm/mod.rs:75-82;
// real activations have groups with |mean| / sigma in the hundreds, and outliers anywhere).
// kMaxThreads / kMinBlocks / kRows: the UNet's GroupNorms (blocks of <= 512 threads, HW < 64k) are compiled for two CTAs per SM,
// so a B = 2 grid of 2 x 132 CTAs runs in one wave; at the 64 registers that allows, a thread keeps 6 rows in flight (8 spill).
// The rest run one CTA per SM with 8 rows in flight (gn_launch).
template <int kMaxThreads, int kMinBlocks, int kRows>
__global__ void __launch_bounds__(kMaxThreads, kMinBlocks)
gn_stats_kernel(const float* __restrict__ x1, int C1, const float* __restrict__ x2, int C2, int HW, int n_group, int R, float eps,
                float* __restrict__ partial, float* __restrict__ final_stats, unsigned* __restrict__ counters) {
  extern __shared__ float sm[];  // [R][C][2]: (mean, m2) of each thread's column
  __shared__ unsigned s_ticket;
  griddep_wait();
  griddep_launch_dependents();
  const int C = C1 + C2;
  const int V = C >> 2;
  const int v = threadIdx.x % V, rr = threadIdx.x / V;
  const int b = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int per = (HW + nchunk - 1) / nchunk;
  const int p0 = chunk * per;
  const int p1 = min(HW, p0 + per);   // p1 <= p0: an empty chunk (nchunk * per may exceed HW by up to per - 1)
  const int c = v * 4;
  const float* src;
  int cc, Cs;
  if (c < C1) { src = x1; cc = c; Cs = C1; } else { src = x2; cc = c - C1; Cs = C2; }
  src += (size_t)b * HW * Cs + cc;
  const int cpg = C / n_group;
  GnRun run;
  int p = p0 + rr;
  run.K = p < p1 ? *reinterpret_cast<const float4*>(src + (size_t)p * Cs) : make_float4(0, 0, 0, 0);   // any start will do
  for (; p < p1; p += kRows * R) {  // kRows independent 128-bit loads in flight per thread; the last block may be partial
    const int k = min(kRows, (p1 - p + R - 1) / R);
    float4 a[kRows];
#pragma unroll
    for (int u = 0; u < kRows; ++u) a[u] = u < k ? *reinterpret_cast<const float4*>(src + (size_t)(p + u * R) * Cs) : make_float4(0, 0, 0, 0);
    run.merge(a, k);
  }
  float* row = sm + ((size_t)rr * C + c) * 2;
  row[0] = run.mean(&float4::x); row[1] = run.m2.x; row[2] = run.mean(&float4::y); row[3] = run.m2.y;
  row[4] = run.mean(&float4::z); row[5] = run.m2.z; row[6] = run.mean(&float4::w); row[7] = run.m2.w;
  __syncthreads();
  if (threadIdx.x < n_group) {
    const int g = threadIdx.x;
    const int np = p1 - p0;   // rows of this chunk; thread row r holds ceil((np - r) / R) of them
    double S = 0.0;
    for (int r = 0; r < R && r < np; ++r) {
      double Sr = 0.0;
      for (int j = 0; j < cpg; ++j) Sr += (double)sm[((size_t)r * C + g * cpg + j) * 2];
      S += (double)((np - r + R - 1) / R) * Sr;
    }
    const double n = (double)cpg * (double)max(np, 0);
    const double m = n > 0.0 ? S / n : 0.0;
    double M2 = 0.0;
    for (int r = 0; r < R && r < np; ++r) {
      const double cnt = (double)((np - r + R - 1) / R);
      for (int j = 0; j < cpg; ++j) {
        const float* e = sm + ((size_t)r * C + g * cpg + j) * 2;
        const double d = (double)e[0] - m;
        M2 += fma(cnt * d, d, (double)e[1]);
      }
    }
    float* o = partial + (((size_t)b * nchunk + chunk) * n_group + g) * 2;
    o[0] = (float)m;
    o[1] = (float)M2;
    __threadfence();  // this CTA's partials are visible device-wide before it takes its ticket
  }
  __syncthreads();
  if (threadIdx.x == 0) s_ticket = atomicAdd(&counters[b], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(nchunk - 1)) return;
  // last CTA of sample b: 8 lanes per group walk the chunk partials in chunk order (deterministic), in double precision: the
  // count-weighted sum of the chunk means, then the chunks' m2 plus count * (chunk mean - mean)^2.
  // Only whole warps take part (blockDim.x >= 32 but not always a multiple of it) and n_group % 4 == 0 (gn_launch), so every
  // warp either reduces four complete groups or skips the loop: the full-mask shuffles below always see all 32 lanes.
  __threadfence();
  const int nred = blockDim.x & ~31;
  for (int g = threadIdx.x >> 3; threadIdx.x < nred && g < n_group; g += nred >> 3) {
    const int sub = threadIdx.x & 7;
    auto load = [&](int k) {   // chunk k's (mean, m2); (0, 0) past the last chunk
      return k < nchunk ? __ldcg(reinterpret_cast<const float2*>(partial + (((size_t)b * nchunk + k) * n_group + g) * 2))
                        : make_float2(0.f, 0.f);
    };
    auto count = [&](int k) { return (double)cpg * (double)max(min(HW - k * per, per), 0); };   // 0 for an empty chunk
    double S = 0.0;
    for (int k0 = sub; k0 < nchunk; k0 += 64) {   // eight independent loads in flight, summed in chunk order
      float2 e[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) e[j] = load(k0 + 8 * j);
#pragma unroll
      for (int j = 0; j < 8; ++j) S = fma(count(k0 + 8 * j), (double)e[j].x, S);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) S += __shfl_xor_sync(0xffffffffu, S, o);
    const double n = (double)cpg * HW;
    const double m = S / n;
    double M2 = 0.0;
    for (int k0 = sub; k0 < nchunk; k0 += 64) {
      float2 e[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) e[j] = load(k0 + 8 * j);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const double d = (double)e[j].x - m;
        M2 += fma(count(k0 + 8 * j) * d, d, (double)e[j].y);
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) M2 += __shfl_xor_sync(0xffffffffu, M2, o);
    if (sub == 0) {
      final_stats[((size_t)b * n_group + g) * 2] = (float)m;
      final_stats[((size_t)b * n_group + g) * 2 + 1] = (float)(1.0 / sqrt(M2 / n + (double)eps));
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
  if (V > 768) return 3002;   // gn_stats_kernel's launch bound (C <= 3072: the refiner's widest concatenation)
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
  static bool optin_narrow[64], optin_wide[64];
  // two CTAs per SM (6 rows in flight) where the grid is short, one with 8 rows in flight where each CTA streams many rows
  // (HW >= 64k: the VAE's larger GroupNorms, HBM-bound) or the block is wider than 512 threads. Chosen by shape only, never by
  // B, so the summation order stays batch-invariant.
  const bool narrow = V * R <= 512 && p.HW < 65536;
  auto kernel = narrow ? gn_stats_kernel<512, 2, 6> : gn_stats_kernel<768, 1, 8>;
  if (int r = smem_optin(kernel, 160 * 1024, narrow ? optin_narrow : optin_wide)) return r;
  float* fin = gn_final(p.partial, p.B, p.n_group);
  unsigned* cnt = gn_counters(p.partial);
  int e = launch_kernel(kernel, dim3(nchunk, p.B), dim3(V * R), smem1, st, true, p.x1, p.C1, p.x2, p.C2, p.HW,
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
