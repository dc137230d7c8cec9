// Fused multi-head attention for the UNet's SpatialTransformer blocks (head dim 64, no mask):
//   out = softmax(q k^T / sqrt(64)) v            (reference src/backend.rs:4-19,32-79,88-128;
//                                                 called from unet/mod.rs:1013-1019)
// Flash-style on Hopper tensor cores (wgmma); scores, probabilities and the output accumulator live in registers:
//   S = Q K^T : wgmma m64n128k16, A = Q tile (K-major, TMA SW128 smem), B = K tile (K-major smem)     -> registers (f32)
//   P         : online softmax on the S registers, packed to f16 in place as the A fragments of the next wgmma
//   O += P V  : wgmma m64n64k16, A = P from registers, B = V tile (MN-major smem: keys are the contraction) -> registers (f32)
// One CTA per (batch, head, 128-query tile): two consumer warpgroups own 64 query rows each, one producer warp streams the
// 128-key K / V blocks through a TMA ring. The running max is exact per key block (the row is rescaled when it grows), so
// every probability is <= 1 before the f16 rounding.
// attention_kernel<true> adds IP-Adapter's image key/value sources (DESIGN.md §9, §13).
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace sdxl {

static constexpr int kTileBytes = 128 * 128;        // 128 rows x 64 halves (Q, K or V tile)
static constexpr int kKvStages = 3;
static constexpr int kConsumerWarps = 8;
static constexpr int kAttnThreads = kConsumerWarps * 32 + 32;
static constexpr int kAttnSmem = 1024 /*align slack*/ + kTileBytes + 2 * kKvStages * kTileBytes + 256;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 t = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// One 128-key block j (key rows kb * 128 .. of a source with S keys, ring stage st) of a consumer warpgroup: S = Q K^T, online
// softmax update of (m, l, o), O += P V, release of the stage.
__device__ __forceinline__ void attn_key_block(float (&o)[32], float (&m)[2], float (&l)[2], uint32_t q_addr, const uint8_t* sK,
                                               const uint8_t* sV, uint64_t* kv_full, uint64_t* kv_empty, int j, int kb, int S,
                                               float sl2e, int lane) {
  const int st = j % kKvStages;
  mbar_wait_nocall(&kv_full[st], (j / kKvStages) & 1);
  float s[64];
  wg_fence();
  const uint32_t k_addr = smem_u32(sK + st * kTileBytes);
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_ss_n128(s, wg_desc_sw128(q_addr + 32 * k), wg_desc_sw128(k_addr + 32 * k), k);
  wg_commit();
  wg_wait<0>();
  if (kb * 128 + 128 > S) {   // ragged last key block: keys past S do not exist
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (kb * 128 + 8 * jj + 2 * (lane & 3) + e >= S) { s[4 * jj + e] = -INFINITY; s[4 * jj + 2 + e] = -INFINITY; }
  }
  uint32_t pa[32];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m[h], mx);
    const float alpha = ex2_approx((m[h] - m_new) * sl2e);
    const float mb = m_new * sl2e;
    float sum = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const float p0 = ex2_approx(fmaf(s[4 * jj + 2 * h], sl2e, -mb));
      const float p1 = ex2_approx(fmaf(s[4 * jj + 2 * h + 1], sl2e, -mb));
      sum += p0 + p1;
      // A fragment of key chunk kk = jj / 2: {row r: keys 0-7, row r+8: keys 0-7, row r: keys 8-15, row r+8: keys 8-15}
      pa[4 * (jj >> 1) + 2 * (jj & 1) + h] = pack_half2(p0, p1);
    }
    l[h] = l[h] * alpha + sum;
    m[h] = m_new;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) { o[4 * jj + 2 * h] *= alpha; o[4 * jj + 2 * h + 1] *= alpha; }
  }
  wg_fence();
  const uint32_t v_addr = smem_u32(sV + st * kTileBytes);
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
    wgmma_rs_n64_tb(o, *reinterpret_cast<const uint32_t(*)[4]>(pa + 4 * kk), wg_desc_sw128(v_addr + 2048 * kk));
  wg_commit();
  wg_wait<0>();
  if (lane == 0) mbar_arrive(&kv_empty[st]);   // this warp is done with K_j / V_j
}

// Image source k of p (source 0 is the AttnParams fields that predate the others; K and V may have separate maps there).
struct IpSrc {
  const CUtensorMap* tk;
  const CUtensorMap* tv;
  int S, k_col0, v_col0;
  const float* scale;
  const float* mask;
};
__device__ __forceinline__ IpSrc ip_source(const AttnParams& p, int k) {
  if (k == 0) return {&p.tmKip, &p.tmVip, p.S_ip, p.k_ip_col0, p.v_ip_col0, p.ip_scale, p.ip_mask};
  const AttnIpSource& s = p.ip_src[k - 1];
  return {&s.tm, &s.tm, s.S, s.k_col0, s.v_col0, s.scale, s.mask};
}

// kIp: decoupled cross-attention (IP-Adapter, DESIGN.md §9, §13). After the text keys the producer streams the keys of each of the
// n_src image sources in turn through the same ring; the consumers keep acc = O_txt / l_txt, restart the online softmax on each
// source's keys and add acc = fmaf(s * m[t], O_k / l_k, acc), s = *scale and m = mask[t] (1 without a mask) read from device
// memory, so rewriting them keeps the CUDA graph valid. One unmasked source is the two-source form: f16(O_txt / l_txt + s O / l).
template <bool kIp>
__global__ void __launch_bounds__(kAttnThreads, 1) attention_kernel(const __grid_constant__ AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kTileBytes;                       // [kKvStages]
  uint8_t* sV = sK + kKvStages * kTileBytes;           // [kKvStages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kKvStages * kTileBytes);
  uint64_t* q_full = bars;
  uint64_t* kv_full = q_full + 1;                      // [kKvStages]
  uint64_t* kv_empty = kv_full + kKvStages;            // [kKvStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nblk = (p.S + 127) / 128;
  const int nqt = (p.T + 127) / 128;
  const int qt = blockIdx.x % nqt, head = (blockIdx.x / nqt) % p.n_head, b = blockIdx.x / (nqt * p.n_head);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK);
    tma_prefetch_desc(&p.tmV);
    if constexpr (kIp) {
      tma_prefetch_desc(&p.tmKip);
      tma_prefetch_desc(&p.tmVip);
      for (int k = 1; k < p.n_src; ++k) tma_prefetch_desc(&p.ip_src[k - 1].tm);
    }
    mbar_init(q_full, 1);
    for (int i = 0; i < kKvStages; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();  // PDL: the prologue above overlapped the previous kernel's tail
  griddep_launch_dependents();

  if (warp == kConsumerWarps) {
    // ===================== TMA producer =====================
    if (lane != 0) return;
    mbar_expect_tx(q_full, kTileBytes);
    tma_load_3d(sQ, &p.tmQ, q_full, p.q_col0 + head * 64, qt * 128, b);
    for (int j = 0; j < nblk; ++j) {
      const int st = j % kKvStages;
      mbar_wait_nocall(&kv_empty[st], ((j / kKvStages) & 1) ^ 1);
      mbar_expect_tx(&kv_full[st], 2 * kTileBytes);
      tma_load_3d(sK + st * kTileBytes, &p.tmK, &kv_full[st], p.k_col0 + head * 64, j * 128, b);
      tma_load_3d(sV + st * kTileBytes, &p.tmV, &kv_full[st], p.v_col0 + head * 64, j * 128, b);
    }
    if constexpr (kIp) {
      int j = nblk;
      for (int k = 0; k < p.n_src; ++k) {
        const IpSrc s = ip_source(p, k);
        const int nb = (s.S + 127) / 128;
        for (int kb = 0; kb < nb; ++kb, ++j) {
          const int st = j % kKvStages;
          mbar_wait_nocall(&kv_empty[st], ((j / kKvStages) & 1) ^ 1);
          mbar_expect_tx(&kv_full[st], 2 * kTileBytes);
          tma_load_3d(sK + st * kTileBytes, s.tk, &kv_full[st], s.k_col0 + head * 64, kb * 128, b);
          tma_load_3d(sV + st * kTileBytes, s.tv, &kv_full[st], s.v_col0 + head * 64, kb * 128, b);
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile =====================
  // Accumulator layout (m64nN): thread holds rows r and r + 8 (h = 0, 1), columns 8 j + 2 (lane & 3) + e at index 4 j + 2 h + e.
  const int wg = warp >> 2;
  const float sl2e = p.scale_log2e;
  const uint32_t q_addr = smem_u32(sQ) + (uint32_t)wg * (64 * 128);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  mbar_wait_nocall(q_full, 0);
  // The text loop is attn_key_block written out: routed through the helper, ptxas allocates registers differently and the
  // kernel without an image prompt would no longer compile to the code it had before the second source existed.
  for (int j = 0; j < nblk; ++j) {
    const int st = j % kKvStages;
    mbar_wait_nocall(&kv_full[st], (j / kKvStages) & 1);
    float s[64];
    wg_fence();
    const uint32_t k_addr = smem_u32(sK + st * kTileBytes);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss_n128(s, wg_desc_sw128(q_addr + 32 * k), wg_desc_sw128(k_addr + 32 * k), k);
    wg_commit();
    wg_wait<0>();
    if (j * 128 + 128 > p.S) {   // ragged last key block: keys past S do not exist
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (j * 128 + 8 * jj + 2 * (lane & 3) + e >= p.S) { s[4 * jj + e] = -INFINITY; s[4 * jj + 2 + e] = -INFINITY; }
    }
    uint32_t pa[32];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx);
      const float alpha = ex2_approx((m[h] - m_new) * sl2e);
      const float mb = m_new * sl2e;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const float p0 = ex2_approx(fmaf(s[4 * jj + 2 * h], sl2e, -mb));
        const float p1 = ex2_approx(fmaf(s[4 * jj + 2 * h + 1], sl2e, -mb));
        sum += p0 + p1;
        // A fragment of key chunk kk = jj / 2: {row r: keys 0-7, row r+8: keys 0-7, row r: keys 8-15, row r+8: keys 8-15}
        pa[4 * (jj >> 1) + 2 * (jj & 1) + h] = pack_half2(p0, p1);
      }
      l[h] = l[h] * alpha + sum;
      m[h] = m_new;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) { o[4 * jj + 2 * h] *= alpha; o[4 * jj + 2 * h + 1] *= alpha; }
    }
    wg_fence();
    const uint32_t v_addr = smem_u32(sV + st * kTileBytes);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wgmma_rs_n64_tb(o, *reinterpret_cast<const uint32_t(*)[4]>(pa + 4 * kk), wg_desc_sw128(v_addr + 2048 * kk));
    wg_commit();
    wg_wait<0>();
    if (lane == 0) mbar_arrive(&kv_empty[st]);   // this warp is done with K_j / V_j
  }
  const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  if constexpr (kIp) {
    float acc[32];   // O_txt / l_txt, then + s_k m_k[t] O_k / l_k per source
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv = 1.0f / lt;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        acc[4 * jj + 2 * h] = o[4 * jj + 2 * h] * inv;
        acc[4 * jj + 2 * h + 1] = o[4 * jj + 2 * h + 1] * inv;
      }
    }
    int j = nblk;
    for (int k = 0; k < p.n_src; ++k) {
#pragma unroll
      for (int h = 0; h < 2; ++h) { m[h] = -INFINITY; l[h] = 0.f; }
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.f;
      const int S = ip_source(p, k).S;
      for (int kb = 0; kb * 128 < S; ++kb, ++j) attn_key_block(o, m, l, q_addr, sK, sV, kv_full, kv_empty, j, kb, S, sl2e, lane);
      const IpSrc s = ip_source(p, k);   // read after the key blocks: nothing but S stays live across them
      const float sk = *s.scale;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float lt = l[h];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const float inv = 1.0f / lt;
        const int t = qt * 128 + r + 8 * h;
        const float w = (s.mask && t < p.T) ? sk * s.mask[t] : sk;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          acc[4 * jj + 2 * h] = fmaf(w, o[4 * jj + 2 * h] * inv, acc[4 * jj + 2 * h]);
          acc[4 * jj + 2 * h + 1] = fmaf(w, o[4 * jj + 2 * h + 1] * inv, acc[4 * jj + 2 * h + 1]);
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = qt * 128 + r + 8 * h;
      if (t < p.T) {
        __half* out = p.out + ((size_t)b * p.T + t) * p.ldo + head * 64 + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
          *reinterpret_cast<__half2*>(out + 8 * jj) = __floats2half2_rn(acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1]);
      }
    }
  } else {
    // ---- write-back: O / l -> f16
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv = 1.0f / lt;
      const int t = qt * 128 + r + 8 * h;
      if (t < p.T) {
        __half* out = p.out + ((size_t)b * p.T + t) * p.ldo + head * 64 + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
          *reinterpret_cast<__half2*>(out + 8 * jj) = __floats2half2_rn(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
      }
    }
  }
}

// Bicubic resize of one f32 mask plane [H, W] to (mh, mw), written flat into out[T]: zero past mh * mw, cut at T. torch's
// F.interpolate(mode="bicubic", align_corners=False): A = -0.75, source x = (W / mw) (ox + 0.5) - 0.5, taps clamped to the
// plane, no antialias, no clamping of the result.
__device__ __forceinline__ float cubic_w1(float x) { return ((-0.75f + 2.f) * x - (-0.75f + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic_w2(float x) { return ((-0.75f * x - 5.f * -0.75f) * x + 8.f * -0.75f) * x - 4.f * -0.75f; }
__device__ __forceinline__ float cubic_1d(float x0, float x1, float x2, float x3, float t) {
  return x0 * cubic_w2(t + 1.f) + x1 * cubic_w1(t) + x2 * cubic_w1(1.f - t) + x3 * cubic_w2(2.f - t);
}
__global__ void ip_mask_resize_kernel(const float* __restrict__ mask, int H, int W, int mh, int mw, int T, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T) return;
  if (i >= mh * mw) { out[i] = 0.f; return; }
  const int oy = i / mw, ox = i % mw;
  const float ry = (float)H / mh * (oy + 0.5f) - 0.5f, rx = (float)W / mw * (ox + 0.5f) - 0.5f;
  const int iy = (int)floorf(ry), ix = (int)floorf(rx);
  const float ty = ry - iy, tx = rx - ix;
  float row[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float* m = mask + (size_t)min(max(iy - 1 + k, 0), H - 1) * W;
    row[k] = cubic_1d(m[min(max(ix - 1, 0), W - 1)], m[min(max(ix, 0), W - 1)], m[min(max(ix + 1, 0), W - 1)],
                      m[min(max(ix + 2, 0), W - 1)], tx);
  }
  out[i] = cubic_1d(row[0], row[1], row[2], row[3], ty);
}

int ip_mask_resize_launch(cudaStream_t st, const float* mask, int H, int W, int mh, int mw, int T, float* out) {
  if (H < 1 || W < 1 || mh < 1 || mw < 1 || T < 1) return 2002;
  ip_mask_resize_kernel<<<(T + 255) / 256, 256, 0, st>>>(mask, H, W, mh, mw, T, out);
  return (int)cudaGetLastError();
}

// Per-device launch state (several devices may be driven from one process: the opt-in to > 48 KB of dynamic shared memory
// is a per-device function attribute).
static bool g_attn_attr[2][64];
int attention_launch(cudaStream_t st, const AttnParams& p) {
  if (p.T < 1 || p.S < 1 || (p.ldo & 1)) return 2002;
  const bool ip = p.S_ip > 0;
  if (ip && (!p.ip_scale || p.n_src < 1 || p.n_src > ATTN_MAX_SRC)) return 2002;
  for (int k = 1; ip && k < p.n_src; ++k)
    if (p.ip_src[k - 1].S < 1 || !p.ip_src[k - 1].scale) return 2002;
  auto kernel = ip ? attention_kernel<true> : attention_kernel<false>;
  int r = smem_optin(kernel, kAttnSmem, g_attn_attr[ip]);
  if (r) return r;
  const long tiles = (long)p.B * p.n_head * ((p.T + 127) / 128);
  return launch_kernel(kernel, dim3((unsigned)tiles), dim3(kAttnThreads), (size_t)kAttnSmem, st, true, p);
}

}  // namespace sdxl
