// FreeU (Si et al. 2023, diffusers' enable_freeu; DESIGN.md §15): at a decoder skip concatenation cat([x, r]) the first half of x's
// channels is scaled by b and the skip r is filtered by diffusers' fourier_filter with threshold 1,
//   r' = ifft2(mask * fft2(r)).real,   mask = s on the frequencies K = {0, -1 mod H} x {0, -1 mod W} (as a set), 1 elsewhere.
// Only the bins of K change, so with N = H * W, theta_k(h, w) = 2 pi (k_h h / H + k_w w / W) and X_k = sum r(h, w) e^{-i theta_k}:
//   r'(h, w) = r(h, w) + (s - 1) / N * sum_{k in K} Re(X_k e^{i theta_k(h, w)})
// which needs one real and up to three complex sums per (row, channel): no FFT.
#include "common.cuh"
#include "kernels.h"

#include <cooperative_groups.h>

#include <cmath>

namespace sdxl {

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

void freeu_twiddles(int H, int W, float* out) {
  // h < H and w < W keep every angle in [0, 2 pi): double precision, rounded once to f32
  const double two_pi = 6.283185307179586476925286766559;
  for (int h = 0; h < H; ++h) {
    out[h] = (float)std::cos(two_pi * h / H);
    out[H + h] = (float)std::sin(two_pi * h / H);
  }
  for (int w = 0; w < W; ++w) {
    out[2 * H + w] = (float)std::cos(two_pi * w / W);
    out[2 * H + W + w] = (float)std::sin(two_pi * w / W);
  }
}

// Work split. A block holds 8 consecutive channels of one row and 64 pixel lanes (512 threads; 8 threads read 32 contiguous bytes of a
// pixel). The pixels of a skip are split between the freeu_cluster(N) blocks of a thread-block cluster: lane l of cluster block q takes
// pixels q * 64 + l, then every (64 * cluster size)-th one. The cluster size and so the order of every sum depend on N only, never on
// the batch; no atomics.
constexpr int FREEU_TC = 8;      // channels per block
constexpr int FREEU_PL = 64;     // pixel lanes per block
static inline int freeu_cluster(long N) { return N >= 8L * 512 ? 8 : N >= 4L * 512 ? 4 : N >= 2L * 512 ? 2 : 1; }

// grid (cluster size, channel tiles, rows). Phase 1: the 7 sums of each channel over the block's pixels (a fixed butterfly within
// the warp, then the 16 warps in order), then over the cluster's blocks in rank order through distributed shared memory. Phase 2:
// r' in place on the block's pixels, and x[:, :Cx / 2] *= *b on them.
__global__ void __launch_bounds__(FREEU_TC * FREEU_PL) freeu_kernel(float* __restrict__ r, int C, float* __restrict__ x, int Cx,
                                                                     int H, int W, const float* __restrict__ tw,
                                                                     const float* __restrict__ s_ptr, const float* __restrict__ b_ptr) {
  namespace cg = cooperative_groups;
  griddep_wait();
  griddep_launch_dependents();
  __shared__ float part[7][FREEU_PL / 4][FREEU_TC];
  __shared__ float blk[7][FREEU_TC];   // this block's sums, read by every block of the cluster
  __shared__ float tot[7][FREEU_TC];
  cg::cluster_group cluster = cg::this_cluster();
  const int ncl = (int)cluster.num_blocks(), q = (int)cluster.block_rank();
  const int t = threadIdx.x, cl = t % FREEU_TC, pl = t / FREEU_TC, warp = t / 32;
  const int c = blockIdx.y * FREEU_TC + cl;
  const long N = (long)H * W, stride = (long)FREEU_PL * ncl;
  const long p0 = (long)q * FREEU_PL + pl;
  const size_t row = blockIdx.z;
  const float* ch = tw;
  const float* sh = tw + H;
  const float* cw = tw + 2 * H;
  const float* sw = tw + 2 * H + W;
  // which of the bins (-1, 0), (0, -1), (-1, -1) are distinct from (0, 0) and each other
  const bool use_h = H > 1, use_w = W > 1;
  if (blockIdx.y * FREEU_TC < C) {   // block-uniform (the whole cluster shares blockIdx.y)
    float* rr = r + row * N * C;
    float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c < C) {
#pragma unroll 4
      for (long p = p0; p < N; p += stride) {
        const int h = (int)(p / W), w = (int)(p - (long)h * W);
        const float v = rr[p * C + c];
        const float a = ch[h], sa = sh[h], bw = cw[w], sb = sw[w];
        const float c11 = a * bw - sa * sb, s11 = sa * bw + a * sb;
        acc[0] += v;
        acc[1] += v * bw;  acc[2] += v * sb;    // X(0, -1)
        acc[3] += v * a;   acc[4] += v * sa;    // X(-1, 0)
        acc[5] += v * c11; acc[6] += v * s11;   // X(-1, -1)
      }
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) {   // the 4 pixel lanes of a warp that share a channel: (l0 + l1) + (l2 + l3) in every lane
      acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 8);
      acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 16);
    }
    if ((t & 31) < FREEU_TC)
#pragma unroll
      for (int k = 0; k < 7; ++k) part[k][warp][cl] = acc[k];
    __syncthreads();
    if (t < 7 * FREEU_TC) {
      float sum = 0.f;
      for (int j = 0; j < FREEU_PL / 4; ++j) sum += part[t / FREEU_TC][j][t % FREEU_TC];
      blk[t / FREEU_TC][t % FREEU_TC] = sum;
    }
    cluster.sync();
    if (t < 7 * FREEU_TC) {
      float sum = 0.f;
      for (int j = 0; j < ncl; ++j) sum += cluster.map_shared_rank(&blk[0][0], j)[t];
      tot[t / FREEU_TC][t % FREEU_TC] = sum;
    }
    cluster.sync();   // every block has read the others' sums before any of them exits; tot is visible block-wide
    const float f = (*s_ptr - 1.f) / (float)N;
    const float X00 = tot[0][cl], A01 = use_w ? tot[1][cl] : 0.f, B01 = use_w ? tot[2][cl] : 0.f,
                A10 = use_h ? tot[3][cl] : 0.f, B10 = use_h ? tot[4][cl] : 0.f, A11 = use_h && use_w ? tot[5][cl] : 0.f,
                B11 = use_h && use_w ? tot[6][cl] : 0.f;
    if (c < C) {
#pragma unroll 4
      for (long p = p0; p < N; p += stride) {
        const int h = (int)(p / W), w = (int)(p - (long)h * W);
        const float a = ch[h], sa = sh[h], bw = cw[w], sb = sw[w];
        const float c11 = a * bw - sa * sb, s11 = sa * bw + a * sb;
        const float corr = X00 + (A01 * bw + B01 * sb) + (A10 * a + B10 * sa) + (A11 * c11 + B11 * s11);
        float* e = rr + p * C + c;
        *e = *e + f * corr;
      }
    }
  }
  const int half = Cx / 2;
  if (c < half) {
    const float bv = *b_ptr;
    float* xr = x + row * N * Cx;
#pragma unroll 4
    for (long p = p0; p < N; p += stride) xr[p * Cx + c] *= bv;
  }
}

int freeu_launch(cudaStream_t st, float* r, int C, float* x, int Cx, int B, int H, int W, const float* tw, const float* s,
                 const float* b) {
  if (B < 1 || H < 1 || W < 1 || C < 1 || Cx < 2) return (int)cudaErrorInvalidValue;
  const int ncl = freeu_cluster((long)H * W);
  const int tiles = cdiv(C > Cx / 2 ? C : Cx / 2, FREEU_TC);
  return launch_kernel_cluster(freeu_kernel, dim3(ncl, tiles, B), dim3(FREEU_TC * FREEU_PL), (size_t)0, st, true, ncl, r, C, x, Cx,
                               H, W, tw, s, b);
}

}  // namespace sdxl
