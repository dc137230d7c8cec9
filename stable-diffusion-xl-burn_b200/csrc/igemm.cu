// Implicit GEMM on Hopper tensor cores (wgmma, f32 accumulators in registers, operands staged by TMA into 128B-swizzled
// shared memory). One kernel serves every dense contraction of the UNet step:
//   * Linear layers (reference unet/mod.rs:830,839,917,944,1009-1011,1021) = 1 segment, 1x1 tap;
//   * 3x3 / 1x1 convolutions (unet/mod.rs:1086,1096,1099,750,767-770,490): one K-segment per filter
//     tap; the tap shift is a TMA box offset on the NHWC activation, zero padding comes from TMA
//     out-of-bounds fill; the ResBlock skip 1x1 conv is just one more K-segment on a second tensor.
//
// Persistent and warp-specialised: grid = min(#tiles, #SMs), every CTA walks the tiles blockIdx.x, + gridDim.x, ...
// (M tiles fastest, so CTAs running at the same time share the weight tile in L2).
//   warpgroup 0     : TMA producer (one lane); gives up registers to the consumers (setmaxnreg)
//   warpgroups 1, 2 : consumers. Each owns 64 rows of the 128 x BN tile (wgmma.m64nNk16, N = 64, 128 or 160 per instruction) and
//                     runs the epilogue straight from its accumulator registers.
// The shared-memory operand ring runs across tile boundaries, so the loads of tile i+1 overlap the epilogue of tile i.
#include "common.cuh"
#include "kernels.h"

#include <stdio.h>
#include <stdlib.h>

namespace sdxl {

static constexpr int kTileM = 128;
static constexpr int kBlockK = 64;                    // 64 halves = 128 B = one swizzle row
static constexpr int kABytes = kTileM * kBlockK * 2;  // 16 KB
static constexpr int kConsumerWarps = 8;
static constexpr int kThreads = 128 + kConsumerWarps * 32;

__device__ __forceinline__ size_t out_pixel(const IgemmParams& p, int tb, int th, int tw, int r, bool& ok, int& bb) {
  const int wt = r % p.Wt, ht = (r / p.Wt) % p.Ht, bt = r / (p.Wt * p.Ht);
  bb = tb * p.Bt + bt;
  const int hh = th * p.Ht + ht, ww = tw * p.Wt + wt;
  ok = (bb < p.Bn) && (hh < p.H) && (ww < p.W);
  return ok ? ((size_t)bb * p.H + hh) * (size_t)p.opix_row + (size_t)ww * p.opix_w + p.opix_off : 0;
}

__device__ __forceinline__ void store2(const IgemmParams& p, size_t off, float x0, float x1, bool two, bool vec) {
  if (p.out_f32) {
    float* o = reinterpret_cast<float*>(p.out) + off;
    if (two && vec) *reinterpret_cast<float2*>(o) = make_float2(x0, x1);
    else { o[0] = x0; if (two) o[1] = x1; }
  } else {
    __half* o = reinterpret_cast<__half*>(p.out) + off;
    if (two && vec) *reinterpret_cast<__half2*>(o) = __floats2half2_rn(x0, x1);
    else { o[0] = __float2half_rn(x0); if (two) o[1] = __float2half_rn(x1); }
  }
}

// Epilogue of one consumer thread: rows r0 and r0 + 8 of the tile, columns 8 j + 2 (lane & 3) + {0, 1} (the wgmma accumulator
// layout: acc[4 j + 2 h + e]).
//   LINEAR: out = acc + bias[batch] (+ f32 residual), f32 or f16.   GEGLU (reference unet/mod.rs:942-956): tile columns [0, BN/2)
//   are values, [BN/2, BN) the matching gates; out = value * gelu_erf(gate), f16, at column nt * BN/2 + c.
// LINEAR runs in chunks of JC column pairs: every bias and residual load of a chunk is issued before the chunk's first add, so
// their latencies overlap. `out` may alias `res` (in-place residual add), so no load can move above an earlier store: without
// the chunks each column pair would pay a full load round trip.
template <int BN>
__device__ __forceinline__ void epilogue(const IgemmParams& p, const float (&acc)[BN / 2], int tb, int th, int tw, int nt, int r0,
                                         int lane) {
  constexpr int JC = BN == 160 ? 10 : 8;
  static_assert((BN / 8) % JC == 0, "column pairs must split into whole chunks");
  const int cq = (lane & 3) * 2;
  const int n0 = nt * BN;
  const bool vec = ((p.ldo | p.ldr | p.bias_bstride) & 1) == 0 && ((reinterpret_cast<uintptr_t>(p.out) | reinterpret_cast<uintptr_t>(p.res) |
                                                                     reinterpret_cast<uintptr_t>(p.bias)) & 7) == 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    bool ok;
    int bb;
    const size_t pix = out_pixel(p, tb, th, tw, r0 + 8 * h, ok, bb);
    if (!ok) continue;
    if (p.mode == IGEMM_LINEAR) {
      const float* bias = p.bias ? p.bias + (size_t)bb * p.bias_bstride : nullptr;
      const float* res = p.res ? p.res + pix * p.ldr : nullptr;
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += JC) {
        float2 bv[JC], rv[JC];
#pragma unroll
        for (int jj = 0; jj < JC; ++jj) {
          const int n = n0 + 8 * (j0 + jj) + cq;
          const bool two = n + 1 < p.N;
          bv[jj] = rv[jj] = make_float2(0.f, 0.f);
          if (n >= p.N) continue;
          if (bias) bv[jj] = (two && vec) ? __ldg(reinterpret_cast<const float2*>(bias + n)) : make_float2(bias[n], two ? bias[n + 1] : 0.f);
          if (res) rv[jj] = (two && vec) ? *reinterpret_cast<const float2*>(res + n) : make_float2(res[n], two ? res[n + 1] : 0.f);
        }
#pragma unroll
        for (int jj = 0; jj < JC; ++jj) {
          const int j = j0 + jj, n = n0 + 8 * j + cq;
          if (n >= p.N) continue;
          float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
          if (bias) { x0 += bv[jj].x; x1 += bv[jj].y; }
          if (res) { x0 += rv[jj].x; x1 += rv[jj].y; }
          store2(p, pix * p.ldo + n, x0, x1, n + 1 < p.N, vec);
        }
      }
    } else {
      constexpr int hb = BN / 2;
#pragma unroll
      for (int j = 0; j < hb / 8; ++j) {
        const int c = 8 * j + cq;
        float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
        float y0 = acc[4 * (j + hb / 8) + 2 * h], y1 = acc[4 * (j + hb / 8) + 2 * h + 1];
        if (p.bias != nullptr) {
          x0 += __ldg(p.bias + n0 + c); x1 += __ldg(p.bias + n0 + c + 1);
          y0 += __ldg(p.bias + n0 + hb + c); y1 += __ldg(p.bias + n0 + hb + c + 1);
        }
        reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.out) + pix * p.ldo + nt * hb + c)[0] =
            __floats2half2_rn(x0 * gelu_erf_f(y0), x1 * gelu_erf_f(y1));
      }
    }
  }
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1) igemm_kernel(const __grid_constant__ IgemmParams p) {
  constexpr int NC = BN == 160 ? 160 : BN >= 128 ? 128 : 64;   // N of one wgmma
  constexpr int NCH = BN / NC;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nst = p.nstages;
  constexpr uint32_t stage_bytes = kABytes + BN * 128;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)nst * stage_bytes);
  uint64_t* empty_bar = full_bar + nst;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = p.tilesW * p.tilesH * p.tilesB;
  const int num_tiles = m_tiles * p.tilesN;
  int total_kb = 0;
  for (int s = 0; s < p.nseg; ++s) total_kb += p.seg[s].nkb;

  if (threadIdx.x == 0) {
    for (int i = 0; i < nst; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kConsumerWarps); }
    fence_barrier_init();
    tma_prefetch_desc(&p.tmA0);
    tma_prefetch_desc(&p.tmA1);
    tma_prefetch_desc(&p.tmB);
  }
  __syncthreads();
  // PDL: everything above overlapped the previous kernel's tail; from here on we touch its outputs.
  griddep_wait();
  griddep_launch_dependents();

  if (warp < 4) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();   // hands registers to the consumers, whose epilogue holds a chunk of loads next to the accumulators
    if (warp != 0 || lane != 0) return;
    uint32_t stage = 0, phase = 0;
    for (int st = blockIdx.x; st < num_tiles; st += gridDim.x) {
      const int mt = st % m_tiles, nt = st / m_tiles;
      const int tw = mt % p.tilesW, th = (mt / p.tilesW) % p.tilesH, tb = mt / (p.tilesW * p.tilesH);
      const int w0 = tw * p.Wt, h0 = th * p.Ht, b0 = tb * p.Bt, n0 = nt * BN;
      int kcol = 0;
      for (int s = 0; s < p.nseg; ++s) {
        const IgemmSeg sg = p.seg[s];
        const void* mapA = sg.map ? (const void*)&p.tmA1 : (const void*)&p.tmA0;
        for (int j = 0; j < sg.nkb; ++j, kcol += kBlockK) {
          mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
          uint8_t* dst = smem + stage * stage_bytes;
          mbar_expect_tx(&full_bar[stage], stage_bytes);
          tma_load_4d(dst, mapA, &full_bar[stage], j * kBlockK, w0 + sg.dw, h0 + sg.dh, b0 + sg.db);
          tma_load_2d(dst + kABytes, &p.tmB, &full_bar[stage], kcol, n0);
          if (++stage == (uint32_t)nst) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<232>();   // 128 x 40 + 256 x 232 registers fit the SM's 64 K
  const int wg = (warp >> 2) - 1;                      // 0 / 1: tile rows [64 wg, 64 wg + 64)
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint32_t smem_base = smem_u32(smem);
  uint32_t stage = 0, phase = 0;
  float acc[BN / 2];
  for (int st = blockIdx.x; st < num_tiles; st += gridDim.x) {
    const int mt = st % m_tiles, nt = st / m_tiles;
    uint32_t prev = 0;
    for (int kb = 0; kb < total_kb; ++kb) {
      mbar_wait_nocall(&full_bar[stage], phase);
      wg_fence();
      const uint32_t a = smem_base + stage * stage_bytes + (uint32_t)wg * (64 * 128);
      const uint32_t b = smem_base + stage * stage_bytes + kABytes;
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k) {
        const uint64_t da = wg_desc_sw128(a + 32 * k);
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const uint64_t db = wg_desc_sw128(b + c * NC * 128 + 32 * k);
          if constexpr (NC == 160) wgmma_ss_n160(*reinterpret_cast<float(*)[80]>(acc), da, db, (kb | k) != 0);
          else if constexpr (NC == 128) wgmma_ss_n128(*reinterpret_cast<float(*)[64]>(acc + 64 * c), da, db, (kb | k) != 0);
          else wgmma_ss_n64(*reinterpret_cast<float(*)[32]>(acc + 32 * c), da, db, (kb | k) != 0);
        }
      }
      wg_commit();
      if (kb > 0) {   // the previous K block's wgmmas have read their stage: hand it back to the producer
        wg_wait<1>();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == (uint32_t)nst) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    if (lane == 0 && total_kb > 0) mbar_arrive(&empty_bar[prev]);
    const int tw = mt % p.tilesW, th = (mt / p.tilesW) % p.tilesH, tb = mt / (p.tilesW * p.tilesH);
    epilogue<BN>(p, acc, tb, th, tw, nt, r0, lane);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(f);
  }
  return fn;
}

static int encode(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                  CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_encodeTiled fn = get_encode();
  if (!fn) return 1001;
  cuuint64_t gd[5];
  cuuint64_t gs[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gs[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = fn(tm, dtype, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "sdxl_b200: cuTensorMapEncodeTiled failed (%d) rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u]\n",
            (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
            (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
            rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return 1002;
  }
  return 0;
}

int make_tmap_act(CUtensorMap* tm, const __half* base, int Bn, int H, int W, int C, int pitch, int Wt, int Ht,
                  int Bt) {
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)Bn};
  uint64_t str[3] = {(uint64_t)pitch * 2, (uint64_t)W * pitch * 2, (uint64_t)H * W * pitch * 2};
  uint32_t box[4] = {64, (uint32_t)Wt, (uint32_t)Ht, (uint32_t)Bt};
  return encode(tm, base, 4, dims, str, box);
}
int make_tmap_wgt(CUtensorMap* tm, const __half* base, int N, int K, int BN) {
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
  uint64_t str[1] = {(uint64_t)K * 2};
  uint32_t box[2] = {64, (uint32_t)BN};
  return encode(tm, base, 2, dims, str, box);
}
int make_tmap_rows(CUtensorMap* tm, const __half* base, int rows_per_batch, int nbatch, int cols, int pitch) {
  uint64_t dims[3] = {(uint64_t)cols, (uint64_t)rows_per_batch, (uint64_t)nbatch};
  uint64_t str[2] = {(uint64_t)pitch * 2, (uint64_t)rows_per_batch * pitch * 2};
  uint32_t box[3] = {64, 128, 1};
  return encode(tm, base, 3, dims, str, box);
}

void igemm_pick_box(int W, int H, int* Wt, int* Ht, int* Bt) {
  int wt = 1;
  while (wt * 2 <= W && wt * 2 <= 128) wt *= 2;
  int ht = 1;
  while (ht * 2 <= H && wt * ht * 2 <= 128) ht *= 2;
  *Wt = wt;
  *Ht = ht;
  *Bt = 128 / (wt * ht);
}

int igemm_pick_bn(int m_tiles, int N, int num_sms, bool geglu) {
  // N tiles the kernel is instantiated for. Cost model: waves * BN (tensor time ~ BN per tile) with a fixed A-operand /
  // epilogue cost per tile; a tile width that divides N wins over padding. 160 divides the UNet's 320 * 2^k widths: at 16 M
  // tiles and N = 1280 it fills 128 of 132 SMs where 256 fills 80. The fixed cost of 48 is the least-squares fit of
  // log(time) to waves * (BN + c) over a sweep of every BN at the SDXL step's GEMM shapes on H100 (DESIGN §4).
  (void)geglu;
  // The one shape the model gets wrong: the base UNet's level-2 QKV (16 M tiles, N = 3840) costs 608 at BN = 256 (2 waves)
  // against 624 at 160 (3 waves), but 160 took 3.8 % off the whole step on H100 (DESIGN §4, §6). The refiner's level-2 QKV
  // (N = 4608) and its N = 1536 GEMMs keep the model's choice. The tile width does not change any result.
  if (m_tiles == 16 && N == 3840) return 160;
  double best = 1e30;
  int best_bn = 0;
  for (int bn : {256, 160, 128, 64}) {
    if (N % bn) continue;
    const long tiles = (long)m_tiles * (N / bn);
    const long waves = (tiles + num_sms - 1) / num_sms;
    const double cost = (double)waves * (bn + 48.0);
    if (cost < best) {
      best = cost;
      best_bn = bn;
    }
  }
  if (!best_bn) best_bn = N <= 64 ? 64 : N <= 128 ? 128 : 256;   // no divisor: cover N with padding
  return best_bn;
}

// Per-device launch state: several devices may be driven from one process (one sdxl_ctx each), and the opt-in to > 48 KB of
// dynamic shared memory and the SM count are per device.
struct IgemmDev { bool attr = false; int num_sms = 0; };
static IgemmDev g_igemm_dev[64];
static IgemmDev* igemm_dev() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  IgemmDev& D = g_igemm_dev[dev];
  if (!D.num_sms) {
    cudaDeviceGetAttribute(&D.num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (D.num_sms <= 0) D.num_sms = 132;
  }
  return &D;
}
static int device_sms() {
  IgemmDev* D = igemm_dev();
  return D ? D->num_sms : 132;
}

static constexpr int kMaxSmem = 227 * 1024;
static size_t igemm_smem_bytes(int nst, int BN) { return (size_t)nst * (kABytes + BN * 128) + 1024 /*align slack*/ + 2 * nst * 8; }

int igemm_configure(IgemmParams& p, const IgemmOperands& o, int outW, int outH, int outB, int mode, int geglu_bn) {
  igemm_pick_box(outW, outH, &p.Wt, &p.Ht, &p.Bt);
  p.W = outW; p.H = outH; p.Bn = outB;
  p.opix_row = outW; p.opix_w = 1; p.opix_off = 0;
  p.tilesW = (outW + p.Wt - 1) / p.Wt;
  p.tilesH = (outH + p.Ht - 1) / p.Ht;
  p.tilesB = (outB + p.Bt - 1) / p.Bt;
  const int m_tiles = p.tilesW * p.tilesH * p.tilesB;
  p.N = o.N;
  p.mode = mode;
  p.BN = (mode == IGEMM_GEGLU) ? geglu_bn : igemm_pick_bn(m_tiles, o.N, device_sms(), false);
  if (p.BN != 64 && p.BN != 128 && p.BN != 160 && p.BN != 256) return 1010;
  p.tilesN = (mode == IGEMM_GEGLU) ? (o.N / p.BN) : ((o.N + p.BN - 1) / p.BN);
  int r = make_tmap_act(&p.tmA0, o.a0, o.a0Bn, o.a0H, o.a0W, o.a0C, o.a0pitch, p.Wt, p.Ht, p.Bt);
  if (!r && o.a1) r = make_tmap_act(&p.tmA1, o.a1, o.a1Bn, o.a1H, o.a1W, o.a1C, o.a1pitch, p.Wt, p.Ht, p.Bt);
  if (!r && !o.a1) p.tmA1 = p.tmA0;
  if (!r) r = make_tmap_wgt(&p.tmB, o.w, o.N, o.Ktot, p.BN);
  if (r) return r;
  const int stage_bytes = kABytes + p.BN * 128;
  int nst = (kMaxSmem - 1024 - 256) / stage_bytes;
  if (nst > 8) nst = 8;
  p.nstages = nst;
  return 0;
}

int igemm_launch(cudaStream_t st, IgemmParams& p) {
  if (p.res != nullptr && p.ldr != p.ldo) return 1003;
  if ((unsigned long long)p.Bn * p.H * (unsigned long long)p.opix_row * (unsigned long long)p.ldo >= (1ull << 32)) return 1004;
  if (p.nstages < 2) return 1011;
  const size_t smem = igemm_smem_bytes(p.nstages, p.BN);
  if (smem > (size_t)kMaxSmem) return 1011;
  IgemmDev* D = igemm_dev();
  if (!D) return 1009;
  if (!D->attr) {
    cudaError_t e = cudaFuncSetAttribute(igemm_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(igemm_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(igemm_kernel<160>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(igemm_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e != cudaSuccess) return (int)e;
    D->attr = true;
  }
  const long tiles = (long)p.tilesW * p.tilesH * p.tilesB * p.tilesN;
  const dim3 grid((unsigned)(tiles < D->num_sms ? (tiles > 0 ? tiles : 1) : D->num_sms));
  switch (p.BN) {
    case 64: return launch_kernel(igemm_kernel<64>, grid, dim3(kThreads), smem, st, true, p);
    case 128: return launch_kernel(igemm_kernel<128>, grid, dim3(kThreads), smem, st, true, p);
    case 160: return launch_kernel(igemm_kernel<160>, grid, dim3(kThreads), smem, st, true, p);
    case 256: return launch_kernel(igemm_kernel<256>, grid, dim3(kThreads), smem, st, true, p);
    default: return 1010;
  }
}

}  // namespace sdxl
