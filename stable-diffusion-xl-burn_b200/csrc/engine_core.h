// Internals shared by the model front ends of libsdxl_b200.so (engine.cu: UNet + sampler + op-level API, vae.cu: latent
// decoder / encoder, clip.cu: text encoders): context, device arena, weight-pack parsing and re-layout helpers, and the
// launch plan (a flat list of kernel launches with pre-built TMA descriptors, run eagerly once and then replayed as a CUDA
// graph). Everything here has internal linkage; the public boundary is include/sdxl_b200.h.
#pragma once
#include "../../include/sdxl_b200.h"
#include "kernels.h"

#include <math.h>
#include <nvtx3/nvToolsExt.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

using namespace sdxl;

// ================================================================================================
// context
// ================================================================================================
struct sdxl_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int num_sms = 132;
  std::string err;
  uint64_t launches = 0;
};

static int fail(sdxl_ctx* c, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code ? code : -1;
}
#define CU(ctx, expr)                                                                         \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return fail(ctx, (int)_e, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)
#define KL(ctx, expr)                                                                         \
  do {                                                                                        \
    int _e = (expr);                                                                          \
    if (_e) return fail(ctx, _e, "%s failed with %d%s%s (%s:%d)", #expr, _e, _e < 1000 ? ": " : "", \
                        _e < 1000 ? cudaGetErrorString((cudaError_t)_e) : "", __FILE__, __LINE__); \
    (ctx)->launches++;                                                                        \
  } while (0)

// ================================================================================================
// fresh-memory fill (SDXL_B200_FILL)
// ================================================================================================
// SDXL_B200_FILL=<byte> (decimal or 0x..): every device buffer the library carves for itself is memset on its stream before
// anything writes to it, so that a read of memory nothing wrote reaches the outputs instead of whatever the allocator left
// there. Floating-point buffers get the byte (0xff: NaN in f16 and f32; 0x7b: large finite values); integer and byte buffers
// get 0, so that an index or a count is never poisoned into an address. -1 when unset or not a byte (sdxl_debug_fill).
static int debug_fill_byte() {
  static const int b = [] {
    const char* s = getenv("SDXL_B200_FILL");
    if (!s || !*s) return -1;
    char* end = nullptr;
    const long v = strtol(s, &end, 0);
    return (*end || v < 0 || v > 255) ? -1 : (int)v;
  }();
  return b;
}
// Queues the fill of n fresh elements of T at p on st; fill = debug_fill_byte(), nothing when it is negative.
template <typename T>
static void debug_fill(T* p, size_t n, cudaStream_t st, int fill) {
  constexpr bool fp = std::is_floating_point<T>::value || std::is_same<T, __half>::value;
  if (fill >= 0 && p && n) cudaMemsetAsync(p, fp ? fill : 0, n * sizeof(T), st);
}

// ================================================================================================
// device arena (bump allocator over one cudaMalloc, freed with the arena)
// ================================================================================================
struct Arena {
  uint8_t* base = nullptr;
  size_t cap = 0, off = 0;
  bool measure = false;  // dry run: only count
  cudaStream_t stream = nullptr;   // the stream that writes the arena: fresh-memory fills are queued on it
  int fill = -1;                   // debug_fill_byte() for a real arena, -1 for none
  Arena() = default;
  Arena(Arena&& o) noexcept : base(o.base), cap(o.cap), off(o.off), measure(o.measure), stream(o.stream), fill(o.fill) { o.base = nullptr; o.cap = o.off = 0; }
  Arena& operator=(Arena&& o) noexcept {
    if (this != &o) {
      release();
      base = o.base; cap = o.cap; off = o.off; measure = o.measure; stream = o.stream; fill = o.fill;
      o.base = nullptr; o.cap = o.off = 0;
    }
    return *this;
  }
  ~Arena() { release(); }
  int init(size_t bytes) {
    release();
    if (cudaMalloc((void**)&base, bytes) != cudaSuccess) {
      base = nullptr;
      cudaGetLastError();   // an oversized request is not sticky: clear it so later launch checks do not report it
      return 1;
    }
    cap = bytes;
    off = 0;
    return 0;
  }
  void release() {
    if (base) cudaFree(base);
    base = nullptr;
    cap = off = 0;
  }
  void* alloc(size_t bytes) {
    const size_t a = (off + 1023) & ~size_t(1023);
    if (!measure && a + bytes > cap) return nullptr;
    off = a + bytes;
    return measure ? (void*)(uintptr_t)(0x1000 + a) : (void*)(base + a);
  }
  template <typename T>
  T* get(size_t n) {
    T* p = (T*)alloc(n * sizeof(T));
    if (fill >= 0 && !measure) debug_fill(p, n, stream, fill);
    return p;
  }
};

// ================================================================================================
// weight pack
// ================================================================================================
#pragma pack(push, 1)
struct PackHeader {
  char magic[8];  // "SDXLPK01"
  uint32_t n_tensors;
  uint32_t reserved;
  uint64_t data_offset;
};
struct PackEntry {
  char name[120];
  uint32_t dtype;  // 0 = f16, 1 = f32
  uint32_t ndim;
  uint64_t shape[4];
  uint64_t offset;  // from pack start
  uint64_t nbytes;
};
#pragma pack(pop)

struct PackView {
  const uint8_t* dev = nullptr;  // pack bytes in device memory
  std::map<std::string, PackEntry> t;
  const PackEntry* find(const std::string& n) const {
    auto it = t.find(n);
    return it == t.end() ? nullptr : &it->second;
  }
};

// ================================================================================================
// layer records + loader
// ================================================================================================
struct Lin {
  __half* w = nullptr; float* b = nullptr; int K = 0, Kpad = 0, N = 0, geglu_bn = 0;
};
struct Conv {
  __half* w = nullptr; float* b = nullptr; int I = 0, O = 0, ks = 0, Ipad = 0, I2 = 0, I2pad = 0, Ktot = 0;
  __half* wup = nullptr;  // upconv(): four 2x2 phase kernels [4][O][4*Ipad] of a 3x3 conv that follows a nearest-2x upsample
};
struct Norm { float* g = nullptr; float* b = nullptr; int C = 0; float eps = 1e-5f; };

// ================================================================================================
// LoRA: registry of the LoRA-able weight slots (filled while loading) and the merge / restore state
// ================================================================================================
// One weight slot = one reference layer inside a re-laid-out weight buffer. Element (n, k) of the layer's [N, I*ks*ks] delta
// (k = i*ks*ks + tap) lives at base[(row0 + geglu_perm(n)) * ld + col0 + tap * Ipad + i] (lora_merge_kernel); `up` slots
// are the phase kernels of an upsample conv ([4][N][4*Ipad], lora_upconv_merge_kernel).
struct WSlot {
  void* base = nullptr;  // weight buffer (key of AdapterState::bufs)
  int conv = 0;          // adapter factors are conv-shaped: down [r, I, ks, ks], up [N, r, 1, 1]; else down [r, I], up [N, r]
  int up = 0, f32 = 0;   // upsample phase kernels; f32 storage (first conv)
  int N = 0, I = 0, ks = 1;
  size_t ld = 0;
  int row0 = 0, col0 = 0, Ipad = 0, geglu_bn = 0;
};
struct AdapterState {
  struct Buf { size_t bytes = 0; void* backup = nullptr; bool dirty = false; };
  std::map<std::string, WSlot> slots;   // by reference layer path
  std::map<void*, Buf> bufs;
  std::vector<void*> allocs;             // backup allocations (one per call that touched new buffers)
  void add(const std::string& path, const WSlot& s, size_t buf_bytes) {
    slots[path] = s;
    Buf& b = bufs[s.base];
    if (buf_bytes > b.bytes) b.bytes = buf_bytes;
  }
  void release() {
    for (void* p : allocs) cudaFree(p);
    allocs.clear();
    for (auto& kv : bufs) { kv.second.backup = nullptr; kv.second.dirty = false; }
  }
  ~AdapterState() { release(); }
};

struct Loader {
  sdxl_ctx* c;
  const PackView* pv;
  Arena* A;
  cudaStream_t st;
  int err = 0;
  AdapterState* reg = nullptr;  // LoRA slot registry (recorded on the real pass only)

  void record(const std::string& path, const WSlot& s, size_t buf_bytes) {
    if (reg && !A->measure) reg->add(path, s, buf_bytes);
  }

  const PackEntry* need(const std::string& name, int ndim) {
    const PackEntry* e = pv->find(name);
    if (!e) { err = fail(c, 4001, "weight pack: missing tensor '%s'", name.c_str()); return nullptr; }
    if (e->dtype != 0) { err = fail(c, 4002, "weight pack: tensor '%s' must be f16", name.c_str()); return nullptr; }
    if ((int)e->ndim != ndim) { err = fail(c, 4003, "weight pack: tensor '%s' has ndim %u, expected %d", name.c_str(), e->ndim, ndim); return nullptr; }
    return e;
  }
  // `path`/weight, an OIHW f16 conv weight of shape [O, I, ks, ks]
  const PackEntry* conv_weight(const std::string& path, int O, int I, int ks) {
    const PackEntry* e = need(path + "/weight", 4);
    if (e && ((int)e->shape[0] != O || (int)e->shape[1] != I || (int)e->shape[2] != ks || (int)e->shape[3] != ks)) {
      err = fail(c, 4007, "weight pack: '%s/weight' has shape [%llu,%llu,%llu,%llu], expected [%d,%d,%d,%d]", path.c_str(),
                 (unsigned long long)e->shape[0], (unsigned long long)e->shape[1], (unsigned long long)e->shape[2],
                 (unsigned long long)e->shape[3], O, I, ks, ks);
      return nullptr;
    }
    return e;
  }
  const __half* ptr(const PackEntry* e) { return (const __half*)(pv->dev + e->offset); }
  bool has(const std::string& name) { return pv->find(name) != nullptr; }

  float* vec_f32(const std::string& name, int expectN, int geglu_bn = 0) {
    const PackEntry* e = need(name, 1);
    if (!e) return nullptr;
    if ((int)e->shape[0] != expectN) { err = fail(c, 4004, "weight pack: '%s' has %llu elements, expected %d", name.c_str(), (unsigned long long)e->shape[0], expectN); return nullptr; }
    float* d = A->get<float>(expectN);
    if (!d) { err = fail(c, 4005, "weight arena exhausted"); return nullptr; }
    if (!A->measure) { int r = bias_to_f32_launch(st, ptr(e), expectN, d, geglu_bn, 0); if (r) err = fail(c, r, "bias_to_f32 failed"); }
    return d;
  }
  // Linear stored [in,out]; produce K-major [N,Kpad]. Rows may be a slice of a fused matrix.
  int lin_into(const std::string& path, __half* dst, int Kpad, int row0, int expectK, int expectN, int geglu_bn) {
    const PackEntry* e = need(path + "/weight", 2);
    if (!e) return err;
    if ((int)e->shape[0] != expectK || (int)e->shape[1] != expectN)
      return err = fail(c, 4006, "weight pack: '%s/weight' is [%llu,%llu], expected [%d,%d]", path.c_str(),
                        (unsigned long long)e->shape[0], (unsigned long long)e->shape[1], expectK, expectN);
    if (!A->measure) { int r = transpose_linear_launch(st, ptr(e), expectK, expectN, dst, Kpad, row0, geglu_bn); if (r) return err = fail(c, r, "transpose_linear failed"); }
    WSlot s;
    s.base = dst; s.N = expectN; s.I = expectK; s.ld = Kpad; s.row0 = row0; s.Ipad = Kpad; s.geglu_bn = geglu_bn;
    record(path, s, (size_t)(row0 + expectN) * Kpad * sizeof(__half));
    return 0;
  }
  static int pad64(int k) { return (k + 63) / 64 * 64; }
  Lin linear(const std::string& path, int K, int N, bool bias, int geglu_bn = 0) {
    Lin L;
    L.K = K; L.N = N; L.Kpad = pad64(K); L.geglu_bn = geglu_bn;
    L.w = A->get<__half>((size_t)N * L.Kpad);
    if (!L.w) { err = fail(c, 4005, "weight arena exhausted"); return L; }
    if (lin_into(path, L.w, L.Kpad, 0, K, N, geglu_bn)) return L;
    if (bias) L.b = vec_f32(path + "/bias", N, geglu_bn);
    return L;
  }
  // 3x3 conv applied to a nearest-2x upsampled image, stored as its four 2x2 phase convolutions on the source image
  // (2.25x fewer MACs, no upsampled copy; elementwise.cu: repack_upconv_kernel)
  Conv upconv(const std::string& path, int I, int O) {
    Conv cv;
    cv.I = I; cv.O = O; cv.ks = 3; cv.Ipad = pad64(I); cv.Ktot = 4 * cv.Ipad;
    cv.wup = A->get<__half>((size_t)4 * O * cv.Ktot);
    if (!cv.wup) { err = fail(c, 4005, "weight arena exhausted"); return cv; }
    const PackEntry* e = conv_weight(path, O, I, 3);
    if (!e) return cv;
    if (!A->measure) { int r = repack_upconv_launch(st, ptr(e), O, I, cv.wup, cv.Ipad); if (r) err = fail(c, r, "repack_upconv failed"); }
    {
      WSlot s;
      s.base = cv.wup; s.conv = 1; s.up = 1; s.N = O; s.I = I; s.ks = 3; s.ld = cv.Ktot; s.Ipad = cv.Ipad;
      record(path, s, (size_t)4 * O * cv.Ktot * sizeof(__half));
    }
    cv.b = vec_f32(path + "/bias", O);
    return cv;
  }
  Norm norm(const std::string& path, int C) {
    Norm n;
    n.C = C;
    n.g = vec_f32(path + "/weight", C);
    n.b = vec_f32(path + "/bias", C);
    return n;
  }
  // 3x3 conv with few input channels for the CUDA-core first-conv kernel: OIHW f16 -> [O][kh][kw][I] f32, bias f32
  int conv_f32(const std::string& path, int I, int O, float*& w, float*& b) {
    const PackEntry* e = conv_weight(path, O, I, 3);
    if (!e) return err;
    const size_t n = (size_t)O * 9 * I;
    __half* tmp = A->get<__half>(n);
    w = A->get<float>(n);
    if (!tmp || !w) return err = fail(c, 4005, "weight arena exhausted");
    if (!A->measure) {
      int r = repack_conv_launch(st, ptr(e), O, I, 3, 3, tmp, 9 * I, 0, I);
      if (!r) r = cast_f16_to_f32_launch(st, tmp, n, w);
      if (r) return err = fail(c, r, "%s repack failed", path.c_str());
    }
    WSlot s;
    s.base = w; s.conv = 1; s.f32 = 1; s.N = O; s.I = I; s.ks = 3; s.ld = 9 * I; s.Ipad = I;
    record(path, s, n * sizeof(float));
    b = vec_f32(path + "/bias", O);
    return err;
  }
  // 1x1 conv OIHW f16 [O, I, 1, 1] -> f32 matrix [O][I], bias f32 (CUDA-core kernels)
  int mat_f32(const std::string& path, int I, int O, float*& w, float*& b) {
    const PackEntry* e = conv_weight(path, O, I, 1);
    if (!e) return err;
    w = A->get<float>((size_t)O * I);
    if (!w) return err = fail(c, 4005, "weight arena exhausted");
    if (!A->measure) { int r = cast_f16_to_f32_launch(st, ptr(e), (size_t)O * I, w); if (r) return err = fail(c, r, "%s cast failed", path.c_str()); }
    b = vec_f32(path + "/bias", O);
    return err;
  }
  // conv OIHW -> [O, ks*ks*Ipad (+ I2pad)]
  // Opad > O: the matrix (and bias) get zero rows up to Opad so the GEMM's N is a multiple of 4 (cv.O = Opad).
  Conv conv(const std::string& path, int I, int O, int ks, const std::string& skip_path = "", int I2 = 0, int Opad = 0) {
    Conv cv;
    cv.I = I; cv.O = O; cv.ks = ks; cv.Ipad = pad64(I); cv.I2 = I2; cv.I2pad = I2 ? pad64(I2) : 0;
    cv.Ktot = ks * ks * cv.Ipad + cv.I2pad;
    const int rows = Opad > O ? Opad : O;
    cv.w = A->get<__half>((size_t)rows * cv.Ktot);
    if (!cv.w) { err = fail(c, 4005, "weight arena exhausted"); return cv; }
    if (rows > O && !A->measure && cudaMemsetAsync(cv.w, 0, (size_t)rows * cv.Ktot * sizeof(__half), st) != cudaSuccess) {
      err = fail(c, 4011, "memset failed");
      return cv;
    }
    const PackEntry* e = conv_weight(path, O, I, ks);
    if (!e) return cv;
    if (!A->measure) { int r = repack_conv_launch(st, ptr(e), O, I, ks, ks, cv.w, cv.Ktot, 0, cv.Ipad); if (r) err = fail(c, r, "repack_conv failed"); }
    {
      WSlot s;
      s.base = cv.w; s.conv = 1; s.N = O; s.I = I; s.ks = ks; s.ld = cv.Ktot; s.Ipad = cv.Ipad;
      record(path, s, (size_t)O * cv.Ktot * sizeof(__half));
    }
    if (rows > O) {
      const PackEntry* be = need(path + "/bias", 1);
      cv.b = A->get<float>(rows);
      if (!be || !cv.b || (int)be->shape[0] != O) { if (!err) err = fail(c, 4012, "weight pack: '%s/bias' missing or mis-sized", path.c_str()); return cv; }
      if (!A->measure) {
        int r = (int)cudaMemsetAsync(cv.b, 0, rows * sizeof(float), st);
        if (!r) r = bias_to_f32_launch(st, ptr(be), O, cv.b, 0, 0);
        if (r) err = fail(c, r, "padded bias failed");
      }
      cv.O = rows;
    } else {
      cv.b = vec_f32(path + "/bias", O);
    }
    if (I2) {
      const PackEntry* s = conv_weight(skip_path, O, I2, 1);
      if (!s) return cv;
      const PackEntry* sb = need(skip_path + "/bias", 1);
      if (!sb) return cv;
      if (!A->measure) {
        int r = repack_conv_launch(st, ptr(s), O, I2, 1, 1, cv.w, cv.Ktot, ks * ks * cv.Ipad, cv.I2pad);
        if (!r) r = bias_to_f32_launch(st, ptr(sb), O, cv.b, 0, 1);
        if (r) err = fail(c, r, "skip repack failed");
      }
      WSlot sk;
      sk.base = cv.w; sk.conv = 1; sk.N = O; sk.I = I2; sk.ks = 1; sk.ld = cv.Ktot; sk.col0 = ks * ks * cv.Ipad; sk.Ipad = cv.I2pad;
      record(skip_path, sk, (size_t)O * cv.Ktot * sizeof(__half));
    }
    return cv;
  }
};

static int parse_pack(sdxl_ctx* c, const void* pack, size_t bytes, int on_device, PackView& pv,
                      std::vector<uint8_t>& host_table) {
  if (bytes < sizeof(PackHeader)) return fail(c, 4100, "weight pack too small");
  PackHeader h;
  if (on_device) CU(c, cudaMemcpy(&h, pack, sizeof h, cudaMemcpyDeviceToHost));
  else memcpy(&h, pack, sizeof h);
  if (memcmp(h.magic, "SDXLPK01", 8) != 0) return fail(c, 4101, "weight pack: bad magic");
  const size_t tbytes = (size_t)h.n_tensors * sizeof(PackEntry);
  if (sizeof h + tbytes > bytes) return fail(c, 4102, "weight pack: truncated table");
  host_table.resize(tbytes);
  if (on_device) CU(c, cudaMemcpy(host_table.data(), (const uint8_t*)pack + sizeof h, tbytes, cudaMemcpyDeviceToHost));
  else memcpy(host_table.data(), (const uint8_t*)pack + sizeof h, tbytes);
  const PackEntry* e = (const PackEntry*)host_table.data();
  for (uint32_t i = 0; i < h.n_tensors; ++i) {
    if (e[i].nbytes > bytes || e[i].offset > bytes - e[i].nbytes) return fail(c, 4103, "weight pack: tensor '%.*s' out of range", 119, e[i].name);
    if (e[i].offset % 16) return fail(c, 4104, "weight pack: tensor '%.*s' not 16B aligned", 119, e[i].name);
    if (e[i].ndim > 4 || e[i].dtype > 1) return fail(c, 4105, "weight pack: tensor '%.*s' has bad rank / dtype", 119, e[i].name);
    {
      uint64_t n = 1;   // element count, overflow-checked against the byte count the entry declares
      bool ok = true;
      for (uint32_t d = 0; d < e[i].ndim && ok; ++d) {
        if (e[i].shape[d] != 0 && n > UINT64_MAX / e[i].shape[d]) ok = false;
        else n *= e[i].shape[d];
      }
      const uint64_t esz = e[i].dtype ? 4 : 2;
      if (!ok || n > UINT64_MAX / esz || n * esz != e[i].nbytes)
        return fail(c, 4106, "weight pack: tensor '%.*s' declares %llu bytes but its shape needs a different size", 119, e[i].name,
                    (unsigned long long)e[i].nbytes);
    }
    std::string name(e[i].name, strnlen(e[i].name, sizeof e[i].name));
    pv.t[name] = e[i];
  }
  return 0;
}

// Parses a weight pack, makes it device-resident for the call (host packs are uploaded to a temporary copy) and runs fn(pv);
// the stream is synchronised before the copy is freed.
template <typename Fn>
static int with_device_pack(sdxl_ctx* c, const void* pack, size_t bytes, int pack_on_device, Fn fn) {
  PackView pv;
  std::vector<uint8_t> table;
  int r = parse_pack(c, pack, bytes, pack_on_device, pv, table);
  if (r) return r;
  void* dev_pack = nullptr;
  if (pack_on_device) {
    pv.dev = (const uint8_t*)pack;
  } else {
    CU(c, cudaMalloc(&dev_pack, bytes));
    cudaError_t e = cudaMemcpyAsync(dev_pack, pack, bytes, cudaMemcpyHostToDevice, c->stream);
    if (e != cudaSuccess) { cudaFree(dev_pack); return fail(c, (int)e, "pack upload failed"); }
    pv.dev = (const uint8_t*)dev_pack;
  }
  r = fn((const PackView&)pv);
  cudaError_t se = cudaStreamSynchronize(c->stream);
  if (dev_pack) cudaFree(dev_pack);
  if (!r && se != cudaSuccess) r = fail(c, (int)se, "weight re-layout failed: %s", cudaGetErrorString(se));
  return r;
}

// Sizes A by measuring: carve(Arena&) runs once against a measuring arena (placeholder pointers, no device work), A is
// allocated to the measured size, and carve runs again against A. carve must take the same buffers on both passes and write
// them on the ctx stream (A's fresh-memory fills are queued there).
template <typename Fn>
static int carve_measured(sdxl_ctx* c, Arena& A, int code, const char* what, Fn carve) {
  Arena meas;
  meas.measure = true;
  if (int r = carve(meas)) return r;
  if (A.init(meas.off)) return fail(c, code, "cannot allocate %zu bytes for %s", meas.off, what);
  A.stream = c->stream;
  A.fill = debug_fill_byte();
  return carve(A);
}

// Loads a model's weights into its weight arena m->warena.
template <typename M>
static int build_two_pass(M* m, const PackView& pv, int (*build)(M*, const PackView&, Arena&)) {
  return carve_measured(m->ctx, m->warena, 4203, "weights", [&](Arena& A) { return build(m, pv, A); });
}

// ================================================================================================
// launch plan
// ================================================================================================
enum OpKind { OP_IGEMM, OP_ATTN, OP_GN, OP_LN, OP_GEMV, OP_TEMB, OP_CONV_IN, OP_UPS, OP_PHASE, OP_CAST16,
              OP_SOFTMAX, OP_TRANSPOSE, OP_PQ, OP_EMBED, OP_ATTN_SMALL, OP_ACT, OP_LN_GATHER, OP_T2I_ADD, OP_PAG_IDENTITY, OP_FREEU,
              OP_COPY, OP_KIND_COUNT };
// the public profile entry points take caller arrays of SDXL_PROFILE_KINDS entries (include/sdxl_b200.h)
static_assert(OP_KIND_COUNT <= SDXL_PROFILE_KINDS, "profile arrays too small for the op kinds");
static const char* const kOpNames[] = {"igemm", "attention", "group_norm", "layer_norm", "gemv", "temb", "conv_in", "upsample",
                                       "phase_split", "cast16", "softmax_rows", "transpose16", "post_quant", "embed_tokens",
                                       "attention_small", "mlp_act", "ln_gather", "t2i_add", "pag_identity", "freeu", "copy"};
static_assert(sizeof(kOpNames) / sizeof(kOpNames[0]) == OP_KIND_COUNT, "one name per op kind");
struct Op {
  OpKind kind;
  double flops = 0;  // algorithmic FLOPs of this launch (igemm / attention), 0 for HBM-bound ops
  double flops_exec = 0;  // FLOPs the launch actually issues to the tensor cores (channel / key padding in, phase-decomposed upsample convs at their real cost)
  int block = -1;    // index into Plan::block_names (NVTX range of the reference block this launch belongs to)
  IgemmParams ig;
  AttnParams at;
  GnParams gn;
  struct { const float* x; const float* g; const float* b; float eps; int rows, C; __half* y; } ln;
  struct { const float* in; int in_bstride, Bv, K; const __half* W; int ldw; const float* bias; const float* add; int add_bstride, N, in_silu, out_silu; float* out; int out_bstride; } gv;
  struct { const float* t; int n, dim; float* out; } te;
  // x2 (nullable): second input source, channels [Cin, Cin + C2) (conv_in_cat_launch)
  struct { const float* x; int Bx, B, Cin, H, W; const float* w; const float* bias; int Cout; float* y; const float* add; int n_add;
           const float* x2; int n2, C2; } ci;
  struct { const float* x; int B, H, W, C; __half* y; } rs;  // upsample / phase split
  struct { const float* x; size_t n; __half* y; } cs;
  struct { const float* S; size_t lds; int rows, cols; float scale; __half* P; size_t ldp; } sm;
  struct { const __half* x; size_t ldx; int rows, cols; __half* y; size_t ldy; } tr;
  struct { const float* x; int B, C, HW; const float* w; const float* bias; float inv_scale; float* y; } pq;
  struct { const int* tokens; int rows, T, C, n_vocab; const __half* tok; const __half* pos; float* x; int* err; } em;
  struct { const __half* q; int q_pitch, q_col0; const __half* k; const __half* v; int kv_pitch, k_col0, v_col0, B, T, S, n_head;
           const __half* mask; int causal; __half* out; int ldo; int head_dim; } as;
  struct { const float* x; size_t n; int quick; __half* y; } ac;
  struct { const float* x; const int* idx; int B, T, C; const float* g; const float* b; float eps; float* y; } lg;
  struct { float* x; const float* F; long per_img; int B, n_hint; const int* t; const int* t_min; } ta;
  struct { const __half* qkv; int C; long rows; __half* out; } pi;   // PAG identity self-attention (pag_identity_launch)
  struct { float* r; int C; float* x; int Cx, B, H, W; const float* tw; const float* s; const float* b; } fu;   // FreeU (freeu_launch)
  struct { const void* src; void* dst; size_t bytes; } cp;   // device-to-device copy (a memcpy node in the graph)
};

struct Plan {
  int Bf = 0, Bx = 0, h = 0, w = 0;
  Arena arena;
  std::vector<Op> ops;
  float* x_in = nullptr;  // [Bx, Cin, h, w] f32 NCHW
  float* eps = nullptr;   // [Bf, h*w, eps_ld] f32 NHWC
  int eps_ld = 4;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t gexec = nullptr;
  int runs = 0;
  double flops = 0;  // algorithmic FLOPs of one run (2*MAC over Linear/conv/attention)
  std::vector<std::string> block_names;   // reference blocks in execution order (input_blocks/3, middle_block, ...)
  // DeepCache's cached forward (engine.cu, DESIGN.md §17): a second op list with its own graph and run count over this plan's
  // buffers. Its arena stays empty; its shapes, x_in and eps are this plan's.
  std::unique_ptr<Plan> cached;
  ~Plan() {
    if (gexec) cudaGraphExecDestroy(gexec);
    if (graph) cudaGraphDestroy(graph);
  }
};

// (Re)builds `plan` for new shapes: build(P, A) fills the plan and takes its buffers from A, P->arena sized by measuring.
// Dims are the plan's cache keys; on failure the plan is dropped.
template <typename Fn>
static int build_plan(sdxl_ctx* c, std::unique_ptr<Plan>& plan, int Bf, int Bx, int h, int w, Fn build) {
  CU(c, cudaStreamSynchronize(c->stream));   // the old plan may still be in flight
  plan.reset(new Plan());
  Plan* P = plan.get();
  P->Bf = Bf; P->Bx = Bx; P->h = h; P->w = w;
  int r = carve_measured(c, P->arena, 5011, "the plan's workspace", [&](Arena& A) { return build(P, &A); });
  if (r) plan.reset();
  return r;
}

struct ActView { const __half* p; int Bn, H, W, C; };

// Taps of a ks x ks stride-1 conv with padding ks/2 on A source `map`, in weight-column order (kh, kw).
static std::vector<IgemmSeg> conv_taps(int ks, int nkb, int map = 0) {
  std::vector<IgemmSeg> segs;
  for (int kh = 0; kh < ks; ++kh)
    for (int kw = 0; kw < ks; ++kw) segs.push_back({(int16_t)map, (int16_t)(kw - ks / 2), (int16_t)(kh - ks / 2), 0, nkb});
  return segs;
}
// Taps of a 3x3 stride-2 pad-1 conv (the UNet's Downsample) on the phase split of its input, [4][Bn][H/2][W/2][C]
// (phase_split_launch): tap kh reads input row 2i + kh - 1, i.e. phase (kh != 1) at row offset -1 for kh = 0; same for kw.
static std::vector<IgemmSeg> stride2_taps(int Bn, int nkb) {
  std::vector<IgemmSeg> segs;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      const int ph = (kh == 1) ? 0 : 1, pw = (kw == 1) ? 0 : 1;
      segs.push_back({0, (int16_t)((kw == 0) ? -1 : 0), (int16_t)((kh == 0) ? -1 : 0), (int16_t)((ph * 2 + pw) * Bn), nkb});
    }
  return segs;
}

// Fills the segments and the epilogue of p and configures it for the operands o (pixel box, N tile, pipeline depth,
// tensor maps). Output image outB x outH x outW, row pitch ldo; bias index b * bias_bstride + n.
static int igemm_setup(sdxl_ctx* c, IgemmParams& p, const IgemmOperands& o, const std::vector<IgemmSeg>& segs, int outH, int outW,
                       int outB, int mode, int geglu_bn, void* out, int out_f32, int ldo, const float* bias, int bias_bstride,
                       const float* res, int ldr) {
  if (segs.size() > (size_t)IGEMM_MAX_SEG) return fail(c, 5002, "too many igemm segments");
  p.nseg = (int)segs.size();
  for (int i = 0; i < p.nseg; ++i) p.seg[i] = segs[i];
  p.out = out; p.out_f32 = out_f32; p.ldo = ldo;
  p.bias = bias; p.bias_bstride = bias_bstride;
  p.res = res; p.ldr = ldr;
  int r = igemm_configure(p, o, outW, outH, outB, mode, geglu_bn);
  if (r) return fail(c, r, "igemm configuration failed (N=%d K=%d)", o.N, o.Ktot);
  return 0;
}
// One eager implicit-GEMM launch on the ctx stream (operator entry points, conditioning hoist, hint encoder).
static int igemm_run(sdxl_ctx* c, const IgemmOperands& o, const std::vector<IgemmSeg>& segs, int outH, int outW, int outB, int mode,
                     int geglu_bn, void* out, int out_f32, int ldo, const float* bias, const float* res, int ldr) {
  IgemmParams p{};
  if (int r = igemm_setup(c, p, o, segs, outH, outW, outB, mode, geglu_bn, out, out_f32, ldo, bias, 0, res, ldr)) return r;
  KL(c, igemm_launch(c->stream, p));
  return 0;
}

struct PlanBuilder {
  sdxl_ctx* c;
  Plan* P;
  Arena* A;
  int Bf;
  int err = 0;
  // shared scratch
  float* gn_partial = nullptr;

  template <typename T>
  T* buf(size_t n) {
    T* p = A->get<T>(n);
    if (!p && !err) err = fail(c, 5001, "plan arena exhausted");
    return p;
  }
  void add_flops(double f) {  // attribute to the op just pushed
    if (err || P->ops.empty()) return;
    P->ops.back().flops += f;
    P->flops += f;
  }
  // generic igemm op; segs reference view a0 (map 0) / a1 (map 1)
  void igemm(const ActView& a0, const ActView* a1, const std::vector<IgemmSeg>& segs, const __half* W, int N, int Ktot,
             int outH, int outW, int outB, int mode, int geglu_bn, void* out, int out_f32, int ldo, const float* bias,
             int bias_bstride, const float* res, int ldr) {
    if (err) return;
    Op op{};
    op.kind = OP_IGEMM;
    if (!A->measure) {   // a measuring arena hands out fake addresses: no tensor maps
      const IgemmOperands o{a0.p, a0.Bn, a0.H, a0.W, a0.C, a0.C, a1 ? a1->p : nullptr, a1 ? a1->Bn : 0, a1 ? a1->H : 0,
                            a1 ? a1->W : 0, a1 ? a1->C : 0, a1 ? a1->C : 0, W, N, Ktot};
      if ((err = igemm_setup(c, op.ig, o, segs, outH, outW, outB, mode, geglu_bn, out, out_f32, ldo, bias, bias_bstride, res, ldr))) return;
    }
    double kb = 0;
    for (const IgemmSeg& s : segs) kb += s.nkb;
    op.flops_exec = 2.0 * outB * outH * (double)outW * N * kb * 64.0;
    P->ops.push_back(op);
  }
  // names the reference block the following launches belong to
  void begin_block(const std::string& name) {
    if (err) return;
    P->block_names.push_back(name);
    cur_block = (int)P->block_names.size() - 1;
    first_op_of_block = P->ops.size();
  }
  void end_block() {
    for (size_t i = first_op_of_block; i < P->ops.size(); ++i) P->ops[i].block = cur_block;
    cur_block = -1;
  }
  int cur_block = -1;
  size_t first_op_of_block = 0;
  void linear(const __half* x, int M, const Lin& L, int mode, void* out, int out_f32, int ldo, const float* res, int ldr) {
    ActView a{x, 1, 1, M, L.K};
    std::vector<IgemmSeg> segs{{0, 0, 0, 0, L.Kpad / 64}};
    igemm(a, nullptr, segs, L.w, L.N, L.Kpad, 1, M, 1, mode, L.geglu_bn, out, out_f32, ldo, L.b, 0, res, ldr);
    add_flops(2.0 * M * (double)L.K * L.N);
  }
  // nearest-2x upsample + 3x3 conv (reference unet/mod.rs:742-751, autoencoder/mod.rs:311-319) as four 2x2 convolutions of the
  // source image x [Bn,H,W,I] (f32 -> f16 copy x16), one per output parity; out is [Bn,2H,2W,O] f32. The algorithmic FLOPs
  // (9 taps on the upsampled image) are what is accounted, a quarter per launch.
  void upconv(const float* x, int Bn, int H, int W, const Conv& cv, __half* x16, float* out) {
    if (err) return;
    {
      Op op{};
      op.kind = OP_CAST16;
      op.cs = {x, (size_t)Bn * H * W * cv.I, x16};
      P->ops.push_back(op);
    }
    ActView a{x16, Bn, H, W, cv.I};
    for (int pa = 0; pa < 2; ++pa)
      for (int pb = 0; pb < 2; ++pb) {
        std::vector<IgemmSeg> segs;
        for (int th = 0; th < 2; ++th)
          for (int tw = 0; tw < 2; ++tw)
            segs.push_back({0, (int16_t)(pb == 0 ? tw - 1 : tw), (int16_t)(pa == 0 ? th - 1 : th), 0, cv.Ipad / 64});
        igemm(a, nullptr, segs, cv.wup + (size_t)(pa * 2 + pb) * cv.O * cv.Ktot, cv.O, cv.Ktot, H, W, Bn, IGEMM_LINEAR, 0, out, 1, cv.O,
              cv.b, 0, nullptr, 0);
        if (err || P->ops.empty()) return;
        IgemmParams& ig = P->ops.back().ig;
        ig.opix_row = 4 * W; ig.opix_w = 2; ig.opix_off = pa * 2 * W + pb;
        add_flops(2.0 * Bn * H * W * 9.0 * cv.I * cv.O);
      }
  }
  // 3x3 stride-1 conv (+ optional fused 1x1 skip segment on a1)
  void conv3(const ActView& a, const ActView* skip, const Conv& cv, float* out, const float* bias, int bias_bstride,
             const float* res) {
    std::vector<IgemmSeg> segs = conv_taps(3, cv.Ipad / 64);
    if (skip) segs.push_back({1, 0, 0, 0, cv.I2pad / 64});
    igemm(a, skip, segs, cv.w, cv.O, cv.Ktot, a.H, a.W, a.Bn, IGEMM_LINEAR, 0, out, 1, cv.O, bias, bias_bstride, res, cv.O);
    add_flops(2.0 * a.Bn * a.H * a.W * (double)cv.O * (9.0 * cv.I + cv.I2));
  }
  void gn(const float* x1, int C1, const float* x2, int C2, int HW, const Norm& n, int silu, __half* y, __half* raw) {
    if (err) return;
    Op op{};
    op.kind = OP_GN;
    op.gn = GnParams{x1, C1, x2, C2, Bf, HW, 32, n.g, n.b, n.eps, silu, y, raw, gn_partial, 0};
    P->ops.push_back(op);
  }
  void ln(const float* x, const Norm& n, int rows, __half* y) {
    if (err) return;
    Op op{};
    op.kind = OP_LN;
    op.ln = {x, n.g, n.b, n.eps, rows, n.C, y};
    P->ops.push_back(op);
  }
  void gemv(const float* in, int in_bstride, int Bv, const Lin& L, const float* add, int add_bstride, int in_silu,
            int out_silu, float* out, int out_bstride) {
    if (err) return;
    for (int b0 = 0; b0 < Bv; b0 += 8) {
      Op op{};
      op.kind = OP_GEMV;
      const int nb = Bv - b0 < 8 ? Bv - b0 : 8;
      op.gv = {in + (size_t)b0 * in_bstride, in_bstride, nb, L.K, L.w, L.Kpad, L.b, add ? add + (size_t)b0 * add_bstride : nullptr,
               add_bstride, L.N, in_silu, out_silu, out + (size_t)b0 * out_bstride, out_bstride};
      P->ops.push_back(op);
    }
    P->flops += 2.0 * Bv * (double)L.K * L.N;
  }

};

static int exec_op(sdxl_ctx* c, Op& op) {
  cudaStream_t st = c->stream;
  switch (op.kind) {
    case OP_IGEMM: KL(c, igemm_launch(st, op.ig)); break;
    case OP_ATTN: KL(c, attention_launch(st, op.at)); break;
    case OP_GN: KL(c, gn_launch(st, op.gn)); c->launches++; break;
    case OP_LN: KL(c, layernorm_launch(st, op.ln.x, op.ln.g, op.ln.b, op.ln.eps, op.ln.rows, op.ln.C, op.ln.y)); break;
    case OP_GEMV:
      KL(c, gemv_launch(st, op.gv.in, op.gv.in_bstride, op.gv.Bv, op.gv.K, op.gv.W, op.gv.ldw, op.gv.bias, op.gv.add, op.gv.add_bstride,
                        op.gv.N, op.gv.in_silu, op.gv.out_silu, op.gv.out, op.gv.out_bstride));
      break;
    case OP_TEMB: KL(c, timestep_embedding_f32_launch(st, op.te.t, op.te.n, op.te.dim, 10000.f, op.te.out)); break;
    case OP_CONV_IN:
      if (op.ci.x2)
        KL(c, conv_in_cat_launch(st, op.ci.x, 1, op.ci.Bx, op.ci.B, op.ci.Cin, op.ci.x2, op.ci.n2, op.ci.C2, op.ci.H, op.ci.W, op.ci.w,
                                 op.ci.bias, op.ci.Cout, op.ci.y, op.ci.add, op.ci.n_add));
      else
        KL(c, conv_in_launch_t(st, op.ci.x, 1, op.ci.Bx, op.ci.B, op.ci.Cin, op.ci.H, op.ci.W, op.ci.w, op.ci.bias, op.ci.Cout, op.ci.y,
                               op.ci.add, op.ci.n_add));
      break;
    case OP_UPS: KL(c, upsample2x_launch(st, op.rs.x, op.rs.B, op.rs.H, op.rs.W, op.rs.C, op.rs.y)); break;
    case OP_PHASE: KL(c, phase_split_launch(st, op.rs.x, op.rs.B, op.rs.H, op.rs.W, op.rs.C, op.rs.y)); break;
    case OP_CAST16: KL(c, cast_f32_to_f16_launch(st, op.cs.x, op.cs.n, op.cs.y)); break;
    case OP_SOFTMAX: KL(c, softmax_rows_launch(st, op.sm.S, op.sm.lds, op.sm.rows, op.sm.cols, op.sm.scale, op.sm.P, op.sm.ldp)); break;
    case OP_TRANSPOSE: KL(c, transpose_f16_launch(st, op.tr.x, op.tr.ldx, op.tr.rows, op.tr.cols, op.tr.y, op.tr.ldy)); break;
    case OP_EMBED: KL(c, embed_tokens_launch(st, op.em.tokens, op.em.rows, op.em.T, op.em.C, op.em.n_vocab, op.em.tok, op.em.pos, op.em.x, op.em.err)); break;
    case OP_ATTN_SMALL:
      KL(c, attention_small_launch(st, op.as.q, op.as.q_pitch, op.as.q_col0, op.as.k, op.as.v, op.as.kv_pitch, op.as.k_col0, op.as.v_col0,
                                   op.as.B, op.as.T, op.as.S, op.as.n_head, op.as.mask, op.as.causal, op.as.out, op.as.ldo, op.as.head_dim));
      break;
    case OP_ACT: KL(c, mlp_act_launch(st, op.ac.x, op.ac.n, op.ac.quick, op.ac.y)); break;
    case OP_LN_GATHER: KL(c, ln_gather_f32_launch(st, op.lg.x, op.lg.idx, op.lg.B, op.lg.T, op.lg.C, op.lg.g, op.lg.b, op.lg.eps, op.lg.y)); break;
    case OP_PQ: KL(c, post_quant_launch(st, op.pq.x, op.pq.B, op.pq.C, op.pq.HW, op.pq.w, op.pq.bias, op.pq.inv_scale, op.pq.y)); break;
    case OP_T2I_ADD: KL(c, t2i_add_launch(st, op.ta.x, op.ta.F, op.ta.per_img, op.ta.B, op.ta.n_hint, op.ta.t, op.ta.t_min)); break;
    case OP_PAG_IDENTITY: KL(c, pag_identity_launch(st, op.pi.qkv, op.pi.C, op.pi.rows, op.pi.out)); break;
    case OP_FREEU:
      KL(c, freeu_launch(st, op.fu.r, op.fu.C, op.fu.x, op.fu.Cx, op.fu.B, op.fu.H, op.fu.W, op.fu.tw, op.fu.s, op.fu.b));
      break;
    case OP_COPY: KL(c, (int)cudaMemcpyAsync(op.cp.dst, op.cp.src, op.cp.bytes, cudaMemcpyDeviceToDevice, st)); break;
  }
  return 0;
}

static int run_plan_ops(sdxl_ctx* c, Plan* P) {
  static const bool no_graph = getenv("SDXL_B200_NO_GRAPH") != nullptr;
  if (P->gexec) {
    CU(c, cudaGraphLaunch(P->gexec, c->stream));
    c->launches += P->ops.size() + [&] { size_t g = 0; for (auto& o : P->ops) g += o.kind == OP_GN; return g; }();
    return 0;
  }
  const bool capture = !no_graph && P->runs >= 1;  // first run eager (sets func attributes), then capture
  if (capture) CU(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
  int r = 0;
  int open_block = -1;   // NVTX range per reference block (host side: visible in eager runs and during graph capture)
  for (auto& op : P->ops) {
    if (op.block != open_block) {
      if (open_block >= 0) nvtxRangePop();
      open_block = op.block;
      if (open_block >= 0) nvtxRangePushA(P->block_names[open_block].c_str());
    }
    r = exec_op(c, op);
    if (r) break;
  }
  if (open_block >= 0) nvtxRangePop();
  if (capture) {
    cudaGraph_t gph = nullptr;
    cudaError_t e = cudaStreamEndCapture(c->stream, &gph);
    if (r) { if (gph) cudaGraphDestroy(gph); return r; }
    if (e != cudaSuccess) return fail(c, (int)e, "graph capture failed: %s", cudaGetErrorString(e));
    P->graph = gph;
    e = cudaGraphInstantiate(&P->gexec, gph, 0);
    if (e != cudaSuccess) { P->gexec = nullptr; return fail(c, (int)e, "graph instantiate failed: %s", cudaGetErrorString(e)); }
    CU(c, cudaGraphLaunch(P->gexec, c->stream));
  }
  P->runs++;
  return r;
}

// Runs every op of the plan eagerly on the ctx stream between CUDA event pairs; ms[i] = device time of op i.
static int time_plan_ops(sdxl_ctx* c, Plan* P, std::vector<float>& ms) {
  const size_t n = P->ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) CU(c, cudaEventCreate(&e));
  int r = 0;
  CU(c, cudaEventRecord(ev[0], c->stream));
  for (size_t i = 0; i < n && !r; ++i) {
    r = exec_op(c, P->ops[i]);
    if (!r && cudaEventRecord(ev[i + 1], c->stream) != cudaSuccess) r = -2;
  }
  cudaError_t se = cudaStreamSynchronize(c->stream);
  ms.assign(n, 0.f);
  if (!r && se == cudaSuccess)
    for (size_t i = 0; i < n; ++i) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  if (se != cudaSuccess) return fail(c, (int)se, "profile run failed: %s", cudaGetErrorString(se));
  return r;
}

// Per-kernel-kind device time of one plan execution (time_plan_ops). kinds: see OpKind. Arrays hold SDXL_PROFILE_KINDS entries.
static int profile_plan_impl(sdxl_ctx* c, Plan* P, double* ms_by_kind, double* flops_by_kind, int* launches_by_kind) {
  std::vector<float> ms;
  const int r = time_plan_ops(c, P, ms);
  for (int k = 0; k < SDXL_PROFILE_KINDS; ++k) { ms_by_kind[k] = 0; flops_by_kind[k] = 0; launches_by_kind[k] = 0; }
  if (r) return r;
  for (size_t i = 0; i < ms.size(); ++i) {
    const int k = (int)P->ops[i].kind;
    if (k < 0 || k >= SDXL_PROFILE_KINDS) continue;
    ms_by_kind[k] += ms[i];
    flops_by_kind[k] += P->ops[i].flops;
    launches_by_kind[k] += (P->ops[i].kind == OP_GN) ? 2 : 1;
  }
  return 0;
}

// Per-op dump of one eager plan execution (time_plan_ops) as CSV: analysis aid for profiles/.
static int profile_dump_impl(sdxl_ctx* c, Plan* P, const char* path) {
  std::vector<float> ms;
  if (int r = time_plan_ops(c, P, ms)) return r;
  FILE* f = fopen(path, "w");
  if (!f) return fail(c, -3, "cannot open %s", path);
  fprintf(f, "op,kind,us,gflop,tflops,M_tiles,N,BN,Kblocks,T,S,heads,mode,out_f32,res\n");
  for (size_t i = 0; i < ms.size(); ++i) {
    const Op& o = P->ops[i];
    int mt = 0, N = 0, BN = 0, kb = 0, T = 0, S = 0, H = 0, mode = 0, of32 = 0, res = 0;
    if (o.kind == OP_IGEMM) {
      mt = o.ig.tilesW * o.ig.tilesH * o.ig.tilesB; N = o.ig.N; BN = o.ig.BN;
      mode = o.ig.mode; of32 = o.ig.out_f32; res = o.ig.res != nullptr;
      for (int s2 = 0; s2 < o.ig.nseg; ++s2) kb += o.ig.seg[s2].nkb;
    } else if (o.kind == OP_ATTN) { T = o.at.T; S = o.at.S; H = o.at.n_head; }
    fprintf(f, "%zu,%s,%.2f,%.3f,%.1f,%d,%d,%d,%d,%d,%d,%d,%d,%d,%d\n", i, kOpNames[o.kind], ms[i] * 1e3, o.flops * 1e-9,
            ms[i] > 0 ? o.flops / (ms[i] * 1e-3) * 1e-12 : 0.0, mt, N, BN, kb, T, S, H, mode, of32, res);
  }
  fclose(f);
  return 0;
}

// Stream-ordered staging buffers of one call, freed on the stream when it returns. get<T>(bytes): T says how a fresh buffer
// is filled under SDXL_B200_FILL (debug_fill).
struct TmpBufs {
  std::vector<void*> p;
  cudaStream_t st;
  int fill = debug_fill_byte();
  explicit TmpBufs(cudaStream_t s) : st(s) {}
  template <typename T>
  T* get(size_t bytes) {
    void* d = nullptr;
    if (cudaMallocAsync(&d, bytes ? bytes : 16, st) != cudaSuccess) return nullptr;
    p.push_back(d);
    if (fill >= 0) debug_fill((T*)d, bytes / sizeof(T), st, fill);
    return (T*)d;
  }
  ~TmpBufs() { for (void* d : p) cudaFreeAsync(d, st); }
};

// One adapter's term of one layer: the merge kernel's term (coef = s * c, or c alone for a DoRA term) and, for DoRA, the
// magnitude m (f32 [N] for axis 0, [I] for axis 1) and the user scale s (DESIGN.md §19).
struct AdapterTerm {
  LoraTerm t{};
  const float* m = nullptr;   // dora_scale; null: not a DoRA term
  int axis = 0;
  float s = 0.f;
};

static std::string shape_str(const PackEntry* e) {
  std::string r = "[";
  for (uint32_t i = 0; i < e->ndim && i < 4; ++i) r += (i ? "," : "") + std::to_string((unsigned long long)e->shape[i]);
  return r + "]";
}

// Replaces the active adapter set of a model whose slots are registered in S (include/sdxl_b200.h: sdxl_unet_set_adapters).
// Phase 1 reads and validates every adapter, expands LoKr factors given as products into scratch and allocates the backups and
// the scratch; nothing in the model is written before it has passed. Phase 2 restores the layers merged by the previous call,
// backs up the newly touched ones and merges. Queued on the ctx stream.
static int adapters_apply(sdxl_ctx* c, AdapterState& S, int n, const sdxl_adapter* ad) {
  if (n < 0 || n > SDXL_MAX_ADAPTERS) return fail(c, 4600, "set_adapters: n = %d outside [0, %d]", n, SDXL_MAX_ADAPTERS);
  if (n > 0 && !ad) return fail(c, 4601, "set_adapters: null adapter array");
  TmpBufs tmp(c->stream);
  std::map<std::string, std::vector<AdapterTerm>> terms;   // by layer path, adapters in call order
  static const char* kLeaves[] = {"lora_down", "lora_up", "alpha", "dora_scale", "diff", "hada_w1_a", "hada_w1_b", "hada_w2_a",
                                  "hada_w2_b", "lokr_w1", "lokr_w1_a", "lokr_w1_b", "lokr_w2", "lokr_w2_a", "lokr_w2_b"};
  for (int a = 0; a < n; ++a) {
    PackView pv;
    std::vector<uint8_t> table;
    if (!ad[a].pack) return fail(c, 4602, "set_adapters: adapter %d has a null pack", a);
    int r = parse_pack(c, ad[a].pack, ad[a].bytes, ad[a].pack_on_device, pv, table);
    if (r) { c->err = "adapter " + std::to_string(a) + ": " + c->err; return r; }
    if (ad[a].pack_on_device) {
      pv.dev = (const uint8_t*)ad[a].pack;
    } else {
      uint8_t* d = tmp.get<uint8_t>(ad[a].bytes);
      if (!d) return fail(c, 4603, "set_adapters: cannot allocate %zu bytes for adapter %d", ad[a].bytes, a);
      CU(c, cudaMemcpyAsync(d, ad[a].pack, ad[a].bytes, cudaMemcpyHostToDevice, c->stream));
      pv.dev = d;
    }
    // group the tensors by layer
    std::map<std::string, std::map<std::string, const PackEntry*>> layers;
    for (auto& kv : pv.t) {
      const size_t slash = kv.first.rfind('/');
      const std::string leaf = slash == std::string::npos ? kv.first : kv.first.substr(slash + 1);
      bool known = false;
      for (const char* l : kLeaves) known |= leaf == l;
      if (slash == std::string::npos || !known)
        return fail(c, 4604, "adapter %d: tensor '%s' is not <layer>/lora_down, <layer>/lora_up or <layer>/alpha, nor a LoHa, LoKr, "
                    "full-delta or dora_scale tensor (DESIGN.md §19)", a, kv.first.c_str());
      layers[kv.first.substr(0, slash)][leaf] = &kv.second;
    }
    for (auto& L : layers) {
      const std::string& path = L.first;
      auto it = S.slots.find(path);
      if (it == S.slots.end()) return fail(c, 4605, "adapter %d: '%s' is not a LoRA-able layer of this model", a, path.c_str());
      const WSlot& s = it->second;
      const int taps = s.ks * s.ks;
      auto get = [&](const char* leaf) -> const PackEntry* { auto f = L.second.find(leaf); return f == L.second.end() ? nullptr : f->second; };
      const char* fams[4][6] = {{"lora_down", "lora_up"}, {"hada_w1_a", "hada_w1_b", "hada_w2_a", "hada_w2_b"},
                                {"lokr_w1", "lokr_w1_a", "lokr_w1_b", "lokr_w2", "lokr_w2_a", "lokr_w2_b"}, {"diff"}};
      int fam = -1;
      const char* first = nullptr;
      for (int f = 0; f < 4; ++f)
        for (int i = 0; i < 6 && fams[f][i]; ++i)
          if (get(fams[f][i])) {
            if (fam >= 0 && fam != f)
              return fail(c, 4615, "adapter %d: '%s' holds two delta families ('%s' and '%s')", a, path.c_str(), first, fams[f][i]);
            fam = f; first = fams[f][i];
          }
      const PackEntry* al = get("alpha");
      const PackEntry* ds = get("dora_scale");
      if (fam < 0 && ds) return fail(c, 4621, "adapter %d: '%s/dora_scale' is on a layer without a delta", a, path.c_str());
      if (fam < 0) fam = 0;   // alpha alone: reported as a LoRA without factors
      for (int f = 0; f < 4; ++f)
        for (int i = 0; i < 6 && fams[f][i]; ++i) {
          const PackEntry* e = get(fams[f][i]);
          if (e && e->dtype != 0) return fail(c, 4607, "adapter %d: '%s/%s' must be f16", a, path.c_str(), fams[f][i]);
        }
      double alpha = 0.0;    // read when have_alpha; a finite negative alpha is used as given
      const bool have_alpha = al != nullptr;
      if (al) {
        const uint64_t esz = al->dtype ? 4 : 2;
        if (al->nbytes != esz) return fail(c, 4611, "adapter %d: '%s/alpha' must have one element", a, path.c_str());
        uint8_t raw[4] = {0, 0, 0, 0};
        if (ad[a].pack_on_device) {
          CU(c, cudaMemcpyAsync(raw, pv.dev + al->offset, esz, cudaMemcpyDeviceToHost, c->stream));
          CU(c, cudaStreamSynchronize(c->stream));
        } else {
          memcpy(raw, (const uint8_t*)ad[a].pack + al->offset, esz);
        }
        if (al->dtype) { float f; memcpy(&f, raw, 4); alpha = f; }
        else { __half_raw hr; memcpy(&hr.x, raw, 2); alpha = (double)__half2float(__half(hr)); }
        if (!isfinite(alpha)) return fail(c, 4612, "adapter %d: '%s/alpha' is not finite", a, path.c_str());
      }
      auto dev16 = [&](const PackEntry* e) { return (const __half*)(pv.dev + e->offset); };
      // columns of a [rows, I(, ks, ks)] factor as input channels: 2-D [rows, I * taps] or (convs) 4-D [rows, I, ks, ks]; -1 otherwise
      auto in_ch = [&](const PackEntry* e) -> long long {
        if (e->ndim == 2) return e->shape[1] % taps ? -1 : (long long)(e->shape[1] / taps);
        if (e->ndim == 4 && s.conv && e->shape[2] == (uint64_t)s.ks && e->shape[3] == (uint64_t)s.ks) return (long long)e->shape[1];
        return -1;
      };
      auto need = [&](const char* leaf) -> const PackEntry* {
        const PackEntry* e = get(leaf);
        if (!e) fail(c, 4616, "adapter %d: '%s/%s' is missing (%s)", a, path.c_str(), leaf, first);
        return e;
      };
      auto bad_shape = [&](const char* leaf, const char* want) {
        return fail(c, 4617, "adapter %d: '%s/%s' has shape %s, expected %s (N = %d, I = %d%s)", a, path.c_str(), leaf,
                    shape_str(get(leaf)).c_str(), want, s.N, s.I, s.conv ? (s.ks == 3 ? ", 3x3 conv" : ", 1x1 conv") : "");
      };
      AdapterTerm T;
      double rank = 1.0;       // the r of alpha / r
      bool use_alpha = true;
      if (fam == 0) {   // LoRA: the original checks and codes
        const PackEntry* dn = get("lora_down");
        const PackEntry* up = get("lora_up");
        if (!dn || !up) return fail(c, 4606, "adapter %d: '%s/%s' is missing", a, path.c_str(), dn ? "lora_up" : "lora_down");
        const uint64_t rk = dn->ndim ? dn->shape[0] : 0;
        const bool dn_ok = s.conv ? (dn->ndim == 4 && dn->shape[1] == (uint64_t)s.I && dn->shape[2] == (uint64_t)s.ks && dn->shape[3] == (uint64_t)s.ks)
                                  : (dn->ndim == 2 && dn->shape[1] == (uint64_t)s.I);
        if (!dn_ok || rk < 1 || rk > 4096)
          return fail(c, 4608, "adapter %d: '%s/lora_down' has shape [%llu,%llu,%llu,%llu] (ndim %u), expected [r, %d%s]", a, path.c_str(),
                      (unsigned long long)dn->shape[0], (unsigned long long)dn->shape[1], (unsigned long long)dn->shape[2],
                      (unsigned long long)dn->shape[3], dn->ndim, s.I, s.conv ? (s.ks == 3 ? ", 3, 3" : ", 1, 1") : "");
        const bool up_ok = s.conv ? (up->ndim == 4 && up->shape[0] == (uint64_t)s.N && up->shape[2] == 1 && up->shape[3] == 1)
                                  : (up->ndim == 2 && up->shape[0] == (uint64_t)s.N);
        if (!up_ok) return fail(c, 4609, "adapter %d: '%s/lora_up' has shape [%llu,%llu,...] (ndim %u), expected [%d, r%s]", a, path.c_str(),
                                (unsigned long long)up->shape[0], (unsigned long long)up->shape[1], up->ndim, s.N, s.conv ? ", 1, 1" : "");
        if (up->shape[1] != rk)
          return fail(c, 4610, "adapter %d: '%s': lora_down has rank %llu but lora_up has rank %llu", a, path.c_str(),
                      (unsigned long long)rk, (unsigned long long)up->shape[1]);
        T.t.kind = LORA_LORA; T.t.up = dev16(up); T.t.down = dev16(dn); T.t.r = (int)rk;
        rank = (double)rk;
      } else if (fam == 1) {   // LoHa
        const PackEntry* f[4];
        const char* nm[4] = {"hada_w1_a", "hada_w1_b", "hada_w2_a", "hada_w2_b"};
        for (int i = 0; i < 4; ++i) if (!(f[i] = need(nm[i]))) return 4616;
        uint64_t rk[2];
        for (int p = 0; p < 2; ++p) {
          const PackEntry* A = f[2 * p];
          const PackEntry* B = f[2 * p + 1];
          if (A->ndim != 2 || A->shape[0] != (uint64_t)s.N || A->shape[1] < 1 || A->shape[1] > 4096) return bad_shape(nm[2 * p], "[N, r]");
          if (in_ch(B) != s.I) return bad_shape(nm[2 * p + 1], s.conv ? "[r, I, kh, kw] or [r, I*kh*kw]" : "[r, I]");
          if (B->shape[0] != A->shape[1])
            return fail(c, 4618, "adapter %d: '%s': %s has rank %llu but %s has rank %llu", a, path.c_str(), nm[2 * p],
                        (unsigned long long)A->shape[1], nm[2 * p + 1], (unsigned long long)B->shape[0]);
          rk[p] = B->shape[0];
        }
        T.t.kind = LORA_LOHA;
        T.t.up = dev16(f[0]); T.t.down = dev16(f[1]); T.t.r = (int)rk[0];
        T.t.up2 = dev16(f[2]); T.t.down2 = dev16(f[3]); T.t.r2 = (int)rk[1];
        rank = (double)rk[0];
      } else if (fam == 2) {   // LoKr: each factor is staged as f32 (a product is expanded with coefficient 1)
        uint64_t prod_rank[2] = {0, 0};
        uint64_t rows[2], cols[2];       // w1 [a, b]; w2 [c, d * taps]
        float* fx[2];
        for (int w = 0; w < 2; ++w) {
          const std::string base = w ? "lokr_w2" : "lokr_w1";
          const PackEntry* full = get(base.c_str());
          const PackEntry* A = get((base + "_a").c_str());
          const PackEntry* B = get((base + "_b").c_str());
          if (full && (A || B))
            return fail(c, 4615, "adapter %d: '%s' holds both '%s' and '%s_%s'", a, path.c_str(), base.c_str(), base.c_str(), A ? "a" : "b");
          if (!full && !(A && B)) return fail(c, 4616, "adapter %d: '%s/%s%s' is missing (%s)", a, path.c_str(), base.c_str(),
                                              A ? "_b" : B ? "_a" : "", first);
          LoraMergeParams q{};
          q.nterm = 1; q.taps = 1; q.term[0].coef = 1.f;
          long long ich;
          if (full) {
            ich = w ? in_ch(full) : (full->ndim == 2 ? (long long)full->shape[1] : -1);
            if (ich < 1) return bad_shape(base.c_str(), w ? (s.conv ? "[c, d, kh, kw] or [c, d*kh*kw]" : "[c, d]") : "[a, b]");
            rows[w] = full->shape[0];
            q.term[0].kind = LORA_FULL; q.term[0].down = dev16(full);
          } else {
            const std::string an = base + "_a", bn = base + "_b";
            if (A->ndim != 2 || A->shape[1] < 1 || A->shape[1] > 4096) return bad_shape(an.c_str(), "[rows, r]");
            ich = w ? in_ch(B) : (B->ndim == 2 ? (long long)B->shape[1] : -1);
            if (ich < 1) return bad_shape(bn.c_str(), w ? (s.conv ? "[r, d, kh, kw] or [r, d*kh*kw]" : "[r, d]") : "[r, b]");
            if (B->shape[0] != A->shape[1])
              return fail(c, 4618, "adapter %d: '%s': %s has rank %llu but %s has rank %llu", a, path.c_str(), an.c_str(),
                          (unsigned long long)A->shape[1], bn.c_str(), (unsigned long long)B->shape[0]);
            rows[w] = A->shape[0];
            prod_rank[w] = A->shape[1];
            q.term[0].kind = LORA_LORA; q.term[0].up = dev16(A); q.term[0].down = dev16(B); q.term[0].r = (int)A->shape[1];
          }
          cols[w] = (uint64_t)ich * (w ? (uint64_t)taps : 1);
          if (rows[w] < 1 || rows[w] > (uint64_t)s.N || cols[w] < 1 || cols[w] > (uint64_t)s.I * taps)
            return fail(c, 4619, "adapter %d: '%s': the LoKr factor %s is larger than the layer (N = %d, I = %d)", a, path.c_str(),
                        base.c_str(), s.N, s.I);
          fx[w] = tmp.get<float>((size_t)rows[w] * cols[w] * sizeof(float));
          if (!fx[w]) return fail(c, 4624, "set_adapters: cannot allocate the LoKr factor %s of '%s'", base.c_str(), path.c_str());
          q.N = (int)rows[w]; q.Kd = (int)cols[w]; q.delta_out = fx[w];
          KL(c, lora_merge_launch(c->stream, q));
        }
        const uint64_t d = cols[1] / taps;
        if (rows[0] * rows[1] != (uint64_t)s.N || cols[0] * d != (uint64_t)s.I)
          return fail(c, 4619, "adapter %d: '%s': kron(lokr_w1 [%llu, %llu], lokr_w2 [%llu, %llu]) is not [N = %d, I = %d]", a, path.c_str(),
                      (unsigned long long)rows[0], (unsigned long long)cols[0], (unsigned long long)rows[1], (unsigned long long)d, s.N, s.I);
        if (prod_rank[0] && prod_rank[1] && prod_rank[0] != prod_rank[1])
          return fail(c, 4618, "adapter %d: '%s': lokr_w1_a has rank %llu but lokr_w2_a has rank %llu (LoKr factors given as "
                      "products must share the rank r of alpha / r)", a, path.c_str(),
                      (unsigned long long)prod_rank[0], (unsigned long long)prod_rank[1]);
        T.t.kind = LORA_LOKR; T.t.w1 = fx[0]; T.t.w2 = fx[1]; T.t.c = (int)rows[1]; T.t.d = (int)d;
        use_alpha = prod_rank[0] || prod_rank[1];
        rank = (double)(prod_rank[0] ? prod_rank[0] : prod_rank[1]);
      } else {   // full delta
        const PackEntry* e = get("diff");
        if (e->shape[0] != (uint64_t)s.N || in_ch(e) != s.I) return bad_shape("diff", s.conv ? "[N, I, kh, kw] or [N, I*kh*kw]" : "[N, I]");
        T.t.kind = LORA_FULL; T.t.down = dev16(e);
        use_alpha = false;
      }
      // c = alpha / r; the LoRA term's coefficient s * alpha / r is evaluated in that order, as before this family table
      const double num = use_alpha ? (have_alpha ? alpha : rank) : 1.0, den = use_alpha ? rank : 1.0;
      T.t.coef = (float)((double)ad[a].scale * num / den);
      if (ds) {
        if (s.up) return fail(c, 4622, "adapter %d: '%s/dora_scale': DoRA on an upsample conv is not supported (its 3x3 weight is not "
                              "retained, so the norm cannot be taken)", a, path.c_str());
        if (ds->dtype != 1) return fail(c, 4623, "adapter %d: '%s/dora_scale' must be f32", a, path.c_str());
        const uint64_t* sh = ds->shape;
        const bool row = (ds->ndim == 1 && sh[0] == (uint64_t)s.N) || (ds->ndim == 2 && sh[0] == (uint64_t)s.N && sh[1] == 1) ||
                         (ds->ndim == 4 && sh[0] == (uint64_t)s.N && sh[1] == 1 && sh[2] == 1 && sh[3] == 1);
        const bool col = (ds->ndim == 2 && sh[0] == 1 && sh[1] == (uint64_t)s.I) ||
                         (ds->ndim == 4 && sh[0] == 1 && sh[1] == (uint64_t)s.I && sh[2] == 1 && sh[3] == 1);
        if (!row && !col)
          return fail(c, 4620, "adapter %d: '%s/dora_scale' has shape %s, expected [%d], [%d,1], [%d,1,1,1] (rows) or [1,%d], [1,%d,1,1] "
                      "(input channels)", a, path.c_str(), shape_str(ds).c_str(), s.N, s.N, s.N, s.I, s.I);
        T.m = (const float*)(pv.dev + ds->offset);
        T.axis = row ? 0 : 1;
        T.s = ad[a].scale;
        T.t.coef = (float)(num / den);
      }
      terms[path].push_back(T);
    }
  }
  // scratch of the layers merged through an f32 delta (upsample convs, DoRA), sized for the largest, reused layer by layer
  float* delta = nullptr;   // the layer's summed delta
  float* ddw = nullptr;     // one DoRA term's delta
  double* dnorm = nullptr;
  {
    size_t nd = 0, nw = 0, nn = 0;
    for (auto& kv : terms) {
      const WSlot& s = S.slots[kv.first];
      const size_t e = (size_t)s.N * s.I * s.ks * s.ks;
      bool dora = false;
      for (auto& T : kv.second) dora |= T.m != nullptr;
      if (s.up || dora) nd = std::max(nd, e);
      if (dora) { nw = std::max(nw, e); nn = std::max(nn, (size_t)std::max(s.N, s.I)); }
    }
    if (nd && !(delta = tmp.get<float>(nd * sizeof(float))))
      return fail(c, 4614, "set_adapters: cannot allocate %zu bytes of merge scratch", nd * sizeof(float));
    if (nw && (!(ddw = tmp.get<float>(nw * sizeof(float))) || !(dnorm = tmp.get<double>(nn * sizeof(double)))))
      return fail(c, 4624, "set_adapters: cannot allocate %zu bytes of DoRA scratch", nw * sizeof(float) + nn * sizeof(double));
  }
  // backups of the buffers touched for the first time, one allocation (a failure leaves the model unchanged)
  {
    std::map<void*, size_t> fresh;   // buffer -> offset in the new allocation
    size_t total = 0;
    for (auto& kv : terms) {
      void* base = S.slots[kv.first].base;
      if (S.bufs[base].backup || fresh.count(base)) continue;
      fresh[base] = total;
      total += (S.bufs[base].bytes + 255) & ~size_t(255);
    }
    if (total) {
      uint8_t* mem = nullptr;
      if (cudaMalloc((void**)&mem, total) != cudaSuccess) return fail(c, 4613, "set_adapters: cannot allocate %zu bytes of weight backup", total);
      S.allocs.push_back(mem);
      for (auto& f : fresh) S.bufs[f.first].backup = mem + f.second;
    }
  }
  // phase 2: writes
  std::map<void*, bool> touched;
  for (auto& kv : terms) touched[S.slots[kv.first].base] = true;
  for (auto& kv : S.bufs) {
    AdapterState::Buf& b = kv.second;
    if (b.dirty) CU(c, cudaMemcpyAsync(kv.first, b.backup, b.bytes, cudaMemcpyDeviceToDevice, c->stream));
    else if (touched.count(kv.first)) CU(c, cudaMemcpyAsync(b.backup, kv.first, b.bytes, cudaMemcpyDeviceToDevice, c->stream));
    b.dirty = touched.count(kv.first) > 0;
  }
  for (auto& kv : terms) {
    const WSlot& s = S.slots[kv.first];
    const void* src = S.bufs[s.base].backup;
    LoraMergeParams p{};
    p.N = s.N; p.taps = s.ks * s.ks; p.Kd = s.I * p.taps;
    p.src = src; p.dst = s.base; p.f32 = s.f32;
    p.ld = s.ld; p.row0 = s.row0; p.col0 = s.col0; p.Ipad = s.Ipad; p.geglu_bn = s.geglu_bn;
    std::vector<const AdapterTerm*> plain, dora;   // non-DoRA terms, then DoRA terms, each in call order
    for (auto& T : kv.second) (T.m ? dora : plain).push_back(&T);
    p.nterm = (int)plain.size();
    for (int i = 0; i < p.nterm; ++i) p.term[i] = plain[i]->t;
    if (dora.empty() && !s.up) {
      KL(c, lora_merge_launch(c->stream, p));
      continue;
    }
    LoraMergeParams q = p;
    q.delta_out = delta;
    if (p.nterm) KL(c, lora_merge_launch(c->stream, q));
    else CU(c, cudaMemsetAsync(delta, 0, (size_t)p.N * p.Kd * sizeof(float), c->stream));
    if (s.up) {
      KL(c, lora_upconv_merge_launch(c->stream, (const __half*)src, delta, s.N, s.I, (__half*)s.base, s.Ipad));
      continue;
    }
    for (const AdapterTerm* T : dora) {
      LoraMergeParams w = p;
      w.nterm = 1; w.term[0] = T->t; w.delta_out = ddw;
      KL(c, lora_merge_launch(c->stream, w));
      KL(c, dora_norm_launch(c->stream, p, ddw, T->axis, dnorm));
      KL(c, dora_accum_launch(c->stream, p, ddw, T->m, dnorm, T->axis, T->s, delta));
    }
    p.nterm = 1;
    p.term[0] = LoraTerm{};
    p.term[0].kind = LORA_F32; p.term[0].w1 = delta; p.term[0].coef = 1.f;
    KL(c, lora_merge_launch(c->stream, p));
  }
  if (n == 0) {   // everything is restored: the backups go
    CU(c, cudaStreamSynchronize(c->stream));
    S.release();
  }
  return 0;
}
