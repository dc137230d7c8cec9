// Text-encoder front end of libsdxl_b200.so (C ABI: sdxl_clip_*). See engine_core.h for the shared machinery.
#include "engine_core.h"

// ================================================================================================
// Text encoders of the Embedder (SURVEY.md §8(f) rank 2): CLIP::{forward_hidden, forward_hidden_pooled}
//   CLIP / ResidualDecoderAttentionBlock / MultiHeadSelfAttention / MLP / QuickGELU
//                                   src/model/clip/mod.rs:82-147, 176-182, 228-245, 289-305, 315-319
//   weight names                    src/model/clip/load.rs:15-115
// 77-token sequences: Linear layers on the wgmma GEMM (one M tile), causal attention / activation / embedding on
// small CUDA-core kernels (clip_kernels.cu). Residual stream f32, GEMM operands f16 (the reference runs f32).
// ================================================================================================
struct CBlock {
  Norm attn_ln, mlp_ln;
  Lin qkv, out, fc1, fc2;
};
struct sdxl_clip {
  sdxl_ctx* ctx = nullptr;
  sdxl_clip_cfg cfg{};
  Arena warena;
  __half* tok_emb = nullptr;
  __half* pos_emb = nullptr;
  std::vector<CBlock> blocks;
  Norm ln_final;
  Lin proj;
  bool has_proj = false;
  // plan (keyed by batch, number of blocks run, captured hidden index, pooled)
  std::unique_ptr<Plan> plan;
  int pB = 0, p_nrun = 0, p_hidden = -1, p_pooled = 0;
  int* tokens_dev = nullptr;
  int* eot_dev = nullptr;
  int* err_dev = nullptr;
  float* hidden = nullptr;   // [B*T, C] result of forward_hidden / h_out
  float* pooled = nullptr;   // [B, embed_dim]
  AdapterState lora;         // LoRA-able weight slots, backups of merged layers (sdxl_clip_set_adapters)
  ~sdxl_clip() { if (tokens_dev) cudaFree(tokens_dev); }
};

static int load_clip_blocks(Loader& L, Arena& A, int n_layer, int C, int mlp, std::vector<CBlock>& blocks);

static int build_clip(sdxl_clip* m, const PackView& pv, Arena& A) {
  sdxl_ctx* c = m->ctx;
  const sdxl_clip_cfg& g = m->cfg;
  Loader L{c, &pv, &A, c->stream};
  L.reg = &m->lora;
  const int C = g.n_state;
  auto table = [&](const std::string& name, int rows, __half*& dst) {
    const PackEntry* e = L.need(name, 2);
    if (!e) return;
    if ((int)e->shape[0] != rows || (int)e->shape[1] != C) { L.err = fail(c, 4401, "weight pack: '%s' is [%llu,%llu], expected [%d,%d]", name.c_str(), (unsigned long long)e->shape[0], (unsigned long long)e->shape[1], rows, C); return; }
    dst = A.get<__half>((size_t)rows * C);
    if (!dst) { L.err = fail(c, 4005, "weight arena exhausted"); return; }
    if (!A.measure && cudaMemcpyAsync(dst, L.ptr(e), (size_t)rows * C * sizeof(__half), cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess)
      L.err = fail(c, 4402, "embedding copy failed");
  };
  table("token_embedding/weight", g.n_vocab, m->tok_emb);
  table("position_embedding/weight", g.n_ctx, m->pos_emb);
  if (L.err) return L.err;
  if (int r = load_clip_blocks(L, A, g.n_layer, C, 4 * C, m->blocks)) return r;
  m->ln_final = L.norm("layer_norm", C);
  m->has_proj = pv.find("text_projection") != nullptr;
  if (m->has_proj) {
    const PackEntry* e = L.need("text_projection", 2);
    if (!e) return L.err;
    if ((int)e->shape[0] != C || (int)e->shape[1] != g.embed_dim) return fail(c, 4404, "text_projection is [%llu,%llu], expected [%d,%d]", (unsigned long long)e->shape[0], (unsigned long long)e->shape[1], C, g.embed_dim);
    Lin& P = m->proj;
    P.K = C; P.Kpad = Loader::pad64(C); P.N = g.embed_dim;
    P.w = A.get<__half>((size_t)g.embed_dim * P.Kpad);
    if (!P.w) return fail(c, 4005, "weight arena exhausted");
    if (!A.measure) { int r = transpose_linear_launch(c->stream, L.ptr(e), C, g.embed_dim, P.w, P.Kpad, 0, 0); if (r) return fail(c, r, "text_projection re-layout failed"); }
  }
  return L.err;
}

// The n_layer pre-LN blocks blocks/<i>/{attn_ln, mlp_ln, attn/{query,key,value,out}, mlp/{fc1,fc2}} of width C, MLP width mlp:
// shared by the text encoders and the vision towers.
static int load_clip_blocks(Loader& L, Arena& A, int n_layer, int C, int mlp, std::vector<CBlock>& blocks) {
  sdxl_ctx* c = L.c;
  blocks.clear();
  const int Cpad = Loader::pad64(C);
  for (int i = 0; i < n_layer && !L.err; ++i) {
    const std::string bp = "blocks/" + std::to_string(i);
    CBlock b;
    b.attn_ln = L.norm(bp + "/attn_ln", C);
    b.mlp_ln = L.norm(bp + "/mlp_ln", C);
    // fused q/k/v projection (clip/mod.rs:229-231: three Linears with bias on the same input)
    b.qkv.K = C; b.qkv.Kpad = Cpad; b.qkv.N = 3 * C;
    b.qkv.w = A.get<__half>((size_t)3 * C * Cpad);
    b.qkv.b = A.get<float>((size_t)3 * C);
    if (!b.qkv.w || !b.qkv.b) { L.err = fail(c, 4005, "weight arena exhausted"); break; }
    const char* names[3] = {"query", "key", "value"};
    for (int j = 0; j < 3 && !L.err; ++j) {
      const std::string lp = bp + "/attn/" + names[j];
      L.lin_into(lp, b.qkv.w, Cpad, j * C, C, C, 0);
      const PackEntry* be = L.need(lp + "/bias", 1);
      if (!be) break;
      if ((int)be->shape[0] != C) { L.err = fail(c, 4403, "weight pack: '%s/bias' mis-sized", lp.c_str()); break; }
      if (!A.measure) { int r = bias_to_f32_launch(c->stream, L.ptr(be), C, b.qkv.b + j * C, 0, 0); if (r) L.err = fail(c, r, "bias_to_f32 failed"); }
    }
    b.out = L.linear(bp + "/attn/out", C, C, true);
    b.fc1 = L.linear(bp + "/mlp/fc1", C, mlp, true);
    b.fc2 = L.linear(bp + "/mlp/fc2", mlp, C, true);
    blocks.push_back(b);
  }
  return L.err;
}

extern "C" void sdxl_clip_destroy(sdxl_clip* m) {
  if (!m) return;
  cudaStreamSynchronize(m->ctx->stream);
  delete m;
}

extern "C" int sdxl_clip_load(sdxl_ctx* c, const sdxl_clip_cfg* cfg, const void* pack, size_t bytes, int pack_on_device, sdxl_clip** out) {
  if (!c || !cfg || !pack || !out) return fail(c, -1, "sdxl_clip_load: null argument");
  *out = nullptr;
  if (cfg->n_head < 1 || cfg->n_state != cfg->n_head * 64) return fail(c, 4410, "text encoder head dim must be 64 (n_state=%d, n_head=%d)", cfg->n_state, cfg->n_head);
  if (cfg->n_ctx < 1 || cfg->n_ctx > 1024 || cfg->n_layer < 1 || cfg->n_vocab < 1 || cfg->embed_dim < 1) return fail(c, 4411, "bad text encoder config");
  CU(c, cudaSetDevice(c->device));
  std::unique_ptr<sdxl_clip> m(new sdxl_clip());
  m->ctx = c;
  m->cfg = *cfg;
  int r = with_device_pack(c, pack, bytes, pack_on_device, [&](const PackView& pv) { return build_two_pass(m.get(), pv, build_clip); });
  if (r) return r;
  if (cudaMalloc((void**)&m->tokens_dev, (size_t)(64 * cfg->n_ctx + 64 + 16) * sizeof(int)) != cudaSuccess) return fail(c, 4412, "cudaMalloc failed");
  m->eot_dev = m->tokens_dev + 64 * cfg->n_ctx;
  m->err_dev = m->eot_dev + 64;
  *out = m.release();
  return 0;
}

// Plan buffers of the residual stream and the block operands.
struct ClipStream { float *xa, *xb; __half *a16, *qkv16, *ao16; float* h32; __half* h16; };

// Emits blocks [0, n_run) on the stream that starts in s.xa (shared by the text encoders and the vision towers). When capture >= 0
// the stream entering block `capture` is preserved and *hidden points at it. Returns the final stream.
static float* clip_block_ops(PlanBuilder& B, const std::vector<CBlock>& blocks, int n_run, int capture, float** hidden, const ClipStream& s,
                             int Bn, int T, int C, int n_head, int head_dim, int mlp, int causal, int quick) {
  Plan* P = B.P;
  const int M = Bn * T;
  float* x = s.xa;
  *hidden = nullptr;
  for (int i = 0; i < n_run && !B.err; ++i) {
    const CBlock& b = blocks[i];
    float* xn = x;
    if (i == capture) {  // keep the input of this block: write the updated stream into the other buffer
      *hidden = x;
      xn = (x == s.xa) ? s.xb : s.xa;
    }
    // x = x + attn(attn_ln(x), causal mask)    (clip/mod.rs:177-179)
    B.ln(x, b.attn_ln, M, s.a16);
    B.linear(s.a16, M, b.qkv, IGEMM_LINEAR, s.qkv16, 0, 3 * C, nullptr, 0);
    {
      Op op{};
      op.kind = OP_ATTN_SMALL;
      op.as = {s.qkv16, 3 * C, 0, s.qkv16, s.qkv16, 3 * C, C, 2 * C, Bn, T, T, n_head, nullptr, causal, s.ao16, C, head_dim};
      P->ops.push_back(op);
      B.add_flops(4.0 * Bn * T * (double)T * C);
    }
    B.linear(s.ao16, M, b.out, IGEMM_LINEAR, xn, 1, C, x, C);
    // x = x + mlp(mlp_ln(x))
    B.ln(xn, b.mlp_ln, M, s.a16);
    B.linear(s.a16, M, b.fc1, IGEMM_LINEAR, s.h32, 1, mlp, nullptr, 0);
    {
      Op op{};
      op.kind = OP_ACT;
      op.ac = {s.h32, (size_t)M * mlp, quick ? 1 : 0, s.h16};
      P->ops.push_back(op);
    }
    B.linear(s.h16, M, b.fc2, IGEMM_LINEAR, xn, 1, C, xn, C);
    x = xn;
  }
  return x;
}

// n_run blocks are executed; when capture >= 0 the stream entering block `capture` is preserved as the hidden output.
static int build_clip_plan(sdxl_clip* m, Plan* P, Arena* A, int n_run, int capture, int pooled) {
  sdxl_ctx* c = m->ctx;
  const sdxl_clip_cfg& g = m->cfg;
  PlanBuilder B{c, P, A, P->Bf};
  P->ops.clear();
  P->flops = 0;
  const int Bn = P->Bf, T = g.n_ctx, C = g.n_state, M = Bn * T;
  float* xa = B.buf<float>((size_t)M * C);
  float* xb = B.buf<float>((size_t)M * C);
  __half* a16 = B.buf<__half>((size_t)M * C);
  __half* qkv16 = B.buf<__half>((size_t)M * 3 * C);
  __half* ao16 = B.buf<__half>((size_t)M * C);
  float* h32 = B.buf<float>((size_t)M * 4 * C);
  __half* h16 = B.buf<__half>((size_t)M * 4 * C);
  float* pin = B.buf<float>((size_t)Bn * C);
  m->pooled = B.buf<float>((size_t)Bn * g.embed_dim);
  if (B.err) return B.err;
  {
    Op op{};
    op.kind = OP_EMBED;
    op.em = {m->tokens_dev, M, T, C, g.n_vocab, m->tok_emb, m->pos_emb, xa, m->err_dev};
    P->ops.push_back(op);
  }
  const ClipStream s{xa, xb, a16, qkv16, ao16, h32, h16};
  float* x = clip_block_ops(B, m->blocks, n_run, capture, &m->hidden, s, Bn, T, C, g.n_head, 64, 4 * C, 1, g.quick_gelu);
  if (capture < 0 || capture >= n_run) m->hidden = x;
  if (pooled && !B.err) {
    // features of the end-of-text position: layer_norm(x)[b, argmax(tokens[b])] (@ text_projection)   (clip/mod.rs:130-141)
    Op op{};
    op.kind = OP_LN_GATHER;
    op.lg = {x, m->eot_dev, Bn, T, C, m->ln_final.g, m->ln_final.b, m->ln_final.eps, m->has_proj ? pin : m->pooled};
    P->ops.push_back(op);
    if (m->has_proj) B.gemv(pin, C, Bn, m->proj, nullptr, 0, 0, 0, m->pooled, g.embed_dim);
  }
  return B.err;
}

static int clip_run(sdxl_clip* m, int Bn, const int32_t* tokens_host, int n_run, int capture, int pooled) {
  sdxl_ctx* c = m->ctx;
  const sdxl_clip_cfg& g = m->cfg;
  if (!tokens_host) return fail(c, -1, "null tokens");
  if (Bn < 1 || Bn > 64) return fail(c, 5201, "text encoder batch must be 1..64 (got %d)", Bn);
  if (n_run < 0 || n_run > g.n_layer) return fail(c, 5202, "hidden_idx %d out of range (n_layer %d)", n_run, g.n_layer);
  CU(c, cudaSetDevice(c->device));
  if (!m->plan || m->pB != Bn || m->p_nrun != n_run || m->p_hidden != capture || m->p_pooled != pooled) {
    if (int r = build_plan(c, m->plan, Bn, Bn, 0, 0, [&](Plan* P, Arena* A) { return build_clip_plan(m, P, A, n_run, capture, pooled); }))
      return r;
    m->pB = Bn; m->p_nrun = n_run; m->p_hidden = capture; m->p_pooled = pooled;
  }
  // eot_indices = tokens.argmax(1): first position of the largest id (clip/mod.rs:130)
  std::vector<int> meta(64 + 1, 0);
  for (int b = 0; b < Bn; ++b) {
    int best = 0;
    for (int t = 1; t < g.n_ctx; ++t)
      if (tokens_host[b * g.n_ctx + t] > tokens_host[b * g.n_ctx + best]) best = t;
    meta[b] = best;
  }
  CU(c, cudaMemcpyAsync(m->tokens_dev, tokens_host, (size_t)Bn * g.n_ctx * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(m->eot_dev, meta.data(), 65 * sizeof(int), cudaMemcpyHostToDevice, c->stream));  // also clears err_dev
  CU(c, cudaStreamSynchronize(c->stream));  // meta / tokens_host are pageable host memory
  int r = run_plan_ops(c, m->plan.get());
  if (r) return r;
  int err = 0;
  CU(c, cudaMemcpyAsync(&err, m->err_dev, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  if (err) return fail(c, 5203, "token id outside [0, %d) (the reference's embedding lookup panics)", g.n_vocab);
  return 0;
}

static int clip_copy_out(sdxl_clip* m, const float* src, size_t n, float* dst, int on_host) {
  sdxl_ctx* c = m->ctx;
  if (!dst) return 0;
  CU(c, cudaMemcpyAsync(dst, src, n * sizeof(float), on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  if (on_host) CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}

extern "C" int sdxl_clip_forward_hidden(sdxl_clip* m, int Bn, const int32_t* tokens_host, int hidden_idx, float* hidden_out, int out_on_host) {
  if (!m || !hidden_out) return fail(m ? m->ctx : nullptr, -1, "sdxl_clip_forward_hidden: null argument");
  int r = clip_run(m, Bn, tokens_host, hidden_idx, -1, 0);
  if (r) return r;
  return clip_copy_out(m, m->hidden, (size_t)Bn * m->cfg.n_ctx * m->cfg.n_state, hidden_out, out_on_host);
}
extern "C" int sdxl_clip_forward_hidden_pooled(sdxl_clip* m, int Bn, const int32_t* tokens_host, int hidden_idx, float* hidden_out,
                                               float* pooled_out, int out_on_host) {
  if (!m || !hidden_out || !pooled_out) return fail(m ? m->ctx : nullptr, -1, "sdxl_clip_forward_hidden_pooled: null argument");
  if (hidden_idx < 0 || hidden_idx >= m->cfg.n_layer) return fail(m->ctx, 5204, "hidden_idx %d out of range: the reference returns an uninitialised tensor there (clip/mod.rs:120-126)", hidden_idx);
  int r = clip_run(m, Bn, tokens_host, m->cfg.n_layer, hidden_idx, 1);
  if (r) return r;
  r = clip_copy_out(m, m->hidden, (size_t)Bn * m->cfg.n_ctx * m->cfg.n_state, hidden_out, out_on_host);
  if (r) return r;
  return clip_copy_out(m, m->pooled, (size_t)Bn * (m->has_proj ? m->cfg.embed_dim : m->cfg.n_state), pooled_out, out_on_host);
}
// LoRA adapters (include/sdxl_b200.h; merge in engine_core.h: adapters_apply). Nothing derived from the weights is cached
// outside the weight arena, so the plan needs no refresh.
extern "C" int sdxl_clip_set_adapters(sdxl_clip* m, int n, const sdxl_adapter* adapters) {
  if (!m) return -1;
  CU(m->ctx, cudaSetDevice(m->ctx->device));
  return adapters_apply(m->ctx, m->lora, n, adapters);
}
extern "C" double sdxl_clip_plan_flops(const sdxl_clip* m) { return (m && m->plan) ? m->plan->flops : 0.0; }


// ================================================================================================
// CLIP vision tower (HF CLIPVisionModelWithProjection; the image encoder of IP-Adapter, DESIGN.md §9):
//   x = pre_layrnorm([class_embedding ; patch_conv(pixels)] + position_embedding)
//   n_layer pre-LN blocks (clip_block_ops: no causal mask, exact-erf GELU unless quick_gelu, head dim n_state / n_head)
//   image_embeds = post_layernorm(x[:, 0]) @ visual_projection
// The p x p stride-p patch conv is one GEMM on igemm over patchify's rows; class / position / pre_layrnorm is one kernel writing
// the f32 residual stream; the pooled token reuses ln_gather_f32 (index 0) and gemv.
// ================================================================================================
struct sdxl_clip_vision {
  sdxl_ctx* ctx = nullptr;
  sdxl_clip_vision_cfg cfg{};
  Arena warena;
  Lin patch;                 // [n_state, Kpad], columns (c, kh, kw)
  __half* cls = nullptr;     // [n_state]
  __half* pos = nullptr;     // [T, n_state]
  Norm pre_ln, post_ln;
  std::vector<CBlock> blocks;
  Lin proj;                  // visual_projection [proj_dim, n_state]
  std::unique_ptr<Plan> plan;
  int pN = 0;
  int p_hidden = -1;         // the plan's hidden_idx (blocks run, no pooled output), or -1: all blocks and image_embeds
  __half* patch16 = nullptr; // plan buffers of the embedding steps, run before the plan
  float* patches = nullptr;
  float* x = nullptr;
  float* hidden = nullptr;   // the stream after the plan's blocks
  float* embeds = nullptr;
  int tokens() const { return (cfg.image_size / cfg.patch_size) * (cfg.image_size / cfg.patch_size) + 1; }
};

static int build_clip_vision(sdxl_clip_vision* m, const PackView& pv, Arena& A) {
  sdxl_ctx* c = m->ctx;
  const sdxl_clip_vision_cfg& g = m->cfg;
  const int C = g.n_state, p = g.patch_size, T = m->tokens(), K = 3 * p * p;
  Loader L{c, &pv, &A, c->stream};
  {
    const PackEntry* e = L.conv_weight("patch_embedding", C, 3, p);
    if (!e) return L.err;
    Lin& P = m->patch;
    P.K = K; P.Kpad = Loader::pad64(K); P.N = C;
    P.w = A.get<__half>((size_t)C * P.Kpad);
    if (!P.w) return fail(c, 4005, "weight arena exhausted");
    if (!A.measure) {   // OIHW rows [C, 3*p*p] into the zero-padded K-major matrix
      CU(c, cudaMemsetAsync(P.w, 0, (size_t)C * P.Kpad * sizeof(__half), c->stream));
      CU(c, cudaMemcpy2DAsync(P.w, (size_t)P.Kpad * sizeof(__half), L.ptr(e), (size_t)K * sizeof(__half), (size_t)K * sizeof(__half), C,
                              cudaMemcpyDeviceToDevice, c->stream));
    }
  }
  auto table = [&](const std::string& name, int ndim, int rows, __half*& dst) {
    const PackEntry* e = L.need(name, ndim);
    if (!e) return;
    if ((ndim == 1 && (int)e->shape[0] != C) || (ndim == 2 && ((int)e->shape[0] != rows || (int)e->shape[1] != C))) {
      L.err = fail(c, 4421, "weight pack: '%s' has the wrong shape (expected %d x %d)", name.c_str(), rows, C);
      return;
    }
    dst = A.get<__half>((size_t)rows * C);
    if (!dst) { L.err = fail(c, 4005, "weight arena exhausted"); return; }
    if (!A.measure && cudaMemcpyAsync(dst, L.ptr(e), (size_t)rows * C * sizeof(__half), cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess)
      L.err = fail(c, 4402, "embedding copy failed");
  };
  table("class_embedding", 1, 1, m->cls);
  table("position_embedding/weight", 2, T, m->pos);
  if (L.err) return L.err;
  m->pre_ln = L.norm("pre_layernorm", C);
  if (int r = load_clip_blocks(L, A, g.n_layer, C, g.mlp_dim, m->blocks)) return r;
  m->post_ln = L.norm("post_layernorm", C);
  if (L.err) return L.err;
  {   // visual_projection [n_state, proj_dim] ([in, out], no bias; named like text_projection, without /weight)
    const PackEntry* e = L.need("visual_projection", 2);
    if (!e) return L.err;
    if ((int)e->shape[0] != C || (int)e->shape[1] != g.proj_dim)
      return fail(c, 4423, "visual_projection is [%llu,%llu], expected [%d,%d]", (unsigned long long)e->shape[0], (unsigned long long)e->shape[1], C, g.proj_dim);
    Lin& P = m->proj;
    P.K = C; P.Kpad = Loader::pad64(C); P.N = g.proj_dim;
    P.w = A.get<__half>((size_t)g.proj_dim * P.Kpad);
    if (!P.w) return fail(c, 4005, "weight arena exhausted");
    if (!A.measure) { int r = transpose_linear_launch(c->stream, L.ptr(e), C, g.proj_dim, P.w, P.Kpad, 0, 0); if (r) return fail(c, r, "visual_projection re-layout failed"); }
  }
  return 0;
}

extern "C" int sdxl_clip_vision_load(sdxl_ctx* c, const sdxl_clip_vision_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                     sdxl_clip_vision** out) {
  if (!c || !cfg || !pack || !out) return fail(c, -1, "sdxl_clip_vision_load: null argument");
  *out = nullptr;
  const int hd = cfg->n_head > 0 ? cfg->n_state / cfg->n_head : 0;
  if (cfg->n_head < 1 || cfg->n_state != cfg->n_head * hd || hd % 8 || hd > 128)
    return fail(c, 4420, "vision encoder head dim must be a multiple of 8 up to 128 (n_state=%d, n_head=%d)", cfg->n_state, cfg->n_head);
  if (cfg->n_layer < 1 || cfg->mlp_dim < 8 || cfg->mlp_dim % 8 || cfg->proj_dim < 1 || cfg->patch_size < 1 ||
      cfg->image_size < cfg->patch_size || cfg->image_size % cfg->patch_size || cfg->n_state % 8)
    return fail(c, 4422, "bad vision encoder config");
  CU(c, cudaSetDevice(c->device));
  std::unique_ptr<sdxl_clip_vision> m(new sdxl_clip_vision());
  m->ctx = c;
  m->cfg = *cfg;
  int r = with_device_pack(c, pack, bytes, pack_on_device, [&](const PackView& pv) { return build_two_pass(m.get(), pv, build_clip_vision); });
  if (r) return r;
  *out = m.release();
  return 0;
}

extern "C" void sdxl_clip_vision_destroy(sdxl_clip_vision* m) {
  if (!m) return;
  cudaStreamSynchronize(m->ctx->stream);
  delete m;
}

// n_run blocks; pooled: then post_layernorm of the class token and visual_projection into m->embeds.
static int build_vision_plan(sdxl_clip_vision* m, Plan* P, Arena* A, int n_run, int pooled) {
  sdxl_ctx* c = m->ctx;
  const sdxl_clip_vision_cfg& g = m->cfg;
  PlanBuilder B{c, P, A, P->Bf};
  P->ops.clear();
  P->flops = 0;
  const int N = P->Bf, T = m->tokens(), C = g.n_state, M = N * T;
  m->patch16 = B.buf<__half>((size_t)N * (T - 1) * m->patch.Kpad);
  m->patches = B.buf<float>((size_t)N * (T - 1) * C);
  const ClipStream s{B.buf<float>((size_t)M * C), B.buf<float>((size_t)M * C), B.buf<__half>((size_t)M * C), B.buf<__half>((size_t)M * 3 * C),
                     B.buf<__half>((size_t)M * C), B.buf<float>((size_t)M * g.mlp_dim), B.buf<__half>((size_t)M * g.mlp_dim)};
  int* idx0 = pooled ? B.buf<int>(N) : nullptr;
  float* pin = pooled ? B.buf<float>((size_t)N * C) : nullptr;
  m->embeds = pooled ? B.buf<float>((size_t)N * g.proj_dim) : nullptr;
  if (B.err) return B.err;
  if (pooled && !A->measure) CU(c, cudaMemsetAsync(idx0, 0, N * sizeof(int), c->stream));   // the class token of every image
  m->x = s.xa;
  float* unused = nullptr;
  float* x = clip_block_ops(B, m->blocks, n_run, -1, &unused, s, N, T, C, g.n_head, C / g.n_head, g.mlp_dim, 0, g.quick_gelu);
  m->hidden = x;
  if (B.err || !pooled) return B.err;
  Op op{};
  op.kind = OP_LN_GATHER;
  op.lg = {x, idx0, N, T, C, m->post_ln.g, m->post_ln.b, m->post_ln.eps, pin};
  P->ops.push_back(op);
  B.gemv(pin, C, N, m->proj, nullptr, 0, 0, 0, m->embeds, g.proj_dim);
  return B.err;
}

// Embeds the pixels and runs the plan for (N, hidden_idx); hidden_idx = -1: every block and image_embeds. The result is m->hidden
// (and m->embeds), queued on the ctx stream.
static int vision_run(sdxl_clip_vision* m, int N, const float* pixels, int on_host, int hidden_idx) {
  sdxl_ctx* c = m->ctx;
  const sdxl_clip_vision_cfg& g = m->cfg;
  if (N < 1 || N > 256) return fail(c, 5205, "vision encoder batch must be 1..256 (got %d)", N);
  CU(c, cudaSetDevice(c->device));
  if (!m->plan || m->pN != N || m->p_hidden != hidden_idx) {
    const int n_run = hidden_idx < 0 ? g.n_layer : hidden_idx;
    if (int r = build_plan(c, m->plan, N, N, 0, 0, [&](Plan* P, Arena* A) { return build_vision_plan(m, P, A, n_run, hidden_idx < 0); }))
      return r;
    m->pN = N;
    m->p_hidden = hidden_idx;
  }
  const int S = g.image_size, T = m->tokens(), C = g.n_state;
  const size_t in_bytes = (size_t)N * 3 * S * S * sizeof(float);
  TmpBufs tmp(c->stream);
  const float* px = pixels;
  if (on_host) {
    float* d = tmp.get<float>(in_bytes);
    if (!d) return fail(c, 5206, "vision encoder: cannot allocate %zu bytes for the pixels", in_bytes);
    CU(c, cudaMemcpyAsync(d, pixels, in_bytes, cudaMemcpyHostToDevice, c->stream));
    px = d;
  }
  const Lin& Pt = m->patch;
  const int rows = N * (T - 1);
  KL(c, patchify_launch(c->stream, px, N, S, g.patch_size, Pt.Kpad, m->patch16));
  const IgemmOperands o{m->patch16, 1, 1, rows, Pt.Kpad, Pt.Kpad, nullptr, 0, 0, 0, 0, 0, Pt.w, Pt.N, Pt.Kpad};
  if (int r = igemm_run(c, o, {{0, 0, 0, 0, Pt.Kpad / 64}}, 1, rows, 1, IGEMM_LINEAR, 0, m->patches, 1, C, nullptr, nullptr, 0)) return r;
  KL(c, vision_embed_ln_launch(c->stream, m->patches, m->cls, m->pos, N, T, C, m->pre_ln.g, m->pre_ln.b, m->pre_ln.eps, m->x));
  return m->plan->ops.empty() ? 0 : run_plan_ops(c, m->plan.get());   // hidden_idx = 0: the embedding alone
}

extern "C" int sdxl_clip_vision_encode(sdxl_clip_vision* m, int N, const float* pixels, int on_host, float* image_embeds_out) {
  if (!m || !pixels || !image_embeds_out) return fail(m ? m->ctx : nullptr, -1, "sdxl_clip_vision_encode: null argument");
  sdxl_ctx* c = m->ctx;
  if (int r = vision_run(m, N, pixels, on_host, -1)) return r;
  const size_t out_bytes = (size_t)N * m->cfg.proj_dim * sizeof(float);
  CU(c, cudaMemcpyAsync(image_embeds_out, m->embeds, out_bytes, on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  if (on_host) CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}

extern "C" int sdxl_clip_vision_encode_hidden(sdxl_clip_vision* m, int N, const float* pixels, int on_host, int hidden_idx, float* hidden_out) {
  if (!m || !pixels || !hidden_out) return fail(m ? m->ctx : nullptr, -1, "sdxl_clip_vision_encode_hidden: null argument");
  sdxl_ctx* c = m->ctx;
  if (hidden_idx < 0 || hidden_idx > m->cfg.n_layer)
    return fail(c, 5207, "hidden_idx %d outside [0, n_layer = %d]", hidden_idx, m->cfg.n_layer);
  if (int r = vision_run(m, N, pixels, on_host, hidden_idx)) return r;
  const size_t out_bytes = (size_t)N * m->tokens() * m->cfg.n_state * sizeof(float);
  CU(c, cudaMemcpyAsync(hidden_out, m->hidden, out_bytes, on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  if (on_host) CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}
