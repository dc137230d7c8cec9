// UNet / sampler front end of libsdxl_b200.so: context entry points, the UNet weight loader (re-layout on device), the
// UNet launch plan, the DDIM/CFG sampler loop and the operator-level entry points of include/sdxl_b200.h. The shared
// machinery (arena, pack parsing, launch plan, CUDA-graph replay) is in engine_core.h; the latent decoder / encoder is
// vae.cu, the text encoders clip.cu, the tokenizers tokenizer.cpp. No torch, no cuBLAS/cuDNN: every device op is one of
// this library's own sm_90a kernels.
//
// Structure mirrored from the reference (file:line relative to the reference root):
//   UNet::forward               src/model/unet/mod.rs:449-493
//   UNetConfig::init (blocks)   src/model/unet/mod.rs:72-430
//   ResBlock / SpatialTransformer / TransformerBlock / MHA / GEGLU
//                               src/model/unet/mod.rs:1082-1106, 820-845, 885-891, 1005-1023, 942-956
//   Diffuser::{sample_latent, sample_latent_with_inpainting, refine_latent, diffuse_latent*,
//              forward_diffuser, get_alpha}
//                               src/model/stablediffusion/mod.rs:317-541
#include "engine_core.h"
#include "schedule.h"

#include <set>

// ================================================================================================
// context
// ================================================================================================
extern "C" int sdxl_ctx_create(int device, void* cuda_stream, sdxl_ctx** out) {
  if (!out) return -1;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device >= n) {
    fprintf(stderr, "sdxl_b200: no CUDA device %d (this library has no CPU fallback)\n", device);
    return -2;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return -3;
  if (prop.major != 9 || prop.minor != 0) {
    fprintf(stderr, "sdxl_b200: device %d is sm_%d%d; this library contains sm_90a code only\n", device,
            prop.major, prop.minor);
    return -4;
  }
  if (cudaSetDevice(device) != cudaSuccess) return -5;
  sdxl_ctx* c = new sdxl_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  if (cuda_stream) {
    c->stream = (cudaStream_t)cuda_stream;
  } else {
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
      delete c;
      return -6;
    }
    c->own_stream = true;
  }
  *out = c;
  return 0;
}
extern "C" void sdxl_ctx_destroy(sdxl_ctx* c) {
  if (!c) return;
  cudaStreamSynchronize(c->stream);
  if (c->own_stream) cudaStreamDestroy(c->stream);
  delete c;
}
extern "C" const char* sdxl_last_error(const sdxl_ctx* c) { return c ? c->err.c_str() : "null ctx"; }
extern "C" int sdxl_ctx_synchronize(sdxl_ctx* c) {
  CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}
extern "C" uint64_t sdxl_ctx_launch_count(const sdxl_ctx* c) { return c ? c->launches : 0; }
extern "C" int sdxl_debug_fill(void) { return debug_fill_byte(); }

// ================================================================================================
// model
// ================================================================================================
struct TBlock {
  Norm n1, n2, n3;
  Lin qkv, out1;      // self-attention (fused [3C, C])
  Lin q2, kv2, out2;  // cross-attention (kv fused [2C, ctx])
  Lin ff1, ff2;
};
struct STrans { Norm norm; Lin proj_in, proj_out; std::vector<TBlock> blocks; int C = 0, n_head = 0; };
struct Res {
  Norm n_in, n_out;
  Conv conv_in, conv_out;  // conv_out carries the fused skip 1x1 segment when Cin != Cout
  int Cin = 0, Cout = 0, temb_off = 0;
  bool has_skip = false;
};
// BT_MID: the middle block (ResBlock, SpatialTransformer, ResBlock); the others are the Block types below.
enum BlockType { BT_CONV, BT_RES, BT_DOWN, BT_REST, BT_RESTU, BT_RESU, BT_MID };
static bool has_transformer(BlockType t) { return t == BT_REST || t == BT_RESTU || t == BT_MID; }
static bool has_upsample(BlockType t) { return t == BT_RESU || t == BT_RESTU; }

struct Block {
  BlockType type = BT_RES;
  Res res;
  STrans st;
  Conv conv;  // BT_DOWN, upsample conv (BT_CONV, the first conv, has its own fields)
};

// One block of the UNet as sdxl_b200/config.py::block_program lists it. `level` is the resolution it runs at (latent >> level);
// a downsample reads its level and writes the next, an upsampling output block writes the previous one.
struct BlockSpec {
  BlockType type;
  std::string path;
  int c_in, c_out;
  int depth;   // transformer depth
  int level;
};
struct BlockProgram { std::vector<BlockSpec> ins; BlockSpec mid; std::vector<BlockSpec> outs; };

// Input / middle / output blocks exactly as UNetConfig::init builds them (reference unet/mod.rs:115-173, 238-248, 250-328).
static BlockProgram block_program(const sdxl_unet_cfg& g) {
  const int mc = g.model_channels, nl = g.n_levels;
  auto ch = [&](int level) { return g.channel_mults[level] * mc; };
  BlockProgram p;
  p.ins.push_back({BT_CONV, "input_blocks/0", g.in_channels, mc, 0, 0});
  int idx = 1;
  for (int level = 0; level < nl; ++level) {
    const int c_in = ch(std::max(level - 1, 0)), c_out = ch(level);
    const bool tr = level == 1 || level == 2;
    for (int k = 0; k < 2; ++k) {
      const int ci = k == 0 ? c_in : c_out;
      if (tr) p.ins.push_back({BT_REST, "input_blocks/" + std::to_string(idx), ci, c_out, g.transformer_depths[level], level});
      else p.ins.push_back({BT_RES, "input_blocks/" + std::to_string(idx), ci, c_out, 0, level});
      idx += 1;
    }
    if (level != nl - 1) {
      p.ins.push_back({BT_DOWN, "input_blocks/" + std::to_string(idx), c_out, c_out, 0, level});
      idx += 1;
    }
  }
  const int cm = ch(nl - 1);
  p.mid = {BT_MID, "middle_block", cm, cm, g.transformer_depths[nl - 1], nl - 1};
  idx = 0;
  for (int level = nl - 1; level >= 0; --level) {
    const int next_level = level != nl - 1 ? level + 1 : level;
    const int c_out = ch(level);
    const int cins[3] = {ch(next_level) + c_out, 2 * c_out, c_out + ch(std::max(level - 1, 0))};
    const bool tr = level == 1 || level == 2;
    for (int k = 0; k < 3; ++k) {
      const bool up = k == 2 && (tr || level != 0);
      if (tr) p.outs.push_back({up ? BT_RESTU : BT_REST, "output_blocks/" + std::to_string(idx), cins[k], c_out, g.transformer_depths[level], level});
      else p.outs.push_back({up ? BT_RESU : BT_RES, "output_blocks/" + std::to_string(idx), cins[k], c_out, 0, level});
      idx += 1;
    }
  }
  return p;
}

// The inpainting UNet (DESIGN.md §12, diffusers' stable-diffusion-xl-1.0-inpainting-0.1): its input is the latent (out_channels),
// the mask (1) and the masked image's latent (out_channels), concatenated. The one-source first conv takes at most 8 channels, so
// no configuration loadable without this layout has it.
static bool inpaint_layout(const sdxl_unet_cfg& g) { return g.in_channels > 8 && g.in_channels == 2 * g.out_channels + 1; }
// The instruction-editing UNet (DESIGN.md §21, diffusers' sdxl-instructpix2pix-768): its input is the latent and the source image's
// latent (out_channels each), concatenated. Only the explicit flag selects it: an 8 -> 4 cfg without it keeps its 8-channel latent.
static bool edit_layout(const sdxl_unet_cfg& g) { return g.edit_layout != 0; }
// Channels of the latent the forward and the sampler take: out_channels on an inpainting or edit UNet (the rest comes from the
// attachment), in_channels otherwise.
static int latent_channels(const sdxl_unet_cfg& g) { return inpaint_layout(g) || edit_layout(g) ? g.out_channels : g.in_channels; }

struct Plan;
struct Sampler;
struct TimeSlot { int t; float tf; };   // one write of the timestep: lround(t) and t
struct ControlAttach;
struct IpAttach;
struct T2IAttach;

// The latent extent (h, w) an attachment was made for, and its row count n: image b of a batch reads its row b % n.
struct Extent {
  int n = 0, h = 0, w = 0;
  bool operator==(const Extent& o) const { return n == o.n && h == o.h && w == o.w; }
};

// An attached inpainting condition (sdxl_unet_set_inpaint_condition): f32 NCHW [n, in_channels - out_channels, h, w], owned.
struct InpaintAttach {
  Extent ext;
  Arena mem;
  float* cond = nullptr;
};

// An attached source image of an edit UNet (sdxl_unet_set_edit_image): its latent f32 NCHW [n, out_channels, h, w], owned, and s_img.
// The first conv reads the plan's per-row copy (sdxl_unet::plan_edit), refreshed from here whenever either changes.
struct EditAttach {
  Extent ext;
  float image_guidance = 0.f;
  Arena mem;
  float* latent = nullptr;
};

// Perturbed-attention guidance (sdxl_unet_set_pag, DESIGN.md §14): the self-attentions that run as the identity on the perturbed
// rows (one flag per transformer block in execution order), the guidance scales, and the perturbed rows of a direct forward.
struct PagAttach {
  float scale = 0.f, adaptive = 0.f;
  std::vector<uint8_t> layers;
  int forward_rows = 0;
};

// FreeU (sdxl_unet_set_freeu, DESIGN.md §15): its four values on the device, [s1, s2, b1, b2], read by every OP_FREEU launch, so
// a change of values keeps the plan and its CUDA graph.
struct FreeuAttach {
  Arena mem;
  float* vals = nullptr;
};

// DeepCache (sdxl_unet_set_deepcache, DESIGN.md §17): the shallow branch the plan's cached list runs, the sampler's full-step interval
// and the kind of forward a direct sdxl_unet_forward* runs.
struct DeepcacheAttach {
  int branch = 0, interval = 1;
  bool forward_cached = false;
};

// Roles of the conditioning rows. The sampler's batch is row groups of n_img rows each: [cond | uncond] with CFG, then a perturbed
// group with PAG ([cond | uncond | ptb]; the refiner: [cond] or [cond | ptb]). The perturbed rows are conditional rows. An edit UNet
// with CFG runs [cond | img | uncond], both of the last two with the negative prompt. n_img = 0: a plain batch, every row conditional.
struct RowLayout {
  int n_img = 0;
  bool uncond = false;   // group 1 is the unconditional one
  bool uncond2 = false;  // so is group 2 (image guidance)
  bool negative(int r) const { return (uncond && r / n_img == 1) || (uncond2 && r / n_img == 2); }
};

// Embeddings, first conv, input blocks and middle block: the part of the UNet a ControlNet copies.
struct EncoderHalf {
  sdxl_ctx* ctx = nullptr;
  sdxl_unet_cfg cfg{};
  Arena warena;  // re-laid-out weights
  Lin t1, t2, l1, l2;      // time / label MLPs
  Lin temb_all;            // concatenated lin_embed of every ResBlock [sumC, 4mc], bias folded with conv_in bias
  float* conv0_w = nullptr;  // first conv [mc][3][3][4] f32
  float* conv0_b = nullptr;
  std::vector<Block> in_blocks;
  Res mid_res1, mid_res2;
  STrans mid_st;
  std::vector<const TBlock*> tblocks;   // every transformer block of the model in execution order (one hoisted K/V each)
};

// The step-invariant conditioning of one model (the UNet or an attached ControlNet) at one (B, n_ctx): the label MLP and the
// cross-attention K/V of every transformer block, hoisted out of the plan by hoist_model.
struct HoistedCond {
  Arena mem;
  int condB = 0, n_ctx = 0;
  float* lab1 = nullptr;       // [B, 4mc]
  float* label_emb = nullptr;  // [B, 4mc]
  std::vector<__half*> kv;     // per transformer block [B*n_ctx, 2C]
};

struct sdxl_controlnet : EncoderHalf {
  sdxl_controlnet_cfg ncfg{};
  float* hint0_w = nullptr;  // first hint conv [c0][3][3][hint_in] f32 (CUDA-core kernel)
  float* hint0_b = nullptr;
  std::vector<Conv> hint;    // the other hint convs in order: c_k -> c_k, c_k -> c_k+1 (stride 2), ..., c_last -> mc
  std::vector<Conv> zero;    // zero_convs/0..n-1 (one per skip tensor), then middle_block_out
};

struct sdxl_unet : EncoderHalf {
  std::vector<Block> out_blocks;
  Norm norm_out;
  Conv conv_out;
  __half* conv_out_w2 = nullptr;   // [O, 2*Ktot] = [W | W]: head conv on the hi/lo-split activation
  std::vector<double> alphas;  // the alphas_cumprod table in effect: alphas_loaded, or the one sdxl_unet_set_prediction gave
  std::vector<double> alphas_loaded;   // host copy of the record's table (f16-stored values widened)
  int prediction = SDXL_PREDICTION_EPSILON;   // sdxl_unet_set_prediction: what the UNet's output is, and guidance rescale's phi
  float guidance_rescale = 0.f;
  // conditioning state: the retained inputs and the hoisted conditioning; cond.condB / cond.n_ctx are its shape (0: not set)
  Arena imem;
  int ctx_pitch = 0;
  __half* ctx16 = nullptr;     // [B*n_ctx, ctx_pitch]
  float* y32 = nullptr;        // [B, adm]
  HoistedCond cond;
  // plan
  std::unique_ptr<Plan> plan;
  std::unique_ptr<Sampler> sampler;
  int* t_dev = nullptr;        // the timestep on the device: the int the T2I-Adapter window compares, then (t_dev + 1) the float the embedding reads
  TimeSlot* t_pinned = nullptr;
  int t_slot = 0;              // ring position in t_pinned (per model: independent contexts never share it)
  AdapterState lora;           // LoRA-able weight slots, backups of merged layers (sdxl_unet_set_adapters)
  std::vector<std::unique_ptr<ControlAttach>> controls;   // sdxl_unet_set_controls, in call order
  std::unique_ptr<IpAttach> ip;   // sdxl_unet_set_image_prompts
  std::unique_ptr<T2IAttach> t2i; // sdxl_unet_set_t2i_adapters
  std::unique_ptr<InpaintAttach> inpaint;   // sdxl_unet_set_inpaint_condition
  std::unique_ptr<EditAttach> edit;         // sdxl_unet_set_edit_image
  std::unique_ptr<PagAttach> pag;           // sdxl_unet_set_pag
  std::unique_ptr<FreeuAttach> freeu;       // sdxl_unet_set_freeu
  std::unique_ptr<DeepcacheAttach> deepcache;   // sdxl_unet_set_deepcache
  uint64_t plan_builds = 0;
  int plan_ptb = 0;               // trailing rows of the current plan that take PAG's identity self-attentions
  int plan_dc = -1;               // DeepCache branch of the current plan's cached list (-1: none)
  bool dc_feature = false;        // a full run of the current plan has kept DeepCache's feature
  float* plan_edit = nullptr;     // edit UNet: the first conv's condition per row of the current plan, f32 NCHW [Bf, out_channels, h, w]
  int plan_edit_zero = 0;         // its trailing rows that are zero (the sampler's unconditional group with image guidance)
  RowLayout rows;                 // roles of the conditioning rows
  ~sdxl_unet() {
    if (t_dev) cudaFree(t_dev);
    if (t_pinned) cudaFreeHost(t_pinned);
  }
};

// One attached ControlNet: its scaled zero convs, the encoded hint and its hoisted conditioning.
struct ControlAttach {
  const sdxl_controlnet* net = nullptr;
  float scale = 1.f;
  Extent ext;                     // n: the hint's n_hint
  Arena mem;                      // zero-conv copies f16(s*W) / s*b, hint_emb f32 NHWC [n_hint, h, w, mc]
  std::vector<Lin> zero;
  float* hint_emb = nullptr;
  HoistedCond cond;               // the net's own conditioning at the UNet's conditioning shape
};

// One perceiver layer of the IP-Adapter Plus Resampler (include/sdxl_b200.h), width W: the attention's LayerNorms of the image
// features (ln1) and of the latents (ln2), its projections without biases, and the feed-forward block.
struct PerceiverLayer {
  Norm ln1, ln2, ln_ff;
  Lin to_q, to_kv, to_out;  // [W, W], [2W, W] (K rows, then V), [W, W]
  Lin fc1, fc2;             // [4W, W], [W, 4W]
};

// IP-Adapter (DESIGN.md §9): the image-token projection (base: proj + norm; Plus: the Resampler) and, per UNet transformer block
// in execution order, the fused [ip_key | ip_value] projection of the image tokens (N = 2C, K = context_dim).
struct sdxl_ip_adapter {
  sdxl_ctx* ctx = nullptr;
  sdxl_ip_adapter_cfg cfg{};
  Arena warena;
  Lin proj;                 // [T * context_dim, D]
  Norm norm;                // over context_dim, eps 1e-5
  // Plus (cfg.resampler_depth > 0)
  float* latents = nullptr; // [Q, W]
  Lin proj_in, proj_out;    // [W, D], [context_dim, W]
  Norm norm_out;            // over context_dim
  std::vector<PerceiverLayer> layers;
  std::vector<Lin> kv;
  bool plus() const { return cfg.resampler_depth > 0; }
};

// One image prompt's token rows for one conditioning batch and their K/V, source-major: [n_sources, condB, S_ip / n_sources, ...]
// (an unmasked prompt is one source of S_ip tokens; a masked one is one source per image), so each source is a dense batch of rows.
struct IpRows {
  Arena mem;
  int condB = 0;
  __half* rows = nullptr;      // [condB * S_ip, context_dim]
  std::vector<__half*> kv;     // per transformer block [condB * S_ip, 2C]
};

// One prompt of the attached image-prompt set: the projected tokens of the prompts and of the negatives, the per-block scales,
// the masks resized to every level's queries, and the image K/V hoisted for the current conditioning rows.
struct IpPrompt {
  const sdxl_ip_adapter* ad = nullptr;
  int n_batch = 0, n_images = 0, S_ip = 0;
  int mask_h = 0, mask_w = 0;  // pixel extent of the masks; 0: unmasked
  __half* tok_pos = nullptr;   // [n_batch, S_ip, context_dim]
  __half* tok_neg = nullptr;   // [n_batch, S_ip, context_dim]
  float* scales = nullptr;     // one per transformer block, read by the attention kernel
  float* masks = nullptr;      // masked: per image, per level l the f32 [(h >> l) * (w >> l)] query weights (ip_mask_off)
  IpRows cond;
  int n_sources() const { return mask_h ? n_images : 1; }
};

// The attached image-prompt set (sdxl_unet_set_image_prompts), in call order.
struct IpAttach {
  Arena mem;                   // every prompt's tokens, scales and masks
  std::vector<IpPrompt> prompts;
};

// Offset in IpPrompt::masks of image i's weights at level l of a UNet with n_levels levels (ip_mask_off(a, n, n_images, 0): the
// floats of all images).
static size_t ip_mask_off(const IpPrompt& a, int n_levels, int i, int l) {
  const int h = a.mask_h / 8, w = a.mask_w / 8;
  size_t per = 0, off = 0;
  for (int k = 0; k < n_levels; ++k) {
    if (k == l) off = per;
    per += (size_t)(h >> k) * (w >> k);
  }
  return (size_t)i * per + off;
}

// T2I-Adapter (DESIGN.md §11, diffusers FullAdapterXL): conv_in on the pixel-unshuffled hint, then per level k an optional 1x1 in_conv
// (k = 1, 2) and n_res_blocks resnets x + block2(relu(block1(x))).
struct T2IRes { Conv block1, block2; };
struct sdxl_t2i_adapter {
  sdxl_ctx* ctx = nullptr;
  sdxl_t2i_adapter_cfg cfg{};
  int ch[4] = {0, 0, 0, 0};   // (mc*m0, mc*m1, mc*m2, mc*m2)
  Arena warena;
  Conv conv_in;
  Conv in_conv[2];            // body/1/in_conv, body/2/in_conv
  std::vector<T2IRes> res[4];
};

// The attached T2I-Adapter set: the scaled sum of the features F_k, f32 NHWC [n_hint, Hk, Wk, Ck], and the timestep window.
struct T2IAttach {
  Extent ext;                       // n: the hints' n_hint
  int C[4] = {}, H[4] = {}, W[4] = {};
  size_t points[3] = {};            // input blocks (indices into the block program) after which F_0..F_2 are added; F_3 after the middle
  Arena mem;
  float* F[4] = {};
  int* t_min = nullptr;             // device: features are added when t >= *t_min
};


static int geglu_bn_for(int n_out /*4C*/) {
  for (int hb = 128; hb >= 32; hb >>= 1)
    if (n_out % hb == 0) return 2 * hb;
  return 0;
}

// temb bookkeeping while building: list of (lin_embed path, Cout, conv_in bias) in block order
struct TembItem { std::string path; int Cout; float* conv_bias; };

static Res load_res(Loader& L, const std::string& path, int Cin, int Cout, std::vector<TembItem>& tembs, int& temb_total) {
  Res r;
  r.Cin = Cin; r.Cout = Cout; r.has_skip = (Cin != Cout);
  r.n_in = L.norm(path + "/norm_in", Cin);
  r.conv_in = L.conv(path + "/conv_in", Cin, Cout, 3);
  r.n_out = L.norm(path + "/norm_out", Cout);
  if (r.has_skip) r.conv_out = L.conv(path + "/conv_out", Cout, Cout, 3, path + "/skip_connection", Cin);
  else r.conv_out = L.conv(path + "/conv_out", Cout, Cout, 3);
  r.temb_off = temb_total;
  tembs.push_back({path + "/lin_embed", Cout, r.conv_in.b});
  temb_total += Cout;
  return r;
}

static STrans load_st(Loader& L, const std::string& path, int C, int ctx_dim, int n_head, int depth) {
  STrans s;
  s.C = C; s.n_head = n_head;
  s.norm = L.norm(path + "/norm", C);
  s.proj_in = L.linear(path + "/proj_in", C, C, true);
  s.proj_out = L.linear(path + "/proj_out", C, C, true);
  const int ctx_pad = Loader::pad64(ctx_dim);
  const int Cpad = Loader::pad64(C);
  for (int j = 0; j < depth && !L.err; ++j) {
    const std::string bp = path + "/transformer_" + std::to_string(j);
    TBlock b;
    b.n1 = L.norm(bp + "/norm1", C);
    b.n2 = L.norm(bp + "/norm2", C);
    b.n3 = L.norm(bp + "/norm3", C);
    // fused QKV for self-attention (reference unet/mod.rs:1009-1011: three bias-free Linears on x)
    b.qkv.K = C; b.qkv.Kpad = Cpad; b.qkv.N = 3 * C;
    b.qkv.w = L.A->get<__half>((size_t)3 * C * Cpad);
    if (!b.qkv.w) { L.err = fail(L.c, 4005, "weight arena exhausted"); break; }
    L.lin_into(bp + "/attn1/query", b.qkv.w, Cpad, 0, C, C, 0);
    L.lin_into(bp + "/attn1/key", b.qkv.w, Cpad, C, C, C, 0);
    L.lin_into(bp + "/attn1/value", b.qkv.w, Cpad, 2 * C, C, C, 0);
    b.out1 = L.linear(bp + "/attn1/out", C, C, true);
    b.q2 = L.linear(bp + "/attn2/query", C, C, false);
    b.kv2.K = ctx_dim; b.kv2.Kpad = ctx_pad; b.kv2.N = 2 * C;
    b.kv2.w = L.A->get<__half>((size_t)2 * C * ctx_pad);
    if (!b.kv2.w) { L.err = fail(L.c, 4005, "weight arena exhausted"); break; }
    L.lin_into(bp + "/attn2/key", b.kv2.w, ctx_pad, 0, ctx_dim, C, 0);
    L.lin_into(bp + "/attn2/value", b.kv2.w, ctx_pad, C, ctx_dim, C, 0);
    b.out2 = L.linear(bp + "/attn2/out", C, C, true);
    const int gbn = geglu_bn_for(4 * C);
    if (!gbn) { L.err = fail(L.c, 4009, "GEGLU width %d not tileable", 4 * C); break; }
    b.ff1 = L.linear(bp + "/mlp/geglu/proj", C, 8 * C, true, gbn);
    b.ff2 = L.linear(bp + "/mlp/lin", 4 * C, C, true);
    s.blocks.push_back(b);
  }
  return s;
}

// An input or output block of the block program (not the first conv).
static Block load_block(Loader& L, const sdxl_unet_cfg& g, const BlockSpec& s, std::vector<TembItem>& tembs, int& temb_total) {
  Block b;
  b.type = s.type;
  if (s.type == BT_DOWN) {
    b.conv = L.conv(s.path, s.c_in, s.c_out, 3);
    return b;
  }
  const bool tr = has_transformer(s.type), up = has_upsample(s.type);
  b.res = load_res(L, tr || up ? s.path + "/res" : s.path, s.c_in, s.c_out, tembs, temb_total);
  if (tr) b.st = load_st(L, s.path + "/transformer", s.c_out, g.context_dim, s.c_out / g.n_head_channels, s.depth);
  if (up) b.conv = L.upconv(s.path + "/upsample/conv", s.c_out, s.c_out);
  return b;
}

// Time / label MLPs, first conv, input blocks and middle block (reference unet/mod.rs:116-248), for the UNet and for a ControlNet.
static int load_encoder(Loader& L, EncoderHalf* u, const BlockProgram& prog, std::vector<TembItem>& tembs, int& temb_total) {
  const sdxl_unet_cfg& g = u->cfg;
  const int mc = g.model_channels, ted = 4 * mc;
  u->in_blocks.clear();
  u->t1 = L.linear("lin1_time_embed", mc, ted, true);
  u->t2 = L.linear("lin2_time_embed", ted, ted, true);
  u->l1 = L.linear("lin1_label_embed", g.adm_in_channels, ted, true);
  u->l2 = L.linear("lin2_label_embed", ted, ted, true);
  if (L.err) return L.err;
  for (const BlockSpec& s : prog.ins) {
    if (L.err) return L.err;
    if (s.type == BT_CONV) {
      if (int r = L.conv_f32(s.path, s.c_in, s.c_out, u->conv0_w, u->conv0_b)) return r;
      Block b0;
      b0.type = BT_CONV;
      u->in_blocks.push_back(std::move(b0));
    } else {
      u->in_blocks.push_back(load_block(L, g, s, tembs, temb_total));
    }
  }
  if (L.err) return L.err;
  const BlockSpec& m = prog.mid;
  u->mid_res1 = load_res(L, m.path + "/res1", m.c_in, m.c_out, tembs, temb_total);
  u->mid_st = load_st(L, m.path + "/transformer", m.c_out, g.context_dim, m.c_out / g.n_head_channels, m.depth);
  u->mid_res2 = load_res(L, m.path + "/res2", m.c_out, m.c_out, tembs, temb_total);
  return L.err;
}

// e->tblocks, after the real build pass (the block vectors no longer move): input blocks, middle, then `outs`.
static void list_tblocks(EncoderHalf* e, const std::vector<Block>& outs) {
  e->tblocks.clear();
  for (auto& b : e->in_blocks) for (auto& t : b.st.blocks) e->tblocks.push_back(&t);
  for (auto& t : e->mid_st.blocks) e->tblocks.push_back(&t);
  for (auto& b : outs) for (auto& t : b.st.blocks) e->tblocks.push_back(&t);
}

// concatenated lin_embed matrix (one GEMV per forward for all ResBlocks); bias += conv_in bias
static int load_temb_all(Loader& L, EncoderHalf* u, const std::vector<TembItem>& tembs, int temb_total) {
  sdxl_ctx* c = L.c;
  Arena& A = *L.A;
  const int ted = 4 * u->cfg.model_channels;
  Lin& T = u->temb_all;
  T.K = ted; T.Kpad = Loader::pad64(ted); T.N = temb_total;
  T.w = A.get<__half>((size_t)temb_total * T.Kpad);
  T.b = A.get<float>(temb_total);
  if (!T.w || !T.b) return fail(c, 4005, "weight arena exhausted");
  int off = 0;
  for (auto& it : tembs) {
    if (L.lin_into(it.path, T.w, T.Kpad, off, ted, it.Cout, 0)) return L.err;
    const PackEntry* e = L.need(it.path + "/bias", 1);
    if (!e) return L.err;
    if (!A.measure) {
      int r = bias_to_f32_launch(c->stream, L.ptr(e), it.Cout, T.b + off, 0, 0);
      // fold the conv_in bias: h = conv_in(..) + b_conv + lin_embed(..)   (unet/mod.rs:1086-1092)
      if (!r) r = vec_add_f32_launch(c->stream, T.b + off, it.conv_bias, it.Cout);
      if (r) return fail(c, r, "temb bias failed");
    }
    off += it.Cout;
  }
  return 0;
}

// Builds every layer (in measure mode only sizes are accumulated).
static int build_model(sdxl_unet* u, const PackView& pv, Arena& A) {
  sdxl_ctx* c = u->ctx;
  const sdxl_unet_cfg& g = u->cfg;
  Loader L{c, &pv, &A, c->stream};
  L.reg = &u->lora;
  const int mc = g.model_channels;
  u->out_blocks.clear();
  std::vector<TembItem> tembs;
  int temb_total = 0;
  const BlockProgram prog = block_program(g);
  if (int r = load_encoder(L, u, prog, tembs, temb_total)) return r;
  for (const BlockSpec& s : prog.outs) {
    if (L.err) return L.err;
    u->out_blocks.push_back(load_block(L, g, s, tembs, temb_total));
  }
  if (L.err) return L.err;
  u->norm_out = L.norm("norm_out", mc);
  u->conv_out = L.conv("conv_out", mc, g.out_channels, 3);
  if (L.err) return L.err;
  // The head conv is the one GEMM whose operand-rounding error reaches eps undamped (every other layer's is averaged by what
  // follows), so its activation operand is split hi + lo (two f16 tensors, ~22 bits): same weights twice along K.
  {
    const Conv& cv = u->conv_out;
    u->conv_out_w2 = A.get<__half>((size_t)cv.O * 2 * cv.Ktot);
    if (!u->conv_out_w2) return fail(c, 4005, "weight arena exhausted");
    if (!A.measure)
      for (int h2 = 0; h2 < 2; ++h2)
        CU(c, cudaMemcpy2DAsync(u->conv_out_w2 + (size_t)h2 * cv.Ktot, (size_t)2 * cv.Ktot * sizeof(__half), cv.w, (size_t)cv.Ktot * sizeof(__half),
                                (size_t)cv.Ktot * sizeof(__half), (size_t)cv.O, cudaMemcpyDeviceToDevice, c->stream));
  }
  if (int r = load_temb_all(L, u, tembs, temb_total)) return r;
  if (!A.measure) list_tblocks(u, u->out_blocks);
  return 0;
}

// ================================================================================================
// load
// ================================================================================================
// The configurations the UNet (and a ControlNet's copy of its encoder) are built for.
static int check_unet_cfg(sdxl_ctx* c, const sdxl_unet_cfg& g) {
  if (g.edit_layout != 0 && g.edit_layout != 1) return fail(c, 5700, "edit_layout = %d must be 0 or 1", g.edit_layout);
  if (edit_layout(g) && g.in_channels != 2 * g.out_channels)
    return fail(c, 5701, "edit_layout: in_channels = %d must be 2 * out_channels = %d", g.in_channels, 2 * g.out_channels);
  if (edit_layout(g) && g.is_refiner) return fail(c, 5702, "edit_layout: not supported with is_refiner");
  if (g.n_head_channels != 64) return fail(c, 4200, "n_head_channels must be 64 (got %d)", g.n_head_channels);
  if (g.n_levels < 1 || g.n_levels > SDXL_MAX_LEVELS) return fail(c, 4201, "bad n_levels");
  if ((g.in_channels > 8 && !inpaint_layout(g)) || g.model_channels % 32) return fail(c, 4202, "unsupported channel config");
  return 0;
}

static int unet_load_impl(sdxl_ctx* c, const sdxl_unet_cfg* cfg, const void* pack, size_t bytes, int pack_on_device, sdxl_unet** out) {
  if (!c || !cfg || !pack || !out) return fail(c, -1, "sdxl_unet_load: null argument");
  *out = nullptr;
  if (int r = check_unet_cfg(c, *cfg)) return r;
  CU(c, cudaSetDevice(c->device));
  std::unique_ptr<sdxl_unet> u(new sdxl_unet());
  u->ctx = c;
  u->cfg = *cfg;
  int r = with_device_pack(c, pack, bytes, pack_on_device, [&](const PackView& pv) {
    int r2 = build_two_pass(u.get(), pv, build_model);
    // alphas_cumprod: f16-stored in the reference's record (HalfPrecisionSettings), read as f64 (mod.rs:485-492)
    if (!r2) {
      const PackEntry* e = pv.find("alphas_cumprod");
      if (!e || e->ndim != 1 || e->dtype != 0) return fail(c, 4204, "weight pack: missing f16 'alphas_cumprod'");
      std::vector<uint16_t> raw(e->shape[0]);
      cudaError_t ce = cudaMemcpyAsync(raw.data(), pv.dev + e->offset, raw.size() * 2, cudaMemcpyDeviceToHost, c->stream);
      if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
      if (ce != cudaSuccess) return fail(c, (int)ce, "alphas download failed");
      u->alphas.resize(raw.size());
      for (size_t i = 0; i < raw.size(); ++i) {
        __half_raw hr;
        hr.x = raw[i];
        u->alphas[i] = (double)__half2float(__half(hr));
      }
      u->alphas_loaded = u->alphas;
    }
    return r2;
  });
  if (r) return r;
  CU(c, cudaMalloc((void**)&u->t_dev, 64));
  CU(c, cudaMallocHost((void**)&u->t_pinned, 4096 * sizeof(TimeSlot)));
  *out = u.release();
  return 0;
}

extern "C" int sdxl_unet_load(sdxl_ctx* c, const sdxl_unet_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                              sdxl_unet** out) {
  return unet_load_impl(c, cfg, pack, bytes, pack_on_device, out);
}

// ---- NCCL, resolved at run time (no link-time dependency: the library must load on machines without it) ----
#include <dlfcn.h>
namespace {
typedef int (*PFN_ncclBroadcast)(const void*, void*, size_t, int /*ncclDataType_t*/, int, void* /*ncclComm_t*/, cudaStream_t);
typedef const char* (*PFN_ncclGetErrorString)(int);
struct NcclApi { PFN_ncclBroadcast bcast = nullptr; PFN_ncclGetErrorString errstr = nullptr; bool tried = false; };
NcclApi& nccl_api() {
  static NcclApi api;
  if (!api.tried) {
    api.tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);   // the copy the host application (e.g. torch) already loaded
    if (!h && getenv("SDXL_B200_NCCL_LIB")) h = dlopen(getenv("SDXL_B200_NCCL_LIB"), RTLD_NOW);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
    if (h) {
      api.bcast = (PFN_ncclBroadcast)dlsym(h, "ncclBroadcast");
      api.errstr = (PFN_ncclGetErrorString)dlsym(h, "ncclGetErrorString");
    }
  }
  return api;
}
}  // namespace

extern "C" int sdxl_unet_load_broadcast(sdxl_ctx* c, const sdxl_unet_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                        void* nccl_comm, int rank, int root, sdxl_unet** out) {
  if (!c || !cfg || !out) return fail(c, -1, "sdxl_unet_load_broadcast: null argument");
  *out = nullptr;
  if (!nccl_comm) return fail(c, 4300, "sdxl_unet_load_broadcast: null NCCL communicator");
  if (rank == root && (!pack || !bytes)) return fail(c, 4301, "sdxl_unet_load_broadcast: the root rank must pass the weight pack");
  NcclApi& N = nccl_api();
  if (!N.bcast) return fail(c, 4302, "sdxl_unet_load_broadcast: libnccl.so.2 not found (set SDXL_B200_NCCL_LIB)");
  CU(c, cudaSetDevice(c->device));
  const int ncclUint8 = 1;
  // 1. the size, so that non-root ranks can allocate
  unsigned long long* dsz = nullptr;
  CU(c, cudaMalloc((void**)&dsz, 8));
  unsigned long long hsz = rank == root ? (unsigned long long)bytes : 0ull;
  cudaError_t e = cudaMemcpyAsync(dsz, &hsz, 8, cudaMemcpyHostToDevice, c->stream);
  int nr = e == cudaSuccess ? N.bcast(dsz, dsz, 8, ncclUint8, root, nccl_comm, c->stream) : 0;
  if (e == cudaSuccess && !nr) e = cudaMemcpyAsync(&hsz, dsz, 8, cudaMemcpyDeviceToHost, c->stream);
  if (e == cudaSuccess && !nr) e = cudaStreamSynchronize(c->stream);
  cudaFree(dsz);
  if (nr) return fail(c, 4303, "ncclBroadcast (pack size) failed: %s", N.errstr ? N.errstr(nr) : "?");
  if (e != cudaSuccess) return fail(c, (int)e, "pack size broadcast failed: %s", cudaGetErrorString(e));
  if (hsz < sizeof(PackHeader)) return fail(c, 4304, "broadcast pack size %llu is not a weight pack", hsz);
  // 2. the pack itself: one flat message
  uint8_t* dpack = nullptr;
  CU(c, cudaMalloc((void**)&dpack, (size_t)hsz));
  if (rank == root)
    e = cudaMemcpyAsync(dpack, pack, (size_t)hsz, pack_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) nr = N.bcast(dpack, dpack, (size_t)hsz, ncclUint8, root, nccl_comm, c->stream);
  if (e == cudaSuccess && !nr) e = cudaStreamSynchronize(c->stream);
  int r = 0;
  if (nr) r = fail(c, 4303, "ncclBroadcast (pack) failed: %s", N.errstr ? N.errstr(nr) : "?");
  else if (e != cudaSuccess) r = fail(c, (int)e, "pack broadcast failed: %s", cudaGetErrorString(e));
  else r = unet_load_impl(c, cfg, dpack, (size_t)hsz, 1, out);
  cudaFree(dpack);
  return r;
}

// ================================================================================================
// ControlNet load
// ================================================================================================
static int build_controlnet(sdxl_controlnet* n, const PackView& pv, Arena& A) {
  const sdxl_unet_cfg& g = n->cfg;
  const sdxl_controlnet_cfg& nc = n->ncfg;
  Loader L{n->ctx, &pv, &A, n->ctx->stream};   // no LoRA registry: adapters on a ControlNet are not supported
  std::vector<TembItem> tembs;
  int temb_total = 0;
  const BlockProgram prog = block_program(g);
  if (int r = load_encoder(L, n, prog, tembs, temb_total)) return r;
  if (int r = load_temb_all(L, n, tembs, temb_total)) return r;
  // hint encoder, SGM's input_hint_block indices: 0 = conv(in -> c0); 2 + 4k = conv(c_k -> c_k), 4 + 4k = conv(c_k -> c_k+1, s2);
  // 4n - 2 = conv(c_last -> mc)
  const int* hc = nc.hint_block_channels;
  const int nb = nc.n_hint_blocks;
  if (int r = L.conv_f32("input_hint_block/0", nc.hint_in_channels, hc[0], n->hint0_w, n->hint0_b)) return r;
  n->hint.clear();
  for (int k = 0; k + 1 < nb && !L.err; ++k) {
    n->hint.push_back(L.conv("input_hint_block/" + std::to_string(2 + 4 * k), hc[k], hc[k], 3));
    n->hint.push_back(L.conv("input_hint_block/" + std::to_string(4 + 4 * k), hc[k], hc[k + 1], 3));
  }
  n->hint.push_back(L.conv("input_hint_block/" + std::to_string(4 * nb - 2), hc[nb - 1], g.model_channels, 3));
  // zero convs: one per skip tensor (the outputs of input_blocks/0, 1, ...), then middle_block_out
  n->zero.clear();
  for (size_t i = 0; i < prog.ins.size() && !L.err; ++i)
    n->zero.push_back(L.conv("zero_convs/" + std::to_string(i), prog.ins[i].c_out, prog.ins[i].c_out, 1));
  n->zero.push_back(L.conv("middle_block_out", prog.mid.c_out, prog.mid.c_out, 1));
  if (!L.err && !A.measure) list_tblocks(n, {});
  return L.err;
}

extern "C" int sdxl_controlnet_load(sdxl_ctx* c, const sdxl_controlnet_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                    sdxl_controlnet** out) {
  if (!c || !cfg || !pack || !out) return fail(c, -1, "sdxl_controlnet_load: null argument");
  *out = nullptr;
  if (int r = check_unet_cfg(c, cfg->unet)) return r;
  if (inpaint_layout(cfg->unet)) return fail(c, 4703, "ControlNet: a UNet cfg with the inpainting layout (in_channels = %d) is not supported", cfg->unet.in_channels);
  if (edit_layout(cfg->unet)) return fail(c, 5703, "ControlNet: a UNet cfg with the edit layout is not supported");
  if (cfg->hint_in_channels < 1 || cfg->hint_in_channels > 8) return fail(c, 4700, "hint_in_channels must be in [1, 8] (got %d)", cfg->hint_in_channels);
  if (cfg->n_hint_blocks != 4) return fail(c, 4701, "n_hint_blocks must be 4 (hint downscale 2^(n-1) = 8), got %d", cfg->n_hint_blocks);
  for (int k = 0; k < cfg->n_hint_blocks; ++k)
    if (cfg->hint_block_channels[k] < 8 || cfg->hint_block_channels[k] % 8)
      return fail(c, 4702, "hint_block_channels[%d] = %d must be a positive multiple of 8", k, cfg->hint_block_channels[k]);
  CU(c, cudaSetDevice(c->device));
  std::unique_ptr<sdxl_controlnet> n(new sdxl_controlnet());
  n->ctx = c;
  n->cfg = cfg->unet;
  n->ncfg = *cfg;
  int r = with_device_pack(c, pack, bytes, pack_on_device,
                           [&](const PackView& pv) { return build_two_pass(n.get(), pv, build_controlnet); });
  if (r) return r;
  *out = n.release();
  return 0;
}

extern "C" void sdxl_controlnet_destroy(sdxl_controlnet* n) {
  if (!n) return;
  cudaStreamSynchronize(n->ctx->stream);
  delete n;
}

// 3x3 pad-1 conv of an NHWC f16 image on the implicit GEMM, stride 1 or 2 (stride 2: `a` is the phase split of the input,
// [4][Bn][H/2][W/2][C], as written by silu_f16_launch / phase_split_launch). Output f32 NHWC at H x W (stride 1) or H/2 x W/2.
static int conv3x3_direct(sdxl_ctx* c, const __half* a, int Bn, int H, int W, int C, const Conv& cv, int stride, float* out) {
  const int Ho = H / stride, Wo = W / stride;
  const IgemmOperands o{a, stride == 2 ? 4 * Bn : Bn, Ho, Wo, C, C, nullptr, 0, 0, 0, 0, 0, cv.w, cv.O, cv.Ktot};
  return igemm_run(c, o, stride == 2 ? stride2_taps(Bn, cv.Ipad / 64) : conv_taps(3, cv.Ipad / 64), Ho, Wo, Bn, IGEMM_LINEAR, 0, out,
                   1, cv.O, cv.b, nullptr, 0);
}

// Points x at a borrowed input of `bytes` in device memory: src itself, or with on_host a copy into T queued on the ctx stream (the
// caller synchronises before it returns: src is the caller's memory). If T cannot allocate the copy, fails with code and fmt.
template <class X, class... A>
static int stage_in(sdxl_ctx* c, TmpBufs& T, const X* src, size_t bytes, int on_host, const X*& x, int code, const char* fmt, A... args) {
  x = src;
  if (!on_host) return 0;
  X* d = T.get<X>(bytes);
  if (!d) return fail(c, code, fmt, args...);
  CU(c, cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, c->stream));
  x = d;
  return 0;
}

// Copies a result from device memory to the caller's host memory and waits for it.
static int stage_out(sdxl_ctx* c, void* host, const void* dev, size_t bytes) {
  CU(c, cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}

// Hint encoder (SGM input_hint_block): hint f32 NCHW [n, in, H, W] (device) -> f32 NHWC [n, H/8, W/8, mc]. Queued on the ctx stream.
static int embed_hint(sdxl_controlnet* net, int n, int H, int W, const float* hint, float* out) {
  sdxl_ctx* c = net->ctx;
  const sdxl_controlnet_cfg& nc = net->ncfg;
  const int* hc = nc.hint_block_channels;
  const int nb = nc.n_hint_blocks;
  if (n < 1 || H < 8 || W < 8 || H % 8 || W % 8) return fail(c, 4710, "hint must be [n >= 1, %d, H, W] with H, W multiples of 8 (got n=%d, %dx%d)", nc.hint_in_channels, n, H, W);
  size_t maxe = 0;
  {
    int h = H, w = W;
    for (int k = 0; k < nb; ++k) { maxe = std::max(maxe, (size_t)n * h * w * hc[k]); h /= 2; w /= 2; }
  }
  TmpBufs T(c->stream);
  float* a = T.get<float>(maxe * sizeof(float));
  __half* a16 = T.get<__half>(maxe * sizeof(__half));
  if (!a || !a16) return fail(c, 4711, "hint encoder: cannot allocate %zu bytes of scratch", maxe * 6);
  KL(c, conv_in_launch_t(c->stream, hint, 1, n, n, nc.hint_in_channels, H, W, net->hint0_w, net->hint0_b, hc[0], a));
  int h = H, w = W;
  for (int k = 0; k + 1 < nb; ++k) {
    KL(c, silu_f16_launch(c->stream, a, n, h, w, hc[k], 0, a16));
    if (int r = conv3x3_direct(c, a16, n, h, w, hc[k], net->hint[2 * k], 1, a)) return r;
    KL(c, silu_f16_launch(c->stream, a, n, h, w, hc[k], 1, a16));
    if (int r = conv3x3_direct(c, a16, n, h, w, hc[k], net->hint[2 * k + 1], 2, a)) return r;
    h /= 2; w /= 2;
  }
  KL(c, silu_f16_launch(c->stream, a, n, h, w, hc[nb - 1], 0, a16));
  return conv3x3_direct(c, a16, n, h, w, hc[nb - 1], net->hint.back(), 1, out);
}

extern "C" int sdxl_controlnet_embed_hint(sdxl_controlnet* net, int n, int H, int W, const float* hint, int on_host, float* out) {
  if (!net || !hint || !out) return -1;
  sdxl_ctx* c = net->ctx;
  CU(c, cudaSetDevice(c->device));
  const int mc = net->cfg.model_channels, h = H / 8, w = W / 8;
  TmpBufs T(c->stream);
  const size_t in_bytes = (size_t)n * net->ncfg.hint_in_channels * H * W * sizeof(float), out_elems = (size_t)n * h * w * mc;
  const float* x;
  if (int r = stage_in(c, T, hint, in_bytes, on_host, x, 4711, "embed_hint: allocation failed")) return r;
  float* e = T.get<float>(out_elems * sizeof(float));
  float* o = on_host ? T.get<float>(out_elems * sizeof(float)) : out;
  if (!e || !o) return fail(c, 4711, "embed_hint: allocation failed");
  if (int r = embed_hint(net, n, H, W, x, e)) return r;
  KL(c, nhwc_to_nchw_f32_launch(c->stream, e, n, h * w, mc, mc, o));
  return on_host ? stage_out(c, out, o, out_elems * sizeof(float)) : 0;
}

// ================================================================================================
// launch plan
// ================================================================================================
// UNet-specific plan pieces on top of the generic PlanBuilder (engine_core.h)
struct UNetPlanBuilder : PlanBuilder {
  sdxl_unet* u = nullptr;
  int kv_index = 0;
  const HoistedCond* cond = nullptr;   // hoisted conditioning of the model being planned (UNet or ControlNet)
  int Bp = 0;                          // trailing perturbed rows: PAG's selected self-attentions of the UNet are the identity there

  struct Scratch { __half *gn1, *raw; float* h; __half *gn2, *a16; float* tok; __half *qkv, *ao, *q, *ff; };
  struct Saved { float* p; int C, H, W; };

  // Time / label MLPs (on the shared timestep embedding te), first conv, input blocks and middle block of UNet::forward
  // (unet/mod.rs:458-482) with the weights of `e` and the conditioning `cond`; every block output is pushed to `saved`, the
  // middle output is returned. hint (nullable): ControlNet hint embedding f32 NHWC [n_hint, h, w, mc] added to the first conv's output.
  // last_in < in_blocks.size(): DeepCache's shallow branch, which stops after input block last_in and returns null.
  float* encoder(const EncoderHalf& e, const float* te, float* t1, float* semb, float* temb_all,
                 const Scratch& s, const float* hint, int n_hint, const std::string& prefix, std::vector<Saved>& saved,
                 size_t last_in) {
    const sdxl_unet_cfg& g = e.cfg;
    const int mc = g.model_channels, ted = 4 * mc, temb_total = e.temb_all.N;
    gemv(te, 0, 1, e.t1, nullptr, 0, 0, 1, t1, 0);
    gemv(t1, 0, Bf, e.t2, cond->label_emb, ted, 0, 1, semb, ted);
    gemv(semb, ted, Bf, e.temb_all, nullptr, 0, 0, 0, temb_all, temb_total);
    int H = P->h, W = P->w;
    float* x = buf<float>((size_t)Bf * H * W * mc);
    int Cx = mc;
    // the inpainting UNet's first conv reads the attached condition as its input channels [out_channels, in_channels)
    const InpaintAttach* ipc = cond == &u->cond ? u->inpaint.get() : nullptr;
    if (inpaint_layout(g) && !ipc && !err) err = fail(c, 5018, "inpainting UNet: no inpainting condition attached");
    if (!err) {
      Op op{};
      op.kind = OP_CONV_IN;
      op.ci = {P->x_in, P->Bx, Bf, latent_channels(g), H, W, e.conv0_w, e.conv0_b, mc, x, hint, n_hint};
      if (inpaint_layout(g)) { op.ci.x2 = ipc->cond; op.ci.n2 = ipc->ext.n; op.ci.C2 = g.in_channels - g.out_channels; }
      if (edit_layout(g) && cond == &u->cond) { op.ci.x2 = u->plan_edit; op.ci.n2 = Bf; op.ci.C2 = g.out_channels; }
      P->ops.push_back(op);
      P->flops += 2.0 * Bf * H * W * 9.0 * g.in_channels * mc;
    }
    saved.push_back({x, Cx, H, W});
    // an attached T2I-Adapter adds its features in the UNet's own encoder (a ControlNet's does not see them)
    const bool t2i = u->t2i && cond == &u->cond;
    for (size_t i = 1; i < e.in_blocks.size() && i <= last_in && !err; ++i) {
      const Block& b = e.in_blocks[i];
      begin_block(prefix + "input_blocks/" + std::to_string(i));
      if (b.type == BT_RES || b.type == BT_REST) {
        x = resblock(b.res, x, Cx, nullptr, 0, H, W, temb_all, temb_total, s.gn1, s.raw, s.h, s.gn2);
        Cx = b.res.Cout;
        if (b.type == BT_REST) x = strans(b.st, x, H, W, s.a16, s.tok, s.qkv, s.ao, s.q, s.ff);
      } else if (b.type == BT_DOWN) {
        // 3x3 stride 2 pad 1 (unet/mod.rs:760-774) on phase-split input
        __half* ph = buf<__half>((size_t)Bf * H * W * Cx);
        Op op{};
        op.kind = OP_PHASE;
        op.rs = {x, Bf, H, W, Cx, ph};
        if (!err) P->ops.push_back(op);
        const int H2 = H / 2, W2 = W / 2;
        ActView a{ph, 4 * Bf, H2, W2, Cx};
        float* y = buf<float>((size_t)Bf * H2 * W2 * Cx);
        igemm(a, nullptr, stride2_taps(Bf, b.conv.Ipad / 64), b.conv.w, b.conv.O, b.conv.Ktot, H2, W2, Bf, IGEMM_LINEAR, 0, y, 1, b.conv.O, b.conv.b, 0, nullptr, 0);
        add_flops(2.0 * Bf * H2 * W2 * 9.0 * Cx * b.conv.O);
        x = y; H = H2; W = W2;
      }
      if (t2i)
        for (int k = 0; k < 3; ++k)
          if (u->t2i->points[k] == i) t2i_add(x, k, Cx, H, W);
      end_block();
      saved.push_back({x, Cx, H, W});
    }
    if (last_in < e.in_blocks.size()) return nullptr;
    // --- middle
    begin_block(prefix + "middle_block");
    x = resblock(e.mid_res1, x, Cx, nullptr, 0, H, W, temb_all, temb_total, s.gn1, s.raw, s.h, s.gn2);
    x = strans(e.mid_st, x, H, W, s.a16, s.tok, s.qkv, s.ao, s.q, s.ff);
    x = resblock(e.mid_res2, x, Cx, nullptr, 0, H, W, temb_all, temb_total, s.gn1, s.raw, s.h, s.gn2);
    if (t2i) t2i_add(x, 3, Cx, H, W);
    end_block();
    return x;
  }

  // FreeU at a decoder skip concatenation cat([x, sk]) of the UNet's level n_levels - 1 - k (k = 0, 1): x[:, :Cx / 2] *= (b1, b2)[k]
  // and sk = fourier_filter(sk, 1, (s1, s2)[k]), both in place (the next resblock is the only reader of either). tw: the level's
  // twiddles.
  void freeu(const Saved& sk, float* x, int Cx, int k, const float* tw) {
    if (err) return;
    Op op{};
    op.kind = OP_FREEU;
    op.fu = {sk.p, sk.C, x, Cx, Bf, sk.H, sk.W, tw, u->freeu->vals + k, u->freeu->vals + 2 + k};
    P->ops.push_back(op);
  }

  // T2I-Adapter injection: x += F_k in place, so the skip saved for the block carries the feature too
  void t2i_add(float* x, int k, int C, int H, int W) {
    if (err) return;
    const T2IAttach& a = *u->t2i;
    if (a.C[k] != C || a.H[k] != H || a.W[k] != W) { err = fail(c, 5017, "T2I-Adapter feature %d shape mismatch", k); return; }
    Op op{};
    op.kind = OP_T2I_ADD;
    op.ta = {x, a.F[k], (long)H * W * C, Bf, a.ext.n, u->t_dev, a.t_min};
    P->ops.push_back(op);
  }

  // ControlNet injection: dst += conv1x1(src) with the scaled zero conv L (f16 operand of src in `a16`, residual add in place)
  void zero_conv(const Saved& src, const Saved& dst, const Lin& L, __half* a16) {
    if (err) return;
    if (src.C != dst.C || src.H != dst.H || src.W != dst.W || L.K != src.C) { err = fail(c, 5006, "control residual shape mismatch"); return; }
    const size_t n = (size_t)Bf * src.H * src.W * src.C;
    Op op{};
    op.kind = OP_CAST16;
    op.cs = {src.p, n, a16};
    P->ops.push_back(op);
    linear(a16, Bf * src.H * src.W, L, IGEMM_LINEAR, dst.p, 1, L.N, dst.p, L.N);
  }

  // ---- ResBlock (reference unet/mod.rs:1082-1106) ----
  float* resblock(const Res& r, const float* xa, int Ca, const float* xb, int Cb, int H, int W, const float* temb_all,
                  int temb_total, __half* s_gn1, __half* s_raw, float* s_h, __half* s_gn2) {
    const int HW = H * W;
    float* out = buf<float>((size_t)Bf * HW * r.Cout);
    gn(xa, Ca, xb, Cb, HW, r.n_in, 1, s_gn1, r.has_skip ? s_raw : nullptr);
    ActView a1{s_gn1, Bf, H, W, r.Cin};
    // h = conv_in(silu(gn(x))) + b + lin_embed(silu(emb))[:, :, None, None]   (bias folded into temb_all)
    conv3(a1, nullptr, r.conv_in, s_h, temb_all + r.temb_off, temb_total, nullptr);
    gn(s_h, r.Cout, nullptr, 0, HW, r.n_out, 1, s_gn2, nullptr);
    ActView a2{s_gn2, Bf, H, W, r.Cout};
    if (r.has_skip) {
      ActView sk{s_raw, Bf, H, W, r.Cin};
      conv3(a2, &sk, r.conv_out, out, r.conv_out.b, 0, nullptr);  // skip 1x1 conv fused as a K segment
    } else {
      conv3(a2, nullptr, r.conv_out, out, r.conv_out.b, 0, xa);   // identity residual in the epilogue
    }
    return out;
  }

  // ---- SpatialTransformer (reference unet/mod.rs:820-845, 885-891, 1005-1023) ----
  float* strans(const STrans& s, const float* x, int H, int W, __half* s_a16, float* s_tok, __half* s_qkv, __half* s_ao,
                __half* s_q, __half* s_ff) {
    const int T = H * W, M = Bf * T, C = s.C;
    float* out = buf<float>((size_t)M * C);
    const float sl2e = (float)(1.4426950408889634 / sqrt(64.0));
    gn(x, C, nullptr, 0, T, s.norm, 0, s_a16, nullptr);
    linear(s_a16, M, s.proj_in, IGEMM_LINEAR, s_tok, 1, C, nullptr, 0);
    for (const TBlock& b : s.blocks) {
      // x = x + attn1(norm1(x))
      ln(s_tok, b.n1, M, s_a16);
      linear(s_a16, M, b.qkv, IGEMM_LINEAR, s_qkv, 0, 3 * C, nullptr, 0);
      if (Bp && cond == &u->cond && u->pag->layers[kv_index]) {
        // PAG: softmax attention over the attended rows, out = v on the perturbed ones (out1 and the residual run on all rows)
        attn(s_qkv, 3 * C, 0, s_qkv, 3 * C, C, 2 * C, T, T, s.n_head, s_ao, C, sl2e, Bf - Bp);
        if (!err) {
          Op op{};
          op.kind = OP_PAG_IDENTITY;
          op.pi = {s_qkv + (size_t)(Bf - Bp) * T * 3 * C, C, (long)Bp * T, s_ao + (size_t)(Bf - Bp) * T * C};
          P->ops.push_back(op);
        }
      } else {
        attn(s_qkv, 3 * C, 0, s_qkv, 3 * C, C, 2 * C, T, T, s.n_head, s_ao, C, sl2e);
      }
      linear(s_ao, M, b.out1, IGEMM_LINEAR, s_tok, 1, C, s_tok, C);
      // x = x + attn2(norm2(x), context)   (K/V hoisted to set_conditioning)
      ln(s_tok, b.n2, M, s_a16);
      linear(s_a16, M, b.q2, IGEMM_LINEAR, s_q, 0, C, nullptr, 0);
      attn(s_q, C, 0, cond->kv[kv_index], 2 * C, 0, C, T, cond->n_ctx, s.n_head, s_ao, C, sl2e);
      P->flops += 2.0 * Bf * cond->n_ctx * (double)b.kv2.K * b.kv2.N;  // hoisted K/V projections (algorithmic work)
      // attached image prompts add their K/V sources to the UNet's own cross-attentions (a ControlNet's see text only)
      if (u->ip && cond == &u->cond)
        for (const IpPrompt& ip : u->ip->prompts) {
          const int ns = ip.n_sources(), S = ip.S_ip / ns;
          int level = 0;
          while (ip.mask_h && level < u->cfg.n_levels && ((ip.mask_h / 8) >> level != H || (ip.mask_w / 8) >> level != W)) ++level;
          if (level == u->cfg.n_levels) { err = fail(c, 5021, "image prompt: its masks do not match the latent"); return out; }
          for (int i = 0; i < ns; ++i)
            attn_ip(ip.cond.kv[kv_index] + (size_t)i * Bf * S * 2 * C, 2 * C, 0, C, S, ip.scales + kv_index,
                    ip.mask_h ? ip.masks + ip_mask_off(ip, u->cfg.n_levels, i, level) : nullptr);
          P->flops += 2.0 * Bf * ip.S_ip * (double)ip.ad->kv[kv_index].K * ip.ad->kv[kv_index].N;
        }
      kv_index++;
      linear(s_ao, M, b.out2, IGEMM_LINEAR, s_tok, 1, C, s_tok, C);
      // x = x + mlp(norm3(x))
      ln(s_tok, b.n3, M, s_a16);
      linear(s_a16, M, b.ff1, IGEMM_GEGLU, s_ff, 0, 4 * C, nullptr, 0);
      // the last block's stream only feeds proj_out: its residual add writes the f16 operand directly (no f32 copy, no cast launch)
      if (&b == &s.blocks.back()) linear(s_ff, M, b.ff2, IGEMM_LINEAR, s_a16, 0, C, s_tok, C);
      else linear(s_ff, M, b.ff2, IGEMM_LINEAR, s_tok, 1, C, s_tok, C);
    }
    if (s.blocks.empty() && !err) {   // no block to fold the cast into
      Op op{};
      op.kind = OP_CAST16;
      op.cs = {s_tok, (size_t)M * C, s_a16};
      P->ops.push_back(op);
    }
    // proj_out(tokens) + x_in
    linear(s_a16, M, s.proj_out, IGEMM_LINEAR, out, 1, C, x, C);
    return out;
  }
  // over the first B rows of the batch (default: all Bf)
  void attn(const __half* qm, int q_pitch, int q_col0, const __half* kvm, int kv_pitch, int k_col0, int v_col0, int T,
            int S, int n_head, __half* out, int ldo, float sl2e, int B = 0) {
    if (err) return;
    if (!B) B = Bf;
    Op op{};
    op.kind = OP_ATTN;
    AttnParams& p = op.at;
    p.T = T; p.S = S; p.n_head = n_head; p.B = B;
    p.q_col0 = q_col0; p.k_col0 = k_col0; p.v_col0 = v_col0;
    p.out = out; p.ldo = ldo; p.scale_log2e = sl2e;
    if (!A->measure) {
      int r = make_tmap_rows(&p.tmQ, qm, T, B, q_pitch, q_pitch);
      if (!r) r = make_tmap_rows(&p.tmK, kvm, S, B, kv_pitch, kv_pitch);
      if (!r) p.tmV = p.tmK;
      if (r) { err = fail(c, r, "tensor map creation failed (attention)"); return; }
    }
    op.flops_exec = 4.0 * B * (double)((T + 127) / 128 * 128) * (double)((S + 127) / 128 * 128) * (n_head * 64);
    P->ops.push_back(op);
    add_flops(4.0 * B * T * (double)S * (n_head * 64));
  }
  // Adds an image source to the attention just pushed: + (*scale) * mask[t] * softmax(q k_ip^T) v_ip (mask nullable: 1), k_ip /
  // v_ip column windows of kvm [Bf * S_ip, kv_pitch].
  void attn_ip(const __half* kvm, int kv_pitch, int k_col0, int v_col0, int S_ip, const float* scale, const float* mask) {
    if (err) return;
    AttnParams& p = P->ops.back().at;
    if (p.n_src == ATTN_MAX_SRC) { err = fail(c, 5022, "image prompt: more than %d image sources", ATTN_MAX_SRC); return; }
    CUtensorMap tm{};
    if (!A->measure)
      if (int r = make_tmap_rows(&tm, kvm, S_ip, Bf, kv_pitch, kv_pitch)) { err = fail(c, r, "tensor map creation failed (attention)"); return; }
    if (p.n_src == 0) {
      p.S_ip = S_ip; p.k_ip_col0 = k_col0; p.v_ip_col0 = v_col0; p.ip_scale = scale; p.ip_mask = mask;
      p.tmKip = p.tmVip = tm;
    } else {
      p.ip_src[p.n_src - 1] = {tm, S_ip, k_col0, v_col0, scale, mask};
    }
    p.n_src++;
    const int C = p.n_head * 64;
    P->ops.back().flops_exec += 4.0 * Bf * (double)((p.T + 127) / 128 * 128) * (double)((S_ip + 127) / 128 * 128) * C;
    add_flops(4.0 * Bf * p.T * (double)S_ip * C);
  }
};



// Transformer blocks that run before output block e in a full forward: the index of e's first one in UNet::tblocks (list_tblocks).
static int tblocks_before_output(const sdxl_unet* u, size_t e) {
  size_t n = u->mid_st.blocks.size();
  for (const Block& b : u->in_blocks) n += b.st.blocks.size();
  for (size_t i = 0; i < e; ++i) n += u->out_blocks[i].st.blocks.size();
  return (int)n;
}

// Buffers that every op list of a plan shares (build_plan_ops).
struct UNetPlanShared {
  UNetPlanBuilder::Scratch scr;
  float *te, *t1, *semb, *temb_all;
  const float* freeu_tw[2] = {nullptr, nullptr};   // FreeU's twiddles of the two deepest levels, made by the first list
};

// Emits one forward into B's op list. branch < 0: no DeepCache. Full list (cached false): UNet::forward (reference
// unet/mod.rs:449-493); with a branch, the backbone input of output block e = 3 * n_levels - 1 - branch is kept in `feature` (a copy
// made before FreeU scales it in place, when FreeU runs there). Cached list: the shallow branch on `feature` (DESIGN.md §17).
static int plan_forward(sdxl_unet* u, UNetPlanBuilder& B, UNetPlanShared& sh, int branch, bool cached, UNetPlanBuilder::Saved& feature) {
  sdxl_ctx* c = u->ctx;
  const sdxl_unet_cfg& g = u->cfg;
  Plan* P = B.P;
  Arena* A = B.A;
  const int Bf = P->Bf, mc = g.model_channels, ted = 4 * mc;
  const int temb_total = u->temb_all.N;
  const int levels = g.n_levels;
  const size_t n_out = u->out_blocks.size();
  const size_t e = branch >= 0 ? n_out - 1 - (size_t)branch : 0;
  const size_t last_in = cached ? (size_t)branch : SIZE_MAX;   // the encoder's bound: SIZE_MAX runs all of it
  const UNetPlanBuilder::Scratch& scr = sh.scr;
  float *te = sh.te, *t1 = sh.t1, *semb = sh.semb, *temb_all = sh.temb_all;

  // --- embeddings (unet/mod.rs:458-468): emb = time_mlp(temb(t)) + label_emb; only SiLU(emb) is consumed
  {
    Op op{};
    op.kind = OP_TEMB;
    op.te = {(const float*)(u->t_dev + 1), 1, mc, te};
    P->ops.push_back(op);
  }
  // --- embeddings, input blocks, middle
  using Saved = UNetPlanBuilder::Saved;
  std::vector<Saved> saved;
  B.cond = &u->cond;
  float* x = B.encoder(*u, te, t1, semb, temb_all, scr, nullptr, 1, "", saved, last_in);
  int H = saved.back().H, W = saved.back().W, Cx = saved.back().C;
  // --- ControlNets (DESIGN.md §8): each runs its own encoder on the same inputs, then skip_i += s * zero_conv_i(h_i) and
  // mid += s * middle_block_out(mid_c), in attachment order. The UNet's own encoder above is untouched. The cached list has no middle.
  for (size_t k = 0; k < u->controls.size() && !B.err; ++k) {
    const ControlAttach& a = *u->controls[k];
    const EncoderHalf& en = *a.net;
    const std::string prefix = "control" + std::to_string(k) + "/";
    const int kv_unet = B.kv_index;
    B.cond = &a.cond;
    B.kv_index = 0;
    float* ct1 = B.buf<float>(ted);
    float* csemb = B.buf<float>((size_t)Bf * ted);
    float* ctemb = B.buf<float>((size_t)Bf * en.temb_all.N);
    std::vector<Saved> cs;
    float* cmid = B.encoder(en, te, ct1, csemb, ctemb, scr, a.hint_emb, a.ext.n, prefix, cs, last_in);
    B.cond = &u->cond;
    B.kv_index = kv_unet;
    if (cs.size() != saved.size() || a.zero.size() != u->in_blocks.size() + 1) return fail(c, 5006, "control %zu: skip count mismatch", k);
    B.begin_block(prefix + "zero_convs");
    for (size_t i = 0; i < saved.size(); ++i) B.zero_conv(cs[i], saved[i], a.zero[i], scr.raw);
    if (!cached) B.zero_conv({cmid, Cx, H, W}, {x, Cx, H, W}, a.zero.back(), scr.raw);
    B.end_block();
  }
  // --- FreeU's twiddle tables of the two deepest levels, computed on the host (freeu_twiddles) into the plan's workspace
  for (int k = 0; k < 2 && u->freeu && !sh.freeu_tw[k] && levels - 1 - k >= 0; ++k) {
    const int th = P->h >> (levels - 1 - k), tw = P->w >> (levels - 1 - k);
    float* d = B.buf<float>((size_t)2 * (th + tw));
    if (B.err) return B.err;
    if (!A->measure) {
      std::vector<float> host((size_t)2 * (th + tw));
      freeu_twiddles(th, tw, host.data());
      CU(c, cudaMemcpyAsync(d, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
      CU(c, cudaStreamSynchronize(c->stream));
    }
    sh.freeu_tw[k] = d;
  }
  if (cached) {   // the deep part is the kept feature
    x = feature.p; Cx = feature.C; H = feature.H; W = feature.W;
    B.kv_index = tblocks_before_output(u, e);
  }
  // DeepCache's copy of a feature that FreeU scales in place: made in the full list, and in the cached list for FreeU to scale
  auto copy = [&](const Saved& src) -> Saved {
    const size_t n = (size_t)Bf * src.H * src.W * src.C;
    float* d = B.buf<float>(n);
    if (!B.err) {
      Op op{};
      op.kind = OP_COPY;
      op.cp = {src.p, d, n * sizeof(float)};
      P->ops.push_back(op);
    }
    return {d, src.C, src.H, src.W};
  };
  // --- output blocks: cat([x, saved.pop()], channel) is never materialised (GN + skip conv read both)
  for (size_t i = cached ? e : 0; i < n_out && !B.err; ++i) {
    const Block& b = u->out_blocks[i];
    if (saved.empty()) return fail(c, 5004, "skip stack underflow");
    Saved sk = saved.back();
    saved.pop_back();
    if (sk.H != H || sk.W != W || Cx + sk.C != b.res.Cin) return fail(c, 5005, "skip shape mismatch at output block %zu", i);
    B.begin_block("output_blocks/" + std::to_string(i));
    // FreeU: the output blocks of the two deepest levels (diffusers' up_blocks[0] and [1]: three each, output block i is at level
    // n_levels - 1 - i / 3), after the ControlNet residuals were added to the skips
    const int k = (int)(i / 3);
    const bool fu = u->freeu && k < 2 && k < levels;
    if (branch >= 0 && i == e) {
      if (cached && fu) x = copy(feature).p;
      else if (!cached) feature = fu ? copy({x, Cx, H, W}) : Saved{x, Cx, H, W};
    }
    if (fu) {
      if (H != P->h >> (levels - 1 - k) || W != P->w >> (levels - 1 - k))
        return fail(c, 5024, "FreeU: output block %zu is not at level %d", i, levels - 1 - k);
      B.freeu(sk, x, Cx, k, sh.freeu_tw[k]);
    }
    x = B.resblock(b.res, x, Cx, sk.p, sk.C, H, W, temb_all, temb_total, scr.gn1, scr.raw, scr.h, scr.gn2);
    Cx = b.res.Cout;
    if (b.type == BT_REST || b.type == BT_RESTU) x = B.strans(b.st, x, H, W, scr.a16, scr.tok, scr.qkv, scr.ao, scr.q, scr.ff);
    if (b.type == BT_RESTU || b.type == BT_RESU) {
      // nearest-2x then 3x3 conv (unet/mod.rs:742-751), as four 2x2 phase convolutions of the source image
      __half* x16 = B.buf<__half>((size_t)Bf * H * W * Cx);
      float* y = B.buf<float>((size_t)Bf * 4 * H * W * Cx);
      B.upconv(x, Bf, H, W, b.conv, x16, y);
      H *= 2; W *= 2;
      x = y;
    }
    B.end_block();
  }
  if (B.err) return B.err;
  B.begin_block("norm_out+conv_out");
  // --- head: GN -> SiLU -> conv 3x3 (unet/mod.rs:488-490)
  B.gn(x, Cx, nullptr, 0, H * W, u->norm_out, 1, scr.gn1, nullptr);
  if (!B.err && !P->ops.empty()) P->ops.back().gn.y_lo = scr.raw;   // rounding residue of the normalised activation (hi/lo split)
  {
    ActView a{scr.gn1, Bf, H, W, Cx}, alo{scr.raw, Bf, H, W, Cx};
    std::vector<IgemmSeg> segs = conv_taps(3, u->conv_out.Ipad / 64, 0), lo = conv_taps(3, u->conv_out.Ipad / 64, 1);
    segs.insert(segs.end(), lo.begin(), lo.end());   // K = [9 taps on hi | 9 taps on lo], weights [W | W]
    B.igemm(a, &alo, segs, u->conv_out_w2, u->conv_out.O, 2 * u->conv_out.Ktot, H, W, Bf, IGEMM_LINEAR, 0, P->eps, 1, P->eps_ld,
            u->conv_out.b, 0, nullptr, 0);
    B.add_flops(2.0 * Bf * H * W * 9.0 * Cx * u->conv_out.O);
  }
  B.end_block();
  return B.err;
}

// Builds the op list for UNet::forward at batch Bf, latent h x w and, with DeepCache attached, the cached list (Plan::cached) after
// it, over the same shared buffers.
static int build_plan_ops(sdxl_unet* u, Plan* P, Arena* A, int Bp) {
  sdxl_ctx* c = u->ctx;
  const sdxl_unet_cfg& g = u->cfg;
  UNetPlanBuilder B{{c, P, A, P->Bf}, u};
  B.Bp = Bp;
  P->ops.clear();
  P->block_names.clear();
  P->flops = 0;
  P->cached.reset();
  const int Bf = P->Bf, mc = g.model_channels, ted = 4 * mc;
  const int temb_total = u->temb_all.N;
  const int levels = g.n_levels;
  if ((P->h % (1 << (levels - 1))) || (P->w % (1 << (levels - 1)))) return fail(c, 5003, "latent %dx%d not divisible by %d", P->h, P->w, 1 << (levels - 1));

  P->x_in = B.buf<float>((size_t)P->Bx * latent_channels(g) * P->h * P->w);
  if (edit_layout(g)) u->plan_edit = B.buf<float>((size_t)Bf * g.out_channels * P->h * P->w);
  P->eps_ld = g.out_channels;
  P->eps = B.buf<float>((size_t)Bf * P->h * P->w * P->eps_ld);
  B.gn_partial = B.buf<float>(gn_scratch_floats(Bf, 32));
  if (B.gn_partial && !A->measure && gn_scratch_init(c->stream, B.gn_partial, Bf, 32)) return fail(c, 5007, "GroupNorm scratch init failed");
  UNetPlanShared sh;
  sh.te = B.buf<float>(mc);
  sh.t1 = B.buf<float>(ted);
  sh.semb = B.buf<float>((size_t)Bf * ted);
  sh.temb_all = B.buf<float>((size_t)Bf * temb_total);

  // maxima for the shared scratch buffers over the ResBlocks and transformers of the block program, each at its level
  size_t max_pixC_cat = 0, max_pixC = 0, max_tokC = 0;
  {
    const BlockProgram prog = block_program(g);
    auto upd = [&](const BlockSpec& s) {
      if (s.type == BT_CONV || s.type == BT_DOWN) return;
      const size_t px = (size_t)(P->h >> s.level) * (P->w >> s.level);
      max_pixC_cat = std::max(max_pixC_cat, px * s.c_in);
      max_pixC = std::max(max_pixC, px * s.c_out);
      if (has_transformer(s.type)) max_tokC = std::max(max_tokC, px * s.c_out);
    };
    for (const BlockSpec& s : prog.ins) upd(s);
    upd(prog.mid);
    for (const BlockSpec& s : prog.outs) upd(s);
  }
  __half* s_gn1 = B.buf<__half>(Bf * max_pixC_cat);
  __half* s_raw = B.buf<__half>(Bf * max_pixC_cat);
  float* s_h = B.buf<float>(Bf * max_pixC);
  __half* s_gn2 = B.buf<__half>(Bf * max_pixC);
  __half* s_a16 = B.buf<__half>(Bf * max_tokC);
  float* s_tok = B.buf<float>(Bf * max_tokC);
  __half* s_qkv = B.buf<__half>(Bf * max_tokC * 3);
  __half* s_ao = B.buf<__half>(Bf * max_tokC);
  __half* s_q = B.buf<__half>(Bf * max_tokC);
  __half* s_ff = B.buf<__half>(Bf * max_tokC * 4);
  if (B.err) return B.err;
  sh.scr = {s_gn1, s_raw, s_h, s_gn2, s_a16, s_tok, s_qkv, s_ao, s_q, s_ff};

  const int branch = u->deepcache ? u->deepcache->branch : -1;
  UNetPlanBuilder::Saved feature{};
  if (int r = plan_forward(u, B, sh, branch, false, feature)) return r;
  if (branch < 0) return 0;
  // DeepCache's cached list: its own ops, graph and run count; every buffer from this plan's arena
  P->cached.reset(new Plan());
  Plan* Q = P->cached.get();
  Q->Bf = P->Bf; Q->Bx = P->Bx; Q->h = P->h; Q->w = P->w;
  Q->x_in = P->x_in; Q->eps = P->eps; Q->eps_ld = P->eps_ld;
  UNetPlanBuilder Bc{{c, Q, A, Bf}, u};
  Bc.Bp = Bp;
  Bc.gn_partial = B.gn_partial;
  return plan_forward(u, Bc, sh, branch, true, feature);
}

// Whether every attachment fits a run of n_img images on an h x w latent: it was made for that latent, and n_img is a multiple of
// its row count (every row group's row of image b reads attachment row b % n). An inpainting UNet runs only with a condition.
static int attachments_fit(sdxl_unet* u, int n_img, int h, int w) {
  sdxl_ctx* c = u->ctx;
  // what: the attachment, subject: what was sized ("its hint"), divisor: the name of its n; codes: extent, then divisor
  auto fit = [&](const std::string& what, const char* subject, const Extent& e, const char* divisor, int code) {
    if (e.h != h || e.w != w)
      return fail(c, code, "%s: %s %dx%d pixels (latent %dx%d) but the latent is %dx%d", what.c_str(), subject, 8 * e.h, 8 * e.w, e.h,
                  e.w, h, w);
    if (n_img % e.n) return fail(c, code + 1, "%s: batch %d is not a multiple of %s = %d", what.c_str(), n_img, divisor, e.n);
    return 0;
  };
  for (size_t k = 0; k < u->controls.size(); ++k)
    if (int r = fit("control " + std::to_string(k), "its hint is", u->controls[k]->ext, "n_hint", 5012)) return r;
  if (u->t2i)
    if (int r = fit("T2I-Adapter", "its hint is", u->t2i->ext, "n_hint", 5015)) return r;
  if (u->ip)
    for (const IpPrompt& a : u->ip->prompts)
      if (a.mask_h && (a.mask_h / 8 != h || a.mask_w / 8 != w))
        return fail(c, 5021, "image prompt: its masks are %dx%d pixels (latent %dx%d) but the latent is %dx%d", a.mask_h, a.mask_w,
                    a.mask_h / 8, a.mask_w / 8, h, w);
  if (edit_layout(u->cfg)) {   // image guidance takes the third row group and the first conv's second source
    if (!u->edit) return fail(c, 5720, "edit UNet: no source image attached (call sdxl_unet_set_edit_image first)");
    if (u->pag) return fail(c, 5723, "edit UNet: PAG is attached; image guidance and PAG would need a fourth row group");
    if (!u->controls.empty()) return fail(c, 5724, "edit UNet: ControlNets are attached; they are not supported with image guidance");
    if (u->t2i) return fail(c, 5725, "edit UNet: T2I-Adapters are attached; they are not supported with image guidance");
    if (u->ip) return fail(c, 5726, "edit UNet: image prompts are attached; they are not supported with image guidance");
    return fit("edit image", "it is", u->edit->ext, "its n", 5721);
  }
  if (!inpaint_layout(u->cfg)) return 0;
  if (!u->inpaint) return fail(c, 5018, "inpainting UNet: no inpainting condition attached (call sdxl_unet_set_inpaint_condition first)");
  return fit("inpainting condition", "it is", u->inpaint->ext, "its n", 5019);
}

// An edit UNet's per-row first-conv condition of the current plan (plan_edit), from the attached image: row r of the first
// Bf - plan_edit_zero reads image r % n, the rest are zero. Called when the plan is built and when the image is rewritten in place.
static int edit_rows_fill(sdxl_unet* u) {
  sdxl_ctx* c = u->ctx;
  if (!edit_layout(u->cfg) || !u->plan || !u->edit) return 0;
  const Plan* P = u->plan.get();
  const size_t img = (size_t)u->cfg.out_channels * P->h * P->w * sizeof(float);
  const int n = u->edit->ext.n, lit = P->Bf - u->plan_edit_zero;
  for (int r = 0; r < lit; r += n)   // lit is a multiple of n (attachments_fit)
    CU(c, cudaMemcpyAsync((uint8_t*)u->plan_edit + r * img, u->edit->latent, n * img, cudaMemcpyDeviceToDevice, c->stream));
  if (u->plan_edit_zero) CU(c, cudaMemsetAsync((uint8_t*)u->plan_edit + lit * img, 0, u->plan_edit_zero * img, c->stream));
  return 0;
}

// Bx: the images of the batch (the direct forward's B, the sampler's Bimg); Bp: the trailing rows that take PAG's identity
// self-attentions (0: none; PAG attached when > 0); Bz: an edit UNet's trailing rows whose first-conv condition is zero.
static int ensure_plan(sdxl_unet* u, int Bf, int Bx, int h, int w, int Bp, int Bz = 0) {
  sdxl_ctx* c = u->ctx;
  if (u->cond.condB != Bf) return fail(c, 5010, "conditioning is set for batch %d but forward batch is %d (call sdxl_unet_set_conditioning first)", u->cond.condB, Bf);
  if (Bp < 0 || Bp >= Bf) return fail(c, 5023, "PAG: %d perturbed rows in a batch of %d (at least one row must be attended)", Bp, Bf);
  if (u->ip)
    for (const IpPrompt& a : u->ip->prompts)
      if (a.cond.condB != Bf) return fail(c, 5014, "image prompt: its K/V are hoisted for batch %d but the batch is %d", a.cond.condB, Bf);
  if (int r = attachments_fit(u, Bx, h, w)) return r;
  // every change of the buffers or attachments a plan reads drops the plan, so the shapes, the perturbed rows and the DeepCache
  // branch are its whole cache key
  const int dc = u->deepcache ? u->deepcache->branch : -1;
  if (u->plan && u->plan->Bf == Bf && u->plan->Bx == Bx && u->plan->h == h && u->plan->w == w && u->plan_ptb == Bp && u->plan_dc == dc &&
      u->plan_edit_zero == Bz)
    return 0;
  u->dc_feature = false;
  if (int r = build_plan(c, u->plan, Bf, Bx, h, w, [&](Plan* P, Arena* A) { return build_plan_ops(u, P, A, Bp); })) return r;
  u->plan_ptb = Bp;
  u->plan_dc = dc;
  u->plan_edit_zero = Bz;
  u->plan_builds++;
  return edit_rows_fill(u);
}

// Refuses DeepCache's cached forward until a full run of the current plan has kept the feature it reads.
static int cached_ready(sdxl_unet* u) {
  if (u->plan && u->plan->cached && u->dc_feature) return 0;
  return fail(u->ctx, 5025, "DeepCache: no full forward has kept a feature since the plan was built (run one with forward_cached = 0)");
}

// Runs the plan's full list, which keeps DeepCache's feature when it is attached, or (cached) its cached list on that feature.
static int run_plan(sdxl_unet* u, bool cached = false) {
  if (cached) {
    if (int r = cached_ready(u)) return r;
    return run_plan_ops(u->ctx, u->plan->cached.get());
  }
  const int r = run_plan_ops(u->ctx, u->plan.get());
  u->dc_feature = !r && u->plan->cached;
  return r;
}

static int set_t(sdxl_unet* u, double t) {
  sdxl_ctx* c = u->ctx;
  const int slot = u->t_slot = (u->t_slot + 1) % 4096;
  u->t_pinned[slot] = {(int)lround(t), (float)t};
  CU(c, cudaMemcpyAsync(u->t_dev, &u->t_pinned[slot], sizeof(TimeSlot), cudaMemcpyHostToDevice, c->stream));
  return 0;
}

// ================================================================================================
// conditioning (step-invariant work hoisted out of UNet::forward)
// ================================================================================================
static int hoist_conditioning(sdxl_unet* u);

// Allocates the conditioning buffers of model e at (B, n_ctx) into h (a fresh object: callers swap it in on success).
static int cond_alloc(sdxl_ctx* c, const EncoderHalf& e, int B, int n_ctx, HoistedCond& h) {
  const int ted = 4 * e.cfg.model_channels;
  h.condB = B;
  h.n_ctx = n_ctx;
  return carve_measured(c, h.mem, 5101, "conditioning buffers", [&](Arena& A) {
    h.lab1 = A.get<float>((size_t)B * ted);
    h.label_emb = A.get<float>((size_t)B * ted);
    h.kv.clear();
    for (const TBlock* t : e.tblocks) h.kv.push_back(A.get<__half>((size_t)B * n_ctx * t->kv2.N));
    return 0;
  });
}

// Allocates an image prompt's row and K/V buffers for conditioning batch B into r (a fresh object, as above).
static int ip_cond_alloc(sdxl_ctx* c, const IpPrompt& a, int B, IpRows& r) {
  const int ctx_dim = a.ad->cfg.unet.context_dim;
  r.condB = B;
  return carve_measured(c, r.mem, 5103, "image-prompt conditioning buffers", [&](Arena& A) {
    r.rows = A.get<__half>((size_t)B * a.S_ip * ctx_dim);
    r.kv.clear();
    for (const Lin& L : a.ad->kv) r.kv.push_back(A.get<__half>((size_t)B * a.S_ip * L.N));
    return 0;
  });
}

// An image prompt's n_batch must divide the number of images the conditioning rows hold.
static int ip_check_batch(sdxl_unet* u, int n_batch /* 0: no prompt */, int B, const RowLayout& L) {
  const int n_img = L.n_img ? L.n_img : B;
  if (n_batch && n_img % n_batch)
    return fail(u->ctx, 5104, "image prompt: batch %d is not a multiple of its n_batch = %d", n_img, n_batch);
  return 0;
}
static int ip_check_batch_all(sdxl_unet* u, int B, const RowLayout& L) {
  if (u->ip)
    for (const IpPrompt& a : u->ip->prompts)
      if (int r = ip_check_batch(u, a.n_batch, B, L)) return r;
  return 0;
}

static int set_conditioning_dev(sdxl_unet* u, int B, int n_ctx, const __half* context_dev, const __half* y_dev, const RowLayout& L) {
  sdxl_ctx* c = u->ctx;
  const sdxl_unet_cfg& g = u->cfg;
  if (B < 1 || n_ctx < 1) return fail(c, 5100, "bad conditioning shape");
  if (int r = ip_check_batch_all(u, B, L)) return r;
  if (u->cond.condB != B || u->cond.n_ctx != n_ctx) {
    // everything sized by (B, n_ctx) is allocated into fresh objects and swapped in only when all of it succeeded: a failure
    // leaves the previous conditioning, and the plan over it, in effect
    const int pitch = (g.context_dim + 7) / 8 * 8;
    Arena imem;
    __half* ctx16 = nullptr;
    float* y32 = nullptr;
    int r = carve_measured(c, imem, 5101, "conditioning inputs", [&](Arena& A) {
      ctx16 = A.get<__half>((size_t)B * n_ctx * pitch);
      y32 = A.get<float>((size_t)B * g.adm_in_channels);
      return 0;
    });
    HoistedCond cond;
    if (!r) r = cond_alloc(c, *u, B, n_ctx, cond);
    std::vector<HoistedCond> ccond(u->controls.size());
    for (size_t k = 0; k < ccond.size() && !r; ++k) r = cond_alloc(c, *u->controls[k]->net, B, n_ctx, ccond[k]);
    std::vector<IpRows> ipc(u->ip ? u->ip->prompts.size() : 0);
    for (size_t k = 0; k < ipc.size() && !r; ++k) r = ip_cond_alloc(c, u->ip->prompts[k], B, ipc[k]);
    if (r) return r;
    CU(c, cudaStreamSynchronize(c->stream));   // the old buffers and the plan over them may still be in flight
    u->plan.reset();
    u->imem = std::move(imem);
    u->ctx_pitch = pitch;
    u->ctx16 = ctx16;
    u->y32 = y32;
    u->cond = std::move(cond);
    for (size_t k = 0; k < ccond.size(); ++k) u->controls[k]->cond = std::move(ccond[k]);
    for (size_t k = 0; k < ipc.size(); ++k) u->ip->prompts[k].cond = std::move(ipc[k]);
    CU(c, cudaMemsetAsync(u->ctx16, 0, (size_t)B * n_ctx * pitch * 2, c->stream));
  }
  u->rows = L;
  CU(c, cudaMemcpy2DAsync(u->ctx16, (size_t)u->ctx_pitch * 2, context_dev, (size_t)g.context_dim * 2, (size_t)g.context_dim * 2,
                          (size_t)B * n_ctx, cudaMemcpyDeviceToDevice, c->stream));
  KL(c, cast_f16_to_f32_launch(c->stream, y_dev, (size_t)B * g.adm_in_channels, u->y32));
  return hoist_conditioning(u);
}

// out[i] = a @ L_i for every Lin (K/V projections of context or image tokens); a f16 [M, K] with row pitch lda.
static int project_kv(sdxl_ctx* c, const __half* a, int M, int K, int lda, const std::vector<const Lin*>& lins, const std::vector<__half*>& out) {
  for (size_t i = 0; i < lins.size(); ++i) {
    const Lin& L = *lins[i];
    const IgemmOperands o{a, 1, 1, M, K, lda, nullptr, 0, 0, 0, 0, 0, L.w, L.N, L.Kpad};
    if (int r = igemm_run(c, o, {{0, 0, 0, 0, L.Kpad / 64}}, 1, M, 1, IGEMM_LINEAR, 0, out[i], 0, L.N, nullptr, nullptr, 0)) return r;
  }
  return 0;
}

// label_emb = lin2(SiLU(lin1(y))) (unet/mod.rs:464-466) and the K/V projections of the context for every cross-attention
// (unet/mod.rs:1010-1011) with the weights of `e` into h, from the UNet's retained conditioning (h has the UNet's shape).
static int hoist_model(sdxl_unet* u, const EncoderHalf& e, const HoistedCond& h) {
  sdxl_ctx* c = u->ctx;
  const sdxl_unet_cfg& g = u->cfg;
  const int ted = 4 * g.model_channels, B = h.condB, n_ctx = h.n_ctx;
  for (int b0 = 0; b0 < B; b0 += 8) {
    const int nb = B - b0 < 8 ? B - b0 : 8;
    KL(c, gemv_launch(c->stream, u->y32 + (size_t)b0 * g.adm_in_channels, g.adm_in_channels, nb, g.adm_in_channels, e.l1.w,
                      e.l1.Kpad, e.l1.b, nullptr, 0, ted, 0, 1, h.lab1 + (size_t)b0 * ted, ted));
    KL(c, gemv_launch(c->stream, h.lab1 + (size_t)b0 * ted, ted, nb, e.l2.K, e.l2.w, e.l2.Kpad, e.l2.b, nullptr, 0, ted, 0, 0,
                      h.label_emb + (size_t)b0 * ted, ted));
  }
  std::vector<const Lin*> lins;
  for (const TBlock* t : e.tblocks) lins.push_back(&t->kv2);
  return project_kv(c, u->ctx16, B * n_ctx, g.context_dim, u->ctx_pitch, lins, h.kv);
}

// An image prompt's token rows for the current conditioning rows (row rule: include/sdxl_b200.h, sdxl_unet_set_image_prompt),
// source-major (IpRows), and their K/V for every UNet cross-attention.
static int ip_hoist(sdxl_unet* u, IpPrompt& a) {
  sdxl_ctx* c = u->ctx;
  const int ctx_dim = u->cfg.context_dim, B = a.cond.condB, ns = a.n_sources();
  const RowLayout& L = u->rows;
  const size_t row = (size_t)a.S_ip * ctx_dim, src_row = row / ns;   // one conditioning row's tokens; one source's part of them
  for (int r = 0; r < B; ++r) {
    // n_batch divides n_img (ip_check_batch), so row r of any group is image r % n_batch
    const __half* src = L.negative(r) ? a.tok_neg + (size_t)(r % a.n_batch) * row : a.tok_pos + (size_t)(r % a.n_batch) * row;
    CU(c, cudaMemcpy2DAsync(a.cond.rows + (size_t)r * src_row, B * src_row * sizeof(__half), src, src_row * sizeof(__half),
                            src_row * sizeof(__half), ns, cudaMemcpyDeviceToDevice, c->stream));
  }
  std::vector<const Lin*> lins;
  for (const Lin& L : a.ad->kv) lins.push_back(&L);
  return project_kv(c, a.cond.rows, B * a.S_ip, ctx_dim, ctx_dim, lins, a.cond.kv);
}

// The step-invariant projections of the retained conditioning (ctx16, y32) under the current weights, for the UNet and every
// attached ControlNet.
static int hoist_conditioning(sdxl_unet* u) {
  if (int r = hoist_model(u, *u, u->cond)) return r;
  for (auto& a : u->controls)
    if (int r = hoist_model(u, *a->net, a->cond)) return r;
  if (u->ip)
    for (IpPrompt& a : u->ip->prompts)
      if (int r = ip_hoist(u, a)) return r;
  return 0;
}

extern "C" int sdxl_unet_set_conditioning(sdxl_unet* u, int B, int n_ctx, const sdxl_half* context, const sdxl_half* y) {
  if (!u || !context || !y) return -1;
  CU(u->ctx, cudaSetDevice(u->ctx->device));
  return set_conditioning_dev(u, B, n_ctx, (const __half*)context, (const __half*)y, RowLayout{});
}

// ================================================================================================
// ControlNet attachment (include/sdxl_b200.h: sdxl_unet_set_controls)
// ================================================================================================
// The first cfg field in which an attachment built for cfg h differs from the UNet's cfg g, or null.
static const char* unet_cfg_mismatch(const sdxl_unet_cfg& g, const sdxl_unet_cfg& h) {
  if (h.model_channels != g.model_channels) return "model_channels";
  if (h.n_levels != g.n_levels) return "n_levels";
  if (h.in_channels != g.in_channels) return "in_channels";
  if (h.context_dim != g.context_dim) return "context_dim";
  if (h.adm_in_channels != g.adm_in_channels) return "adm_in_channels";
  if (h.n_head_channels != g.n_head_channels) return "n_head_channels";
  for (int l = 0; l < g.n_levels; ++l) {
    if (h.channel_mults[l] != g.channel_mults[l]) return "channel_mults";
    if (h.transformer_depths[l] != g.transformer_depths[l]) return "transformer_depths";
  }
  return nullptr;
}

static const sdxl_unet_cfg& unet_cfg_of(const sdxl_controlnet& n) { return n.cfg; }
template <class O> static const sdxl_unet_cfg& unet_cfg_of(const O& o) { return o.cfg.unet; }

// Refuses an object that cannot be attached to u: null, made on another sdxl_ctx, or built for another UNet cfg. what, k: the
// entry point and the item, for the messages; codes: the three refusals' codes in that order.
template <class O>
static int attachable(sdxl_unet* u, const char* what, int k, const O* obj, const int (&codes)[3]) {
  sdxl_ctx* c = u->ctx;
  if (!obj) return fail(c, codes[0], "%s %d: null object", what, k);
  if (obj->ctx != c) return fail(c, codes[1], "%s %d: created on another sdxl_ctx", what, k);
  if (const char* field = unet_cfg_mismatch(u->cfg, unet_cfg_of(*obj)))
    return fail(c, codes[2], "%s %d: cfg field '%s' differs from the UNet's", what, k, field);
  return 0;
}

// Moves a new attachment into its slot of u. The plan reads the old one and may still be in flight: the stream is drained and the
// plan dropped first.
template <class S>
static int attach_install(sdxl_unet* u, S& slot, S fresh) {
  CU(u->ctx, cudaStreamSynchronize(u->ctx->stream));
  u->plan.reset();
  slot = std::move(fresh);
  return 0;
}

template <class T> static bool slot_empty(const std::unique_ptr<T>& s) { return !s; }
template <class T> static bool slot_empty(const std::vector<T>& s) { return s.empty(); }

// Empties a slot of u; an empty slot keeps the plan.
template <class S>
static int attach_detach(sdxl_unet* u, S& slot) {
  return slot_empty(slot) ? 0 : attach_install(u, slot, S());
}

// Writes the per-attachment buffers that depend on scale and hint values: f16(s*W) / s*b of every zero conv, and hint_emb.
static int control_write(sdxl_ctx* c, ControlAttach& a, const sdxl_control& ctl) {
  const sdxl_controlnet* n = a.net;
  for (size_t i = 0; i < n->zero.size(); ++i) {
    const Conv& z = n->zero[i];
    KL(c, scale_weights_launch(c->stream, z.w, (size_t)z.O * z.Ktot, z.b, z.O, ctl.scale, a.zero[i].w, a.zero[i].b));
  }
  a.scale = ctl.scale;
  TmpBufs T(c->stream);
  const size_t bytes = (size_t)ctl.n_hint * n->ncfg.hint_in_channels * ctl.height * ctl.width * sizeof(float);
  const float* hint;
  if (int r = stage_in(c, T, ctl.hint, bytes, ctl.hint_on_host, hint, 4720, "set_controls: cannot allocate %zu bytes for the hint", bytes))
    return r;
  int r = embed_hint(const_cast<sdxl_controlnet*>(n), ctl.n_hint, ctl.height, ctl.width, hint, a.hint_emb);
  if (!r && ctl.hint_on_host) CU(c, cudaStreamSynchronize(c->stream));   // the caller may reuse its host memory
  return r;
}

extern "C" int sdxl_unet_set_controls(sdxl_unet* u, int n, const sdxl_control* ctl) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  // validate everything first: on failure the attached set is unchanged
  if (n < 0 || n > SDXL_MAX_CONTROLS) return fail(c, 4730, "set_controls: n = %d outside [0, %d]", n, SDXL_MAX_CONTROLS);
  if (n > 0 && !ctl) return fail(c, 4731, "set_controls: null control array");
  const sdxl_unet_cfg& g = u->cfg;
  for (int k = 0; k < n; ++k) {
    if (int r = attachable(u, "set_controls: control", k, ctl[k].net, {4732, 4733, 4734})) return r;
    if (ctl[k].n_hint < 1) return fail(c, 4735, "set_controls: control %d: n_hint = %d must be >= 1", k, ctl[k].n_hint);
    if (!ctl[k].hint) return fail(c, 4736, "set_controls: control %d: null hint", k);
    if (ctl[k].height < 8 || ctl[k].width < 8 || ctl[k].height % 8 || ctl[k].width % 8)
      return fail(c, 4737, "set_controls: control %d: hint size %dx%d must be a positive multiple of 8", k, ctl[k].height, ctl[k].width);
    if (!isfinite(ctl[k].scale)) return fail(c, 4738, "set_controls: control %d: scale is not finite", k);
  }
  if (n == 0) return attach_detach(u, u->controls);
  // same nets, n_hint and sizes: only scales and hint values change, the launch plan stays valid
  auto extent = [&](int k) { return Extent{ctl[k].n_hint, ctl[k].height / 8, ctl[k].width / 8}; };
  bool in_place = (size_t)n == u->controls.size();
  for (int k = 0; k < n && in_place; ++k) in_place = u->controls[k]->net == ctl[k].net && u->controls[k]->ext == extent(k);
  if (in_place) {   // not staged: a runtime failure of control k leaves 0..k-1 rewritten (documented in include/sdxl_b200.h)
    for (int k = 0; k < n; ++k)
      if (int r = control_write(c, *u->controls[k], ctl[k])) return r;
    return 0;
  }
  std::vector<std::unique_ptr<ControlAttach>> fresh;
  for (int k = 0; k < n; ++k) {
    std::unique_ptr<ControlAttach> a(new ControlAttach());
    const sdxl_controlnet* net = ctl[k].net;
    a->net = net;
    a->ext = extent(k);
    if (int r = carve_measured(c, a->mem, 4739, "set_controls: control buffers", [&](Arena& A) {
          a->zero.clear();
          for (const Conv& z : net->zero) {
            Lin L;
            L.K = z.I; L.Kpad = z.Ktot; L.N = z.O;
            L.w = A.get<__half>((size_t)z.O * z.Ktot);
            L.b = A.get<float>(z.O);
            a->zero.push_back(L);
          }
          a->hint_emb = A.get<float>((size_t)a->ext.n * a->ext.h * a->ext.w * g.model_channels);
          return 0;
        }))
      return r;
    if (int r = control_write(c, *a, ctl[k])) return r;
    if (u->cond.condB > 0) {
      if (int r = cond_alloc(c, *net, u->cond.condB, u->cond.n_ctx, a->cond)) return r;
      if (int r = hoist_model(u, *net, a->cond)) return r;
    }
    fresh.push_back(std::move(a));
  }
  return attach_install(u, u->controls, std::move(fresh));
}


// ================================================================================================
// IP-Adapter (include/sdxl_b200.h: sdxl_ip_adapter_load, sdxl_unet_set_image_prompt; DESIGN.md §9)
// ================================================================================================
static int build_ip_adapter(sdxl_ip_adapter* a, const PackView& pv, Arena& A) {
  const sdxl_ip_adapter_cfg& g = a->cfg;
  const int ctx_dim = g.unet.context_dim;
  Loader L{a->ctx, &pv, &A, a->ctx->stream};
  std::set<std::string> names;
  auto lin = [&](const std::string& path, int K, int N, bool bias) {
    names.insert(path + "/weight");
    if (bias) names.insert(path + "/bias");
    return L.linear(path, K, N, bias);
  };
  auto norm = [&](const std::string& path, int C) {
    names.insert(path + "/weight");
    names.insert(path + "/bias");
    return L.norm(path, C);
  };
  if (!a->plus()) {
    a->proj = lin("image_proj/proj", g.image_embed_dim, g.tokens_per_image * ctx_dim, true);
    a->norm = norm("image_proj/norm", ctx_dim);
  } else {
    const int W = 64 * g.resampler_heads, Q = g.tokens_per_image;
    {   // latents [Q, W] f16 -> f32
      const PackEntry* e = L.need("image_proj/latents", 2);
      if (!e) return L.err;
      if ((int)e->shape[0] != Q || (int)e->shape[1] != W)
        return fail(a->ctx, 4006, "weight pack: 'image_proj/latents' is [%llu,%llu], expected [%d,%d]", (unsigned long long)e->shape[0],
                    (unsigned long long)e->shape[1], Q, W);
      names.insert("image_proj/latents");
      a->latents = A.get<float>((size_t)Q * W);
      if (!a->latents) return fail(a->ctx, 4005, "weight arena exhausted");
      if (!A.measure) KL(a->ctx, cast_f16_to_f32_launch(a->ctx->stream, L.ptr(e), (size_t)Q * W, a->latents));
    }
    a->proj_in = lin("image_proj/proj_in", g.image_embed_dim, W, true);
    a->layers.clear();
    for (int i = 0; i < g.resampler_depth && !L.err; ++i) {
      const std::string lp = "image_proj/layers/" + std::to_string(i);
      PerceiverLayer l;
      l.ln1 = norm(lp + "/attn/norm1", W);
      l.ln2 = norm(lp + "/attn/norm2", W);
      l.to_q = lin(lp + "/attn/to_q", W, W, false);
      l.to_kv = lin(lp + "/attn/to_kv", W, 2 * W, false);
      l.to_out = lin(lp + "/attn/to_out", W, W, false);
      l.ln_ff = norm(lp + "/ff/norm", W);
      l.fc1 = lin(lp + "/ff/fc1", W, 4 * W, false);
      l.fc2 = lin(lp + "/ff/fc2", 4 * W, W, false);
      a->layers.push_back(l);
    }
    a->proj_out = lin("image_proj/proj_out", W, ctx_dim, true);
    a->norm_out = norm("image_proj/norm_out", ctx_dim);
  }
  if (L.err) return L.err;
  a->kv.clear();
  // one fused [ip_key | ip_value] per UNet transformer block, in the order of the UNet's tblocks
  const BlockProgram prog = block_program(g.unet);
  std::vector<BlockSpec> blocks = prog.ins;
  blocks.push_back(prog.mid);
  blocks.insert(blocks.end(), prog.outs.begin(), prog.outs.end());
  for (const BlockSpec& s : blocks) {
    if (!has_transformer(s.type)) continue;
    const int C = s.c_out;
    for (int j = 0; j < s.depth; ++j) {
      if (L.err) return L.err;
      const std::string bp = s.path + "/transformer/transformer_" + std::to_string(j);
      Lin kv;
      kv.K = ctx_dim; kv.Kpad = Loader::pad64(ctx_dim); kv.N = 2 * C;
      kv.w = A.get<__half>((size_t)kv.N * kv.Kpad);
      if (!kv.w) return fail(a->ctx, 4005, "weight arena exhausted");
      L.lin_into(bp + "/attn2/ip_key", kv.w, kv.Kpad, 0, ctx_dim, C, 0);
      L.lin_into(bp + "/attn2/ip_value", kv.w, kv.Kpad, C, ctx_dim, C, 0);
      names.insert(bp + "/attn2/ip_key/weight");
      names.insert(bp + "/attn2/ip_value/weight");
      a->kv.push_back(kv);
    }
  }
  if (L.err) return L.err;
  for (const auto& t : pv.t)   // e.g. a pack for a UNet with more transformer blocks
    if (!names.count(t.first)) return fail(a->ctx, 4804, "IP-Adapter pack: tensor '%s' is not part of an adapter for this UNet cfg", t.first.c_str());
  return 0;
}

extern "C" int sdxl_ip_adapter_load(sdxl_ctx* c, const sdxl_ip_adapter_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                    sdxl_ip_adapter** out) {
  if (!c || !cfg || !pack || !out) return fail(c, -1, "sdxl_ip_adapter_load: null argument");
  *out = nullptr;
  if (int r = check_unet_cfg(c, cfg->unet)) return r;
  if (cfg->unet.is_refiner) return fail(c, 4800, "IP-Adapter: the refiner is not supported");
  if (cfg->unet.context_dim < 8 || cfg->unet.context_dim % 8)
    return fail(c, 4801, "IP-Adapter: context_dim = %d must be a positive multiple of 8", cfg->unet.context_dim);
  if (cfg->image_embed_dim < 1) return fail(c, 4802, "IP-Adapter: image_embed_dim = %d must be >= 1", cfg->image_embed_dim);
  if (cfg->tokens_per_image < 1 || cfg->tokens_per_image > 64)
    return fail(c, 4803, "IP-Adapter: tokens_per_image = %d outside [1, 64]", cfg->tokens_per_image);
  if (cfg->resampler_depth < 0 || cfg->resampler_depth > 64)
    return fail(c, 4805, "IP-Adapter: resampler_depth = %d outside [0, 64]", cfg->resampler_depth);
  if (cfg->resampler_depth > 0) {   // Plus: the LayerNorm over the width takes up to 2048 columns; the hidden states are f16 GEMM rows
    if (cfg->resampler_heads < 1 || cfg->resampler_heads > 32)
      return fail(c, 4806, "IP-Adapter Plus: resampler_heads = %d outside [1, 32]", cfg->resampler_heads);
    if (cfg->image_embed_dim % 8)
      return fail(c, 4807, "IP-Adapter Plus: image_embed_dim = %d must be a multiple of 8", cfg->image_embed_dim);
  }
  CU(c, cudaSetDevice(c->device));
  std::unique_ptr<sdxl_ip_adapter> a(new sdxl_ip_adapter());
  a->ctx = c;
  a->cfg = *cfg;
  int r = with_device_pack(c, pack, bytes, pack_on_device,
                           [&](const PackView& pv) { return build_two_pass(a.get(), pv, build_ip_adapter); });
  if (r) return r;
  *out = a.release();
  return 0;
}

extern "C" void sdxl_ip_adapter_destroy(sdxl_ip_adapter* a) {
  if (!a) return;
  cudaStreamSynchronize(a->ctx->stream);
  delete a;
}

// tokens f16 [n * T, context_dim] = LayerNorm(e @ proj + b) of embeds f32 [n, D] in device memory. Queued on the ctx stream.
static int ip_project(const sdxl_ip_adapter* a, int n, const float* e, __half* tokens) {
  sdxl_ctx* c = a->ctx;
  const Lin& P = a->proj;
  TmpBufs T(c->stream);
  float* y = T.get<float>((size_t)n * P.N * sizeof(float));
  if (!y) return fail(c, 4810, "IP-Adapter projection: cannot allocate %zu bytes", (size_t)n * P.N * sizeof(float));
  for (int b0 = 0; b0 < n; b0 += 8)
    KL(c, gemv_launch(c->stream, e + (size_t)b0 * P.K, P.K, std::min(8, n - b0), P.K, P.w, P.Kpad, P.b, nullptr, 0, P.N, 0, 0,
                      y + (size_t)b0 * P.N, P.N));
  KL(c, layernorm_launch(c->stream, y, a->norm.g, a->norm.b, a->norm.eps, n * a->cfg.tokens_per_image, a->cfg.unet.context_dim, tokens));
  return 0;
}

// IP-Adapter Plus: tokens f16 [n * Q, context_dim] = Resampler(h) of hidden states f32 [n, L, D] in device memory (include/sdxl_b200.h).
// Eager launches on the ctx stream: the GEMMs on igemm (f32 residuals into the latent stream for to_out and fc2), the per-layer
// LayerNorms in one perceiver_ln launch, the attention of the Q latents over L + Q keys per image on attention_small.
static int ip_resample(const sdxl_ip_adapter* a, int n, int L, const float* h, __half* tokens) {
  sdxl_ctx* c = a->ctx;
  const sdxl_ip_adapter_cfg& g = a->cfg;
  const int D = g.image_embed_dim, Q = g.tokens_per_image, W = 64 * g.resampler_heads, S = L + Q, ctx_dim = g.unet.context_dim;
  TmpBufs T(c->stream);
  __half* h16 = T.get<__half>((size_t)n * L * D * sizeof(__half));
  float* x = T.get<float>((size_t)n * L * W * sizeof(float));          // proj_in(h), read by every layer
  float* lat = T.get<float>((size_t)n * Q * W * sizeof(float));        // the latent stream
  __half* kv_in = T.get<__half>((size_t)n * S * W * sizeof(__half));   // per image [LN1(x) ; LN2(lat)]
  __half* a16 = T.get<__half>((size_t)n * Q * W * sizeof(__half));     // the f16 operand of the next GEMM on the latent rows
  __half* q16 = T.get<__half>((size_t)n * Q * W * sizeof(__half));
  __half* kv16 = T.get<__half>((size_t)n * S * 2 * W * sizeof(__half));
  float* f32 = T.get<float>((size_t)n * Q * std::max(4 * W, ctx_dim) * sizeof(float));   // fc1 output, then proj_out output
  __half* f16 = T.get<__half>((size_t)n * Q * 4 * W * sizeof(__half));
  if (!h16 || !x || !lat || !kv_in || !a16 || !q16 || !kv16 || !f32 || !f16)
    return fail(c, 4812, "IP-Adapter Plus Resampler: cannot allocate its buffers (n = %d, seq_len = %d)", n, L);
  // out [M, Lw.N] (row pitch Lw.N) = in [M, Lw.K] (row pitch lda) @ Lw + bias (+ res, f32 output only)
  auto linear = [&](const __half* in, int M, int lda, const Lin& Lw, void* out, int out_f32, const float* res) {
    const IgemmOperands o{in, 1, 1, M, Lw.K, lda, nullptr, 0, 0, 0, 0, 0, Lw.w, Lw.N, Lw.Kpad};
    return igemm_run(c, o, {{0, 0, 0, 0, Lw.Kpad / 64}}, 1, M, 1, IGEMM_LINEAR, 0, out, out_f32, Lw.N, Lw.b, res, Lw.N);
  };
  KL(c, cast_f32_to_f16_launch(c->stream, h, (size_t)n * L * D, h16));
  if (int r = linear(h16, n * L, D, a->proj_in, x, 1, nullptr)) return r;
  for (int i = 0; i < n; ++i)
    CU(c, cudaMemcpyAsync(lat + (size_t)i * Q * W, a->latents, (size_t)Q * W * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  for (const PerceiverLayer& l : a->layers) {
    KL(c, perceiver_ln_launch(c->stream, x, lat, n, L, Q, W, l.ln1.g, l.ln1.b, l.ln2.g, l.ln2.b, l.ln1.eps, kv_in, a16));
    if (int r = linear(a16, n * Q, W, l.to_q, q16, 0, nullptr)) return r;
    if (int r = linear(kv_in, n * S, W, l.to_kv, kv16, 0, nullptr)) return r;
    KL(c, attention_small_launch(c->stream, q16, W, 0, kv16, kv16, 2 * W, 0, W, n, Q, S, g.resampler_heads, nullptr, 0, a16, W, 64));
    if (int r = linear(a16, n * Q, W, l.to_out, lat, 1, lat)) return r;
    KL(c, layernorm_launch(c->stream, lat, l.ln_ff.g, l.ln_ff.b, l.ln_ff.eps, n * Q, W, a16));
    if (int r = linear(a16, n * Q, W, l.fc1, f32, 1, nullptr)) return r;
    KL(c, mlp_act_launch(c->stream, f32, (size_t)n * Q * 4 * W, 0, f16));
    if (int r = linear(f16, n * Q, 4 * W, l.fc2, lat, 1, lat)) return r;
  }
  KL(c, cast_f32_to_f16_launch(c->stream, lat, (size_t)n * Q * W, a16));
  if (int r = linear(a16, n * Q, W, a->proj_out, f32, 1, nullptr)) return r;
  KL(c, layernorm_launch(c->stream, f32, a->norm_out.g, a->norm_out.b, a->norm_out.eps, n * Q, ctx_dim, tokens));
  return 0;
}

extern "C" int sdxl_ip_adapter_resample(sdxl_ip_adapter* a, int n, int seq_len, const float* hidden, int on_host, sdxl_half* tokens_out) {
  if (!a || !hidden || !tokens_out) return fail(a ? a->ctx : nullptr, -1, "sdxl_ip_adapter_resample: null argument");
  sdxl_ctx* c = a->ctx;
  if (!a->plus()) return fail(c, 4813, "ip_adapter_resample: the adapter is a base IP-Adapter (use sdxl_ip_adapter_project)");
  if (n < 1 || seq_len < 1 || seq_len > 4096) return fail(c, 4814, "ip_adapter_resample: n = %d must be >= 1 and seq_len = %d in [1, 4096]", n, seq_len);
  CU(c, cudaSetDevice(c->device));
  TmpBufs T(c->stream);
  const size_t in_bytes = (size_t)n * seq_len * a->cfg.image_embed_dim * sizeof(float);
  const size_t out_bytes = (size_t)n * a->cfg.tokens_per_image * a->cfg.unet.context_dim * sizeof(__half);
  const float* e;
  if (int r = stage_in(c, T, hidden, in_bytes, on_host, e, 4811, "ip_adapter_resample: allocation failed")) return r;
  __half* o = on_host ? T.get<__half>(out_bytes) : (__half*)tokens_out;
  if (!o) return fail(c, 4811, "ip_adapter_resample: allocation failed");
  if (int r = ip_resample(a, n, seq_len, e, o)) return r;
  return on_host ? stage_out(c, tokens_out, o, out_bytes) : 0;
}

extern "C" int sdxl_ip_adapter_project(sdxl_ip_adapter* a, int n, const float* embeds, int on_host, sdxl_half* tokens_out) {
  if (!a || !embeds || !tokens_out || n < 1) return -1;
  sdxl_ctx* c = a->ctx;
  if (a->plus()) return fail(c, 4813, "ip_adapter_project: the adapter is an IP-Adapter Plus (use sdxl_ip_adapter_resample)");
  CU(c, cudaSetDevice(c->device));
  TmpBufs T(c->stream);
  const size_t in_bytes = (size_t)n * a->cfg.image_embed_dim * sizeof(float);
  const size_t out_bytes = (size_t)n * a->cfg.tokens_per_image * a->cfg.unet.context_dim * sizeof(__half);
  const float* e;
  if (int r = stage_in(c, T, embeds, in_bytes, on_host, e, 4811, "ip_adapter_project: allocation failed")) return r;
  __half* o = on_host ? T.get<__half>(out_bytes) : (__half*)tokens_out;
  if (!o) return fail(c, 4811, "ip_adapter_project: allocation failed");
  if (int r = ip_project(a, n, e, o)) return r;
  return on_host ? stage_out(c, tokens_out, o, out_bytes) : 0;
}

// One prompt's values computed into temporaries: the tokens of prompts and negatives, the per-block scales and the masks resized
// to every level. A set is copied into its attachment (ip_commit) only when every prompt's work has succeeded, so a failure leaves
// the attached set unchanged.
struct IpStaged {
  __half* tp = nullptr;
  __half* tn = nullptr;
  float* ts = nullptr;
  float* tm = nullptr;
  size_t tok_bytes = 0, mask_floats = 0;
};

// diffusers' IPAdapterMaskProcessor.downsample grid (mh, mw) for T queries and a mask of H x W pixels, computed in double; both
// are kept >= 1 where diffusers would divide by zero or make an empty grid (levels of a few latent pixels).
static void ip_mask_grid(int H, int W, int T, int& mh, int& mw) {
  const double ratio = (double)W / H;
  mh = std::max(1, (int)sqrt(T / ratio));
  mh += T % mh != 0;
  mw = std::max(1, T / mh);
}

static int ip_stage(sdxl_ctx* c, int n_levels, const IpPrompt& a, const sdxl_image_prompt& p, const std::vector<float>& mask,
                    TmpBufs& T, IpStaged& s) {
  const int n = p.n_batch * p.n_images, n_tb = (int)a.ad->kv.size();
  s.tok_bytes = (size_t)a.n_batch * a.S_ip * a.ad->cfg.unet.context_dim * sizeof(__half);
  const int rows = a.ad->plus() ? p.seq_len : 1;   // input rows per image: Plus hidden states, or one embedding
  const size_t bytes = (size_t)n * rows * a.ad->cfg.image_embed_dim * sizeof(float);
  const char* alloc_failed = "set_image_prompt: cannot allocate %zu bytes for the embeddings";
  const float *e, *neg;
  if (int r = stage_in(c, T, p.embeds, bytes, p.on_host, e, 4820, alloc_failed, bytes)) return r;
  if (p.negative_embeds) {
    if (int r = stage_in(c, T, p.negative_embeds, bytes, p.on_host, neg, 4820, alloc_failed, bytes)) return r;
  } else {   // diffusers' default negative: zeros
    float* z = T.get<float>(bytes);
    if (!z) return fail(c, 4820, alloc_failed, bytes);
    CU(c, cudaMemsetAsync(z, 0, bytes, c->stream));
    neg = z;
  }
  s.tp = T.get<__half>(s.tok_bytes);
  s.tn = T.get<__half>(s.tok_bytes);
  s.ts = T.get<float>(n_tb * sizeof(float));
  if (!s.tp || !s.tn || !s.ts) return fail(c, 4820, "set_image_prompt: cannot allocate the token staging buffers");
  if (a.ad->plus()) {
    if (int r = ip_resample(a.ad, n, p.seq_len, e, s.tp)) return r;
    if (int r = ip_resample(a.ad, n, p.seq_len, neg, s.tn)) return r;
  } else {
    if (int r = ip_project(a.ad, n, e, s.tp)) return r;
    if (int r = ip_project(a.ad, n, neg, s.tn)) return r;
  }
  std::vector<float> sc(n_tb, p.scale);
  if (p.block_scales_host) sc.assign(p.block_scales_host, p.block_scales_host + n_tb);
  CU(c, cudaMemcpyAsync(s.ts, sc.data(), sc.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  if (a.mask_h) {
    const int H = a.mask_h, W = a.mask_w;
    s.mask_floats = ip_mask_off(a, n_levels, a.n_images, 0);
    float* pix = T.get<float>(mask.size() * sizeof(float));
    s.tm = T.get<float>(s.mask_floats * sizeof(float));
    if (!pix || !s.tm) return fail(c, 4820, "set_image_prompt: cannot allocate the mask staging buffers");
    CU(c, cudaMemcpyAsync(pix, mask.data(), mask.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    for (int i = 0; i < a.n_images; ++i)
      for (int l = 0; l < n_levels; ++l) {
        const int Tl = ((H / 8) >> l) * ((W / 8) >> l);
        if (Tl < 1) continue;
        int mh, mw;
        ip_mask_grid(H, W, Tl, mh, mw);
        KL(c, ip_mask_resize_launch(c->stream, pix + (size_t)i * H * W, H, W, mh, mw, Tl, s.tm + ip_mask_off(a, n_levels, i, l)));
      }
  }
  CU(c, cudaStreamSynchronize(c->stream));   // sc, the mask and the caller's host memory; any failure of the work above surfaces here
  return 0;
}

static int ip_commit(sdxl_ctx* c, IpPrompt& a, const IpStaged& s) {
  CU(c, cudaMemcpyAsync(a.tok_pos, s.tp, s.tok_bytes, cudaMemcpyDeviceToDevice, c->stream));
  CU(c, cudaMemcpyAsync(a.tok_neg, s.tn, s.tok_bytes, cudaMemcpyDeviceToDevice, c->stream));
  CU(c, cudaMemcpyAsync(a.scales, s.ts, a.ad->kv.size() * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  if (a.mask_h) CU(c, cudaMemcpyAsync(a.masks, s.tm, s.mask_floats * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  return 0;
}

// The checks of one prompt that need no device work.
static int ip_prompt_check(sdxl_unet* u, int k, const sdxl_image_prompt* p) {
  sdxl_ctx* c = u->ctx;
  const sdxl_ip_adapter* ad = p->adapter;
  if (u->cfg.is_refiner) return fail(c, 4832, "set_image_prompt: IP-Adapter on the refiner is not supported");
  if (int r = attachable(u, "set_image_prompt: prompt", k, ad, {4830, 4831, 4833})) return r;
  // equal cfgs: the adapter's K/V were laid out by the same block program as the UNet's transformer blocks
  const int n_tb = (int)ad->kv.size();
  if (!p->embeds) return fail(c, 4835, "set_image_prompt: null embeds");
  if (ad->plus()) {
    if (!p->negative_embeds)
      return fail(c, 4839, "set_image_prompt: an IP-Adapter Plus prompt needs negative_embeds (the hidden states of an all-zero "
                           "pixel tensor; the library cannot compute them)");
    if (p->seq_len < 1 || p->seq_len > 4096) return fail(c, 4840, "set_image_prompt: seq_len = %d outside [1, 4096]", p->seq_len);
  }
  if (p->n_batch < 1 || p->n_images < 1 || p->n_images > 64)
    return fail(c, 4836, "set_image_prompt: n_batch = %d must be >= 1 and n_images = %d in [1, 64]", p->n_batch, p->n_images);
  if (!isfinite(p->scale)) return fail(c, 4837, "set_image_prompt: scale is not finite");
  if (p->block_scales_host)
    for (int i = 0; i < n_tb; ++i)
      if (!isfinite(p->block_scales_host[i])) return fail(c, 4837, "set_image_prompt: block scale %d is not finite", i);
  if (u->cond.condB > 0)
    if (int r = ip_check_batch(u, p->n_batch, u->cond.condB, u->rows)) return r;
  return 0;
}

// Reads prompt k's mask planes [n_images, height, width] into host memory and checks them.
static int ip_mask_read(sdxl_ctx* c, const sdxl_ip_mask& m, int n_images, int k, std::vector<float>& host) {
  if (m.height < 8 || m.width < 8 || m.height % 8 || m.width % 8 || m.height > 16384 || m.width > 16384)
    return fail(c, 4843, "set_image_prompts: mask %d is %dx%d pixels; height and width must be positive multiples of 8 up to 16384", k,
                m.height, m.width);
  host.resize((size_t)n_images * m.height * m.width);
  if (m.on_host) {
    memcpy(host.data(), m.mask, host.size() * sizeof(float));
  } else {
    CU(c, cudaMemcpyAsync(host.data(), m.mask, host.size() * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
  }
  for (size_t i = 0; i < host.size(); ++i)
    if (!isfinite(host[i])) return fail(c, 4844, "set_image_prompts: mask %d has a non-finite value at element %zu", k, i);
  return 0;
}

extern "C" int sdxl_unet_set_image_prompts(sdxl_unet* u, int n, const sdxl_image_prompt* prompts, const sdxl_ip_mask* masks) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  if (n < 0 || n > SDXL_MAX_IMAGE_PROMPTS)
    return fail(c, 4841, "set_image_prompts: n = %d outside [0, %d]", n, SDXL_MAX_IMAGE_PROMPTS);
  if (n == 0) return attach_detach(u, u->ip);
  if (!prompts) return fail(c, -1, "set_image_prompts: null prompts");
  // validate everything first: on failure the attached set is unchanged
  const int nl = u->cfg.n_levels;
  std::vector<IpPrompt> shape(n);
  std::vector<std::vector<float>> mask(n);
  int n_src = 0;
  for (int k = 0; k < n; ++k) {
    const sdxl_image_prompt& p = prompts[k];
    if (int r = ip_prompt_check(u, k, &p)) return r;
    const sdxl_ip_mask* m = masks && masks[k].mask ? &masks[k] : nullptr;
    IpPrompt& a = shape[k];
    a.ad = p.adapter;
    a.n_batch = p.n_batch;
    a.n_images = p.n_images;
    a.S_ip = p.n_images * p.adapter->cfg.tokens_per_image;
    if (m) {
      if (int r = ip_mask_read(c, *m, p.n_images, k, mask[k])) return r;
      a.mask_h = m->height;
      a.mask_w = m->width;
    }
    n_src += a.n_sources();
  }
  if (n_src > SDXL_MAX_IP_SOURCES)
    return fail(c, 4842, "set_image_prompts: %d image sources (one per unmasked prompt, one per image of a masked prompt); at most %d",
                n_src, SDXL_MAX_IP_SOURCES);
  const int condB = u->cond.condB;
  TmpBufs T(c->stream);
  std::vector<IpStaged> st(n);
  bool same = u->ip && u->ip->prompts.size() == (size_t)n;
  for (int k = 0; same && k < n; ++k) {
    const IpPrompt &o = u->ip->prompts[k], &a = shape[k];
    same = o.ad == a.ad && o.n_batch == a.n_batch && o.n_images == a.n_images && o.mask_h == a.mask_h && o.mask_w == a.mask_w;
  }
  if (same) {   // same buffers: plan stays
    for (int k = 0; k < n; ++k)
      if (int r = ip_stage(c, nl, u->ip->prompts[k], prompts[k], mask[k], T, st[k])) return r;
    for (int k = 0; k < n; ++k)
      if (int r = ip_commit(c, u->ip->prompts[k], st[k])) return r;
    if (condB > 0)
      for (IpPrompt& a : u->ip->prompts)
        if (int r = ip_hoist(u, a)) return r;
    return 0;
  }
  std::unique_ptr<IpAttach> a(new IpAttach());
  a->prompts = std::move(shape);
  if (int r = carve_measured(c, a->mem, 4838, "set_image_prompt: token buffers", [&](Arena& A) {
        for (IpPrompt& q : a->prompts) {
          const size_t tok = (size_t)q.n_batch * q.S_ip * u->cfg.context_dim;
          q.tok_pos = A.get<__half>(tok);
          q.tok_neg = A.get<__half>(tok);
          q.scales = A.get<float>(q.ad->kv.size());
          q.masks = q.mask_h ? A.get<float>(ip_mask_off(q, nl, q.n_images, 0)) : nullptr;
        }
        return 0;
      }))
    return r;
  for (int k = 0; k < n; ++k) {
    IpPrompt& q = a->prompts[k];
    if (condB > 0)
      if (int r = ip_cond_alloc(c, q, condB, q.cond)) return r;
    if (int r = ip_stage(c, nl, q, prompts[k], mask[k], T, st[k])) return r;
  }
  for (int k = 0; k < n; ++k)
    if (int r = ip_commit(c, a->prompts[k], st[k])) return r;
  if (condB > 0)
    for (IpPrompt& q : a->prompts)
      if (int r = ip_hoist(u, q)) return r;
  return attach_install(u, u->ip, std::move(a));
}

extern "C" int sdxl_unet_set_image_prompt(sdxl_unet* u, const sdxl_image_prompt* p) {
  return sdxl_unet_set_image_prompts(u, p ? 1 : 0, p, nullptr);
}

// ================================================================================================
// T2I-Adapter (include/sdxl_b200.h: sdxl_t2i_adapter_load, sdxl_unet_set_t2i_adapters; DESIGN.md §11)
// ================================================================================================
// Why a UNet cfg cannot take a T2I-Adapter, or null: FullAdapterXL's four features fit SDXL base's encoder only.
static const char* t2i_unet_problem(const sdxl_unet_cfg& g) {
  if (g.is_refiner) return "the refiner is not supported";
  if (g.n_levels != 3) return "the UNet must have 3 levels";
  if (g.transformer_depths[0] != 0) return "the UNet must have no transformer on level 0";
  if (g.channel_mults[0] == g.channel_mults[1] || g.channel_mults[1] == g.channel_mults[2])
    return "the widths of levels 0, 1 and 2 must differ (every in_conv of the adapter is present)";
  return nullptr;
}

// The input blocks after which F_0, F_1, F_2 are added: per level its last block with a transformer or, on a level without one,
// its last block (the Downsample where it has one) -- where diffusers' CrossAttnDownBlock2D and DownBlock2D add them.
static void t2i_points(const BlockProgram& p, size_t out[3]) {
  for (int level = 0; level < 3; ++level) {
    size_t last = 0, last_tr = 0;
    for (size_t i = 1; i < p.ins.size(); ++i)
      if (p.ins[i].level == level) {
        last = i;
        if (has_transformer(p.ins[i].type)) last_tr = i;
      }
    out[level] = last_tr ? last_tr : last;
  }
}

static int build_t2i_adapter(sdxl_t2i_adapter* a, const PackView& pv, Arena& A) {
  const int* ch = a->ch;
  Loader L{a->ctx, &pv, &A, a->ctx->stream};
  std::set<std::string> names;
  auto conv = [&](const std::string& path, int I, int O, int ks) {
    names.insert(path + "/weight");
    names.insert(path + "/bias");
    return L.conv(path, I, O, ks);
  };
  a->conv_in = conv("conv_in", a->cfg.in_channels * 256, ch[0], 3);
  for (int k = 1; k < 3; ++k) a->in_conv[k - 1] = conv("body/" + std::to_string(k) + "/in_conv", ch[k - 1], ch[k], 1);
  for (int k = 0; k < 4 && !L.err; ++k) {
    a->res[k].clear();
    for (int j = 0; j < a->cfg.n_res_blocks; ++j) {
      const std::string p = "body/" + std::to_string(k) + "/resnets/" + std::to_string(j);
      T2IRes r;
      r.block1 = conv(p + "/block1", ch[k], ch[k], 3);
      r.block2 = conv(p + "/block2", ch[k], ch[k], 1);
      a->res[k].push_back(r);
    }
  }
  if (L.err) return L.err;
  for (const auto& t : pv.t)
    if (!names.count(t.first)) return fail(a->ctx, 4904, "T2I-Adapter pack: tensor '%s' is not part of an adapter for this cfg", t.first.c_str());
  return 0;
}

extern "C" int sdxl_t2i_adapter_load(sdxl_ctx* c, const sdxl_t2i_adapter_cfg* cfg, const void* pack, size_t bytes, int pack_on_device,
                                     sdxl_t2i_adapter** out) {
  if (!c || !cfg || !pack || !out) return fail(c, -1, "sdxl_t2i_adapter_load: null argument");
  *out = nullptr;
  if (int r = check_unet_cfg(c, cfg->unet)) return r;
  if (const char* why = t2i_unet_problem(cfg->unet)) return fail(c, 4900, "T2I-Adapter: %s", why);
  if (cfg->in_channels < 1 || cfg->in_channels > 4) return fail(c, 4901, "T2I-Adapter: in_channels = %d outside [1, 4]", cfg->in_channels);
  if (cfg->n_res_blocks < 1 || cfg->n_res_blocks > 8) return fail(c, 4902, "T2I-Adapter: n_res_blocks = %d outside [1, 8]", cfg->n_res_blocks);
  CU(c, cudaSetDevice(c->device));
  std::unique_ptr<sdxl_t2i_adapter> a(new sdxl_t2i_adapter());
  a->ctx = c;
  a->cfg = *cfg;
  const sdxl_unet_cfg& g = cfg->unet;
  for (int k = 0; k < 4; ++k) a->ch[k] = g.model_channels * g.channel_mults[k < 3 ? k : 2];
  int r = with_device_pack(c, pack, bytes, pack_on_device,
                           [&](const PackView& pv) { return build_two_pass(a.get(), pv, build_t2i_adapter); });
  if (r) return r;
  *out = a.release();
  return 0;
}

extern "C" void sdxl_t2i_adapter_destroy(sdxl_t2i_adapter* a) {
  if (!a) return;
  cudaStreamSynchronize(a->ctx->stream);
  delete a;
}

// ks x ks pad ks/2 conv of an f16 NHWC image [Bn, H, W, cv.I] on the implicit GEMM: out f32 NHWC = conv + bias (+ res, may be out).
static int conv_nhwc(sdxl_ctx* c, const __half* a, int Bn, int H, int W, const Conv& cv, float* out, const float* res) {
  const IgemmOperands o{a, Bn, H, W, cv.I, cv.I, nullptr, 0, 0, 0, 0, 0, cv.w, cv.O, cv.Ktot};
  return igemm_run(c, o, conv_taps(cv.ks, cv.Ipad / 64), H, W, Bn, IGEMM_LINEAR, 0, out, 1, cv.O, cv.b, res, cv.O);
}

// Elements of F_k for n hints of H x W pixels.
static size_t t2i_feature_elems(const sdxl_t2i_adapter* a, int k, int n, int H, int W) {
  const int d = k < 2 ? 16 : 32;
  return (size_t)n * (H / d) * (W / d) * a->ch[k];
}

// Adapter forward of hint f32 NCHW [n, in_channels, H, W] (device) into F[k] f32 NHWC at scale 1. Eager on the ctx stream.
static int t2i_forward(const sdxl_t2i_adapter* a, int n, int H, int W, const float* hint, float* const F[4]) {
  sdxl_ctx* c = a->ctx;
  const int h2 = H / 16, w2 = W / 16, h4 = H / 32, w4 = W / 32;
  size_t max16 = (size_t)n * h2 * w2 * a->cfg.in_channels * 256, max32 = 0;
  for (int k = 0; k < 4; ++k) {
    max16 = std::max(max16, t2i_feature_elems(a, k, n, H, W));
    max32 = std::max(max32, t2i_feature_elems(a, k, n, H, W));
  }
  TmpBufs T(c->stream);
  __half* a16 = T.get<__half>(max16 * sizeof(__half));   // the f16 operand of the next conv
  float* t32 = T.get<float>(max32 * sizeof(float));      // block1 output
  __half* t16 = T.get<__half>(max32 * sizeof(__half));   // relu(block1)
  if (!a16 || !t32 || !t16) return fail(c, 4910, "T2I-Adapter: cannot allocate its scratch (n = %d, %dx%d)", n, H, W);
  KL(c, pixel_unshuffle_launch(c->stream, hint, n, a->cfg.in_channels, H, W, a16));
  if (int r = conv_nhwc(c, a16, n, h2, w2, a->conv_in, F[0], nullptr)) return r;
  for (int k = 0; k < 4; ++k) {
    const int hk = k < 2 ? h2 : h4, wk = k < 2 ? w2 : w4;
    const size_t e = t2i_feature_elems(a, k, n, H, W);
    if (k == 1) {
      KL(c, cast_f32_to_f16_launch(c->stream, F[0], t2i_feature_elems(a, 0, n, H, W), a16));
      if (int r = conv_nhwc(c, a16, n, hk, wk, a->in_conv[0], F[1], nullptr)) return r;
    } else if (k == 2) {
      KL(c, avg_pool2_f16_launch(c->stream, F[1], n, h2, w2, a->ch[1], a16));
      if (int r = conv_nhwc(c, a16, n, hk, wk, a->in_conv[1], F[2], nullptr)) return r;
    } else if (k == 3) {
      CU(c, cudaMemcpyAsync(F[3], F[2], e * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
    }
    for (const T2IRes& rb : a->res[k]) {   // x = x + block2(relu(block1(x))), the residual added in block2's epilogue
      KL(c, cast_f32_to_f16_launch(c->stream, F[k], e, a16));
      if (int r = conv_nhwc(c, a16, n, hk, wk, rb.block1, t32, nullptr)) return r;
      KL(c, relu_f16_launch(c->stream, t32, e, t16));
      if (int r = conv_nhwc(c, t16, n, hk, wk, rb.block2, F[k], F[k])) return r;
    }
  }
  return 0;
}

static int t2i_check_size(sdxl_ctx* c, int n, int H, int W) {
  if (n < 1 || H < 32 || W < 32 || H % 32 || W % 32)
    return fail(c, 4920, "T2I-Adapter: hint must be [n >= 1, C, H, W] with H, W positive multiples of 32 (got n=%d, %dx%d)", n, H, W);
  return 0;
}

extern "C" int sdxl_t2i_adapter_features(sdxl_t2i_adapter* a, int n, int H, int W, const float* hint, int on_host, float* out) {
  if (!a || !hint || !out) return fail(a ? a->ctx : nullptr, -1, "sdxl_t2i_adapter_features: null argument");
  sdxl_ctx* c = a->ctx;
  if (int r = t2i_check_size(c, n, H, W)) return r;
  CU(c, cudaSetDevice(c->device));
  TmpBufs T(c->stream);
  size_t total = 0;
  float* F[4];
  for (int k = 0; k < 4; ++k) {
    total += t2i_feature_elems(a, k, n, H, W);
    F[k] = T.get<float>(t2i_feature_elems(a, k, n, H, W) * sizeof(float));
  }
  const size_t in_bytes = (size_t)n * a->cfg.in_channels * H * W * sizeof(float);
  const float* x;
  if (int r = stage_in(c, T, hint, in_bytes, on_host, x, 4911, "t2i_adapter_features: allocation failed")) return r;
  float* o = on_host ? T.get<float>(total * sizeof(float)) : out;
  if (!o || !F[0] || !F[1] || !F[2] || !F[3]) return fail(c, 4911, "t2i_adapter_features: allocation failed");
  if (int r = t2i_forward(a, n, H, W, x, F)) return r;
  size_t off = 0;
  for (int k = 0; k < 4; ++k) {
    const int d = k < 2 ? 16 : 32;
    KL(c, nhwc_to_nchw_f32_launch(c->stream, F[k], n, (H / d) * (W / d), a->ch[k], a->ch[k], o + off));
    off += t2i_feature_elems(a, k, n, H, W);
  }
  return on_host ? stage_out(c, out, o, total * sizeof(float)) : 0;
}

extern "C" int sdxl_unet_set_t2i_adapters(sdxl_unet* u, int n, const sdxl_t2i_control* ctl, int32_t t_min) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  // validate everything first: on failure the attached set is unchanged
  if (n < 0 || n > SDXL_MAX_T2I_ADAPTERS) return fail(c, 4930, "set_t2i_adapters: n = %d outside [0, %d]", n, SDXL_MAX_T2I_ADAPTERS);
  if (n > 0 && !ctl) return fail(c, 4931, "set_t2i_adapters: null control array");
  if (n > 0)
    if (const char* why = t2i_unet_problem(u->cfg)) return fail(c, 4932, "set_t2i_adapters: %s", why);
  for (int k = 0; k < n; ++k) {
    if (int r = attachable(u, "set_t2i_adapters: item", k, ctl[k].adapter, {4933, 4934, 4935})) return r;
    if (!ctl[k].hint) return fail(c, 4936, "set_t2i_adapters: item %d: null hint", k);
    if (ctl[k].n_hint < 1) return fail(c, 4937, "set_t2i_adapters: item %d: n_hint = %d must be >= 1", k, ctl[k].n_hint);
    if (ctl[k].n_hint != ctl[0].n_hint || ctl[k].height != ctl[0].height || ctl[k].width != ctl[0].width)
      return fail(c, 4938, "set_t2i_adapters: item %d: n_hint and size (%d, %dx%d) differ from item 0's (%d, %dx%d)", k, ctl[k].n_hint,
                  ctl[k].height, ctl[k].width, ctl[0].n_hint, ctl[0].height, ctl[0].width);
    if (int r = t2i_check_size(c, ctl[k].n_hint, ctl[k].height, ctl[k].width)) return r;
    if (!isfinite(ctl[k].scale)) return fail(c, 4939, "set_t2i_adapters: item %d: scale is not finite", k);
  }
  if (n == 0) return attach_detach(u, u->t2i);
  const int n_hint = ctl[0].n_hint, H = ctl[0].height, W = ctl[0].width;
  const Extent ext{n_hint, H / 8, W / 8};
  const sdxl_t2i_adapter* a0 = ctl[0].adapter;
  // the sum is formed in temporaries and copied into the attachment only when all of it succeeded
  TmpBufs T(c->stream);
  float* S[4];
  float* Fa[4];
  bool ok = true;
  for (int k = 0; k < 4; ++k) {
    S[k] = T.get<float>(t2i_feature_elems(a0, k, n_hint, H, W) * sizeof(float));
    Fa[k] = T.get<float>(t2i_feature_elems(a0, k, n_hint, H, W) * sizeof(float));
    ok = ok && S[k] && Fa[k];
  }
  if (!ok) return fail(c, 4940, "set_t2i_adapters: cannot allocate the feature staging buffers");
  for (int k = 0; k < 4; ++k) CU(c, cudaMemsetAsync(S[k], 0, t2i_feature_elems(a0, k, n_hint, H, W) * sizeof(float), c->stream));
  for (int i = 0; i < n; ++i) {
    const size_t bytes = (size_t)n_hint * ctl[i].adapter->cfg.in_channels * H * W * sizeof(float);
    const float* hint;
    if (int r = stage_in(c, T, ctl[i].hint, bytes, ctl[i].hint_on_host, hint, 4940, "set_t2i_adapters: cannot allocate %zu bytes for hint %d",
                         bytes, i))
      return r;
    if (int r = t2i_forward(ctl[i].adapter, n_hint, H, W, hint, Fa)) return r;
    for (int k = 0; k < 4; ++k)   // S += s_i * F_i, adapters in array order
      KL(c, axpby_launch(c->stream, S[k], Fa[k], t2i_feature_elems(a0, k, n_hint, H, W), 1.f, ctl[i].scale));
  }
  CU(c, cudaStreamSynchronize(c->stream));   // the caller's host hints; any failure of the work above surfaces here
  T2IAttach* cur = u->t2i.get();
  std::unique_ptr<T2IAttach> fresh;
  if (!cur || !(cur->ext == ext)) {   // new shapes: new buffers and a new plan
    fresh.reset(new T2IAttach());
    T2IAttach& f = *fresh;
    f.ext = ext;
    t2i_points(block_program(u->cfg), f.points);
    for (int k = 0; k < 4; ++k) {
      const int d = k < 2 ? 16 : 32;
      f.C[k] = a0->ch[k]; f.H[k] = H / d; f.W[k] = W / d;
    }
    if (int r = carve_measured(c, f.mem, 4941, "set_t2i_adapters: feature buffers", [&](Arena& A) {
          for (int k = 0; k < 4; ++k) f.F[k] = A.get<float>(t2i_feature_elems(a0, k, n_hint, H, W));
          f.t_min = A.get<int>(1);
          return 0;
        }))
      return r;
    cur = fresh.get();
  }
  for (int k = 0; k < 4; ++k)
    CU(c, cudaMemcpyAsync(cur->F[k], S[k], t2i_feature_elems(a0, k, n_hint, H, W) * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  CU(c, cudaMemcpyAsync(cur->t_min, &t_min, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  if (fresh) return attach_install(u, u->t2i, std::move(fresh));
  CU(c, cudaStreamSynchronize(c->stream));   // t_min is on the stack
  return 0;
}

// ================================================================================================
// inpainting UNet (include/sdxl_b200.h: sdxl_unet_set_inpaint_condition; DESIGN.md §12)
// ================================================================================================
extern "C" int sdxl_unet_set_inpaint_condition(sdxl_unet* u, const sdxl_inpaint_condition* ic) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  const sdxl_unet_cfg& g = u->cfg;
  if (!ic) return attach_detach(u, u->inpaint);
  // validate everything first: on failure the attached condition is unchanged
  if (!inpaint_layout(g))
    return fail(c, 4960, "set_inpaint_condition: the UNet does not have the inpainting layout (in_channels = %d, out_channels = %d; "
                "it needs in_channels = 2 * out_channels + 1 > 8)", g.in_channels, g.out_channels);
  if (!ic->cond) return fail(c, 4961, "set_inpaint_condition: null cond");
  if (ic->n < 1) return fail(c, 4962, "set_inpaint_condition: n = %d must be >= 1", ic->n);
  if (ic->height < 8 || ic->width < 8 || ic->height % 8 || ic->width % 8)
    return fail(c, 4963, "set_inpaint_condition: size %dx%d must be a positive multiple of 8", ic->height, ic->width);
  const Extent ext{ic->n, ic->height / 8, ic->width / 8};
  const size_t bytes = (size_t)ext.n * (g.in_channels - g.out_channels) * ext.h * ext.w * sizeof(float);
  InpaintAttach* cur = u->inpaint.get();
  std::unique_ptr<InpaintAttach> fresh;
  if (!cur || !(cur->ext == ext)) {   // new shape: a new buffer and a new plan
    fresh.reset(new InpaintAttach());
    fresh->ext = ext;
    if (int r = carve_measured(c, fresh->mem, 4964, "set_inpaint_condition: condition buffer", [&](Arena& A) {
          fresh->cond = A.get<float>(bytes / sizeof(float));
          return 0;
        }))
      return r;
    cur = fresh.get();
  }
  CU(c, cudaMemcpyAsync(cur->cond, ic->cond, bytes, ic->on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
  if (fresh) return attach_install(u, u->inpaint, std::move(fresh));
  CU(c, cudaStreamSynchronize(c->stream));   // the caller's memory
  return 0;
}

// ================================================================================================
// instruction-based editing (include/sdxl_b200.h: sdxl_unet_set_edit_image; DESIGN.md §21)
// ================================================================================================
extern "C" int sdxl_unet_set_edit_image(sdxl_unet* u, const sdxl_edit_image* e) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  const sdxl_unet_cfg& g = u->cfg;
  if (!e) return attach_detach(u, u->edit);
  // validate everything first: on failure the attached image is unchanged
  if (!edit_layout(g)) return fail(c, 5710, "set_edit_image: the UNet does not have the edit layout (cfg edit_layout = 0)");
  if (!e->latent) return fail(c, 5711, "set_edit_image: null latent");
  if (e->n < 1) return fail(c, 5712, "set_edit_image: n = %d must be >= 1", e->n);
  if (e->height < 8 || e->width < 8 || e->height % 8 || e->width % 8)
    return fail(c, 5713, "set_edit_image: size %dx%d must be a positive multiple of 8", e->height, e->width);
  if (!isfinite(e->image_guidance)) return fail(c, 5714, "set_edit_image: image_guidance = %g must be finite", e->image_guidance);
  const Extent ext{e->n, e->height / 8, e->width / 8};
  const size_t bytes = (size_t)ext.n * g.out_channels * ext.h * ext.w * sizeof(float);
  EditAttach* cur = u->edit.get();
  std::unique_ptr<EditAttach> fresh;
  if (!cur || !(cur->ext == ext)) {   // new shape: a new buffer and a new plan
    fresh.reset(new EditAttach());
    fresh->ext = ext;
    if (int r = carve_measured(c, fresh->mem, 5715, "set_edit_image: image buffer", [&](Arena& A) {
          fresh->latent = A.get<float>(bytes / sizeof(float));
          return 0;
        }))
      return r;
    cur = fresh.get();
  }
  cur->image_guidance = e->image_guidance;
  CU(c, cudaMemcpyAsync(cur->latent, e->latent, bytes, e->on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
  if (fresh) return attach_install(u, u->edit, std::move(fresh));
  if (int r = edit_rows_fill(u)) return r;   // the same plan and graph read the new values
  CU(c, cudaStreamSynchronize(c->stream));   // the caller's memory
  return 0;
}

// ================================================================================================
// LoRA adapters (include/sdxl_b200.h; merge in engine_core.h: adapters_apply)
// ================================================================================================
extern "C" int sdxl_unet_set_adapters(sdxl_unet* u, int n, const sdxl_adapter* adapters) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  int r = adapters_apply(c, u->lora, n, adapters);
  if (r) return r;
  // the head conv's duplicated [W | W] copy follows conv_out
  const Conv& cv = u->conv_out;
  for (int h2 = 0; h2 < 2; ++h2)
    CU(c, cudaMemcpy2DAsync(u->conv_out_w2 + (size_t)h2 * cv.Ktot, (size_t)2 * cv.Ktot * sizeof(__half), cv.w, (size_t)cv.Ktot * sizeof(__half),
                            (size_t)cv.Ktot * sizeof(__half), (size_t)cv.O, cudaMemcpyDeviceToDevice, c->stream));
  // cross-attention K/V and the label MLP were computed from the previous weights
  return u->cond.condB > 0 ? hoist_conditioning(u) : 0;
}

// ================================================================================================
// perturbed-attention guidance (include/sdxl_b200.h: sdxl_unet_set_pag; DESIGN.md §14)
// ================================================================================================
extern "C" int sdxl_unet_num_self_attentions(const sdxl_unet* u) { return u ? (int)u->tblocks.size() : -1; }

extern "C" int sdxl_unet_set_pag(sdxl_unet* u, const sdxl_pag* p) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  if (!p) return attach_detach(u, u->pag);
  // validate everything first: on failure the attached state is unchanged
  const int n = (int)u->tblocks.size();
  if (!(isfinite(p->scale) && p->scale > 0.f)) return fail(c, 4970, "set_pag: scale = %g must be finite and > 0 (detach with NULL)", p->scale);
  if (!(isfinite(p->adaptive_scale) && p->adaptive_scale >= 0.f))
    return fail(c, 4971, "set_pag: adaptive_scale = %g must be finite and >= 0", p->adaptive_scale);
  if (p->n_layers != n) return fail(c, 4972, "set_pag: n_layers = %d but the UNet has %d self-attentions", p->n_layers, n);
  if (!p->layers_host) return fail(c, 4973, "set_pag: null layers_host");
  int n_sel = 0;
  for (int i = 0; i < n; ++i) n_sel += p->layers_host[i] != 0;
  if (!n_sel) return fail(c, 4974, "set_pag: no self-attention selected");
  if (p->forward_perturbed_rows < 0) return fail(c, 4975, "set_pag: forward_perturbed_rows = %d is negative", p->forward_perturbed_rows);
  std::vector<uint8_t> layers(n);
  for (int i = 0; i < n; ++i) layers[i] = p->layers_host[i] != 0;
  if (!u->pag || u->pag->layers != layers) {   // a new layer set changes the plan; the scales and the row count do not (ensure_plan)
    std::unique_ptr<PagAttach> fresh(new PagAttach());
    fresh->layers = std::move(layers);
    if (int r = attach_install(u, u->pag, std::move(fresh))) return r;
  }
  u->pag->scale = p->scale;
  u->pag->adaptive = p->adaptive_scale;
  u->pag->forward_rows = p->forward_perturbed_rows;
  return 0;
}

// ================================================================================================
// FreeU (include/sdxl_b200.h: sdxl_unet_set_freeu; DESIGN.md §15)
// ================================================================================================
extern "C" int sdxl_unet_set_freeu(sdxl_unet* u, const sdxl_freeu* f) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  if (!f) return attach_detach(u, u->freeu);
  // validate everything first: on failure the attached state is unchanged
  const float v[4] = {f->s1, f->s2, f->b1, f->b2};
  static const char* const names[4] = {"s1", "s2", "b1", "b2"};
  for (int i = 0; i < 4; ++i)
    if (!isfinite(v[i])) return fail(c, 4980 + i, "set_freeu: %s = %g must be finite", names[i], v[i]);
  // diffusers runs FreeU only when all four values are nonzero
  for (int i = 0; i < 4; ++i)
    if (v[i] == 0.f) return attach_detach(u, u->freeu);
  if (u->freeu) {   // new values only: the plan and its graph read them from the device
    CU(c, cudaMemcpyAsync(u->freeu->vals, v, sizeof(v), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));   // v is on this stack
    return 0;
  }
  std::unique_ptr<FreeuAttach> fresh(new FreeuAttach());
  if (int r = carve_measured(c, fresh->mem, 4984, "set_freeu: value buffer", [&](Arena& A) {
        fresh->vals = A.get<float>(4);
        return 0;
      }))
    return r;
  CU(c, cudaMemcpyAsync(fresh->vals, v, sizeof(v), cudaMemcpyHostToDevice, c->stream));
  return attach_install(u, u->freeu, std::move(fresh));   // drains the stream before v goes
}

// ================================================================================================
// DeepCache (include/sdxl_b200.h: sdxl_unet_set_deepcache; DESIGN.md §17)
// ================================================================================================
extern "C" int sdxl_unet_set_deepcache(sdxl_unet* u, const sdxl_deepcache* d) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  if (!d) return attach_detach(u, u->deepcache);
  // validate everything first: on failure the attached state is unchanged
  const int n = (int)u->out_blocks.size();
  if (d->interval < 1) return fail(c, 4990, "set_deepcache: interval = %d must be >= 1", d->interval);
  if (d->branch < 0 || d->branch >= n) return fail(c, 4991, "set_deepcache: branch = %d outside [0, %d]", d->branch, n - 1);
  if (d->forward_cached != 0 && d->forward_cached != 1)
    return fail(c, 4992, "set_deepcache: forward_cached = %d must be 0 or 1", d->forward_cached);
  if (!u->deepcache || u->deepcache->branch != d->branch) {   // a new branch changes the plan; the interval and the forward kind do not
    std::unique_ptr<DeepcacheAttach> fresh(new DeepcacheAttach());
    fresh->branch = d->branch;
    if (int r = attach_install(u, u->deepcache, std::move(fresh))) return r;
  }
  u->deepcache->interval = d->interval;
  u->deepcache->forward_cached = d->forward_cached != 0;
  return 0;
}

// ================================================================================================
// prediction type, guidance rescale and the noise table (include/sdxl_b200.h: sdxl_unet_set_prediction; DESIGN.md §18)
// ================================================================================================
extern "C" int sdxl_unet_set_prediction(sdxl_unet* u, const sdxl_prediction* p) {
  if (!u) return -1;
  sdxl_ctx* c = u->ctx;
  if (!p) {
    u->prediction = SDXL_PREDICTION_EPSILON;
    u->guidance_rescale = 0.f;
    u->alphas = u->alphas_loaded;
    return 0;
  }
  // validate everything first: on failure the previous state is unchanged
  const int N = (int)u->alphas_loaded.size();
  if (p->type != SDXL_PREDICTION_EPSILON && p->type != SDXL_PREDICTION_V)
    return fail(c, 5600, "set_prediction: type = %d must be SDXL_PREDICTION_EPSILON (0) or SDXL_PREDICTION_V (1)", p->type);
  if (!(p->guidance_rescale >= 0.f && p->guidance_rescale <= 1.f))   // also refuses NaN
    return fail(c, 5601, "set_prediction: guidance_rescale = %g outside [0, 1]", p->guidance_rescale);
  if (p->n_alphas != 0 && p->n_alphas != N)
    return fail(c, 5602, "set_prediction: n_alphas = %d must be 0 (the loaded table) or the UNet's %d timesteps", p->n_alphas, N);
  if (p->n_alphas && !p->alphas_cumprod_host) return fail(c, 5603, "set_prediction: null alphas_cumprod_host with n_alphas = %d", p->n_alphas);
  for (int i = 0; i < p->n_alphas; ++i) {
    const double a = p->alphas_cumprod_host[i];
    if (!(a > 0.0 && a < 1.0) || (i && !(a < p->alphas_cumprod_host[i - 1])))
      return fail(c, 5604, "set_prediction: alphas_cumprod_host[%d] = %g is not inside (0, 1) and below its predecessor", i, a);
  }
  u->prediction = p->type;
  u->guidance_rescale = p->guidance_rescale;
  if (p->n_alphas) u->alphas.assign(p->alphas_cumprod_host, p->alphas_cumprod_host + N);
  else u->alphas = u->alphas_loaded;
  return 0;
}

// ================================================================================================
// UNet::forward
// ================================================================================================
// The direct forwards' body: x NCHW [B, C, h, w] in, eps NCHW out, both f16 (sdxl_unet_forward) or both f32.
static int unet_forward(sdxl_unet* u, int B, int h, int w, const void* x, bool f16, double t, void* eps_out) {
  sdxl_ctx* c = u->ctx;
  int r = ensure_plan(u, B, B, h, w, u->pag ? u->pag->forward_rows : 0);
  if (r) return r;
  const bool cached = u->deepcache && u->deepcache->forward_cached;
  if (cached && (r = cached_ready(u))) return r;
  Plan* P = u->plan.get();
  const size_t n = (size_t)B * latent_channels(u->cfg) * h * w;
  if (f16) KL(c, cast_f16_to_f32_launch(c->stream, (const __half*)x, n, P->x_in));
  else CU(c, cudaMemcpyAsync(P->x_in, x, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
  if ((r = set_t(u, t))) return r;
  if ((r = run_plan(u, cached))) return r;
  if (f16) KL(c, nhwc_to_nchw_f16_launch(c->stream, P->eps, B, h * w, u->cfg.out_channels, P->eps_ld, (__half*)eps_out));
  else KL(c, nhwc_to_nchw_f32_launch(c->stream, P->eps, B, h * w, u->cfg.out_channels, P->eps_ld, (float*)eps_out));
  return 0;
}
extern "C" int sdxl_unet_forward(sdxl_unet* u, int B, int h, int w, const sdxl_half* x, int32_t t_host, sdxl_half* eps_out) {
  if (!u || !x || !eps_out) return -1;
  CU(u->ctx, cudaSetDevice(u->ctx->device));
  return unet_forward(u, B, h, w, x, true, t_host, eps_out);
}
extern "C" int sdxl_unet_forward_f32(sdxl_unet* u, int B, int h, int w, const float* x, int32_t t_host, float* eps_out) {
  return sdxl_unet_forward_f32_at(u, B, h, w, x, (double)t_host, eps_out);
}
extern "C" int sdxl_unet_forward_f32_at(sdxl_unet* u, int B, int h, int w, const float* x, double t_host, float* eps_out) {
  if (!u || !x || !eps_out) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  if (!(t_host >= 0.0 && t_host <= (double)(u->cfg.n_steps - 1)))   // also refuses NaN
    return fail(c, 5024, "forward: timestep %g outside [0, %d]", t_host, u->cfg.n_steps - 1);
  return unet_forward(u, B, h, w, x, false, t_host, eps_out);
}
// Per-kernel-kind device time of one plan execution, measured with CUDA events on the ctx stream
// (eager launches, one event pair per op). kinds: see OpKind. Arrays hold SDXL_PROFILE_KINDS entries.
extern "C" int sdxl_unet_profile_plan(sdxl_unet* u, double* ms_by_kind, double* flops_by_kind, int* launches_by_kind) {
  if (!u || !u->plan) return -1;
  return profile_plan_impl(u->ctx, u->plan.get(), ms_by_kind, flops_by_kind, launches_by_kind);
}
// Per-op dump of one eager plan execution (CUDA-event time per launch) as CSV: analysis aid for profiles/.
extern "C" int sdxl_unet_profile_dump(sdxl_unet* u, const char* path) {
  if (!u || !u->plan || !path) return -1;
  return profile_dump_impl(u->ctx, u->plan.get(), path);
}
extern "C" double sdxl_unet_alpha(const sdxl_unet* u, int i) {
  if (!u || i < 0 || i >= (int)u->alphas.size()) return NAN;
  return u->alphas[i];
}
// algorithmic FLOPs of the current plan (debug / bench helper, not in the public header)
extern "C" double sdxl_unet_plan_flops(const sdxl_unet* u) { return (u && u->plan) ? u->plan->flops : 0.0; }
extern "C" int sdxl_unet_plan_num_ops(const sdxl_unet* u) { return (u && u->plan) ? (int)u->plan->ops.size() : 0; }
extern "C" uint64_t sdxl_unet_plan_builds(const sdxl_unet* u) { return u ? u->plan_builds : 0; }
// FLOPs the plan's tensor-core launches actually execute (see Op::flops_exec): excludes the hoisted K/V projections (not in
// the plan), counts the phase-decomposed upsample convs at 4/9 of the algorithmic figure, includes channel / key padding.
extern "C" double sdxl_unet_plan_flops_executed(const sdxl_unet* u) {
  if (!u || !u->plan) return 0.0;
  double f = 0;
  for (const Op& o : u->plan->ops) f += o.flops_exec;
  return f;
}

// ================================================================================================
// sampler (Diffuser)
// ================================================================================================
struct Sampler {
  int Bimg = 0, nfwd = 1, h = 0, w = 0, n_ctx = 0;   // nfwd: row groups of Bimg rows, [cond | uncond] or [cond], then [ptb] with PAG
  bool cfg = false, pag = false;
  bool img = false;        // image guidance: the rows are [cond | img | uncond] (an edit UNet with CFG)
  int evals = 0;           // UNet evaluations since sampler_begin (DeepCache: evaluation j is full when j % interval == 0)
  float guidance = 1.f;
  float* noise = nullptr;  // scratch [Bimg,4,h,w]
  float* xh = nullptr;     // scheduled samplers: the state x / sqrt(alpha), the denoised-latent history slots H1 and H2 and the
  float* hist = nullptr;   // saved state xs (DESIGN.md §16, §20)
  float* h2 = nullptr;
  float* xs = nullptr;
  float* ref = nullptr;
  uint8_t* mask = nullptr;
  float* rescale = nullptr;    // guidance rescale: the per-image factors [Bimg] and the statistics kernel's scratch
  void* stats = nullptr;
  __half* cond_ctx = nullptr;  // staged [nfwd*Bimg, n_ctx, ctx]
  __half* cond_y = nullptr;
  float* host_stage = nullptr;  // pinned
  size_t latent_elems = 0;
  Arena arena;
  ~Sampler() {
    if (host_stage) cudaFreeHost(host_stage);
  }
};

// Uploads/assembles the batched conditioning: rows [0,Bimg) conditional, rows [Bimg,2*Bimg) the
// unconditional context repeated (reference stablediffusion/mod.rs:506-537). With PAG attached a last group of Bimg rows repeats
// the conditional rows (the refiner, without CFG: [cond | ptb]); an edit UNet with CFG repeats the unconditional rows there
// ([cond | img | uncond], DESIGN.md §21), its first-conv condition zero. no_cfg: the base model runs its conditional rows alone too.
static int sampler_begin(sdxl_unet* u, const sdxl_conditioning* cond, double guidance, bool no_cfg = false) {
  sdxl_ctx* c = u->ctx;
  const sdxl_unet_cfg& g = u->cfg;
  if (!cond) return fail(c, 5200, "null conditioning");
  const int Bimg = cond->n_batch, n_ctx = cond->n_ctx;
  const int h = cond->resolution[0] / 8, w = cond->resolution[1] / 8;
  const bool use_cfg = !g.is_refiner && !no_cfg, pag = u->pag != nullptr, img = edit_layout(g) && use_cfg;
  const int nfwd = (use_cfg ? 2 : 1) + (pag || img ? 1 : 0);   // attachments_fit refuses PAG on an edit UNet
  const RowLayout layout{Bimg, use_cfg, img};
  const sdxl_half* ctx_c = g.is_refiner ? cond->context_open_clip : cond->context_full;
  const sdxl_half* ctx_u = g.is_refiner ? cond->unconditional_context_open_clip : cond->unconditional_context_full;
  const sdxl_half* y_c = g.is_refiner ? cond->channel_context_refiner : cond->channel_context;
  const sdxl_half* y_u = g.is_refiner ? cond->unconditional_channel_context_refiner : cond->unconditional_channel_context;
  if (!ctx_c || !y_c || (use_cfg && (!ctx_u || !y_u))) return fail(c, 5201, "conditioning tensors for this model are null");
  if (Bimg < 1 || h < 1 || w < 1) return fail(c, 5202, "bad conditioning batch/resolution");
  if (int r = attachments_fit(u, Bimg, h, w)) return r;
  if (int r = ip_check_batch_all(u, nfwd * Bimg, layout)) return r;
  Sampler* S = u->sampler.get();
  const size_t lat = (size_t)Bimg * latent_channels(g) * h * w;
  if (n_ctx < 1) return fail(c, 5202, "bad conditioning context length");
  // new shapes: a fresh sampler, installed only when the conditioning and the plan for it are in place (the steps pair its
  // shapes with the plan's buffers)
  std::unique_ptr<Sampler> fresh;
  if (!S || S->Bimg != Bimg || S->h != h || S->w != w || S->nfwd != nfwd || S->n_ctx != n_ctx) {   // staging buffers are sized by all five
    fresh.reset(new Sampler());
    S = fresh.get();
    S->Bimg = Bimg; S->nfwd = nfwd; S->h = h; S->w = w; S->n_ctx = n_ctx; S->latent_elems = lat;
    const size_t ctx_elems = (size_t)nfwd * Bimg * n_ctx * g.context_dim;
    const size_t y_elems = (size_t)nfwd * Bimg * g.adm_in_channels;
    if (int r = carve_measured(c, S->arena, 5203, "sampler buffers", [&](Arena& A) {
          S->noise = A.get<float>(lat);
          S->xh = A.get<float>(lat);
          S->hist = A.get<float>(lat);
          S->h2 = A.get<float>(lat);
          S->xs = A.get<float>(lat);
          S->ref = A.get<float>(lat);
          S->mask = A.get<uint8_t>(lat);
          S->rescale = A.get<float>(Bimg);
          S->stats = A.get<uint8_t>(guidance_stats_scratch_bytes(Bimg));
          S->cond_ctx = A.get<__half>(ctx_elems);
          S->cond_y = A.get<__half>(y_elems);
          return 0;
        }))
      return r;
    KL(c, guidance_stats_scratch_init(c->stream, S->stats, Bimg));
    CU(c, cudaMallocHost((void**)&S->host_stage, lat * sizeof(float)));
  }
  S->guidance = (float)guidance;
  S->cfg = use_cfg;
  S->pag = pag;
  S->img = img;
  S->evals = 0;
  const cudaMemcpyKind kind = cond->on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  const size_t ctx_row = (size_t)n_ctx * g.context_dim * 2, y_row = (size_t)g.adm_in_channels * 2;
  CU(c, cudaMemcpyAsync(S->cond_ctx, ctx_c, ctx_row * Bimg, kind, c->stream));
  CU(c, cudaMemcpyAsync(S->cond_y, y_c, y_row * Bimg, kind, c->stream));
  if (use_cfg)
    for (int b = 0; b < Bimg; ++b) {  // unsqueeze().repeat(0, n_batch)
      CU(c, cudaMemcpyAsync((uint8_t*)S->cond_ctx + ctx_row * (Bimg + b), ctx_u, ctx_row, kind, c->stream));
      CU(c, cudaMemcpyAsync((uint8_t*)S->cond_y + y_row * (Bimg + b), y_u, y_row, kind, c->stream));
    }
  if (pag || img) {   // the perturbed group repeats the conditional rows, image guidance's third group the unconditional ones
    const int g0 = (nfwd - 1) * Bimg, src = pag ? 0 : Bimg;
    CU(c, cudaMemcpyAsync((uint8_t*)S->cond_ctx + ctx_row * g0, (uint8_t*)S->cond_ctx + ctx_row * src, ctx_row * Bimg, cudaMemcpyDeviceToDevice,
                          c->stream));
    CU(c, cudaMemcpyAsync((uint8_t*)S->cond_y + y_row * g0, (uint8_t*)S->cond_y + y_row * src, y_row * Bimg, cudaMemcpyDeviceToDevice,
                          c->stream));
  }
  int r = set_conditioning_dev(u, nfwd * Bimg, n_ctx, S->cond_ctx, S->cond_y, layout);
  if (!r) r = ensure_plan(u, nfwd * Bimg, Bimg, h, w, pag ? Bimg : 0, img ? Bimg : 0);
  if (r || !fresh) return r;
  CU(c, cudaStreamSynchronize(c->stream));   // the old sampler's buffers may still be in flight
  u->sampler = std::move(fresh);
  return 0;
}

// One UNet evaluation of a sampling loop: with DeepCache, the full list on every interval-th evaluation since sampler_begin and the
// cached list between.
static int run_sampler_plan(sdxl_unet* u) {
  Sampler* S = u->sampler.get();
  const int r = run_plan(u, u->deepcache && S->evals % u->deepcache->interval != 0);
  if (!r) S->evals++;
  return r;
}

// s_img of a sampler with image guidance (0 otherwise: the kernels do not read it)
static float img_scale(const sdxl_unet* u) { return u->sampler->img ? u->edit->image_guidance : 0.f; }

// PAG's scale at timestep t, with diffusers' adaptive scaling: p_t = max(scale - adaptive * (n_steps - t), 0)
static float pag_scale(const sdxl_unet* u, double t) {
  return std::max(u->pag->scale - u->pag->adaptive * (float)(u->cfg.n_steps - t), 0.f);
}

// What the step kernel after this evaluation reads the UNet's output as (kernels.h: Prediction), at noise level sigma for the guided
// step. With guidance rescale on a call that has CFG rows, the statistics kernel first writes the per-image factors.
static int step_prediction(sdxl_unet* u, float p_t, double sigma, Prediction& pr) {
  sdxl_ctx* c = u->ctx;
  Sampler* S = u->sampler.get();
  Plan* P = u->plan.get();
  pr = Prediction{};
  if (u->guidance_rescale > 0.f && S->cfg) {
    KL(c, guidance_stats_launch(c->stream, P->eps, P->eps_ld, S->Bimg, latent_channels(u->cfg), S->h * S->w, S->pag, S->guidance, p_t,
                                u->guidance_rescale, S->stats, S->rescale, S->img, img_scale(u)));
    pr.factor = S->rescale;
  }
  if (u->prediction == SDXL_PREDICTION_V) {
    const DScale q = d_scale(SDXL_PREDICTION_V, sigma);
    pr.v = 1;
    pr.dx = q.dx;
    pr.de = q.de;
  }
  return 0;
}

// one loop-body iteration (reference stablediffusion/mod.rs:406-429)
static int sampler_step(sdxl_unet* u, int t, int t_prev) {
  sdxl_ctx* c = u->ctx;
  Sampler* S = u->sampler.get();
  Plan* P = u->plan.get();
  if (!S || !P) return fail(c, 5210, "sampler not initialised (call sdxl_sampler_begin)");
  if (t < 0 || t >= (int)u->alphas.size() || t_prev >= (int)u->alphas.size()) return fail(c, 5211, "timestep out of range");
  const double a = u->alphas[t];
  const double ap = t_prev >= 0 ? u->alphas[t_prev] : 1.0;
  int r = set_t(u, t);
  if (r) return r;
  if ((r = run_sampler_plan(u))) return r;
  const float p_t = S->pag ? pag_scale(u, t) : 0.f;
  Prediction pr;
  if ((r = step_prediction(u, p_t, sqrt((1.0 - a) / a), pr))) return r;
  KL(c, cfg_ddim_launch(c->stream, P->eps, P->eps_ld, S->Bimg, latent_channels(u->cfg), S->h * S->w, S->cfg, S->pag, S->guidance, p_t,
                        (float)sqrt(a), (float)sqrt(1.0 - a), (float)sqrt(ap), (float)sqrt(1.0 - ap), P->x_in, pr, S->img, img_scale(u)));
  return 0;
}

extern "C" int sdxl_sampler_begin(sdxl_unet* u, const sdxl_conditioning* cond, double guidance_scale) {
  if (!u) return -1;
  CU(u->ctx, cudaSetDevice(u->ctx->device));
  return sampler_begin(u, cond, guidance_scale);
}
extern "C" int sdxl_sampler_step(sdxl_unet* u, int t, int t_prev) {
  if (!u) return -1;
  CU(u->ctx, cudaSetDevice(u->ctx->device));
  return sampler_step(u, t, t_prev);
}
extern "C" int sdxl_sampler_set_latent(sdxl_unet* u, const float* latent, int on_host) {
  if (!u || !u->sampler || !u->plan) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  CU(c, cudaMemcpyAsync(u->plan->x_in, latent, u->sampler->latent_elems * 4, on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c->stream));
  if (on_host) CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}
extern "C" int sdxl_sampler_get_latent(sdxl_unet* u, float* latent, int on_host) {
  if (!u || !u->sampler || !u->plan) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  CU(c, cudaMemcpyAsync(latent, u->plan->x_in, u->sampler->latent_elems * 4, on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  if (on_host) CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}
extern "C" int sdxl_sampler_step_host(sdxl_unet* u, int t, int t_prev, float* latent_host) {
  if (!u || !u->sampler || !u->plan || !latent_host) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  Sampler* S = u->sampler.get();
  const size_t bytes = S->latent_elems * 4;
  memcpy(S->host_stage, latent_host, bytes);  // caller memory may be pageable: stage through pinned
  CU(c, cudaMemcpyAsync(u->plan->x_in, S->host_stage, bytes, cudaMemcpyHostToDevice, c->stream));
  int r = sampler_step(u, t, t_prev);
  if (r) return r;
  CU(c, cudaMemcpyAsync(S->host_stage, u->plan->x_in, bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  memcpy(latent_host, S->host_stage, bytes);
  return 0;
}
extern "C" int sdxl_randn(sdxl_ctx* c, float* out, size_t n, uint64_t seed, uint64_t subsequence) {
  if (!c || !out) return -1;
  CU(c, cudaSetDevice(c->device));
  KL(c, randn_launch(c->stream, out, n, seed, subsequence));
  return 0;
}

// The noise draws of a sampling call, in the call's order: the injected tensors first, then subsequences 0, 1, 2, ... of the
// seeded Philox stream. Injected tensors from the host are staged on the device once, so that every draw is read in place.
struct NoiseFeed {
  const float* injected = nullptr;   // device, n_injected tensors of lat elements
  int n_injected = 0, used = 0;
  size_t lat = 0;
  uint64_t seed = 0, subseq = 0;
  int init(sdxl_ctx* c, TmpBufs& tmp, const float* noise, int n_noise, bool on_host, size_t lat_, uint64_t seed_) {
    lat = lat_; seed = seed_;
    injected = noise; n_injected = noise ? n_noise : 0;
    if (n_injected > 0 && on_host) {
      const size_t bytes = (size_t)n_injected * lat * sizeof(float);
      float* d = tmp.get<float>(bytes);
      if (!d) return fail(c, 5235, "cannot allocate %zu bytes to stage the injected noise", bytes);
      CU(c, cudaMemcpyAsync(d, noise, bytes, cudaMemcpyHostToDevice, c->stream));
      injected = d;
    }
    return 0;
  }
  // the next draw: an injected tensor z, or (z null) subsequence sub of the seeded stream
  void next(const float*& z, uint64_t& sub) {
    z = nullptr;
    sub = 0;
    if (used < n_injected) z = injected + (size_t)used++ * lat;
    else sub = subseq++;
  }
  // the next draw in memory, for kernels that read their noise: an injected tensor in place, or the seeded one generated into dst
  int next_in(sdxl_ctx* c, float* dst, const float*& z) {
    uint64_t sub;
    next(z, sub);
    if (!z) {
      KL(c, randn_launch(c->stream, dst, lat, seed, sub));
      z = dst;
    }
    return 0;
  }
};

// The start of a sampling call whose arguments have been checked: the sampler, then the inpainting reference and mask.
static int sample_begin(sdxl_unet* u, const sdxl_conditioning* cond, double guidance, bool no_cfg, const float* inpaint_ref,
                        const uint8_t* inpaint_mask) {
  if (int r = sampler_begin(u, cond, guidance, no_cfg)) return r;
  if (inpaint_ref) {
    sdxl_ctx* c = u->ctx;
    Sampler* S = u->sampler.get();
    const cudaMemcpyKind kind = cond->on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    CU(c, cudaMemcpyAsync(S->ref, inpaint_ref, S->latent_elems * sizeof(float), kind, c->stream));
    CU(c, cudaMemcpyAsync(S->mask, inpaint_mask, S->latent_elems, kind, c->stream));
  }
  return 0;
}
// The end of a sampling call: the latent to the caller's memory, synchronised when that is host memory.
static int sample_end(sdxl_unet* u, const sdxl_conditioning* cond, const float* latent, float* latent_out) {
  sdxl_ctx* c = u->ctx;
  CU(c, cudaMemcpyAsync(latent_out, latent, u->sampler->latent_elems * sizeof(float),
                        cond->on_host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, c->stream));
  if (cond->on_host) CU(c, cudaStreamSynchronize(c->stream));
  return 0;
}

extern "C" int sdxl_sample_latent(sdxl_unet* u, const sdxl_conditioning* cond, double guidance_scale, int n_steps,
                                  int step_start, const float* init_latent, const float* noise, int n_noise, uint64_t seed,
                                  const float* inpaint_ref, const uint8_t* inpaint_mask, float* latent_out) {
  if (!u || !cond || !latent_out) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  const int total = u->cfg.n_steps;
  if (n_steps < 1 || n_steps > total) return fail(c, 5220, "n_steps must be in [1,%d]", total);
  if (step_start < 0 || step_start >= total) return fail(c, 5221, "bad step_start");
  if ((inpaint_ref == nullptr) != (inpaint_mask == nullptr)) return fail(c, 5222, "inpaint_ref and inpaint_mask must be given together");
  if (inpaint_ref && edit_layout(u->cfg)) return fail(c, 5727, "edit UNet: the latent-blend inpainting arguments are not supported");
  if (step_start > 0 && !init_latent) return fail(c, 5223, "refine (step_start>0) needs init_latent");
  int r = sample_begin(u, cond, guidance_scale, false, inpaint_ref, inpaint_mask);
  if (r) return r;
  Sampler* S = u->sampler.get();
  Plan* P = u->plan.get();
  const size_t lat = S->latent_elems, bytes = lat * 4;
  const cudaMemcpyKind in_kind = cond->on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  const int step_size = total / n_steps;      // mod.rs:400
  const int t_begin = total - step_start;     // mod.rs:404
  TmpBufs tmp(c->stream);
  NoiseFeed feed;
  if ((r = feed.init(c, tmp, noise, n_noise, cond->on_host, lat, seed))) return r;
  const float* z;
  // initial latent
  if (init_latent) {
    CU(c, cudaMemcpyAsync(P->x_in, init_latent, bytes, in_kind, c->stream));
  } else {
    if ((r = feed.next_in(c, P->x_in, z))) return r;
    if (z != P->x_in) CU(c, cudaMemcpyAsync(P->x_in, z, bytes, cudaMemcpyDeviceToDevice, c->stream));
  }
  if (step_start > 0) {
    // refine_latent entry (mod.rs:363-367): x = x*sqrt(a_t0) + noise*sqrt(1-a_t0), t0 = n_steps_total - step_start
    const double a0 = u->alphas[t_begin];
    if ((r = feed.next_in(c, S->noise, z))) return r;
    KL(c, axpby_launch(c->stream, P->x_in, z, lat, (float)sqrt(a0), (float)sqrt(1.0 - a0)));
  }
  // for t in (0..t_begin).rev().step_by(step_size)   (mod.rs:406, 452)
  for (int t = t_begin - 1; t >= 0; t -= step_size) {
    const int t_prev = (t >= step_size) ? t - step_size : -1;
    if (inpaint_ref) {
      const double a = u->alphas[t];
      if ((r = feed.next_in(c, S->noise, z))) return r;
      KL(c, inpaint_blend_launch(c->stream, P->x_in, S->ref, z, S->mask, lat, (float)sqrt(a), (float)sqrt(1.0 - a)));
    }
    if ((r = sampler_step(u, t, t_prev))) return r;
  }
  return sample_end(u, cond, P->x_in, latent_out);
}

// ================================================================================================
// scheduled samplers (include/sdxl_b200.h: sdxl_schedule; DESIGN.md §16)
// ================================================================================================
static thread_local std::string g_schedule_err;
extern "C" const char* sdxl_schedule_last_error(void) { return g_schedule_err.c_str(); }
extern "C" int sdxl_schedule_build(const double* alphas_cumprod, int n_train, const sdxl_schedule* s, double* timesteps, double* sigmas) {
  g_schedule_err.clear();
  if (!alphas_cumprod || !timesteps || !sigmas) g_schedule_err = "schedule_build: null argument";
  else if (n_train < 1) g_schedule_err = "schedule_build: n_train must be >= 1";
  else g_schedule_err = schedule_problem(s, n_train);
  if (g_schedule_err.empty())
    for (int i = 0; i < n_train; ++i)
      if (!(alphas_cumprod[i] > 0.0 && alphas_cumprod[i] < 1.0) || (i && !(alphas_cumprod[i] < alphas_cumprod[i - 1]))) {
        g_schedule_err = "schedule_build: alphas_cumprod[" + std::to_string(i) + "] is not inside (0, 1) and below its predecessor";
        break;
      }
  if (!g_schedule_err.empty()) return 5230;
  schedule_fill(SigmaTable(alphas_cumprod, n_train), *s, timesteps, sigmas);
  return 0;
}

extern "C" int sdxl_sample_latent_scheduled(sdxl_unet* u, const sdxl_conditioning* cond, double guidance_scale, const sdxl_schedule* sch,
                                            const float* init_latent, const float* noise, int n_noise, uint64_t seed,
                                            const float* inpaint_ref, const uint8_t* inpaint_mask, float* latent_out) {
  if (!u || !cond || !latent_out) return -1;
  sdxl_ctx* c = u->ctx;
  CU(c, cudaSetDevice(c->device));
  // everything is validated before any state changes
  const int N = (int)u->alphas.size();
  const std::string why = schedule_problem(sch, N);
  if (!why.empty()) return fail(c, 5230, "%s", why.c_str());
  if ((inpaint_ref == nullptr) != (inpaint_mask == nullptr)) return fail(c, 5231, "inpaint_ref and inpaint_mask must be given together");
  if (inpaint_ref && edit_layout(u->cfg)) return fail(c, 5727, "edit UNet: the latent-blend inpainting arguments are not supported");
  if (sch->first_step > 0 && !init_latent) return fail(c, 5232, "schedule: first_step = %d needs init_latent", sch->first_step);
  if (n_noise < 0 || (n_noise > 0 && !noise)) return fail(c, 5233, "n_noise = %d with %s noise", n_noise, noise ? "a" : "null");
  const int n = sch->n_steps, k0 = sch->first_step, k1 = sch->last_step ? sch->last_step : n;
  std::vector<double> ts(n), sig(n + 1);
  const SigmaTable table(u->alphas.data(), N);
  schedule_fill(table, *sch, ts.data(), sig.data());
  for (int k = 0; k < n; ++k)
    if (!(sig[k + 1] < sig[k])) return fail(c, 5234, "schedule: n_steps = %d gives sigmas that do not decrease at step %d", n, k);

  int r = sample_begin(u, cond, guidance_scale, sch->no_cfg != 0, inpaint_ref, inpaint_mask);
  if (r) return r;
  Sampler* S = u->sampler.get();
  Plan* P = u->plan.get();
  const size_t lat = S->latent_elems, bytes = lat * 4;
  const cudaMemcpyKind in_kind = cond->on_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
  TmpBufs tmp(c->stream);
  NoiseFeed feed;   // the step kernel reads an injected draw in place and generates a seeded one
  if ((r = feed.init(c, tmp, noise, n_noise, cond->on_host, lat, seed))) return r;
  GuidedStepParams p{};
  p.Bimg = S->Bimg; p.C = latent_channels(u->cfg); p.HW = S->h * S->w;
  p.xh = S->xh; p.x_in = P->x_in; p.hist = S->hist;
  p.seed = seed;
  if (inpaint_ref) { p.mask = S->mask; p.ref = S->ref; }
  // entry: xh at sigma_k0, blended for the first forward
  float* init_dev = nullptr;
  if (init_latent && (k0 == 0 && cond->on_host)) {   // the initial noise from the host: read by the kernel as z
    init_dev = tmp.get<float>(bytes);
    if (!init_dev) return fail(c, 5235, "cannot allocate %zu bytes to stage the initial noise", bytes);
    CU(c, cudaMemcpyAsync(init_dev, init_latent, bytes, cudaMemcpyHostToDevice, c->stream));
  }
  if (k0 == 0) {
    CU(c, cudaMemsetAsync(S->xh, 0, bytes, c->stream));
    p.cx = 0.f;
    p.cn = (float)sqrt(sig[0] * sig[0] + 1.0);
    if (init_latent) p.z = init_dev ? init_dev : init_latent;
    else feed.next(p.z, p.z_subseq);
  } else {
    CU(c, cudaMemcpyAsync(S->xh, init_latent, bytes, in_kind, c->stream));
    p.cx = 1.f;
    if (sch->renoise) {
      p.cn = (float)sig[k0];
      feed.next(p.z, p.z_subseq);
    }
  }
  p.c_in = (float)(1.0 / sqrt(sig[k0] * sig[k0] + 1.0));
  if (inpaint_ref) {
    p.sigma_blend = (float)sig[k0];
    feed.next(p.zb, p.zb_subseq);
  }
  KL(c, guided_step_launch(c->stream, p));
  // the steps: per evaluation, write t, replay the plan, one launch
  p.eps = P->eps; p.ld = P->eps_ld; p.use_cfg = S->cfg; p.use_pag = S->pag; p.guidance = S->guidance;
  StepRows rows;
  rows.xs = S->xs; rows.h2 = S->h2;
  for (int k = k0; k < k1; ++k) {
    const StepStages ss = step_stages(&table, *sch, k, ts.data(), sig.data(), std::min(k - k0, 2));
    for (int i = 0; i < ss.n; ++i) {
      const Stage& q = ss.st[i];
      if ((r = set_t(u, q.t))) return r;
      if ((r = run_sampler_plan(u))) return r;
      p.sigma = (float)q.sigma;
      p.cx = q.cx; p.cd = q.cd; p.ch = q.ch; p.cn = q.cn; p.c_in = q.c_in;
      p.write_hist = q.write_hist;
      rows.cs = q.cs; rows.ch2 = q.ch2;
      rows.sx = q.sx; rows.ss = q.ss; rows.sd = q.sd; rows.sh = q.sh; rows.sh2 = q.sh2;
      rows.write_xs = q.write_xs; rows.shift = q.shift;
      if (S->pag) p.p_t = pag_scale(u, q.t);
      p.z = p.zb = nullptr;
      p.mask = nullptr;
      if (q.cn != 0.f) feed.next(p.z, p.z_subseq);
      if (inpaint_ref && (i + 1 < ss.n || k + 1 < k1)) {   // the blend before the next forward: its noise follows this launch's
        p.mask = S->mask;
        p.sigma_blend = (float)q.sigma_next;
        feed.next(p.zb, p.zb_subseq);
      }
      Prediction pr;
      if ((r = step_prediction(u, p.p_t, q.sigma, pr))) return r;
      KL(c, guided_step_launch(c->stream, p, pr, q.rows() ? &rows : nullptr, S->img, img_scale(u)));
    }
  }
  return sample_end(u, cond, S->xh, latent_out);
}

// ================================================================================================
// inpainting mask of the `sample` front end (reference src/bin/sample/main.rs:144-190)
// ================================================================================================
// Crop window in PIXELS -> Bool mask [1, n_channels, h/8... ] in latent coordinates: pixel coordinates are divided by
// scale = image height / latent height (integer division, main.rs:164-169), ones inside [top,bottom) x [left,right), zero padding
// outside, inverted by crop_out (main.rs:183-187). mask = 1 keeps the GENERATED latent (mask_where, stablediffusion/mod.rs:465).
// A negative bound means "not given" (the reference's Option defaults: 0 / image extent). Host memory, [n_channels, lat_h, lat_w].
extern "C" int sdxl_make_inpaint_mask(int img_w, int img_h, int lat_w, int lat_h, int crop_left, int crop_right, int crop_top,
                                      int crop_bottom, int crop_out, int n_channels, uint8_t* mask_out_host) {
  if (!mask_out_host || img_w <= 0 || img_h <= 0 || lat_w <= 0 || lat_h <= 0 || n_channels <= 0 || lat_h > img_h) return -1;
  const int l = crop_left < 0 ? 0 : crop_left, r = crop_right < 0 ? img_w : crop_right;
  const int t = crop_top < 0 ? 0 : crop_top, b = crop_bottom < 0 ? img_h : crop_bottom;
  // the reference asserts `right <= w && bottom <= h && left < right || top < bottom` (operator precedence makes it weaker than
  // intended); here every condition must hold
  if (r > img_w || b > img_h || l >= r || t >= b) return 5500;
  const int scale = img_h / lat_h;
  if (scale <= 0) return 5501;
  const int cl = l / scale, cr = r / scale, ct = t / scale, cb = b / scale;
  if (cr > lat_w || cb > lat_h) return 5502;
  for (int c = 0; c < n_channels; ++c)
    for (int y = 0; y < lat_h; ++y)
      for (int x = 0; x < lat_w; ++x) {
        const bool inside = y >= ct && y < cb && x >= cl && x < cr;
        mask_out_host[((size_t)c * lat_h + y) * lat_w + x] = (uint8_t)(inside != (crop_out != 0));
      }
  return 0;
}

extern "C" void sdxl_unet_destroy(sdxl_unet* u) {
  if (!u) return;
  cudaStreamSynchronize(u->ctx->stream);
  delete u;
}

// ================================================================================================
// operator-level entry points
// ================================================================================================

extern "C" int sdxl_qkv_attention(sdxl_ctx* c, const sdxl_half* q, const sdxl_half* k, const sdxl_half* v, const sdxl_half* mask,
                                  int B, int T, int S, int C, int n_head, sdxl_half* out) {
  if (!c || !q || !k || !v || !out) return -1;
  if (n_head < 1 || C != n_head * 64) return fail(c, 5301, "sdxl_qkv_attention: head dim must be 64 (C=%d, n_head=%d)", C, n_head);
  if (mask) {
    // additive [T,S] mask (the text encoders' causal mask, clip/mod.rs:88): short sequences, CUDA-core kernel
    KL(c, attention_small_launch(c->stream, (const __half*)q, C, 0, (const __half*)k, (const __half*)v, C, 0, 0, B, T, S, n_head,
                                 (const __half*)mask, 0, (__half*)out, C));
    return 0;
  }
  AttnParams p{};
  p.T = T; p.S = S; p.n_head = n_head; p.B = B;
  p.q_col0 = p.k_col0 = p.v_col0 = 0;
  p.out = (__half*)out; p.ldo = C;
  p.scale_log2e = (float)(1.4426950408889634 / sqrt(64.0));
  int r = make_tmap_rows(&p.tmQ, (const __half*)q, T, B, C, C);
  if (!r) r = make_tmap_rows(&p.tmK, (const __half*)k, S, B, C, C);
  if (!r) r = make_tmap_rows(&p.tmV, (const __half*)v, S, B, C, C);
  if (r) return fail(c, r, "tensor map creation failed");
  KL(c, attention_launch(c->stream, p));
  return 0;
}

extern "C" int sdxl_op_ip_attention(sdxl_ctx* c, const sdxl_half* q, const sdxl_half* k, const sdxl_half* v, const sdxl_half* k_ip,
                                    const sdxl_half* v_ip, int B, int T, int S, int S_ip, int C, int n_head, float scale, sdxl_half* out) {
  if (!c || !q || !k || !v || !k_ip || !v_ip || !out) return -1;
  if (n_head < 1 || C != n_head * 64) return fail(c, 5302, "sdxl_op_ip_attention: head dim must be 64 (C=%d, n_head=%d)", C, n_head);
  if (B < 1 || S_ip < 1) return fail(c, 5303, "sdxl_op_ip_attention: B = %d and S_ip = %d must be >= 1", B, S_ip);
  CU(c, cudaSetDevice(c->device));
  TmpBufs tmp(c->stream);
  float* s = tmp.get<float>(sizeof(float));
  if (!s) return fail(c, 5304, "temporary allocation failed");
  CU(c, cudaMemcpyAsync(s, &scale, sizeof(float), cudaMemcpyHostToDevice, c->stream));
  AttnParams p{};
  p.T = T; p.S = S; p.n_head = n_head; p.B = B;
  p.out = (__half*)out; p.ldo = C;
  p.scale_log2e = (float)(1.4426950408889634 / sqrt(64.0));
  p.S_ip = S_ip; p.ip_scale = s; p.n_src = 1;
  int r = make_tmap_rows(&p.tmQ, (const __half*)q, T, B, C, C);
  if (!r) r = make_tmap_rows(&p.tmK, (const __half*)k, S, B, C, C);
  if (!r) r = make_tmap_rows(&p.tmV, (const __half*)v, S, B, C, C);
  if (!r) r = make_tmap_rows(&p.tmKip, (const __half*)k_ip, S_ip, B, C, C);
  if (!r) r = make_tmap_rows(&p.tmVip, (const __half*)v_ip, S_ip, B, C, C);
  if (r) return fail(c, r, "tensor map creation failed");
  KL(c, attention_launch(c->stream, p));
  CU(c, cudaStreamSynchronize(c->stream));   // `scale` lives on the caller's stack
  return 0;
}

extern "C" int sdxl_op_linear(sdxl_ctx* c, const sdxl_half* x, const sdxl_half* w, const sdxl_half* bias, const float* residual,
                              int M, int K, int N, int geglu, int out_f16, void* out) {
  if (!c || !x || !w || !out) return -1;
  if (K % 8) return fail(c, 5310, "sdxl_op_linear: K must be a multiple of 8");
  TmpBufs T(c->stream);
  const int Kpad = (K + 63) / 64 * 64;
  int gbn = 0;
  if (geglu) {
    gbn = geglu_bn_for(N / 2);
    if (!gbn || (N & 1)) return fail(c, 5311, "sdxl_op_linear: GEGLU width not tileable");
  }
  __half* wt = T.get<__half>((size_t)N * Kpad * 2);
  float* b32 = bias ? T.get<float>((size_t)N * 4) : nullptr;
  if (!wt || (bias && !b32)) return fail(c, 5312, "temporary allocation failed");
  KL(c, transpose_linear_launch(c->stream, (const __half*)w, K, N, wt, Kpad, 0, gbn));
  if (bias) KL(c, bias_to_f32_launch(c->stream, (const __half*)bias, N, b32, gbn, 0));
  const IgemmOperands o{(const __half*)x, 1, 1, M, K, K, nullptr, 0, 0, 0, 0, 0, wt, N, Kpad};
  return igemm_run(c, o, {{0, 0, 0, 0, Kpad / 64}}, 1, M, 1, geglu ? IGEMM_GEGLU : IGEMM_LINEAR, gbn, out, geglu ? 0 : !out_f16,
                   geglu ? N / 2 : N, b32, geglu ? nullptr : residual, N);
}

extern "C" int sdxl_op_conv2d(sdxl_ctx* c, const float* x, const sdxl_half* w, const sdxl_half* bias, int B, int H, int W, int Cin,
                              int Cout, int ksize, int stride, int upsample, float* out) {
  if (!c || !x || !w || !out) return -1;
  if ((ksize != 1 && ksize != 3) || (stride != 1 && stride != 2) || (stride == 2 && (upsample || ksize != 3)))
    return fail(c, 5320, "sdxl_op_conv2d: unsupported ksize/stride/upsample combination");
  if (Cin % 8) return fail(c, 5321, "sdxl_op_conv2d: Cin must be a multiple of 8");
  TmpBufs T(c->stream);
  const int Ipad = (Cin + 63) / 64 * 64, Ktot = ksize * ksize * Ipad;
  __half* wt = T.get<__half>((size_t)Cout * Ktot * 2);
  float* b32 = bias ? T.get<float>((size_t)Cout * 4) : nullptr;
  const int Hi = upsample ? 2 * H : H, Wi = upsample ? 2 * W : W;  // conv input extent
  __half* a16 = T.get<__half>((size_t)B * Hi * Wi * Cin * 2);
  if (!wt || !a16 || (bias && !b32)) return fail(c, 5322, "temporary allocation failed");
  KL(c, repack_conv_launch(c->stream, (const __half*)w, Cout, Cin, ksize, ksize, wt, Ktot, 0, Ipad));
  if (bias) KL(c, bias_to_f32_launch(c->stream, (const __half*)bias, Cout, b32, 0, 0));
  int Ho = Hi, Wo = Wi, Ba = B;   // output extent; images of the A operand
  std::vector<IgemmSeg> segs;
  if (stride == 2) {
    if ((H & 1) || (W & 1)) return fail(c, 5323, "sdxl_op_conv2d: stride 2 needs even H, W");
    KL(c, phase_split_launch(c->stream, x, B, H, W, Cin, a16));
    Ho = H / 2; Wo = W / 2; Ba = 4 * B;
    segs = stride2_taps(B, Ipad / 64);
  } else {
    if (upsample) KL(c, upsample2x_launch(c->stream, x, B, H, W, Cin, a16));
    else KL(c, cast_f32_to_f16_launch(c->stream, x, (size_t)B * H * W * Cin, a16));
    segs = conv_taps(ksize, Ipad / 64);
  }
  const IgemmOperands o{a16, Ba, Ho, Wo, Cin, Cin, nullptr, 0, 0, 0, 0, 0, wt, Cout, Ktot};
  return igemm_run(c, o, segs, Ho, Wo, B, IGEMM_LINEAR, 0, out, 1, Cout, b32, nullptr, 0);
}

extern "C" int sdxl_op_group_norm(sdxl_ctx* c, const float* x1, int C1, const float* x2, int C2, int B, int HW, int n_group,
                                  const float* gamma, const float* beta, float eps, int silu, sdxl_half* out) {
  if (!c || !x1 || !gamma || !beta || !out) return -1;
  TmpBufs T(c->stream);
  float* part = T.get<float>(gn_scratch_floats(B, n_group) * 4);
  if (part && gn_scratch_init(c->stream, part, B, n_group)) return fail(c, 5007, "GroupNorm scratch init failed");
  if (!part) return fail(c, 5330, "temporary allocation failed");
  GnParams p{x1, C1, x2, x2 ? C2 : 0, B, HW, n_group, gamma, beta, eps, silu, (__half*)out, nullptr, part, 0};
  KL(c, gn_launch(c->stream, p));
  c->launches++;
  return 0;
}
extern "C" int sdxl_op_layer_norm(sdxl_ctx* c, const float* x, const float* gamma, const float* beta, float eps, int rows, int C,
                                  sdxl_half* out) {
  if (!c || !x || !gamma || !beta || !out) return -1;
  KL(c, layernorm_launch(c->stream, x, gamma, beta, eps, rows, C, (__half*)out));
  return 0;
}
extern "C" int sdxl_op_timestep_embedding(sdxl_ctx* c, const int32_t* t_host, int n, int dim, int max_period, float* out) {
  if (!c || !t_host || !out || n < 1 || (dim & 1)) return -1;
  TmpBufs T(c->stream);
  int* td = T.get<int>((size_t)n * 4);
  if (!td) return fail(c, 5340, "temporary allocation failed");
  CU(c, cudaMemcpyAsync(td, t_host, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
  KL(c, timestep_embedding_launch(c->stream, td, n, dim, (float)max_period, out));
  CU(c, cudaStreamSynchronize(c->stream));  // t_host is pageable caller memory
  return 0;
}
