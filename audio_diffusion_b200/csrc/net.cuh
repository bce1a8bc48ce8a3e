// Shared host-side machinery of the model handles.  An architecture is one list of blocks (Block); the parameter table,
// the packed-weight arena layout and the launch plan (ResnetBlock2D / attention with the GroupNorm apply fused into the
// consuming conv) are each one loop over it, and one executor runs the forward and backward plans of both models.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200ad.h"
#include "taps.cuh"

namespace b200ad {

int set_err(const char* fmt, ...);
#define CK(call)                                                                  \
  do {                                                                            \
    cudaError_t e__ = (call);                                                     \
    if (e__ != cudaSuccess) return set_err("%s: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

struct Param {
  std::string name;
  std::vector<int64_t> shape;
};

struct Act {  // PF8 activation tensor
  __nv_bfloat16* p = nullptr;
  int C = 0, H = 0, W = 0;
  stat_t* stats = nullptr;
  size_t off = 0;  // byte offset of p in its arena: known in a size-only pass too, where p is null
};

// The forward values are reported per launch by b200ad_unet_profile_step (4 was the unfolded nearest-2x upsample); the
// backward's follow them.
enum OpKind { OP_TEMB = 0, OP_CONV_IN = 1, OP_GN = 2, OP_CONV = 3, OP_PARITY = 5, OP_ATTN = 6, OP_CONV_OUT = 7,
              OP_ATTN1 = 8 /* single head of dim C */, OP_VAE_SAMPLE = 9, OP_MIX1X1 = 10,
              OP_LN = 11 /* LayerNorm over channels */, OP_GEGLU = 12, OP_MHA = 13 /* multi-head attention, head_dim 16/32/64 */,
              OP_XVEC = 14 /* cross-attention against a one-token encoding = per-sample vector */,
              OP_GNAPPLY = 15 /* materialised GroupNorm (attention input: the q/k/v projection has 12 cout tiles) */,
              OP_PACK_T /* transposed weight packs of a backward plan */, OP_DGRAD, OP_WGRAD, OP_GN_BWD, OP_CHANSUM,
              OP_REDUCE_N, OP_SCATTER, OP_PF8ADD, OP_ATTN_BWD, OP_UNFOLD, OP_SCALAR_WGRAD, OP_CONV_IN_BWD, OP_FLIP, OP_SUMADD,
              OP_LIN_IN, OP_LIN_W, OP_SILU_BWD, OP_SILU_FWD, OP_MEMSET, OP_LN_BWD, OP_GEGLU_BWD, OP_XVEC_BWD, OP_MHA_BWD,
              OP_ATTN1_BWD, OP_QUANT_BWD, OP_LATENT_IN_BWD,
              OP_XKV /* cross-attention K / V projections of an S > 1 encoding */, OP_XATTN /* cross-attention, S > 1 */,
              OP_XATTN_BWD, OP_XKV_BWD, OP_NKINDS };
// by OpKind: error messages and the backward profile's keys (tools/cond_train_bench.py matches "mha_bwd x<count>")
static const char* const op_names[] = {
    "temb", "conv_in", "gn_finalize", "conv_tc", "", "parity_split", "attention", "conv_out", "attention_1head", "vae_sample",
    "mix1x1", "layernorm", "geglu", "mha", "cross_attn_vec", "gn_apply", "pack_transposed", "conv_tc(dgrad)", "wgrad_tc",
    "gn_bwd", "chan_sum", "reduce_n", "scatter", "pf8_add", "attention_bwd", "unfold_up2", "scalar_wgrad", "conv_in(dgrad)",
    "flip", "sum_add", "lin_in", "lin_w", "silu_bwd", "silu_fwd", "memset", "layernorm_bwd", "geglu_bwd",
    "cross_attn_vec_bwd", "mha_bwd", "attention_1head_bwd", "quant_conv_bwd", "latent_in_bwd", "cross_attn_kv", "cross_attn",
    "cross_attn_bwd", "cross_attn_kv_wgrad"};
static_assert(sizeof(op_names) / sizeof(op_names[0]) == OP_NKINDS, "one name per OpKind");

struct RunArgs {                        // the per-call inputs of a plan
  const float* in = nullptr;            // U-Net: the sample x; autoencoder: the image (encode) or the latents (decode)
  const float* t = nullptr;             // U-Net: timesteps [N]
  const float* noise = nullptr;         // U-Net: the scheduler's noise z; autoencoder encode: the sampling noise
  float* out = nullptr;                 // U-Net: eps (optional); autoencoder: z (encode) or the image (decode)
  float* moments = nullptr;             // autoencoder encode (optional)
  float* x_out = nullptr;               // U-Net: the scheduler update (optional), with coef or coef_dev
  const b200ad_step_coef* coef = nullptr;
  const b200ad_step_coef* coef_dev = nullptr;
  // backward (`in`: the forward's input)
  const float* g_eps = nullptr;         // the gradient of the model output (U-Net: eps; autoencoder decoder: the image)
  const float* g_mom = nullptr;         // autoencoder encoder: the gradient of the moments
  float* g_z = nullptr;                 // autoencoder decoder: the gradient w.r.t. the latents (written)
};

using OpFn = std::function<cudaError_t(const RunArgs&, cudaStream_t)>;
// One entry of a plan.  A closure must not capture its builder (a temporary that the plan outlives): op closures use
// explicit capture lists, never [=] or [&].
struct Op {
  OpKind kind;
  int launches = 1;   // what this op adds to the plan's launch count
  ConvParams conv;    // OP_CONV / OP_DGRAD (launch_conv_tc): data, because gn_attach edits the last conv of a forward plan
                      // and b200ad_unet_conv_plan / b200ad_unet_profile_step read it
  OpFn run;           // every other kind
};

struct Bump {  // two-pass bump allocator: base == nullptr computes sizes only
  uint8_t* base = nullptr;
  size_t off = 0;
  void* take(size_t bytes) {
    off = (off + 255) & ~(size_t)255;
    void* r = base ? base + off : nullptr;
    off += bytes;
    return r;
  }
};
static size_t take_off(Bump& b, size_t bytes) {  // size-only pass: returns the aligned offset
  b.take(0);
  const size_t o = (b.off + 255) & ~(size_t)255;
  b.take(bytes);
  return o;
}
static Act take_act(Bump& b, int N, int C, int H, int W) {  // a PF8 tensor (no statistics)
  Act a;
  a.C = C; a.H = H; a.W = W;
  a.off = take_off(b, (size_t)N * (C / 8) * make_geom(N, H, W).PL * 16);
  a.p = b.base ? (__nv_bfloat16*)(b.base + a.off) : nullptr;
  return a;
}

struct PackJob {  // one K-segment's packed weights
  int w_param;      // index of the fp32 weight in the table
  int cout, cin_total, KH, KW, cin_off, ksteps;
  PackTaps taps;
  size_t off;       // byte offset in the packed arena
  int cout_real = -1;  // < cout when the output channels are zero-padded up to the 128-channel tile
};

struct FusedBias {  // a bias vector of the packed arena made from one or more parameters
  enum Kind { SUM2,     // conv2.bias + conv_shortcut.bias
              QKV,      // to_q | to_k | to_v biases
              PAD128 }  // bias zero-padded to 128 output channels
    kind;
  int p[3];         // parameter indices (-1: unused)
  size_t off;       // byte offset in the packed arena
};

// One block of an architecture, in forward order.  Every block reads the output of the block before it (`in`); a U-Net
// up-block resnet also reads the output of a down block (`skip`).
enum BlockKind {
  BK_UNET_HEAD,    // conv_in + the timestep-embedding MLP
  BK_CONV_IN,      // conv_in on the caller's image (autoencoder encoder)
  BK_LATENT_IN,    // post_quant_conv + conv_in on the caller's latents (autoencoder decoder)
  BK_RESNET,       // ResnetBlock2D over cat(input, skip)
  BK_ATTN,         // self-attention block (head_dim 8; the autoencoder: one head)
  BK_TRANSFORMER,  // Transformer2DModel with one BasicTransformerBlock (conditional U-Net)
  BK_DOWN,         // Downsample2D, padding 1
  BK_DOWN_ASYM,    // Downsample2D, padding (0, 1, 0, 1) (autoencoder encoder)
  BK_UP,           // Upsample2D: nearest 2x + 3x3 conv
  BK_CONV_OUT,     // conv_norm_out + SiLU + conv_out (U-Net: + the scheduler update)
  BK_LATENT_OUT,   // conv_norm_out + SiLU + conv_out + quant_conv + latent sampling (autoencoder encoder)
};
struct Block {
  BlockKind kind;
  std::string name;        // diffusers name prefix (heads and tails: of the model part, "", "encoder." or "decoder.")
  int in = -1, skip = -1;  // indices of the blocks whose outputs are the input and the skip connection (-1: none)
  int cin = 0, cskip = 0, cout = 0;
  int temb = 0;            // U-Net head and resnets: width of the time embedding
  int cross = 0;           // transformer: width of the cross-attention encoding
  std::string pool;        // output buffer: pooled under this tag ("": a buffer of its own)
  // byte offsets in the packed arena, assigned by the layout pass
  size_t conv1[2] = {}, conv2 = 0, shortcut[2] = {};    // resnet K-segments: conv1 over (input, skip), conv2, 1x1 shortcut
  size_t qkv = 0, out = 0;                              // attention / attn1: q | k | v projection, to_out
  size_t q2 = 0, out2 = 0;                              // transformer attn2 (encodings of S > 1 tokens): to_q, to_out
  size_t proj_in = 0, ff1 = 0, ff2 = 0, proj_out = 0;   // transformer
  size_t seg[4] = {};                                   // down / up: one K-segment per parity; latent out: conv_out
  size_t ident = 0;                                     // identity block of the residual K-segment
  size_t bias = 0;                                      // fused bias vector
  int temb_row = -1;                                    // resnet: its rows in the concatenated time_emb_proj
};
static Block& add_block(std::vector<Block>& bl, BlockKind kind, const std::string& name, int cin, int cout,
                        const char* pool) {
  Block b;
  b.kind = kind; b.name = name; b.in = (int)bl.size() - 1; b.cin = cin; b.cout = cout; b.pool = pool;
  bl.push_back(b);
  return bl.back();
}

struct OpList {  // one launch sequence and the GroupNorm statistics it accumulates (zeroed before every run)
  std::vector<Op> ops;
  stat_t* stats = nullptr;
  size_t stats_bytes = 0;
};
struct Plan {    // everything a plan builder derives from the workspace and (N, H, W)
  std::vector<OpList> lists;         // U-Net: the forward; autoencoder: encoder, decoder
  std::map<std::string, Act> taps;   // activations by name (debug_tensor; the U-Net backward reads its inputs here)
  float* temb_act = nullptr;
  float* temb_proj = nullptr;
  int* temb_lead = nullptr;          // [N] first sample with the same timestep (inference only)
  float* temb_emb = nullptr;         // training: [N][dim0]   sinusoid
  float* temb_u1 = nullptr;          // training: [N][4 dim0] linear_1 output before SiLU
  float* temb_u2 = nullptr;          // training: [N][4 dim0] linear_2 output before SiLU
  float* zq = nullptr;               // autoencoder: post_quant_conv(z), [N][L][h][w]
  std::map<std::string, float*> lse; // training, conditional U-Net: attn1's row log-sum-exp [N][heads][H*W] by block name
                                     // (attn2's, S > 1: by block name + ".attn2")
  std::map<std::string, __nv_bfloat16*> xkv; // training, S > 1: attn2's K | V, bf16 [N][S][C] each, by block name
  std::map<std::string, float*> probs; // training, autoencoder: the single-head attention's softmax P [N][HW][HW] by block name
  float* z_in = nullptr;             // training, autoencoder: the decoder's input latents [N][L][h][w] (post_quant_conv wgrad)
  size_t ws_bytes = 0;
};

struct Backward;   // a backward plan (unet_bwd.cu)

// State shared by the model handles (U-Net, VAE): parameter table, packed-weight arena layout, workspace plan, backward
// plans.
struct NetBase {
  int norm_groups = 32;
  float norm_eps = 1e-5f;
  std::vector<Param> params;
  std::map<std::string, int> pidx;
  std::vector<const float*> pptr;
  // packed arena layout
  std::vector<PackJob> jobs;
  std::map<int, size_t> ident_off;         // channels -> identity weight blocks
  std::vector<FusedBias> fused;
  size_t packed_bytes = 0;
  size_t off_wcat = 0, off_bcat = 0;       // U-Net: concatenated time_emb_proj weights / biases
  int temb_rows = 0;
  uint8_t* packed = nullptr;
  // workspace / plan
  int N = 0, H = 0, W = 0;
  uint8_t* ws = nullptr;
  size_t ws_bytes = 0;
  Plan plan;
  bool training = false;            // keep every activation (no pooling) and the timestep-MLP pre-activations for backward
  int num_sms = 132;
  const float* enc = nullptr;       // conditional U-Net: encoder_hidden_states [N][enc_S][X] of the next forward
  int enc_S = 0;
  int enc_len = 1;                  // conditional U-Net: the encoder sequence length the next workspace plan is built for
  int plan_enc_len = 1;             // ... and the one the bound plan was built for
  int last_launches = 0;
  PackBatch pack_batch;             // device job table of the weight packing (one launch for all K-segments)
  std::vector<PackJob> xjobs;       // conditional U-Net: the K-segments only S > 1 plans read (layout_attn2)
  PackBatch xpack_batch;
  bool xpacked = false;             // xjobs packed from the current parameters
  // backward: one plan per part (U-Net: the whole model; autoencoder: encoder, decoder), built by bind_backward
  int nparts = 1;
  Backward* bwd[2] = {};
};
void release_backward(NetBase* h);   // frees h->bwd (unet_bwd.cu)

static PackItem make_pack_item(const NetBase* h, const PackJob& j, uint8_t* arena) {
  PackItem it;
  memset(&it, 0, sizeof(it));       // padding included: the table is compared bytewise
  it.w = h->pptr[j.w_param];
  it.dst = (__nv_bfloat16*)(arena + j.off);
  it.cout = j.cout; it.cin_total = j.cin_total; it.KH = j.KH; it.KW = j.KW; it.cin_off = j.cin_off; it.ksteps = j.ksteps;
  it.cout_real = j.cout_real < 0 ? j.cout : j.cout_real;
  it.taps = j.taps;
  it.nvec = (long long)(j.cout / 128) * j.ksteps * j.taps.ntaps * 256;
  return it;
}

// The configuration checks of both models' create; 0, or -1 with the error set.
static int check_net_config(int num_blocks, const int* ch, int out_channels, int groups) {
  if (num_blocks < 1 || num_blocks > B200AD_MAX_BLOCKS) return set_err("num_blocks out of range");
  for (int i = 0; i < num_blocks; ++i)
    if (ch[i] % 128) return set_err("block_out_channels must be multiples of 128");
  if (out_channels > 4) return set_err("out_channels > 4 not implemented");
  if (groups < 1 || groups > 64) return set_err("norm_num_groups must be in 1..64");
  for (int i = 0; i < num_blocks; ++i)   // GroupNorm partial sums are kept per 4-channel quad: a group must be whole quads
    if (ch[i] % groups || (ch[i] / groups) % 4)
      return set_err("channels per GroupNorm group must be a multiple of 4 for every block");
  return 0;
}

static std::string S(const char* fmt, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return buf;
}

// ================================================================================= parameter table
static int param_shape(const NetBase* h, int i, int64_t* dims) {
  const auto& s = h->params[i].shape;
  for (size_t k = 0; k < s.size(); ++k) dims[k] = s[k];
  return (int)s.size();
}
static void add_param(NetBase* h, const std::string& name, std::vector<int64_t> shape) {
  h->pidx[name] = (int)h->params.size();
  h->params.push_back({name, std::move(shape)});
}
static void p_conv(NetBase* h, const std::string& n, int cin, int cout, int k) {
  add_param(h, n + ".weight", {cout, cin, k, k});
  add_param(h, n + ".bias", {cout});
}
static void p_lin(NetBase* h, const std::string& n, int cin, int cout) {
  add_param(h, n + ".weight", {cout, cin});
  add_param(h, n + ".bias", {cout});
}
static void p_gn(NetBase* h, const std::string& n, int c) {
  add_param(h, n + ".weight", {c});
  add_param(h, n + ".bias", {c});
}
static void p_resnet(NetBase* h, const std::string& n, int cin, int cout, int temb) {  // temb == 0: no time embedding
  p_gn(h, n + ".norm1", cin);
  p_conv(h, n + ".conv1", cin, cout, 3);
  if (temb) p_lin(h, n + ".time_emb_proj", temb, cout);
  p_gn(h, n + ".norm2", cout);
  p_conv(h, n + ".conv2", cout, cout, 3);
  if (cin != cout) p_conv(h, n + ".conv_shortcut", cin, cout, 1);
}
static void p_attn(NetBase* h, const std::string& n, int c) {
  p_gn(h, n + ".group_norm", c);
  p_lin(h, n + ".to_q", c, c);
  p_lin(h, n + ".to_k", c, c);
  p_lin(h, n + ".to_v", c, c);
  p_lin(h, n + ".to_out.0", c, c);
}
// Transformer2DModel + BasicTransformerBlock of the conditional U-Net (diffusers naming)
static void p_transformer(NetBase* h, const std::string& n, int c, int X) {
  p_gn(h, n + ".norm", c);
  p_conv(h, n + ".proj_in", c, c, 1);
  const std::string b = n + ".transformer_blocks.0";
  p_gn(h, b + ".norm1", c);
  add_param(h, b + ".attn1.to_q.weight", {c, c});
  add_param(h, b + ".attn1.to_k.weight", {c, c});
  add_param(h, b + ".attn1.to_v.weight", {c, c});
  p_lin(h, b + ".attn1.to_out.0", c, c);
  p_gn(h, b + ".norm2", c);
  add_param(h, b + ".attn2.to_q.weight", {c, c});
  add_param(h, b + ".attn2.to_k.weight", {c, X});
  add_param(h, b + ".attn2.to_v.weight", {c, X});
  p_lin(h, b + ".attn2.to_out.0", c, c);
  p_gn(h, b + ".norm3", c);
  p_lin(h, b + ".ff.net.0.proj", c, 8 * c);
  p_lin(h, b + ".ff.net.2", 4 * c, c);
  p_conv(h, n + ".proj_out", c, c, 1);
}
static void p_block(NetBase* h, const Block& k) {
  const std::string& n = k.name;
  switch (k.kind) {
    case BK_UNET_HEAD:
      p_conv(h, n + "conv_in", k.cin, k.cout, 3);
      p_lin(h, "time_embedding.linear_1", k.cout, k.temb);
      p_lin(h, "time_embedding.linear_2", k.temb, k.temb);
      break;
    case BK_CONV_IN: p_conv(h, n + "conv_in", k.cin, k.cout, 3); break;
    case BK_LATENT_IN:
      p_conv(h, "post_quant_conv", k.cin, k.cin, 1);
      p_conv(h, n + "conv_in", k.cin, k.cout, 3);
      break;
    case BK_RESNET: p_resnet(h, n, k.cin + k.cskip, k.cout, k.temb); break;
    case BK_ATTN: p_attn(h, n, k.cout); break;
    case BK_TRANSFORMER: p_transformer(h, n, k.cout, k.cross); break;
    case BK_DOWN: case BK_DOWN_ASYM: case BK_UP: p_conv(h, n, k.cout, k.cout, 3); break;
    case BK_CONV_OUT:
      p_gn(h, n + "conv_norm_out", k.cin);
      p_conv(h, n + "conv_out", k.cin, k.cout, 3);
      break;
    case BK_LATENT_OUT:
      p_gn(h, n + "conv_norm_out", k.cin);
      p_conv(h, n + "conv_out", k.cin, k.cout, 3);
      p_conv(h, "quant_conv", k.cout, k.cout, 1);
      break;
  }
}

// ================================================================================= packed-weight arena layout
static size_t add_job(NetBase* h, Bump& b, const std::string& wname, int cout, int cin_total, int K, int cin_off,
                      int cin_cnt, const TapSet& taps, int cout_real = -1, std::vector<PackJob>* list = nullptr) {
  PackJob j;
  j.w_param = h->pidx.at(wname);
  j.cout = cout; j.cin_total = cin_total; j.KH = K; j.KW = K; j.cin_off = cin_off; j.ksteps = cin_cnt / 16;
  j.taps = taps.pack;
  j.cout_real = cout_real;
  j.off = take_off(b, (size_t)(cout / 128) * j.ksteps * taps.pack.ntaps * CONV_B_TAP);
  (list ? *list : h->jobs).push_back(j);
  return j.off;
}
static size_t add_ident(NetBase* h, Bump& b, int ch) {  // identity weight blocks for residual-as-K-segment
  auto it = h->ident_off.find(ch);
  if (it == h->ident_off.end()) it = h->ident_off.emplace(ch, take_off(b, (size_t)(ch / 128) * (ch / 16) * CONV_B_TAP)).first;
  return it->second;
}
static size_t add_bias(NetBase* h, Bump& b, FusedBias::Kind kind, size_t floats, const std::string& p0,
                       const std::string& p1 = "", const std::string& p2 = "") {
  FusedBias f;
  f.kind = kind;
  f.p[0] = h->pidx.at(p0);
  f.p[1] = p1.empty() ? -1 : h->pidx.at(p1);
  f.p[2] = p2.empty() ? -1 : h->pidx.at(p2);
  f.off = take_off(b, floats * 4);
  h->fused.push_back(f);
  return f.off;
}
static TapSet down_taps(const Block& k, int a, int b) {
  return k.kind == BK_DOWN ? taps_parity(a, b) : taps_parity_asym(a, b);
}
// ResnetBlock2D over cat(a, b): conv1 is one K-segment per source (each with its own fused GroupNorm scale/shift slice),
// conv2 carries the shortcut (1x1 conv or identity) as extra K-segments.
static void layout_resnet(NetBase* h, Bump& b, Block& k) {
  const std::string& n = k.name;
  const int ca = k.cin, cb = k.cskip, co = k.cout, cin = ca + cb;
  k.conv1[0] = add_job(h, b, n + ".conv1.weight", co, cin, 3, 0, ca, taps_conv(3));
  if (cb) k.conv1[1] = add_job(h, b, n + ".conv1.weight", co, cin, 3, ca, cb, taps_conv(3));
  k.conv2 = add_job(h, b, n + ".conv2.weight", co, co, 3, 0, co, taps_conv(3));
  if (cin == co) {
    k.ident = add_ident(h, b, co);
  } else {
    k.shortcut[0] = add_job(h, b, n + ".conv_shortcut.weight", co, cin, 1, 0, ca, taps_conv(1));
    if (cb) k.shortcut[1] = add_job(h, b, n + ".conv_shortcut.weight", co, cin, 1, ca, cb, taps_conv(1));
    k.bias = add_bias(h, b, FusedBias::SUM2, co, n + ".conv2.bias", n + ".conv_shortcut.bias");
  }
  if (k.temb) {
    k.temb_row = h->temb_rows;
    h->temb_rows += co;
  }
}
static void layout_attn(NetBase* h, Bump& b, Block& k) {
  const std::string& n = k.name;
  const int ch = k.cout;
  k.qkv = add_job(h, b, n + ".to_q.weight", ch, ch, 1, 0, ch, taps_conv(1));   // q | k | v blocks are contiguous
  add_job(h, b, n + ".to_k.weight", ch, ch, 1, 0, ch, taps_conv(1));
  add_job(h, b, n + ".to_v.weight", ch, ch, 1, 0, ch, taps_conv(1));
  k.out = add_job(h, b, n + ".to_out.0.weight", ch, ch, 1, 0, ch, taps_conv(1));
  k.bias = add_bias(h, b, FusedBias::QKV, (size_t)3 * ch, n + ".to_q.bias", n + ".to_k.bias", n + ".to_v.bias");
  k.ident = add_ident(h, b, ch);
}
static void layout_transformer(NetBase* h, Bump& b, Block& k) {
  const std::string& n = k.name;
  const std::string t = n + ".transformer_blocks.0";
  const int c = k.cout;
  k.proj_in = add_job(h, b, n + ".proj_in.weight", c, c, 1, 0, c, taps_conv(1));
  k.qkv = add_job(h, b, t + ".attn1.to_q.weight", c, c, 1, 0, c, taps_conv(1));   // q | k | v blocks are contiguous
  add_job(h, b, t + ".attn1.to_k.weight", c, c, 1, 0, c, taps_conv(1));
  add_job(h, b, t + ".attn1.to_v.weight", c, c, 1, 0, c, taps_conv(1));
  k.out = add_job(h, b, t + ".attn1.to_out.0.weight", c, c, 1, 0, c, taps_conv(1));
  k.ff1 = add_job(h, b, t + ".ff.net.0.proj.weight", 8 * c, c, 1, 0, c, taps_conv(1));
  k.ff2 = add_job(h, b, t + ".ff.net.2.weight", c, 4 * c, 1, 0, 4 * c, taps_conv(1));
  k.proj_out = add_job(h, b, n + ".proj_out.weight", c, c, 1, 0, c, taps_conv(1));
  k.ident = add_ident(h, b, c);
}
// attn2's to_q and to_out of a transformer block, read only by plans for encodings of S > 1 tokens: their own job list
// at the end of the arena, packed only while such a plan is bound (pack_xattn), so a one-token model packs what it did
// before this path existed.
static void layout_attn2(NetBase* h, Bump& b, Block& k) {
  const std::string t = k.name + ".transformer_blocks.0";
  const int c = k.cout;
  k.q2 = add_job(h, b, t + ".attn2.to_q.weight", c, c, 1, 0, c, taps_conv(1), -1, &h->xjobs);
  k.out2 = add_job(h, b, t + ".attn2.to_out.0.weight", c, c, 1, 0, c, taps_conv(1), -1, &h->xjobs);
}
static void layout_block(NetBase* h, Bump& b, Block& k) {
  switch (k.kind) {
    case BK_RESNET: layout_resnet(h, b, k); break;
    case BK_ATTN: layout_attn(h, b, k); break;
    case BK_TRANSFORMER: layout_transformer(h, b, k); break;
    case BK_DOWN: case BK_DOWN_ASYM:   // one K-segment per parity plane of the input
      for (int a = 0; a < 2; ++a)
        for (int c = 0; c < 2; ++c)
          k.seg[a * 2 + c] = add_job(h, b, k.name + ".weight", k.cout, k.cout, 3, 0, k.cout, down_taps(k, a, c));
      break;
    case BK_UP:                        // one folded 2x2 conv per output parity
      for (int a = 0; a < 2; ++a)
        for (int c = 0; c < 2; ++c)
          k.seg[a * 2 + c] = add_job(h, b, k.name + ".weight", k.cout, k.cout, 3, 0, k.cout, taps_up2(a, c));
      break;
    case BK_LATENT_OUT:                // conv_out: 2L output channels zero-padded to one 128-channel tile
      k.seg[0] = add_job(h, b, k.name + "conv_out.weight", 128, k.cin, 3, 0, k.cin, taps_conv(3), k.cout);
      k.bias = add_bias(h, b, FusedBias::PAD128, 128, k.name + "conv_out.bias");
      break;
    default: break;                    // fp32 weights read as they are
  }
}

static __global__ void add_vec_kernel(const float* a, const float* b, float* o, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] + (b ? b[i] : 0.f);
}

// Pack every conv K-segment, the identity blocks and the fused bias vectors into the arena (after pptr/packed are set).
static int pack_common(NetBase* h, cudaStream_t st) {
  {
    std::vector<PackItem> items;
    items.reserve(h->jobs.size());
    for (const PackJob& j : h->jobs) items.push_back(make_pack_item(h, j, h->packed));
    CK(launch_pack_batch(h->pack_batch, items, st));
  }
  for (const auto& kv : h->ident_off) CK(launch_pack_identity(kv.first, (__nv_bfloat16*)(h->packed + kv.second), st));
  for (const FusedBias& f : h->fused) {
    float* dst = (float*)(h->packed + f.off);
    const int c = (int)h->params[f.p[0]].shape[0];
    const float* const* src = h->pptr.data();
    switch (f.kind) {
      case FusedBias::SUM2:
        add_vec_kernel<<<(c + 255) / 256, 256, 0, st>>>(src[f.p[0]], src[f.p[1]], dst, c);
        CK(cudaGetLastError());
        break;
      case FusedBias::QKV:
        for (int i = 0; i < 3; ++i) CK(cudaMemcpyAsync(dst + i * c, src[f.p[i]], c * 4, cudaMemcpyDeviceToDevice, st));
        break;
      case FusedBias::PAD128:
        CK(cudaMemsetAsync(dst, 0, 128 * 4, st));
        CK(cudaMemcpyAsync(dst, src[f.p[0]], c * 4, cudaMemcpyDeviceToDevice, st));
        break;
    }
  }
  return 0;
}

// Packs the K-segments only plans for S > 1 encoder tokens read (after pptr / packed are set).
static int pack_xattn(NetBase* h, cudaStream_t st) {
  if (!h->xjobs.empty()) {
    std::vector<PackItem> items;
    items.reserve(h->xjobs.size());
    for (const PackJob& j : h->xjobs) items.push_back(make_pack_item(h, j, h->packed));
    CK(launch_pack_batch(h->xpack_batch, items, st));
  }
  h->xpacked = true;
  return 0;
}

// ================================================================================= launch plan
// a conv writing `out` (its work decomposition, tiles per item and item count, is filled in by launch_conv_tc)
static ConvParams conv_geom(int N, const Act& out) {
  const Geom g = make_geom(N, out.H, out.W);
  ConvParams p{};
  p.N = N; p.H = out.H; p.W = out.W; p.Wp = g.Wp; p.lead = g.lead; p.PL = g.PL;
  p.cout = out.C;
  p.out = out.p;
  p.stats = out.stats;
  return p;
}
// GroupNorm(+SiLU) over cat(a, b) into dst; dst null: the parameters of the scale/shift finalize (gn_finalize)
static GnApplyParams gn_params(const NetBase* h, int N, const Act& a, const Act* b, const std::string& norm,
                               __nv_bfloat16* dst, bool silu, float eps = -1.f) {
  GnApplyParams p{};
  p.src[0] = a.p; p.stats[0] = a.stats; p.C[0] = a.C;
  p.src[1] = b ? b->p : nullptr; p.stats[1] = b ? b->stats : nullptr; p.C[1] = b ? b->C : 0;
  p.gamma = h->pptr[h->pidx.at(norm + ".weight")]; p.beta = h->pptr[h->pidx.at(norm + ".bias")];
  p.dst = dst;
  p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = eps < 0.f ? h->norm_eps : eps; p.silu = silu ? 1 : 0;
  return p;
}

struct Builder {
  const NetBase* h;
  Plan* built;
  Bump ws;
  Bump st;  // stats arena (floats, offsets in bytes)
  std::vector<Op>* ops;
  std::map<std::string, Act> pool;  // reusable transient buffers keyed by tag
  int N, H = 0, W = 0;              // H, W: input size of the block list being planned
  int heads = 8;                    // transformer: attention heads
  bool nopool = false;  // B200AD_DEBUG_NOPOOL=1: every activation gets its own buffer (per-layer parity taps)
  bool single_head = false;  // attention with one head of dim C (AutoencoderKL mid block) instead of head_dim 8
  std::map<size_t, size_t> kv_pool;  // the workspace offsets of attn2's K | V buffers (S > 1) by size: shared unless nopool

  Act alloc(int C, int H, int W, bool stats) {
    Act a = take_act(ws, N, C, H, W);
    if (stats) a.stats = (stat_t*)st.take((size_t)N * (C / 4) * 2 * sizeof(stat_t));
    return a;
  }
  Act pooled(const std::string& tag, int C, int H, int W, bool stats) {
    const std::string key = S("%s:%d:%d:%d", tag.c_str(), C, H, W);
    if (nopool) return alloc(C, H, W, stats);
    auto it = pool.find(key);
    if (it == pool.end()) it = pool.emplace(key, alloc(C, H, W, false)).first;
    Act a = it->second;
    if (stats) a.stats = (stat_t*)st.take((size_t)N * (C / 4) * 2 * sizeof(stat_t));
    return a;
  }
  Act output(const Block& k, int C, int H, int W) {  // a block's output (raw + stats)
    return k.pool.empty() ? alloc(C, H, W, true) : pooled(k.pool, C, H, W, true);
  }
  const float* P(const std::string& name) const { return h->pptr[h->pidx.at(name)]; }
  template <class T> const T* PK(size_t off) const { return h->packed ? (const T*)(h->packed + off) : nullptr; }

  void emit(OpKind kind, OpFn run, int launches = 1) { ops->push_back(Op{kind, launches, {}, std::move(run)}); }
  void conv(const ConvParams& p) {
    Op op{OP_CONV};
    op.conv = p;
    ops->push_back(op);
  }
  void seg(ConvSeg& s, const __nv_bfloat16* src, int C, int H, int W, size_t woff, const TapSet& t) {
    set_seg(s, src, C / 8, C, H, W, PK<__nv_bfloat16>(woff), t);
  }
  void seg(ConvSeg& s, const Act& a, size_t woff, const TapSet& t) { seg(s, a.p, a.C, a.H, a.W, woff, t); }

  // Let the launch just planned (the producer of `a`; `b`, a skip connection, is older) finalize the GroupNorm over
  // cat(a, b) in its last CTA.  Returns the [N][Ca + Cb] (scale, shift) array, or nullptr if the last op cannot do it
  // (conv_in, an op of another kind, a batch too large for the scratch).
  float2* gn_attach(const Act& a, const Act* b, const std::string& norm, float2* ss = nullptr, float eps = -1.f) {
    const int Ct = a.C + (b ? b->C : 0);
    if (ops->empty() || ops->back().kind != OP_CONV || ops->back().conv.out != a.p || ops->back().conv.fin.ss ||
        (size_t)N * h->norm_groups * 2 * sizeof(float) > 32768)
      return nullptr;
    if (!ss) ss = (float2*)ws.take((size_t)N * Ct * sizeof(float2));
    ConvGnFin& f = ops->back().conv.fin;
    f.stats[0] = a.stats; f.C[0] = a.C;
    f.stats[1] = b ? b->stats : nullptr; f.C[1] = b ? b->C : 0;
    f.gamma = P(norm + ".weight"); f.beta = P(norm + ".bias");
    f.ss = ss;
    f.counter = (unsigned*)ws.take(sizeof(unsigned));
    f.groups = h->norm_groups; f.HW = a.H * a.W; f.eps = eps < 0.f ? h->norm_eps : eps;
    return ss;
  }

  // GroupNorm over cat(a, b): statistics -> per-(sample, channel) scale/shift; the apply itself is fused into the consumer
  // conv's transform warps. Returns the [N][Ca + Cb] scale/shift array.
  float2* gn_finalize(const Act& a, const Act* b, const std::string& norm, float eps = -1.f) {
    const int Ct = a.C + (b ? b->C : 0);
    float2* ss = (float2*)ws.take((size_t)N * Ct * sizeof(float2));
    if (gn_attach(a, b, norm, ss, eps)) return ss;
    const GnApplyParams p = gn_params(h, N, a, b, norm, nullptr, false, eps);
    emit(OP_GN, [p, ss](const RunArgs&, cudaStream_t s) { return launch_gn_finalize(p, ss, s); });
    return ss;
  }
  static void seg_norm(ConvSeg& s, const float2* ss, int stride, bool silu) {
    s.ss = ss; s.ss_stride = stride; s.silu = silu ? 1 : 0;
  }

  // conv_in of a model part, on the caller's fp32 input or on `src`
  Act conv_in(const Block& k, const float* src) {
    Act x = output(k, k.cout, H, W);
    emit(OP_CONV_IN, [src, w = P(k.name + "conv_in.weight"), b = P(k.name + "conv_in.bias"), N = N, cin = k.cin, H = H,
                      W = W, x](const RunArgs& a, cudaStream_t s) {
      return launch_conv_in(src ? src : a.in, w, b, N, cin, H, W, x.C, x.p, x.stats, s);
    });
    built->taps[k.name + "conv_in"] = x;
    return x;
  }

  // timestep embedding (one op for the MLP and every resnet's projection), then conv_in
  Act unet_head(const Block& k) {
    built->temb_act = (float*)ws.take((size_t)N * k.temb * 4);
    built->temb_proj = (float*)ws.take((size_t)N * h->temb_rows * 4);
    built->temb_lead = (int*)ws.take((size_t)N * 4);
    if (h->training) {
      built->temb_emb = (float*)ws.take((size_t)N * k.cout * 4);
      built->temb_u1 = (float*)ws.take((size_t)N * k.temb * 4);
      built->temb_u2 = (float*)ws.take((size_t)N * k.temb * 4);
    }
    const Plan& pl = *built;
    emit(OP_TEMB, [h = h, dim0 = k.cout, act = pl.temb_act, proj = pl.temb_proj, emb = pl.temb_emb, u1 = pl.temb_u1,
                   u2 = pl.temb_u2, lead = h->training ? nullptr : pl.temb_lead](const RunArgs& a, cudaStream_t s) {
      auto P = [h](const char* name) { return h->pptr[h->pidx.at(name)]; };
      return launch_temb(a.t, h->N, dim0, P("time_embedding.linear_1.weight"), P("time_embedding.linear_1.bias"),
                         P("time_embedding.linear_2.weight"), P("time_embedding.linear_2.bias"), act,
                         (const float*)(h->packed + h->off_wcat), (const float*)(h->packed + h->off_bcat), h->temb_rows,
                         proj, s, emb, u1, u2, lead);
    }, 2);   // the MLP, then every resnet's projection
    return conv_in(k, nullptr);
  }

  // post_quant_conv on the caller's latents, then conv_in
  Act latent_in(const Block& k) {
    float* zq = built->zq = (float*)ws.take((size_t)N * k.cin * H * W * 4);
    float* z_in = h->training ? built->z_in = (float*)ws.take((size_t)N * k.cin * H * W * 4) : nullptr;
    emit(OP_MIX1X1, [zq, z_in, w = P("post_quant_conv.weight"), b = P("post_quant_conv.bias"), N = N, L = k.cin, H = H,
                     W = W](const RunArgs& a, cudaStream_t s) {
      if (z_in) {   // training: the input is kept for the weight gradient
        const cudaError_t e = cudaMemcpyAsync(z_in, a.in, (size_t)N * L * H * W * 4, cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return e;
      }
      return launch_mix1x1(a.in, w, b, zq, N, L, H * W, s);
    });
    return conv_in(k, zq);
  }

  // ResnetBlock2D on x = cat(a, b) (b optional) -> out (raw + stats)
  Act resnet(const Block& k, const Act& a, const Act* b) {
    const std::string& n = k.name;
    const int cin = a.C + (b ? b->C : 0), cout = k.cout;
    const int H = a.H, W = a.W;
    const float2* ss1 = gn_finalize(a, b, n + ".norm1");
    Act h1 = pooled("h1", cout, H, W, true);
    {
      ConvParams p = conv_geom(N, h1);
      p.nseg = 1;
      seg(p.seg[0], a, k.conv1[0], taps_conv(3));
      seg_norm(p.seg[0], ss1, cin, true);
      if (b) {
        seg(p.seg[1], *b, k.conv1[1], taps_conv(3));
        seg_norm(p.seg[1], ss1 + a.C, cin, true);
        p.nseg = 2;
      }
      p.bias = P(n + ".conv1.bias");
      if (k.temb_row >= 0) {
        p.temb = built->temb_proj + k.temb_row;
        p.temb_stride = h->temb_rows;
      }
      conv(p);
    }
    const float2* ss2 = gn_finalize(h1, nullptr, n + ".norm2");
    Act out = output(k, cout, H, W);
    {
      ConvParams p = conv_geom(N, out);
      p.nseg = 1;
      seg(p.seg[0], h1, k.conv2, taps_conv(3));
      seg_norm(p.seg[0], ss2, cout, true);
      if (cin != cout) {  // 1x1 conv_shortcut over the raw input(s): extra K-segments into the same accumulators
        seg(p.seg[1], a, k.shortcut[0], taps_conv(1));
        p.nseg = 2;
        if (b) {
          seg(p.seg[2], *b, k.shortcut[1], taps_conv(1));
          p.nseg = 3;
        }
        p.bias = PK<float>(k.bias);
      } else {            // identity shortcut: residual add as a 1-tap identity-weight segment over the raw input
        seg(p.seg[1], a, k.ident, taps_conv(1));
        p.nseg = 2;
        p.bias = P(n + ".conv2.bias");
      }
      conv(p);
    }
    built->taps[n + ".h1"] = h1;
    built->taps[n] = out;
    return out;
  }

  // plain 1-tap conv (a linear layer over the pixel tokens) with optional fused GroupNorm of the source, identity residual
  // and per-sample additive vector
  void linear(const Act& out, const Act& src, size_t woff, const float* bias, const float2* ss = nullptr,
              const Act* residual = nullptr, size_t ident = 0, const float* vec = nullptr, int vec_stride = 0) {
    ConvParams p = conv_geom(N, out);
    p.nseg = 1;
    seg(p.seg[0], src, woff, taps_conv(1));
    if (ss) seg_norm(p.seg[0], ss, src.C, false);
    if (residual) {
      seg(p.seg[1], *residual, ident, taps_conv(1));
      p.nseg = 2;
    }
    p.bias = bias;
    p.temb = vec; p.temb_stride = vec_stride;
    conv(p);
  }

  // LayerNorm over channels (eps 1e-5) of src into dst
  void layer_norm(const Act& src, const Act& dst, const std::string& nm) {
    emit(OP_LN, [x = src.p, y = dst.p, g = P(nm + ".weight"), b = P(nm + ".bias"), N = N, C = src.C, H = src.H,
                 W = src.W](const RunArgs&, cudaStream_t s) { return launch_layernorm_pf8(x, y, g, b, N, C, H, W, 1e-5f, s); });
  }

  // attn2 of a transformer block against an encoding of S > 1 tokens, on h1 = h0 + attn1(LN1(h0)):
  //   h2 = h1 + to_out(xattn(to_q(LN2(h1)), enc Wk^T, enc Wv^T))
  Act cross_attention(const Block& k, const Act& h1, int S) {
    const std::string& n = k.name;
    const std::string t = n + ".transformer_blocks.0";
    const int C = h1.C, H = h1.H, W = h1.W;
    Act n2 = pooled("tf_ln", C, H, W, false);
    layer_norm(h1, n2, t + ".norm2");
    Act q2 = pooled("tf_q2", C, H, W, false);
    linear(q2, n2, k.q2, nullptr);
    const size_t kv_bytes = (size_t)2 * N * S * C * sizeof(__nv_bfloat16);
    auto it = kv_pool.find(kv_bytes);
    if (nopool || it == kv_pool.end()) it = kv_pool.insert_or_assign(kv_bytes, take_off(ws, kv_bytes)).first;
    __nv_bfloat16* kv = ws.base ? (__nv_bfloat16*)(ws.base + it->second) : nullptr;
    if (h->training) built->xkv[n] = kv;
    emit(OP_XKV, [h = h, wk = P(t + ".attn2.to_k.weight"), wv = P(t + ".attn2.to_v.weight"), kv, N = N, S, C,
                  X = k.cross](const RunArgs&, cudaStream_t s) {
      return launch_xattn_kv(h->enc, wk, wv, kv, kv + (size_t)N * S * C, N, S, C, X, s);
    });
    Act ao2 = pooled("tf_ao", C, H, W, false);    // attn1's output is dead after h1
    float* lse = h->training ? built->lse[n + ".attn2"] = (float*)ws.take((size_t)N * heads * H * W * sizeof(float)) : nullptr;
    emit(OP_XATTN, [q = q2.p, kv, o = ao2.p, N = N, C, heads = heads, H, W, S, lse](const RunArgs&, cudaStream_t s) {
      return launch_xattn(q, kv, kv + (size_t)N * S * C, o, N, C, heads, H, W, S, s, lse);
    });
    Act h2 = pooled("tf_h2", C, H, W, false);
    linear(h2, ao2, k.out2, P(t + ".attn2.to_out.0.bias"), nullptr, &h1, k.ident);
    if (h->training) {
      built->taps[n + ".n2"] = n2;
      built->taps[n + ".q2"] = q2;
      built->taps[n + ".ao2"] = ao2;
    }
    return h2;
  }

  // Transformer2DModel with one BasicTransformerBlock (conditional U-Net):
  //   h0 = proj_in(GroupNorm(x));  h1 = h0 + attn1(LN1(h0));  h2 = h1 + attn2(LN2(h1), enc);  h3 = h2 + ff(LN3(h2));
  //   out = proj_out(h3) + x
  // Encoder sequence length S = 1: attn2 with ONE key is the per-sample vector to_out(to_v(enc)) (softmax over a single
  // key is 1): it rides on the per-sample additive term of the attn1 output projection, and h1 is never formed.
  // S > 1: cross_attention.
  Act transformer(const Block& k, const Act& x) {
    const std::string& n = k.name;
    const int C = x.C, H = x.H, W = x.W, S = h->enc_len;
    const std::string t = n + ".transformer_blocks.0";
    const float2* ssx = gn_finalize(x, nullptr, n + ".norm", 1e-6f);
    float* vec = nullptr;
    if (S == 1) {
      vec = (float*)ws.take((size_t)N * C * sizeof(float));
      emit(OP_XVEC, [h = h, wv = P(t + ".attn2.to_v.weight"), wo = P(t + ".attn2.to_out.0.weight"),
                     bo = P(t + ".attn2.to_out.0.bias"), vec, N = N, C, X = k.cross](const RunArgs&, cudaStream_t s) {
        return launch_cross_attn_vec(h->enc, wv, wo, bo, vec, N, C, X, s);
      });
    }
    Act h0 = pooled("tf_h0", C, H, W, false);
    linear(h0, x, k.proj_in, P(n + ".proj_in.bias"), ssx);
    Act n1 = pooled("tf_ln", C, H, W, false);
    layer_norm(h0, n1, t + ".norm1");
    Act qkv = pooled("tf_qkv", 3 * C, H, W, false);
    linear(qkv, n1, k.qkv, nullptr);
    Act ao = pooled("tf_ao", C, H, W, false);
    float* lse = h->training ? built->lse[n] = (float*)ws.take((size_t)N * heads * H * W * sizeof(float)) : nullptr;
    emit(OP_MHA, [q = qkv.p, o = ao.p, N = N, C, heads = heads, H, W, lse](const RunArgs&, cudaStream_t s) {
      return launch_mha_flash(q, o, N, C, heads, H, W, s, lse);
    });
    Act h2;
    if (S == 1) {
      h2 = pooled("tf_h2", C, H, W, false);
      linear(h2, ao, k.out, P(t + ".attn1.to_out.0.bias"), nullptr, &h0, k.ident, vec, C);
    } else {
      Act h1 = pooled("tf_h1", C, H, W, false);
      linear(h1, ao, k.out, P(t + ".attn1.to_out.0.bias"), nullptr, &h0, k.ident);
      built->taps[n + ".attn1"] = h1;
      h2 = cross_attention(k, h1, S);
    }
    Act n3 = pooled("tf_ln", C, H, W, false);     // the same buffer as n1 unless training
    layer_norm(h2, n3, t + ".norm3");
    Act ff1 = pooled("tf_ff1", 8 * C, H, W, false);
    linear(ff1, n3, k.ff1, P(t + ".ff.net.0.proj.bias"));
    Act gg = pooled("tf_gg", 4 * C, H, W, false);
    emit(OP_GEGLU, [x = ff1.p, y = gg.p, N = N, C, H, W](const RunArgs&, cudaStream_t s) {
      return launch_geglu_pf8(x, y, N, 4 * C, H, W, s);
    });
    Act h3 = pooled("tf_h0", C, H, W, false);     // h0 is dead after h2 (S > 1: after h1)
    linear(h3, gg, k.ff2, P(t + ".ff.net.2.bias"), nullptr, &h2, k.ident);
    Act out = output(k, C, H, W);
    linear(out, h3, k.proj_out, P(n + ".proj_out.bias"), nullptr, &x, k.ident);
    built->taps[n + ".attn2"] = h2;
    built->taps[n] = out;
    if (h->training) {   // no pooling: every intermediate has its own buffer, kept for BwdBuilder::transformer_bwd
      built->taps[n + ".h0"] = h0;
      built->taps[n + ".n1"] = n1;
      built->taps[n + ".qkv"] = qkv;
      built->taps[n + ".ao"] = ao;
      built->taps[n + ".n3"] = n3;
      built->taps[n + ".ff1"] = ff1;
      built->taps[n + ".gg"] = gg;
      built->taps[n + ".h3"] = h3;
    }
    return out;
  }

  // Downsample2D: 3x3 stride-2 conv = four K-segments over the parity planes of the input
  Act down2(const Block& k, const Act& x) {
    const int C = x.C, Ho = x.H / 2, Wo = x.W / 2;
    const Geom go = make_geom(N, Ho, Wo);
    const size_t tsz = (size_t)N * (C / 8) * go.PL * 8;  // elements per parity tensor
    Act par = pooled("parity", 4 * C, Ho, Wo, false);     // 4 tensors back to back (same bytes as 4C channels)
    built->taps[k.name + ".parity"] = par;
    emit(OP_PARITY, [x, par = par.p, N = N](const RunArgs&, cudaStream_t s) {
      return launch_parity_split(x.p, par, N, x.C, x.H, x.W, s);
    });
    Act y = output(k, C, Ho, Wo);
    ConvParams p = conv_geom(N, y);
    p.nseg = 4;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b)
        seg(p.seg[a * 2 + b], par.p + (size_t)(a * 2 + b) * tsz, C, Ho, Wo, k.seg[a * 2 + b], down_taps(k, a, b));
    p.bias = P(k.name + ".bias");
    conv(p);
    built->taps[k.name] = y;
    return y;
  }

  // Upsample2D(use_conv): nearest-2x + 3x3 conv folded into four 2x2 convs on the low-res tensor (one launch per parity)
  Act up2(const Block& k, const Act& x) {
    const int C = x.C, hh = x.H, ww = x.W;
    Act y = output(k, C, hh * 2, ww * 2);
    for (int pa = 0; pa < 2; ++pa)
      for (int pb = 0; pb < 2; ++pb) {
        Act lo = y;                       // item geometry = low-res input geometry, output tensor = y
        lo.H = hh; lo.W = ww;
        ConvParams p = conv_geom(N, lo);
        p.up2 = 1; p.oy = pa; p.ox = pb;
        p.nseg = 1;
        seg(p.seg[0], x, k.seg[pa * 2 + pb], taps_up2(pa, pb));
        p.bias = P(k.name + ".bias");
        conv(p);
      }
    built->taps[k.name] = y;
    return y;
  }

  Act attention(const Block& k, const Act& x) {
    const std::string& n = k.name;
    const int C = x.C, H = x.H, W = x.W;
    // The q/k/v projection is a 1-tap conv with 3C/128 (= 12) cout tiles: fused, every one of those tiles would re-normalise
    // the same window in its transform warps, and a 1-tap k-step (192 MMA cycles) cannot hide that (measured 187 us per
    // launch at 16x16, batch 64).  The normalised tensor is tiny here (16 MB): materialise it once, project the plain tensor.
    Act xn = pooled("attn_xn", C, H, W, false);
    const GnApplyParams g = gn_params(h, N, x, nullptr, n + ".group_norm", xn.p, false);
    emit(OP_GNAPPLY, [g](const RunArgs&, cudaStream_t s) { return launch_gn_apply(g, s); });
    Act qkv = pooled("qkv", 3 * C, H, W, false);
    linear(qkv, xn, k.qkv, PK<float>(k.bias));   // q|k|v blocks are contiguous
    Act ao = pooled("attn_o", C, H, W, false);
    if (single_head) {
      float* scores = (float*)ws.take((size_t)N * H * W * H * W * sizeof(float));
      if (h->training) built->probs[n] = scores;
      emit(OP_ATTN1, [q = qkv.p, o = ao.p, scores, N = N, C, H, W](const RunArgs&, cudaStream_t s) {
        return launch_attention_1head(q, o, scores, N, C, H, W, s);
      }, 3);   // scores, softmax, output
    } else {
      emit(OP_ATTN, [q = qkv.p, o = ao.p, N = N, C, H, W](const RunArgs&, cudaStream_t s) {
        return launch_attention(q, o, N, C, H, W, s);
      });
    }
    Act out = output(k, C, H, W);
    linear(out, ao, k.out, P(n + ".to_out.0.bias"), nullptr, &x, k.ident);   // + residual
    built->taps[n + ".qkv"] = qkv;
    built->taps[n + ".ao"] = ao;
    built->taps[n] = out;
    return out;
  }

  // conv_norm_out + SiLU + conv_out, fused with the scheduler update; the GroupNorm is finalised by the last conv's last
  // CTA (null: in conv_out)
  Act conv_out(const Block& k, const Act& x) {
    const std::string& n = k.name;
    ConvOutParams p{};
    p.src = x.p; p.stats = x.stats;
    p.ss = gn_attach(x, nullptr, n + "conv_norm_out");
    p.gamma = P(n + "conv_norm_out.weight"); p.beta = P(n + "conv_norm_out.bias");
    p.w = P(n + "conv_out.weight"); p.b = P(n + "conv_out.bias");
    p.N = N; p.C = x.C; p.H = x.H; p.W = x.W; p.cout = k.cout; p.groups = h->norm_groups; p.eps = h->norm_eps;
    emit(OP_CONV_OUT, [p](const RunArgs& a, cudaStream_t s) {
      ConvOutParams q = p;
      q.eps_out = a.out;
      q.x = a.in; q.z = a.noise; q.x_out = a.x_out;
      static_assert(sizeof(b200ad_step_coef) == sizeof(StepCoef), "step-coefficient layouts differ");
      q.coef_dev = reinterpret_cast<const StepCoef*>(a.coef_dev);
      if (a.coef) memcpy(&q.coef, a.coef, sizeof(StepCoef));
      return launch_conv_out(q, s);
    });
    built->taps[n + "pre_out"] = x;
    return x;
  }

  // conv_norm_out + SiLU + conv_out on the tensor cores (output padded to 128 channels), then quant_conv + sampling
  Act latent_out(const Block& k, const Act& x) {
    const std::string& n = k.name;
    Act eo = pooled("enc_out", 128, x.H, x.W, false);
    {
      const float2* ss = gn_finalize(x, nullptr, n + "conv_norm_out");
      ConvParams p = conv_geom(N, eo);
      p.nseg = 1;
      seg(p.seg[0], x, k.seg[0], taps_conv(3));
      seg_norm(p.seg[0], ss, x.C, true);
      p.bias = PK<float>(k.bias);
      conv(p);
    }
    built->taps[n + "conv_out"] = eo;
    emit(OP_VAE_SAMPLE, [eo = eo.p, w = P("quant_conv.weight"), b = P("quant_conv.bias"), N = N, L = k.cout / 2, H = x.H,
                         W = x.W](const RunArgs& a, cudaStream_t s) {
      return launch_vae_sample(eo, w, b, a.noise, a.out, a.moments, N, 128, L, H, W, s);
    });
    return eo;
  }

  // Appends the plan of a block list.
  void run(const std::vector<Block>& blocks) {
    std::vector<Act> outs(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) {
      const Block& k = blocks[i];
      const Act* x = k.in >= 0 ? &outs[k.in] : nullptr;
      const Act* skip = k.skip >= 0 ? &outs[k.skip] : nullptr;
      switch (k.kind) {
        case BK_UNET_HEAD: outs[i] = unet_head(k); break;
        case BK_CONV_IN: outs[i] = conv_in(k, nullptr); break;
        case BK_LATENT_IN: outs[i] = latent_in(k); break;
        case BK_RESNET: outs[i] = resnet(k, *x, skip); break;
        case BK_ATTN: outs[i] = attention(k, *x); break;
        case BK_TRANSFORMER: outs[i] = transformer(k, *x); break;
        case BK_DOWN: case BK_DOWN_ASYM: outs[i] = down2(k, *x); break;
        case BK_UP: outs[i] = up2(k, *x); break;
        case BK_CONV_OUT: outs[i] = conv_out(k, *x); break;
        case BK_LATENT_OUT: outs[i] = latent_out(k, *x); break;
      }
    }
  }
};

static bool debug_nopool() {
  const char* e = getenv("B200AD_DEBUG_NOPOOL");
  return e && e[0] == '1';
}

// Binds the plan `build` makes for (N, H, W) over a caller-owned workspace: a size pass, the workspace zeroed, the bound pass.
template <class Net>
static int bind_workspace(Net* h, Plan (*build)(const Net*, uint8_t*, int, int, int), void* workspace, size_t bytes, int N,
                          int H, int W, cudaStream_t st) {
  if (!h->packed) return set_err("set_params must be called before bind_workspace");
  const int down = 1 << (h->cfg.num_blocks - 1);
  if (H % down || W % down) return set_err("H and W must be multiples of %d", down);
  const size_t need = build(h, nullptr, N, H, W).ws_bytes;
  if (bytes < need) return set_err("workspace too small: %zu < %zu", bytes, need);
  CK(cudaMemsetAsync(workspace, 0, need, st));
  h->plan = build(h, (uint8_t*)workspace, N, H, W);
  h->N = N; h->H = H; h->W = W;
  h->ws = (uint8_t*)workspace; h->ws_bytes = need;
  int dev = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

static int set_training(NetBase* h, int on) {
  if (!h) return set_err("null handle");
  if (h->training != (on != 0)) {
    h->training = on != 0;
    h->plan.lists.clear();    // the workspace layout changes: bind_workspace must be called again
  }
  return 0;
}

// ================================================================================= plan executor
struct OpEvents {   // per-op timing: an event before the first op of a run and one after every op
  std::vector<cudaEvent_t> ev;
  ~OpEvents() {
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
  }
  int ms(size_t i, float* out) const {   // device time of op i (after the stream has synchronised)
    CK(cudaEventElapsedTime(out, ev[i], ev[i + 1]));
    return 0;
  }
};

// Zeroes the plan's GroupNorm statistics and launches its ops in order; on success stores the launch count.
static int run_ops(const NetBase* h, const OpList& l, const RunArgs& a, cudaStream_t st, int* launches,
                   OpEvents* timing = nullptr) {
  if (l.stats_bytes) CK(cudaMemsetAsync(l.stats, 0, l.stats_bytes, st));
  if (timing) {
    timing->ev.assign(l.ops.size() + 1, nullptr);
    for (cudaEvent_t& e : timing->ev) CK(cudaEventCreate(&e));
    CK(cudaEventRecord(timing->ev[0], st));
  }
  int n = 0;
  for (size_t i = 0; i < l.ops.size(); ++i) {
    const Op& op = l.ops[i];
    const cudaError_t e = op.run ? op.run(a, st) : launch_conv_tc(op.conv, h->num_sms, st);
    if (e != cudaSuccess) return set_err("%s: %s", op_names[op.kind], cudaGetErrorString(e));
    if (timing) CK(cudaEventRecord(timing->ev[i + 1], st));
    n += op.launches;
  }
  *launches = n;
  return 0;
}

static int debug_tensor(const NetBase* h, const char* name, float* dst, int* dims, cudaStream_t st) {
  auto it = h->plan.taps.find(name);
  if (it == h->plan.taps.end()) return set_err("unknown tap '%s'", name);
  const Act& a = it->second;
  if (dims) { dims[0] = a.C; dims[1] = a.H; dims[2] = a.W; }
  if (dst) CK(launch_pf8_to_nchw(a.p, dst, h->N, a.C, a.H, a.W, st));
  return a.C;
}

}  // namespace b200ad
