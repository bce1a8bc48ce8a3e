// Shared host-side machinery of the model handles: parameter table, packed-weight arena, activation workspace and the
// launch-plan builder (ResnetBlock2D / attention with the GroupNorm apply fused into the consuming conv).
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200ad.h"
#include "conv_tc.cuh"
#include "kernels.cuh"

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
};

enum OpKind { OP_TEMB, OP_CONV_IN, OP_GN, OP_CONV, OP_UPSAMPLE, OP_PARITY, OP_ATTN, OP_CONV_OUT,
              OP_ATTN1 /* single head of dim C */, OP_VAE_SAMPLE, OP_MIX1X1,
              OP_LN /* LayerNorm over channels */, OP_GEGLU, OP_MHA /* multi-head attention, head_dim 16/32/64 */,
              OP_XVEC /* cross-attention against a one-token encoding = per-sample vector */,
              OP_GNAPPLY /* materialised GroupNorm (attention input: the q/k/v projection has 12 cout tiles) */ };
struct Op {
  OpKind kind;
  ConvParams conv;
  GnApplyParams gn;
  // generic slots
  const __nv_bfloat16* src = nullptr;
  __nv_bfloat16* dst = nullptr;
  int C = 0, H = 0, W = 0;
  ConvOutParams co;
  float2* ss = nullptr;  // OP_GN: output of gn_finalize
  float* f0 = nullptr;   // OP_ATTN1: score scratch; OP_MIX1X1: fp32 destination
  const float* fw = nullptr;  // OP_CONV_IN / OP_VAE_SAMPLE / OP_MIX1X1: fp32 weight and bias
  const float* fb = nullptr;
  const float* fc = nullptr;  // OP_XVEC: to_out bias
  float* f1 = nullptr;        // OP_XVEC: destination [N][C]
  int cin = 0;
  float eps = 0.f;            // OP_LN
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

struct PackJob {  // one K-segment's packed weights
  int w_param;      // index of the fp32 weight in the table
  int cout, cin_total, KH, KW, cin_off, ksteps;
  PackTaps taps;
  size_t off;       // byte offset in the packed arena
  int cout_real = -1;  // < cout when the output channels are zero-padded up to the 128-channel tile
};

// State shared by the model handles (U-Net, VAE): parameter table, packed-weight arena layout, workspace plan.
struct NetBase {
  int norm_groups = 32;
  float norm_eps = 1e-5f;
  std::vector<Param> params;
  std::map<std::string, int> pidx;
  std::vector<const float*> pptr;
  // packed arena layout
  std::vector<PackJob> jobs;
  std::map<std::string, size_t> seg_off;  // "<conv name>#<seg>" -> byte offset
  size_t packed_bytes = 0;
  size_t off_wcat = 0, off_bcat = 0, off_misc = 0;
  std::map<std::string, size_t> misc_off;  // fused bias vectors (floats)
  std::map<int, size_t> ident_off;         // channels -> identity weight blocks
  int temb_rows = 0;
  std::map<std::string, int> temb_row_off;
  uint8_t* packed = nullptr;
  // workspace / plan
  int N = 0, H = 0, W = 0;
  uint8_t* ws = nullptr;
  size_t ws_bytes = 0;
  std::vector<Op> plan;
  std::map<std::string, Act> taps;
  stat_t* stats_arena = nullptr;
  size_t stats_bytes = 0;
  float* temb_act = nullptr;
  float* temb_proj = nullptr;
  int* temb_lead = nullptr;         // [N] first sample with the same timestep (inference only)
  bool training = false;            // keep every activation (no pooling) and the timestep-MLP pre-activations for backward
  float* temb_emb = nullptr;        // [N][dim0]      sinusoid
  float* temb_u1 = nullptr;         // [N][4 dim0]    linear_1 output before SiLU
  float* temb_u2 = nullptr;         // [N][4 dim0]    linear_2 output before SiLU
  int num_sms = 132;
  const float* enc = nullptr;       // conditional U-Net: encoder_hidden_states [N][enc_S][X] of the next forward
  int enc_S = 0;
  int last_launches = 0;
  PackBatch pack_batch;             // device job table of the weight packing (one launch for all K-segments)
};

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

static const char* check_groups(const int* ch, int n, int groups) {
  if (groups < 1 || groups > 64) return "norm_num_groups must be in 1..64";
  for (int i = 0; i < n; ++i)   // GroupNorm partial sums are kept per 4-channel quad: a group must be whole quads
    if (ch[i] % groups || (ch[i] / groups) % 4) return "channels per GroupNorm group must be a multiple of 4 for every block";
  return nullptr;
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

static std::string S(const char* fmt, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return buf;
}

static PackTaps taps_3x3() {
  PackTaps t{};
  t.ntaps = 9;
  for (int k = 0; k < 9; ++k) { t.kh[k] = k / 3; t.kw[k] = k % 3; }
  return t;
}
static PackTaps taps_1x1() {
  PackTaps t{};
  t.ntaps = 1;
  t.kh[0] = 0; t.kw[0] = 0;
  return t;
}
// stride-2 3x3 conv on parity plane (a, b): the taps that read input rows of parity a and columns of parity b
static PackTaps taps_parity(int a, int b) {
  PackTaps t{};
  t.ntaps = 0;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      const int pa = (kh == 1) ? 0 : 1, pb = (kw == 1) ? 0 : 1;
      if (pa == a && pb == b) { t.kh[t.ntaps] = kh; t.kw[t.ntaps] = kw; ++t.ntaps; }
    }
  return t;
}

static void add_job(NetBase* h, Bump& b, const std::string& key, const std::string& wname, int cout, int cin_total,
                    int K, int cin_off, int cin_cnt, const PackTaps& taps) {
  PackJob j;
  j.w_param = h->pidx.at(wname);
  j.cout = cout; j.cin_total = cin_total; j.KH = K; j.KW = K; j.cin_off = cin_off; j.ksteps = cin_cnt / 16;
  j.taps = taps;
  j.cout_real = -1;
  const size_t bytes = (size_t)(cout / 128) * j.ksteps * taps.ntaps * CONV_B_TAP;
  b.take(0);
  j.off = (b.off + 255) & ~(size_t)255;
  b.take(bytes);
  h->seg_off[key] = j.off;
  h->jobs.push_back(j);
}

static size_t take_off(Bump& b, size_t bytes) {  // size-only pass: returns the aligned offset
  b.take(0);
  const size_t o = (b.off + 255) & ~(size_t)255;
  b.take(bytes);
  return o;
}
static void need_ident(NetBase* h, Bump& b, int ch) {  // identity weight blocks for residual-as-K-segment
  if (!h->ident_off.count(ch)) h->ident_off[ch] = take_off(b, (size_t)(ch / 128) * (ch / 16) * CONV_B_TAP);
}
// ResnetBlock2D over cat(a, b): conv1 is one K-segment per source (each with its own fused GroupNorm scale/shift slice),
// conv2 carries the shortcut (1x1 conv or identity) as extra K-segments.
static void layout_resnet(NetBase* h, Bump& b, const std::string& n, int ca, int cb, int co, bool temb) {
  const int cin = ca + cb;
  add_job(h, b, n + ".conv1#0", n + ".conv1.weight", co, cin, 3, 0, ca, taps_3x3());
  if (cb) add_job(h, b, n + ".conv1#1", n + ".conv1.weight", co, cin, 3, ca, cb, taps_3x3());
  add_job(h, b, n + ".conv2#0", n + ".conv2.weight", co, co, 3, 0, co, taps_3x3());
  if (cin == co) need_ident(h, b, co);
  if (cin != co) {
    add_job(h, b, n + ".conv2#1", n + ".conv_shortcut.weight", co, cin, 1, 0, ca, taps_1x1());
    if (cb) add_job(h, b, n + ".conv2#2", n + ".conv_shortcut.weight", co, cin, 1, ca, cb, taps_1x1());
    h->misc_off[n + ".bias2"] = take_off(b, (size_t)co * 4);
  }
  if (temb) {
    h->temb_row_off[n] = h->temb_rows;
    h->temb_rows += co;
  }
}
static void layout_attn(NetBase* h, Bump& b, const std::string& n, int ch) {
  add_job(h, b, n + ".qkv#q", n + ".to_q.weight", ch, ch, 1, 0, ch, taps_1x1());
  add_job(h, b, n + ".qkv#k", n + ".to_k.weight", ch, ch, 1, 0, ch, taps_1x1());
  add_job(h, b, n + ".qkv#v", n + ".to_v.weight", ch, ch, 1, 0, ch, taps_1x1());
  add_job(h, b, n + ".out#0", n + ".to_out.0.weight", ch, ch, 1, 0, ch, taps_1x1());
  h->misc_off[n + ".bias_qkv"] = take_off(b, (size_t)3 * ch * 4);
  need_ident(h, b, ch);
}

// Transformer2DModel + BasicTransformerBlock of the conditional U-Net (diffusers naming): packed 1x1 projections
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
static void layout_transformer(NetBase* h, Bump& b, const std::string& n, int c) {
  const std::string t = n + ".transformer_blocks.0";
  add_job(h, b, n + ".proj_in#0", n + ".proj_in.weight", c, c, 1, 0, c, taps_1x1());
  add_job(h, b, t + ".qkv#q", t + ".attn1.to_q.weight", c, c, 1, 0, c, taps_1x1());   // q | k | v blocks are contiguous
  add_job(h, b, t + ".qkv#k", t + ".attn1.to_k.weight", c, c, 1, 0, c, taps_1x1());
  add_job(h, b, t + ".qkv#v", t + ".attn1.to_v.weight", c, c, 1, 0, c, taps_1x1());
  add_job(h, b, t + ".attn1.out#0", t + ".attn1.to_out.0.weight", c, c, 1, 0, c, taps_1x1());
  add_job(h, b, t + ".ff1#0", t + ".ff.net.0.proj.weight", 8 * c, c, 1, 0, c, taps_1x1());
  add_job(h, b, t + ".ff2#0", t + ".ff.net.2.weight", c, 4 * c, 1, 0, 4 * c, taps_1x1());
  add_job(h, b, n + ".proj_out#0", n + ".proj_out.weight", c, c, 1, 0, c, taps_1x1());
  need_ident(h, b, c);
}

static __global__ void add_vec_kernel(const float* a, const float* b, float* o, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) o[i] = a[i] + (b ? b[i] : 0.f);
}

static bool ends_with(const std::string& s, const char* suf) {
  const size_t n = strlen(suf);
  return s.size() > n && s.compare(s.size() - n, n, suf) == 0;
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
  for (const auto& kv : h->misc_off) {
    const std::string& key = kv.first;
    float* dst = (float*)(h->packed + kv.second);
    if (ends_with(key, ".bias2")) {            // conv2.bias + conv_shortcut.bias
      const std::string n = key.substr(0, key.size() - 6);
      const int co = (int)h->params[h->pidx.at(n + ".conv2.bias")].shape[0];
      add_vec_kernel<<<(co + 255) / 256, 256, 0, st>>>(h->pptr[h->pidx.at(n + ".conv2.bias")],
                                                       h->pptr[h->pidx.at(n + ".conv_shortcut.bias")], dst, co);
      CK(cudaGetLastError());
    } else if (ends_with(key, ".bias_qkv")) {  // to_q | to_k | to_v biases
      const std::string n = key.substr(0, key.size() - 9);
      const int c = (int)h->params[h->pidx.at(n + ".to_q.bias")].shape[0];
      CK(cudaMemcpyAsync(dst, h->pptr[h->pidx.at(n + ".to_q.bias")], c * 4, cudaMemcpyDeviceToDevice, st));
      CK(cudaMemcpyAsync(dst + c, h->pptr[h->pidx.at(n + ".to_k.bias")], c * 4, cudaMemcpyDeviceToDevice, st));
      CK(cudaMemcpyAsync(dst + 2 * c, h->pptr[h->pidx.at(n + ".to_v.bias")], c * 4, cudaMemcpyDeviceToDevice, st));
    } else if (ends_with(key, ".bias_pad")) {  // bias zero-padded to 128 output channels
      const std::string n = key.substr(0, key.size() - 9);
      const int co = (int)h->params[h->pidx.at(n + ".bias")].shape[0];
      CK(cudaMemsetAsync(dst, 0, 128 * 4, st));
      CK(cudaMemcpyAsync(dst, h->pptr[h->pidx.at(n + ".bias")], co * 4, cudaMemcpyDeviceToDevice, st));
    } else {
      return set_err("unknown fused-bias key %s", key.c_str());
    }
  }
  return 0;
}

struct Builder {
  NetBase* h;
  Bump ws;
  Bump st;  // stats arena (floats, offsets in bytes)
  std::vector<Op>* plan;
  std::map<std::string, Act> pool;  // reusable transient buffers keyed by tag
  int N;
  bool nopool = false;  // B200AD_DEBUG_NOPOOL=1: every activation gets its own buffer (per-layer parity taps)
  bool single_head = false;  // attention with one head of dim C (AutoencoderKL mid block) instead of head_dim 8

  Act alloc(int C, int H, int W, bool stats) {
    Act a;
    a.C = C; a.H = H; a.W = W;
    const Geom g = make_geom(N, H, W);
    a.p = (__nv_bfloat16*)ws.take((size_t)N * (C / 8) * g.PL * 16);
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
  const float* P(const std::string& name) const { return h->pptr[h->pidx.at(name)]; }
  const __nv_bfloat16* WP(const std::string& key) const {
    return h->packed ? (const __nv_bfloat16*)(h->packed + h->seg_off.at(key)) : nullptr;
  }
  const float* MISC(const std::string& key) const { return h->packed ? (const float*)(h->packed + h->misc_off.at(key)) : nullptr; }

  void conv_common(ConvParams& p, const Act& out) {
    const Geom g = make_geom(N, out.H, out.W);
    p.N = N; p.H = out.H; p.W = out.W; p.Wp = g.Wp; p.lead = g.lead; p.PL = g.PL;
    p.cout = out.C;  // work decomposition (tiles per item, item count) is filled in by launch_conv_tc
    p.out = out.p;
    p.stats = out.stats;
  }
  static void seg_taps(ConvSeg& s, const PackTaps& t, bool parity, int a, int b) {
    s.ntaps = t.ntaps;
    s.ht = s.hb = s.hl = s.hr = 0;
    for (int k = 0; k < t.ntaps; ++k) {
      if (parity) {
        s.dh[k] = (t.kh[k] == 0) ? -1 : 0;
        s.dw[k] = (t.kw[k] == 0) ? -1 : 0;
      } else if (t.ntaps == 9) {
        s.dh[k] = (signed char)(t.kh[k] - 1);
        s.dw[k] = (signed char)(t.kw[k] - 1);
      } else {
        s.dh[k] = 0; s.dw[k] = 0;
      }
      if (s.dh[k] < 0) s.ht = 1;
      if (s.dh[k] > 0) s.hb = 1;
      if (s.dw[k] < 0) s.hl = 1;
      if (s.dw[k] > 0) s.hr = 1;
    }
    (void)a; (void)b;
  }
  void set_seg(ConvSeg& s, const __nv_bfloat16* src, int C, int H, int W, const __nv_bfloat16* wpack, const PackTaps& t,
               bool parity = false) {
    const Geom g = make_geom(N, H, W);
    s.src = src;
    s.wpack = wpack;
    s.img_stride = (long long)(C / 8) * g.PL * 8;
    s.ksteps = C / 16;
    s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
    seg_taps(s, t, parity, 0, 0);
  }

  // GroupNorm over cat(a, b): statistics -> per-(sample, channel) scale/shift; the apply itself is fused into the consumer
  // conv's transform warps. Returns the [N][Ca + Cb] scale/shift array.
  // Let the launch just planned (the producer of `a`; `b`, a skip connection, is older) finalize the GroupNorm over
  // cat(a, b) in its last CTA.  Returns the [N][Ca + Cb] (scale, shift) array, or nullptr if the last op cannot do it
  // (conv_in, an op of another kind, a batch too large for the scratch).
  float2* gn_attach(const Act& a, const Act* b, const std::string& norm, float2* ss = nullptr, float eps = -1.f) {
    const int Ct = a.C + (b ? b->C : 0);
    static const bool off = [] { const char* e = getenv("B200AD_NO_GNFOLD"); return e && e[0] == '1'; }();   // A/B switch
    if (off) return nullptr;
    if (plan->empty() || plan->back().kind != OP_CONV || plan->back().conv.out != a.p || plan->back().conv.fin.ss ||
        (size_t)N * h->norm_groups * 2 * sizeof(float) > 32768)
      return nullptr;
    if (!ss) ss = (float2*)ws.take((size_t)N * Ct * sizeof(float2));
    ConvGnFin& f = plan->back().conv.fin;
    f.stats[0] = a.stats; f.C[0] = a.C;
    f.stats[1] = b ? b->stats : nullptr; f.C[1] = b ? b->C : 0;
    f.gamma = P(norm + ".weight"); f.beta = P(norm + ".bias");
    f.ss = ss;
    f.counter = (unsigned*)ws.take(sizeof(unsigned));
    f.groups = h->norm_groups; f.HW = a.H * a.W; f.eps = eps < 0.f ? h->norm_eps : eps;
    return ss;
  }
  float2* gn_attach(const Act& a, const std::string& norm) { return gn_attach(a, nullptr, norm); }

  float2* gn_finalize(const Act& a, const Act* b, const std::string& norm, float eps = -1.f) {
    const int Ct = a.C + (b ? b->C : 0);
    float2* ss = (float2*)ws.take((size_t)N * Ct * sizeof(float2));
    if (gn_attach(a, b, norm, ss, eps)) return ss;
    Op op{};
    op.kind = OP_GN;
    GnApplyParams& p = op.gn;
    p.src[0] = a.p; p.stats[0] = a.stats; p.C[0] = a.C;
    p.src[1] = b ? b->p : nullptr; p.stats[1] = b ? b->stats : nullptr; p.C[1] = b ? b->C : 0;
    p.gamma = P(norm + ".weight"); p.beta = P(norm + ".bias");
    p.dst = nullptr;
    p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = eps < 0.f ? h->norm_eps : eps; p.silu = 0;
    op.ss = ss;
    plan->push_back(op);
    return ss;
  }
  static void seg_norm(ConvSeg& s, const float2* ss, int stride, bool silu) {
    s.ss = ss; s.ss_stride = stride; s.silu = silu ? 1 : 0;
  }
  const __nv_bfloat16* IDENT(int ch) const {
    return h->packed ? (const __nv_bfloat16*)(h->packed + h->ident_off.at(ch)) : nullptr;
  }

  // ResnetBlock2D on x = cat(a, b) (b optional) -> out (raw + stats)
  Act resnet(const std::string& n, const Act& a, const Act* b, int cout, bool out_pooled, const std::string& out_tag) {
    const int cin = a.C + (b ? b->C : 0);
    const int H = a.H, W = a.W;
    const float2* ss1 = gn_finalize(a, b, n + ".norm1");
    Act h1 = pooled("h1", cout, H, W, true);
    {
      Op op{};
      op.kind = OP_CONV;
      ConvParams& p = op.conv;
      conv_common(p, h1);
      p.nseg = 1;
      set_seg(p.seg[0], a.p, a.C, H, W, WP(n + ".conv1#0"), taps_3x3());
      seg_norm(p.seg[0], ss1, cin, true);
      if (b) {
        set_seg(p.seg[1], b->p, b->C, H, W, WP(n + ".conv1#1"), taps_3x3());
        seg_norm(p.seg[1], ss1 + a.C, cin, true);
        p.nseg = 2;
      }
      p.bias = P(n + ".conv1.bias");
      if (h->temb_rows) {
        p.temb = h->temb_proj + h->temb_row_off.at(n);
        p.temb_stride = h->temb_rows;
      } else {
        p.temb = nullptr;
        p.temb_stride = 0;
      }
      plan->push_back(op);
    }
    const float2* ss2 = gn_finalize(h1, nullptr, n + ".norm2");
    Act out = out_pooled ? pooled(out_tag, cout, H, W, true) : alloc(cout, H, W, true);
    {
      Op op{};
      op.kind = OP_CONV;
      ConvParams& p = op.conv;
      conv_common(p, out);
      p.nseg = 1;
      set_seg(p.seg[0], h1.p, cout, H, W, WP(n + ".conv2#0"), taps_3x3());
      seg_norm(p.seg[0], ss2, cout, true);
      p.temb = nullptr;
      p.temb_stride = 0;
      if (cin != cout) {  // 1x1 conv_shortcut over the raw input(s): extra K-segments into the same accumulators
        set_seg(p.seg[1], a.p, a.C, H, W, WP(n + ".conv2#1"), taps_1x1());
        p.nseg = 2;
        if (b) {
          set_seg(p.seg[2], b->p, b->C, H, W, WP(n + ".conv2#2"), taps_1x1());
          p.nseg = 3;
        }
        p.bias = MISC(n + ".bias2");
      } else {            // identity shortcut: residual add as a 1-tap identity-weight segment over the raw input
        set_seg(p.seg[1], a.p, a.C, H, W, IDENT(cout), taps_1x1());
        p.nseg = 2;
        p.bias = P(n + ".conv2.bias");
      }
      plan->push_back(op);
    }
    h->taps[n + ".h1"] = h1;
    h->taps[n] = out;
    return out;
  }

  // plain 1-tap conv (a linear layer over the pixel tokens) with optional fused GroupNorm of the source, identity residual
  // and per-sample additive vector
  void linear(const Act& out, const Act& src, const std::string& wkey, const float* bias, const float2* ss = nullptr,
              const Act* residual = nullptr, const float* vec = nullptr, int vec_stride = 0) {
    Op op{};
    op.kind = OP_CONV;
    ConvParams& p = op.conv;
    conv_common(p, out);
    p.nseg = 1;
    set_seg(p.seg[0], src.p, src.C, src.H, src.W, WP(wkey), taps_1x1());
    if (ss) seg_norm(p.seg[0], ss, src.C, false);
    if (residual) {
      set_seg(p.seg[1], residual->p, residual->C, residual->H, residual->W, IDENT(residual->C), taps_1x1());
      p.nseg = 2;
    }
    p.bias = bias;
    p.temb = vec; p.temb_stride = vec_stride;
    plan->push_back(op);
  }

  // Transformer2DModel with one BasicTransformerBlock (conditional U-Net), encoder sequence length 1:
  //   h0 = proj_in(GroupNorm(x));  h2 = h0 + attn1(LN1(h0)) + attn2(enc);  h3 = h2 + ff(LN3(h2));  out = proj_out(h3) + x
  // attn2 with ONE key is the per-sample vector to_out(to_v(enc)) (softmax over a single key is 1): it rides on the
  // per-sample additive term of the attn1 output projection.
  Act transformer(const std::string& n, const Act& x, int heads, int X, bool out_pooled, const std::string& out_tag) {
    const int C = x.C, H = x.H, W = x.W;
    const std::string t = n + ".transformer_blocks.0";
    const float2* ssx = gn_finalize(x, nullptr, n + ".norm", 1e-6f);
    float* vec = (float*)ws.take((size_t)N * C * sizeof(float));
    {
      Op op{};
      op.kind = OP_XVEC;
      op.C = C; op.cin = X;
      op.fw = P(t + ".attn2.to_v.weight"); op.fb = P(t + ".attn2.to_out.0.weight"); op.fc = P(t + ".attn2.to_out.0.bias");
      op.f1 = vec;
      plan->push_back(op);
    }
    Act h0 = pooled("tf_h0", C, H, W, false);
    linear(h0, x, n + ".proj_in#0", P(n + ".proj_in.bias"), ssx);
    Act n1 = pooled("tf_ln", C, H, W, false);
    auto layer_norm = [&](const Act& src, const Act& dst, const std::string& nm) {
      Op op{};
      op.kind = OP_LN;
      op.src = src.p; op.dst = dst.p; op.C = C; op.H = H; op.W = W;
      op.fw = P(nm + ".weight"); op.fb = P(nm + ".bias"); op.eps = 1e-5f;
      plan->push_back(op);
    };
    layer_norm(h0, n1, t + ".norm1");
    Act qkv = pooled("tf_qkv", 3 * C, H, W, false);
    linear(qkv, n1, t + ".qkv#q", nullptr);
    Act ao = pooled("tf_ao", C, H, W, false);
    {
      Op op{};
      op.kind = OP_MHA;
      op.src = qkv.p; op.dst = ao.p; op.C = C; op.H = H; op.W = W; op.cin = heads;
      plan->push_back(op);
    }
    Act h2 = pooled("tf_h2", C, H, W, false);
    linear(h2, ao, t + ".attn1.out#0", P(t + ".attn1.to_out.0.bias"), nullptr, &h0, vec, C);
    layer_norm(h2, n1, t + ".norm3");
    Act ff1 = pooled("tf_ff1", 8 * C, H, W, false);
    linear(ff1, n1, t + ".ff1#0", P(t + ".ff.net.0.proj.bias"));
    Act gg = pooled("tf_gg", 4 * C, H, W, false);
    {
      Op op{};
      op.kind = OP_GEGLU;
      op.src = ff1.p; op.dst = gg.p; op.C = 4 * C; op.H = H; op.W = W;
      plan->push_back(op);
    }
    Act h3 = pooled("tf_h0", C, H, W, false);     // h0 is dead after h2
    linear(h3, gg, t + ".ff2#0", P(t + ".ff.net.2.bias"), nullptr, &h2);
    Act out = out_pooled ? pooled(out_tag, C, H, W, true) : alloc(C, H, W, true);
    linear(out, h3, n + ".proj_out#0", P(n + ".proj_out.bias"), nullptr, &x);
    h->taps[n + ".attn2"] = h2;
    h->taps[n] = out;
    return out;
  }

  // Downsample2D(use_conv, padding 1): 3x3 stride-2 conv = four K-segments over the parity planes of the input
  Act down2(const std::string& n, const Act& x) {
    const int C = x.C, Ho = x.H / 2, Wo = x.W / 2;
    const Geom go = make_geom(N, Ho, Wo);
    const size_t tsz = (size_t)N * (C / 8) * go.PL * 8;  // elements per parity tensor
    Act par = pooled("parity", 4 * C, Ho, Wo, false);     // 4 tensors back to back (same bytes as 4C channels)
    h->taps[n + ".parity"] = par;
    {
      Op op{};
      op.kind = OP_PARITY;
      op.src = x.p; op.dst = par.p; op.C = C; op.H = x.H; op.W = x.W;
      plan->push_back(op);
    }
    Act y = alloc(C, Ho, Wo, true);
    Op op{};
    op.kind = OP_CONV;
    ConvParams& p = op.conv;
    conv_common(p, y);
    p.nseg = 4;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b)
        set_seg(p.seg[a * 2 + b], par.p + (size_t)(a * 2 + b) * tsz, C, Ho, Wo, WP(n + S("#%d", a * 2 + b)), taps_parity(a, b), true);
    p.bias = P(n + ".bias");
    p.temb = nullptr; p.temb_stride = 0;
    plan->push_back(op);
    h->taps[n] = y;
    return y;
  }

  // Upsample2D(use_conv): nearest-2x + 3x3 conv folded into four 2x2 convs on the low-res tensor (one launch per parity)
  Act up2(const std::string& nm, const Act& x) {
    const int C = x.C, hh = x.H, ww = x.W;
    Act y = pooled("up_conv", C, hh * 2, ww * 2, true);
    for (int pa = 0; pa < 2; ++pa)
      for (int pb = 0; pb < 2; ++pb) {
        const UpTaps ut = taps_up2(pa, pb);
        Op op{};
        op.kind = OP_CONV;
        ConvParams& p = op.conv;
        Act lo = y;                       // item geometry = low-res input geometry, output tensor = y
        lo.H = hh; lo.W = ww;
        conv_common(p, lo);
        p.up2 = 1; p.oy = pa; p.ox = pb;
        p.nseg = 1;
        ConvSeg& sgm = p.seg[0];
        set_seg(sgm, x.p, C, hh, ww, WP(nm + S("#p%d", pa * 2 + pb)), ut.pack);
        sgm.ht = sgm.hb = sgm.hl = sgm.hr = 0;
        for (int t = 0; t < 4; ++t) {
          sgm.dh[t] = ut.dh[t]; sgm.dw[t] = ut.dw[t];
          if (ut.dh[t] < 0) sgm.ht = 1;
          if (ut.dh[t] > 0) sgm.hb = 1;
          if (ut.dw[t] < 0) sgm.hl = 1;
          if (ut.dw[t] > 0) sgm.hr = 1;
        }
        p.bias = P(nm + ".bias");
        p.temb = nullptr; p.temb_stride = 0;
        plan->push_back(op);
      }
    h->taps[nm] = y;
    return y;
  }

  Act attention(const std::string& n, const Act& x, bool out_pooled, const std::string& out_tag) {
    const int C = x.C, H = x.H, W = x.W;
    // The q/k/v projection is a 1-tap conv with 3C/128 (= 12) cout tiles: fused, every one of those tiles would re-normalise
    // the same window in its transform warps, and a 1-tap k-step (192 MMA cycles) cannot hide that (measured 187 us per
    // launch at 16x16, batch 64).  The normalised tensor is tiny here (16 MB): materialise it once, project the plain tensor.
    Act xn = pooled("attn_xn", C, H, W, false);
    {
      Op op{};
      op.kind = OP_GNAPPLY;
      GnApplyParams& g = op.gn;
      g.src[0] = x.p; g.stats[0] = x.stats; g.C[0] = C;
      g.src[1] = nullptr; g.stats[1] = nullptr; g.C[1] = 0;
      g.gamma = P(n + ".group_norm.weight"); g.beta = P(n + ".group_norm.bias");
      g.dst = xn.p;
      g.N = N; g.H = H; g.W = W; g.groups = h->norm_groups; g.eps = h->norm_eps; g.silu = 0;
      plan->push_back(op);
    }
    Act qkv = pooled("qkv", 3 * C, H, W, false);
    {
      Op op{};
      op.kind = OP_CONV;
      ConvParams& p = op.conv;
      conv_common(p, qkv);
      p.nseg = 1;
      set_seg(p.seg[0], xn.p, C, H, W, WP(n + ".qkv#q"), taps_1x1());  // q|k|v blocks are contiguous
      p.bias = MISC(n + ".bias_qkv");
      p.temb = nullptr; p.temb_stride = 0; p.stats = nullptr;
      plan->push_back(op);
    }
    Act ao = pooled("attn_o", C, H, W, false);
    {
      Op op{};
      op.kind = single_head ? OP_ATTN1 : OP_ATTN;
      op.src = qkv.p; op.dst = ao.p; op.C = C; op.H = H; op.W = W;
      if (single_head) op.f0 = (float*)ws.take((size_t)N * H * W * H * W * sizeof(float));
      plan->push_back(op);
    }
    Act out = out_pooled ? pooled(out_tag, C, H, W, true) : alloc(C, H, W, true);
    {
      Op op{};
      op.kind = OP_CONV;
      ConvParams& p = op.conv;
      conv_common(p, out);
      p.nseg = 2;
      set_seg(p.seg[0], ao.p, C, H, W, WP(n + ".out#0"), taps_1x1());
      set_seg(p.seg[1], x.p, C, H, W, IDENT(C), taps_1x1());          // + residual
      p.bias = P(n + ".to_out.0.bias");
      p.temb = nullptr; p.temb_stride = 0;
      plan->push_back(op);
    }
    h->taps[n + ".qkv"] = qkv;
    h->taps[n + ".ao"] = ao;
    h->taps[n] = out;
    return out;
  }
};

}  // namespace b200ad
