// Host side of the U-Net: parameter table (diffusers naming), weight packing, activation workspace layout and
// the launch plan that walks UNet2DModel.forward (reference call sites: audiodiffusion/pipeline_audio_diffusion.py:163,
// :237; architecture: scripts/train_unet.py:115-137).  No tensor math happens on the host.
#include "unet.cuh"

namespace b200ad {

thread_local char g_err[512] = "";
int set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return -1;
}

}  // namespace b200ad

using namespace b200ad;


namespace b200ad {

// UNet2DModel.forward as a block list: conv_in, down blocks (each output a skip connection), mid block, up blocks (each
// resnet consuming one skip, last first), conv_out.  The pool tags decide which outputs may share a buffer: a resnet
// followed by attention writes the transient "res_tmp"; the up path alternates "up_a" / "up_b".
static std::vector<Block> unet_blocks(const b200ad_unet_config& c) {
  const int nb = c.num_blocks, D = c.block_out_channels[0] * 4, X = c.cross_attention_dim;
  const int* boc = c.block_out_channels;
  std::vector<Block> bl;
  add_block(bl, BK_UNET_HEAD, "", c.in_channels, boc[0], "").temb = D;
  std::vector<int> skips{0};
  auto attn = [&](const std::string& n, bool self, bool cross, int ch, const char* pool) {
    if (self || cross) add_block(bl, cross ? BK_TRANSFORMER : BK_ATTN, n, ch, ch, pool).cross = cross ? X : 0;
  };
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < c.layers_per_block; ++j) {
      const bool att = c.down_attn[i] || c.down_cross[i];
      add_block(bl, BK_RESNET, S("down_blocks.%d.resnets.%d", i, j), bl.back().cout, boc[i], att ? "res_tmp" : "").temb = D;
      attn(S("down_blocks.%d.attentions.%d", i, j), c.down_attn[i], c.down_cross[i], boc[i], "");
      skips.push_back((int)bl.size() - 1);
    }
    if (i != nb - 1) {
      add_block(bl, BK_DOWN, S("down_blocks.%d.downsamplers.0.conv", i), boc[i], boc[i], "");
      skips.push_back((int)bl.size() - 1);
    }
  }
  const int mid = boc[nb - 1];
  add_block(bl, BK_RESNET, "mid_block.resnets.0", mid, mid, "res_tmp").temb = D;
  attn("mid_block.attentions.0", !X, X != 0, mid, "up_a");
  add_block(bl, BK_RESNET, "mid_block.resnets.1", mid, mid, "up_b").temb = D;
  int flip = 0;
  for (int i = 0; i < nb; ++i) {
    const int out_c = boc[nb - 1 - i];
    for (int j = 0; j < c.layers_per_block + 1; ++j) {
      const bool att = c.up_attn[i] || c.up_cross[i];
      const int sk = skips.back();
      skips.pop_back();
      Block& r = add_block(bl, BK_RESNET, S("up_blocks.%d.resnets.%d", i, j), bl.back().cout, out_c,
                           att ? "res_tmp" : (flip++ & 1) ? "up_b" : "up_a");
      r.skip = sk;
      r.cskip = bl[sk].cout;
      r.temb = D;
      if (att) attn(S("up_blocks.%d.attentions.%d", i, j), c.up_attn[i], c.up_cross[i], out_c, (flip++ & 1) ? "up_b" : "up_a");
    }
    if (i != nb - 1) add_block(bl, BK_UP, S("up_blocks.%d.upsamplers.0.conv", i), out_c, out_c, "up_conv");
  }
  add_block(bl, BK_CONV_OUT, "", boc[0], c.out_channels, "");
  return bl;
}

}  // namespace b200ad

// ================================================================================= C ABI: U-Net
extern "C" const char* b200ad_last_error(void) { return g_err; }
extern "C" int b200ad_version(void) { return 1; }

extern "C" int b200ad_unet_create(const b200ad_unet_config* cfg, b200ad_unet** out) {
  if (!cfg || !out) return set_err("null argument");
  if (check_net_config(cfg->num_blocks, cfg->block_out_channels, cfg->out_channels, cfg->norm_num_groups)) return -1;
  if (cfg->attention_head_dim != 8) return set_err("only attention_head_dim == 8 is implemented");
  if (cfg->cross_attention_dim < 0 || cfg->cross_attention_dim > 4096) return set_err("cross_attention_dim out of range");
  for (int i = 0; i < cfg->num_blocks; ++i) {
    if ((cfg->down_cross[i] || cfg->up_cross[i]) && !cfg->cross_attention_dim) return set_err("cross-attention blocks need cross_attention_dim");
    if ((cfg->down_cross[i] && cfg->down_attn[i]) || (cfg->up_cross[i] && cfg->up_attn[i])) return set_err("a block is either Attn or CrossAttn");
    const int d = cfg->block_out_channels[i] / 8;    // conditional model: 8 heads, head_dim = channels / 8
    if ((cfg->down_cross[i] || cfg->up_cross[i]) && d != 16 && d != 32 && d != 64) return set_err("cross-attention blocks need channels / 8 in {16, 32, 64}");
  }
  b200ad_unet* h = new b200ad_unet();
  h->cfg = *cfg;
  h->norm_groups = cfg->norm_num_groups;
  h->norm_eps = cfg->norm_eps;
  h->heads = cfg->attention_head_dim;
  std::vector<Block>& bl = h->parts[0] = unet_blocks(*cfg);
  for (const Block& k : bl) p_block(h, k);
  Bump b;
  for (Block& k : bl) layout_block(h, b, k);
  const int D = cfg->block_out_channels[0] * 4;
  h->off_wcat = take_off(b, (size_t)h->temb_rows * D * 4);
  h->off_bcat = take_off(b, (size_t)h->temb_rows * 4);
  for (Block& k : bl)
    if (k.kind == BK_TRANSFORMER) layout_attn2(h, b, k);
  h->packed_bytes = (b.off + 255) & ~(size_t)255;
  h->pptr.assign(h->params.size(), nullptr);
  *out = h;
  return 0;
}
extern "C" void b200ad_unet_destroy(b200ad_unet* h) {
  if (!h) return;
  release_backward(h);
  delete h;
}
extern "C" int b200ad_unet_num_params(const b200ad_unet* h) { return (int)h->params.size(); }
extern "C" const char* b200ad_unet_param_name(const b200ad_unet* h, int i) { return h->params[i].name.c_str(); }
extern "C" int b200ad_unet_param_shape(const b200ad_unet* h, int i, int64_t* dims) { return param_shape(h, i, dims); }
extern "C" size_t b200ad_unet_packed_bytes(const b200ad_unet* h) { return h->packed_bytes; }

extern "C" int b200ad_unet_set_params(b200ad_unet* h, const float* const* params, void* packed, size_t packed_bytes,
                                      void* stream) {
  if (packed_bytes < h->packed_bytes) return set_err("packed buffer too small: %zu < %zu", packed_bytes, h->packed_bytes);
  cudaStream_t st = (cudaStream_t)stream;
  for (size_t i = 0; i < h->params.size(); ++i) h->pptr[i] = params[i];
  h->packed = (uint8_t*)packed;
  if (pack_common(h, st)) return -1;
  h->xpacked = false;
  if ((h->plan_enc_len > 1 || h->enc_len > 1) && pack_xattn(h, st)) return -1;   // else packed when such a plan is bound
  // concatenated time_emb_proj weights / biases
  const int D = h->cfg.block_out_channels[0] * 4;
  for (const Block& k : h->parts[0]) {
    if (k.temb_row < 0) continue;
    CK(cudaMemcpyAsync(h->packed + h->off_wcat + (size_t)k.temb_row * D * 4,
                       h->pptr[h->pidx.at(k.name + ".time_emb_proj.weight")], (size_t)k.cout * D * 4,
                       cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(h->packed + h->off_bcat + (size_t)k.temb_row * 4,
                       h->pptr[h->pidx.at(k.name + ".time_emb_proj.bias")], (size_t)k.cout * 4, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

// ================================================================================= plan builder
namespace b200ad {

// Two passes: the stats arena lives at the start of the workspace; its size is found by a dry run.
Plan build_plan(const b200ad_unet* h, uint8_t* ws_base, int N, int H, int W) {
  Plan pl;
  pl.lists.resize(1);
  OpList& l = pl.lists[0];
  Builder B;
  B.h = h; B.built = &pl; B.ops = &l.ops;
  B.N = N; B.H = H; B.W = W;
  B.ckpt = pl.checkpoint = h->training && h->checkpointing;
  B.nopool = debug_nopool() || (h->training && !B.ckpt);
  B.ws.base = ws_base;
  for (int pass = 0; pass < 2; ++pass) {
    l.ops.clear();
    B.reset();
    B.st.base = pass == 0 ? nullptr : ws_base;
    B.st.off = 0;
    B.ws.off = pass == 0 ? 0 : ((l.stats_bytes + 255) & ~(size_t)255);
    B.run(h->parts[0], &l.recompute);
    if (pass == 0) l.stats_bytes = B.st.off;
  }
  l.stats = (stat_t*)ws_base;
  pl.ws_bytes = (B.ws.off + 255) & ~(size_t)255;
  return pl;
}

}  // namespace b200ad

extern "C" size_t b200ad_unet_workspace_bytes(const b200ad_unet* h, int N, int H, int W) {
  return build_plan(h, nullptr, N, H, W).ws_bytes;
}

extern "C" int b200ad_unet_bind_workspace(b200ad_unet* h, void* workspace, size_t bytes, int N, int H, int W, void* stream) {
  if (bind_workspace(h, build_plan, workspace, bytes, N, H, W, (cudaStream_t)stream)) return -1;
  h->plan_enc_len = h->enc_len;
  if (h->plan_enc_len > 1 && !h->xpacked && pack_xattn(h, (cudaStream_t)stream)) return -1;
  return 0;
}

extern "C" int b200ad_unet_set_encoder_len(b200ad_unet* h, int S) {
  if (!h) return set_err("null handle");
  if (!h->cfg.cross_attention_dim) return set_err("set_encoder_len: this U-Net is unconditional");
  if (S < 1 || S > XATTN_MAX_S) return set_err("set_encoder_len: encoder sequence length %d outside [1, %d]", S, XATTN_MAX_S);
  h->enc_len = S;
  return 0;
}

// The bound encoding must have the token count the bound plan was built for (its K / V buffers, its op list).
static int check_encoding(const b200ad_unet* h, const char* what) {
  if (!h->cfg.cross_attention_dim) return 0;
  if (!h->enc) return set_err("conditional U-Net: call b200ad_unet_set_encoding before %s", what);
  if (h->plan_enc_len > 1 && !h->xpacked) return set_err("conditional U-Net: weights not packed for the bound plan");
  if (h->enc_S != h->plan_enc_len)
    return set_err("conditional U-Net: the encoding has %d tokens but the workspace is planned for %d (call "
                   "b200ad_unet_set_encoder_len(%d) and bind the workspace again)", h->enc_S, h->plan_enc_len, h->enc_S);
  return 0;
}

static int run_plan(b200ad_unet* h, const RunArgs& a, cudaStream_t st, OpEvents* timing = nullptr) {
  if (h->plan.lists.empty()) return set_err("bind_workspace must be called before forward");
  if (check_encoding(h, "forward")) return -1;   // the transformer blocks read the encoding
  return run_ops(h, h->plan.lists[0], a, st, &h->last_launches, timing);
}

// One step with a CUDA event pair around every launch of the plan (device time per op, on `stream`).
extern "C" int b200ad_unet_profile_step(b200ad_unet* h, const float* x, const float* t, const float* z,
                                        const b200ad_step_coef* coef, float* x_out, float* op_ms, int* op_kind,
                                        double* op_flops, int max_ops, void* stream) {
  if (h->plan.lists.empty()) return set_err("bind_workspace must be called before profile_step");
  cudaStream_t st = (cudaStream_t)stream;
  const std::vector<Op>& ops = h->plan.lists[0].ops;
  const int nops = (int)ops.size();
  if (nops > max_ops) return set_err("profile_step: %d ops > max_ops %d", nops, max_ops);
  const b200ad_multistep_coef mc = {*coef, 0.f, 0.f};
  RunArgs a;
  a.in = x; a.t = t; a.noise = z; a.coef = &mc; a.x_out = x_out;
  OpEvents ev;
  if (run_plan(h, a, st, &ev)) return -1;
  CK(cudaStreamSynchronize(st));
  for (int i = 0; i < nops; ++i) {
    if (ev.ms(i, &op_ms[i])) return -1;
    op_kind[i] = (int)ops[i].kind;
    double fl = 0;
    if (ops[i].kind == OP_CONV) {
      const ConvParams& p = ops[i].conv;
      double k = 0;
      // algorithmic taps: a folded upsample launch stands for the 3x3 conv on its quarter of the output pixels; a residual
      // add carried as an identity-weight K-segment is an addition, not a convolution: no algorithmic FLOPs
      for (int s = 0; s < p.nseg; ++s) {
        bool ident = false;
        for (const auto& kv : h->ident_off)
          if ((const uint8_t*)p.seg[s].wpack == h->packed + kv.second) ident = true;
        if (!ident) k += (double)(p.up2 ? 9 : p.seg[s].ntaps) * p.seg[s].ksteps * 16;
      }
      fl = 2.0 * p.N * p.H * p.W * p.cout * k;
    }
    op_flops[i] = fl;
  }
  return nops;
}

extern "C" int b200ad_unet_conv_plan(const b200ad_unet* h, int N, int H, int W, int num_sms, int* rows, int max_rows) {
  const Plan pl = build_plan(h, nullptr, N, H, W);
  const int dbg = conv_dbg_env();
  int n = 0;
  for (const Op& op : pl.lists[0].ops) {
    if (op.kind != OP_CONV) continue;
    if (n >= max_rows) return set_err("conv_plan: more than %d conv launches", max_rows);
    ConvParams p = op.conv;
    p.dbg = dbg;
    if (plan_conv_tc(p, num_sms) != cudaSuccess) return set_err("conv_plan: launch %d cannot be planned", n);
    const int row[B200AD_CONV_PLAN_COLS] = {p.H, p.W, p.seg[0].ksteps * 16, p.cout, p.nseg, p.up2,
                                             p.pack, p.tw, p.th, p.total_work, p.as, p.bs};
    for (int c = 0; c < B200AD_CONV_PLAN_COLS; ++c) rows[n * B200AD_CONV_PLAN_COLS + c] = row[c];
    ++n;
  }
  return n;
}

extern "C" int b200ad_unet_set_encoding(b200ad_unet* h, const float* enc, int S) {
  if (!h->cfg.cross_attention_dim) return set_err("set_encoding: this U-Net is unconditional");
  if (S < 1) return set_err("set_encoding: empty encoder sequence");
  h->enc = enc;
  h->enc_S = S;
  return 0;
}

extern "C" int b200ad_unet_forward(b200ad_unet* h, const float* x, const float* t, float* eps_out, void* stream) {
  RunArgs a;
  a.in = x; a.t = t; a.out = eps_out;
  return run_plan(h, a, (cudaStream_t)stream);
}
// The DDPM / DDIM step is the multistep step without history.
extern "C" int b200ad_unet_forward_multistep(b200ad_unet* h, const float* x, const float* t, const float* z,
                                             const b200ad_multistep_coef* coef, float* hist1, float* hist2, float* x_out,
                                             float* eps_out, void* stream) {
  if (!coef || !x_out) return set_err("coef and x_out are required");
  if (hist2 && !hist1) return set_err("forward_multistep: hist2 needs hist1");
  RunArgs a;
  a.in = x; a.t = t; a.noise = z; a.coef = coef; a.x_out = x_out; a.out = eps_out; a.hist1 = hist1; a.hist2 = hist2;
  return run_plan(h, a, (cudaStream_t)stream);
}
extern "C" int b200ad_unet_forward_step(b200ad_unet* h, const float* x, const float* t, const float* z,
                                        const b200ad_step_coef* coef, float* x_out, float* eps_out, void* stream) {
  if (!coef) return set_err("coef and x_out are required");
  const b200ad_multistep_coef mc = {*coef, 0.f, 0.f};
  return b200ad_unet_forward_multistep(h, x, t, z, &mc, nullptr, nullptr, x_out, eps_out, stream);
}
// per-step scalars -> device (kernel ARGUMENTS are copied at launch time, so the host may run any number of steps ahead)
template <typename Coef>
__global__ void step_scalars_kernel(Coef coef, float t, Coef* coef_dev, float* t_dev, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *coef_dev = coef;
  if (i < n) t_dev[i] = t;
}
template <typename Coef>
static int step_scalars_upload(const Coef* coef, float t, Coef* coef_dev, float* t_dev, int n, void* stream) {
  if (!coef || !coef_dev || !t_dev || n < 1) return set_err("step_scalars_upload: bad arguments");
  step_scalars_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*coef, t, coef_dev, t_dev, n);
  CK(cudaGetLastError());
  return 0;
}
extern "C" int b200ad_step_scalars_upload(const b200ad_step_coef* coef, float t, b200ad_step_coef* coef_dev, float* t_dev, int n,
                                          void* stream) {
  return step_scalars_upload(coef, t, coef_dev, t_dev, n, stream);
}
extern "C" int b200ad_multistep_scalars_upload(const b200ad_multistep_coef* coef, float t, b200ad_multistep_coef* coef_dev,
                                               float* t_dev, int n, void* stream) {
  return step_scalars_upload(coef, t, coef_dev, t_dev, n, stream);
}
extern "C" int b200ad_unet_forward_multistep_dev(b200ad_unet* h, const float* x, const float* t, const float* z,
                                                 const b200ad_multistep_coef* coef_dev, float* hist1, float* hist2,
                                                 float* x_out, void* stream) {
  if (!coef_dev || !x_out) return set_err("coef_dev and x_out are required");
  if (hist2 && !hist1) return set_err("forward_multistep_dev: hist2 needs hist1");
  RunArgs a;
  a.in = x; a.t = t; a.noise = z; a.coef_dev = coef_dev; a.x_out = x_out; a.hist1 = hist1; a.hist2 = hist2;
  return run_plan(h, a, (cudaStream_t)stream);
}
// Without history the kernel reads only the leading b200ad_step_coef of *coef_dev, so a plain one may stand in for it.
extern "C" int b200ad_unet_forward_step_dev(b200ad_unet* h, const float* x, const float* t, const float* z,
                                            const b200ad_step_coef* coef_dev, float* x_out, void* stream) {
  return b200ad_unet_forward_multistep_dev(h, x, t, z, reinterpret_cast<const b200ad_multistep_coef*>(coef_dev), nullptr,
                                           nullptr, x_out, stream);
}
extern "C" int b200ad_unet_last_launch_count(const b200ad_unet* h) { return h->last_launches; }

extern "C" int b200ad_unet_debug_tensor(b200ad_unet* h, const char* name, float* dst, int* dims, void* stream) {
  return debug_tensor(h, name, dst, dims, (cudaStream_t)stream);
}
