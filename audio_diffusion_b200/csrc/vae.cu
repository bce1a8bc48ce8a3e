// Host side of the latent autoencoder: diffusers `AutoencoderKL` in the shape of config/ldm_autoencoder_kl.yaml:18-28
// (ch 128, ch_mult [1,2,4,4], 2 res blocks, z_channels 1), as the pipeline calls it:
//   audiodiffusion/pipeline_audio_diffusion.py:143-147   vqvae.encode(x).latent_dist.sample(generator) * scaling_factor
//   audiodiffusion/pipeline_audio_diffusion.py:187-190   vqvae.decode(1 / scaling_factor * z)["sample"]
// Parameter names are the diffusers state-dict keys that audiodiffusion/utils.py:156-303 (convert_ldm_to_hf_vae) emits.
// The resnets, attention and up/down-samplers run on the same wgmma implicit-GEMM kernel as the U-Net (net.cuh).
#include "net.cuh"

using namespace b200ad;

struct b200ad_vae : NetBase {
  b200ad_vae_config cfg;
  std::vector<Op> enc_plan, dec_plan;
  stat_t* enc_stats = nullptr;
  stat_t* dec_stats = nullptr;
  size_t enc_stats_bytes = 0, dec_stats_bytes = 0;
  float* zq = nullptr;           // post_quant_conv(z), [N][L][h][w]
  int launches = 0;
};

namespace b200ad {

static void p_mid(NetBase* h, const std::string& n, int c) {
  p_resnet(h, n + ".resnets.0", c, c, 0);
  p_attn(h, n + ".attentions.0", c);
  p_resnet(h, n + ".resnets.1", c, c, 0);
}

static void vae_param_table(b200ad_vae* h) {
  const b200ad_vae_config& c = h->cfg;
  const int nb = c.num_blocks, L = c.latent_channels;
  const int* boc = c.block_out_channels;
  p_conv(h, "encoder.conv_in", c.in_channels, boc[0], 3);
  int out_c = boc[0];
  for (int i = 0; i < nb; ++i) {
    const int in_c = out_c;
    out_c = boc[i];
    for (int j = 0; j < c.layers_per_block; ++j)
      p_resnet(h, S("encoder.down_blocks.%d.resnets.%d", i, j), j == 0 ? in_c : out_c, out_c, 0);
    if (i != nb - 1) p_conv(h, S("encoder.down_blocks.%d.downsamplers.0.conv", i), out_c, out_c, 3);
  }
  p_mid(h, "encoder.mid_block", boc[nb - 1]);
  p_gn(h, "encoder.conv_norm_out", boc[nb - 1]);
  p_conv(h, "encoder.conv_out", boc[nb - 1], 2 * L, 3);
  p_conv(h, "quant_conv", 2 * L, 2 * L, 1);
  p_conv(h, "post_quant_conv", L, L, 1);
  p_conv(h, "decoder.conv_in", L, boc[nb - 1], 3);
  p_mid(h, "decoder.mid_block", boc[nb - 1]);
  out_c = boc[nb - 1];
  for (int i = 0; i < nb; ++i) {
    const int prev = out_c;
    out_c = boc[nb - 1 - i];
    for (int j = 0; j < c.layers_per_block + 1; ++j)
      p_resnet(h, S("decoder.up_blocks.%d.resnets.%d", i, j), j == 0 ? prev : out_c, out_c, 0);
    if (i != nb - 1) p_conv(h, S("decoder.up_blocks.%d.upsamplers.0.conv", i), out_c, out_c, 3);
  }
  p_gn(h, "decoder.conv_norm_out", boc[0]);
  p_conv(h, "decoder.conv_out", boc[0], c.out_channels, 3);
}

// Downsample2D(padding=0): F.pad(x, (0,1,0,1)) then a stride-2 3x3 conv without padding, i.e.
// out[y][x] = sum w[kh][kw] * in[2y+kh][2x+kw].  On parity plane (a, b)[y][x] = in[2y+a][2x+b] that is the taps with
// kh % 2 == a, kw % 2 == b read at row offset kh / 2, column offset kw / 2.
static PackTaps taps_parity_asym(int a, int b) {
  PackTaps t{};
  t.ntaps = 0;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw)
      if ((kh & 1) == a && (kw & 1) == b) { t.kh[t.ntaps] = kh; t.kw[t.ntaps] = kw; ++t.ntaps; }
  return t;
}

static void layout_mid(NetBase* h, Bump& b, const std::string& n, int c) {
  layout_resnet(h, b, n + ".resnets.0", c, 0, c, false);
  layout_attn(h, b, n + ".attentions.0", c);
  layout_resnet(h, b, n + ".resnets.1", c, 0, c, false);
}

static void vae_packed_layout(b200ad_vae* h) {
  const b200ad_vae_config& c = h->cfg;
  const int nb = c.num_blocks;
  const int* boc = c.block_out_channels;
  Bump b;
  h->jobs.clear();
  h->ident_off.clear();
  int out_c = boc[0];
  for (int i = 0; i < nb; ++i) {
    const int in_c = out_c;
    out_c = boc[i];
    for (int j = 0; j < c.layers_per_block; ++j)
      layout_resnet(h, b, S("encoder.down_blocks.%d.resnets.%d", i, j), j == 0 ? in_c : out_c, 0, out_c, false);
    if (i != nb - 1) {
      const std::string n = S("encoder.down_blocks.%d.downsamplers.0.conv", i);
      for (int a = 0; a < 2; ++a)
        for (int bb = 0; bb < 2; ++bb)
          add_job(h, b, n + S("#%d", a * 2 + bb), n + ".weight", out_c, out_c, 3, 0, out_c, taps_parity_asym(a, bb));
    }
  }
  layout_mid(h, b, "encoder.mid_block", boc[nb - 1]);
  // encoder.conv_out: 2L output channels zero-padded to one 128-channel tile of the tensor-core kernel
  add_job(h, b, "encoder.conv_out#0", "encoder.conv_out.weight", 128, boc[nb - 1], 3, 0, boc[nb - 1], taps_3x3());
  h->jobs.back().cout_real = 2 * c.latent_channels;
  h->misc_off["encoder.conv_out.bias_pad"] = take_off(b, 128 * 4);
  layout_mid(h, b, "decoder.mid_block", boc[nb - 1]);
  out_c = boc[nb - 1];
  for (int i = 0; i < nb; ++i) {
    const int prev = out_c;
    out_c = boc[nb - 1 - i];
    for (int j = 0; j < c.layers_per_block + 1; ++j)
      layout_resnet(h, b, S("decoder.up_blocks.%d.resnets.%d", i, j), j == 0 ? prev : out_c, 0, out_c, false);
    if (i != nb - 1) {
      const std::string nm = S("decoder.up_blocks.%d.upsamplers.0.conv", i);
      for (int pa = 0; pa < 2; ++pa)
        for (int pb = 0; pb < 2; ++pb)
          add_job(h, b, nm + S("#p%d", pa * 2 + pb), nm + ".weight", out_c, out_c, 3, 0, out_c, taps_up2(pa, pb).pack);
    }
  }
  h->packed_bytes = (b.off + 255) & ~(size_t)255;
}

static void set_taps_explicit(ConvSeg& s, int ntaps, const signed char* dh, const signed char* dw) {
  s.ntaps = ntaps;
  s.ht = s.hb = s.hl = s.hr = 0;
  for (int t = 0; t < ntaps; ++t) {
    s.dh[t] = dh[t]; s.dw[t] = dw[t];
    if (dh[t] < 0) s.ht = 1;
    if (dh[t] > 0) s.hb = 1;
    if (dw[t] < 0) s.hl = 1;
    if (dw[t] > 0) s.hr = 1;
  }
}

// Transient activations ping-pong between two pooled buffers per (C, H, W): every block reads its input from one and
// writes its output to the other (the shortcut K-segment re-reads the input while the output is being written).
struct PingPong {
  int flip = 0;
  std::string operator()() { return (flip++ & 1) ? "pp1" : "pp0"; }
};

static Act build_mid(Builder& B, PingPong& tag, const std::string& n, Act x, int c) {
  x = B.resnet(n + ".resnets.0", x, nullptr, c, true, tag());
  x = B.attention(n + ".attentions.0", x, true, tag());
  return B.resnet(n + ".resnets.1", x, nullptr, c, true, tag());
}

// Builds both plans (encoder, then decoder) into one workspace. Layout: [enc stats | dec stats | activations ...].
static int vae_build_plan(b200ad_vae* h, uint8_t* ws_base, int N, int H, int W, size_t* ws_bytes_out) {
  const b200ad_vae_config& c = h->cfg;
  const int nb = c.num_blocks, L = c.latent_channels;
  const int* boc = c.block_out_channels;
  const int f = 1 << (nb - 1);
  const int lh = H / f, lw = W / f;
  std::vector<Op> enc, dec;
  Builder B;
  B.h = h; B.N = N;
  B.single_head = true;
  {
    const char* e = getenv("B200AD_DEBUG_NOPOOL");
    B.nopool = e && e[0] == '1';
  }
  B.ws.base = ws_base;
  size_t enc_sb = 0, dec_sb = 0;
  for (int pass = 0; pass < 2; ++pass) {
    enc.clear(); dec.clear();
    B.pool.clear();
    h->taps.clear();
    B.st.off = 0;
    B.st.base = pass == 0 ? nullptr : ws_base;
    B.ws.off = pass == 0 ? 0 : ((enc_sb + dec_sb + 511) & ~(size_t)255);
    // ------------------------------------------------------------------ encoder
    B.plan = &enc;
    int hh = H, ww = W, out_c = boc[0];
    PingPong tag;
    Act x = B.pooled(tag(), out_c, hh, ww, true);
    {
      Op op{};
      op.kind = OP_CONV_IN;
      op.dst = x.p; op.C = out_c; op.H = hh; op.W = ww; op.cin = c.in_channels;
      op.fw = B.P("encoder.conv_in.weight"); op.fb = B.P("encoder.conv_in.bias");
      op.conv.stats = x.stats;
      enc.push_back(op);
    }
    h->taps["encoder.conv_in"] = x;
    for (int i = 0; i < nb; ++i) {
      out_c = boc[i];
      for (int j = 0; j < c.layers_per_block; ++j)
        x = B.resnet(S("encoder.down_blocks.%d.resnets.%d", i, j), x, nullptr, out_c, true, tag());
      if (i != nb - 1) {
        const std::string n = S("encoder.down_blocks.%d.downsamplers.0.conv", i);
        const int Ho = hh / 2, Wo = ww / 2;
        const Geom go = make_geom(N, Ho, Wo);
        const size_t tsz = (size_t)N * (out_c / 8) * go.PL * 8;
        Act par = B.pooled("parity", 4 * out_c, Ho, Wo, false);
        {
          Op op{};
          op.kind = OP_PARITY;
          op.src = x.p; op.dst = par.p; op.C = out_c; op.H = hh; op.W = ww;
          enc.push_back(op);
        }
        Act y = B.pooled(tag(), out_c, Ho, Wo, true);
        {
          Op op{};
          op.kind = OP_CONV;
          ConvParams& p = op.conv;
          B.conv_common(p, y);
          p.nseg = 4;
          for (int a = 0; a < 2; ++a)
            for (int b = 0; b < 2; ++b) {
              const PackTaps pt = taps_parity_asym(a, b);
              ConvSeg& sg = p.seg[a * 2 + b];
              B.set_seg(sg, par.p + (size_t)(a * 2 + b) * tsz, out_c, Ho, Wo, B.WP(n + S("#%d", a * 2 + b)), pt);
              signed char dh[9], dw[9];
              for (int t = 0; t < pt.ntaps; ++t) { dh[t] = (signed char)(pt.kh[t] >> 1); dw[t] = (signed char)(pt.kw[t] >> 1); }
              set_taps_explicit(sg, pt.ntaps, dh, dw);
            }
          p.bias = B.P(n + ".bias");
          p.temb = nullptr; p.temb_stride = 0;
          enc.push_back(op);
        }
        h->taps[n] = y;
        x = y;
        hh = Ho; ww = Wo;
      }
    }
    x = build_mid(B, tag, "encoder.mid_block", x, out_c);
    Act eo = B.pooled("enc_out", 128, hh, ww, false);
    {
      const float2* ss = B.gn_finalize(x, nullptr, "encoder.conv_norm_out");
      Op op{};
      op.kind = OP_CONV;
      ConvParams& p = op.conv;
      B.conv_common(p, eo);
      p.nseg = 1;
      B.set_seg(p.seg[0], x.p, x.C, hh, ww, B.WP("encoder.conv_out#0"), taps_3x3());
      Builder::seg_norm(p.seg[0], ss, x.C, true);
      p.bias = B.MISC("encoder.conv_out.bias_pad");
      p.temb = nullptr; p.temb_stride = 0; p.stats = nullptr;
      enc.push_back(op);
    }
    h->taps["encoder.conv_out"] = eo;
    {
      Op op{};
      op.kind = OP_VAE_SAMPLE;
      op.src = eo.p; op.C = 128; op.H = hh; op.W = ww;
      op.fw = B.P("quant_conv.weight"); op.fb = B.P("quant_conv.bias");
      enc.push_back(op);
    }
    if (pass == 0) enc_sb = (B.st.off + 255) & ~(size_t)255;
    // ------------------------------------------------------------------ decoder
    B.plan = &dec;
    B.st.base = (pass == 1 && ws_base) ? ws_base + enc_sb : nullptr;
    B.st.off = 0;
    h->zq = (float*)B.ws.take((size_t)N * L * lh * lw * 4);
    {
      Op op{};
      op.kind = OP_MIX1X1;
      op.f0 = h->zq; op.C = L; op.H = lh; op.W = lw;
      op.fw = B.P("post_quant_conv.weight"); op.fb = B.P("post_quant_conv.bias");
      dec.push_back(op);
    }
    hh = lh; ww = lw; out_c = boc[nb - 1];
    x = B.pooled(tag(), out_c, hh, ww, true);
    {
      Op op{};
      op.kind = OP_CONV_IN;
      op.dst = x.p; op.C = out_c; op.H = hh; op.W = ww; op.cin = L;
      op.f0 = h->zq;  // reads post_quant_conv(z), not the caller's tensor
      op.fw = B.P("decoder.conv_in.weight"); op.fb = B.P("decoder.conv_in.bias");
      op.conv.stats = x.stats;
      dec.push_back(op);
    }
    h->taps["decoder.conv_in"] = x;
    x = build_mid(B, tag, "decoder.mid_block", x, out_c);
    for (int i = 0; i < nb; ++i) {
      out_c = boc[nb - 1 - i];
      for (int j = 0; j < c.layers_per_block + 1; ++j)
        x = B.resnet(S("decoder.up_blocks.%d.resnets.%d", i, j), x, nullptr, out_c, true, tag());
      if (i != nb - 1) {
        const std::string nm = S("decoder.up_blocks.%d.upsamplers.0.conv", i);
        Act y = B.pooled(tag(), out_c, hh * 2, ww * 2, true);
        for (int pa = 0; pa < 2; ++pa)
          for (int pb = 0; pb < 2; ++pb) {
            const UpTaps ut = taps_up2(pa, pb);
            Op op{};
            op.kind = OP_CONV;
            ConvParams& p = op.conv;
            Act lo = y;
            lo.H = hh; lo.W = ww;
            B.conv_common(p, lo);
            p.up2 = 1; p.oy = pa; p.ox = pb;
            p.nseg = 1;
            B.set_seg(p.seg[0], x.p, out_c, hh, ww, B.WP(nm + S("#p%d", pa * 2 + pb)), ut.pack);
            set_taps_explicit(p.seg[0], 4, ut.dh, ut.dw);
            p.bias = B.P(nm + ".bias");
            p.temb = nullptr; p.temb_stride = 0;
            dec.push_back(op);
          }
        hh *= 2; ww *= 2;
        h->taps[nm] = y;
        x = y;
      }
    }
    {
      Op op{};
      op.kind = OP_CONV_OUT;
      ConvOutParams& p = op.co;
      p.src = x.p; p.stats = x.stats;
      p.ss = B.gn_attach(x, "decoder.conv_norm_out");
      p.gamma = B.P("decoder.conv_norm_out.weight"); p.beta = B.P("decoder.conv_norm_out.bias");
      p.w = B.P("decoder.conv_out.weight"); p.b = B.P("decoder.conv_out.bias");
      p.N = N; p.C = x.C; p.H = hh; p.W = ww; p.cout = c.out_channels; p.groups = c.norm_num_groups; p.eps = c.norm_eps;
      dec.push_back(op);
    }
    if (pass == 0) dec_sb = (B.st.off + 255) & ~(size_t)255;
  }
  if (ws_bytes_out) *ws_bytes_out = (B.ws.off + 255) & ~(size_t)255;
  if (ws_base) {
    h->enc_plan = enc; h->dec_plan = dec;
    h->enc_stats = (stat_t*)ws_base; h->enc_stats_bytes = enc_sb;
    h->dec_stats = (stat_t*)(ws_base + enc_sb); h->dec_stats_bytes = dec_sb;
  }
  return 0;
}

static int vae_run(b200ad_vae* h, std::vector<Op>& plan, const float* in, const float* noise, float* out, float* moments,
                   cudaStream_t st) {
  const b200ad_vae_config& c = h->cfg;
  int launches = 0;
  for (Op& op : plan) {
    switch (op.kind) {
      case OP_CONV_IN:
        CK(launch_conv_in(op.f0 ? op.f0 : in, op.fw, op.fb, h->N, op.cin, op.H, op.W, op.C, op.dst, op.conv.stats, st));
        break;
      case OP_GN: CK(launch_gn_finalize(op.gn, op.ss, st)); break;
      case OP_GNAPPLY: CK(launch_gn_apply(op.gn, st)); break;
      case OP_CONV: CK(launch_conv_tc(op.conv, h->num_sms, st)); break;
      case OP_PARITY: CK(launch_parity_split(op.src, op.dst, h->N, op.C, op.H, op.W, st)); break;
      case OP_ATTN1:
        CK(launch_attention_1head(op.src, op.dst, op.f0, h->N, op.C, op.H, op.W, st));
        launches += 2;
        break;
      case OP_VAE_SAMPLE:
        CK(launch_vae_sample(op.src, op.fw, op.fb, noise, out, moments, h->N, op.C, c.latent_channels,
                             op.H, op.W, st));
        break;
      case OP_MIX1X1: CK(launch_mix1x1(in, op.fw, op.fb, op.f0, h->N, op.C, op.H * op.W, st)); break;
      case OP_CONV_OUT: {
        ConvOutParams p = op.co;
        p.eps_out = out;
        p.x = nullptr; p.z = nullptr; p.x_out = nullptr;
        CK(launch_conv_out(p, st));
        break;
      }
      default: return set_err("vae plan: unexpected op kind %d", (int)op.kind);
    }
    ++launches;
  }
  h->launches = launches;
  return 0;
}

}  // namespace b200ad

// ================================================================================= C ABI: AutoencoderKL
extern "C" int b200ad_vae_create(const b200ad_vae_config* cfg, b200ad_vae** out) {
  if (!cfg || !out) return set_err("null argument");
  if (cfg->num_blocks < 1 || cfg->num_blocks > B200AD_MAX_BLOCKS) return set_err("num_blocks out of range");
  for (int i = 0; i < cfg->num_blocks; ++i)
    if (cfg->block_out_channels[i] % 128) return set_err("block_out_channels must be multiples of 128");
  if (cfg->latent_channels < 1 || cfg->latent_channels > 4) return set_err("latent_channels must be 1..4");
  if (cfg->out_channels > 4) return set_err("out_channels > 4 not implemented");
  if (const char* e = check_groups(cfg->block_out_channels, cfg->num_blocks, cfg->norm_num_groups)) return set_err("%s", e);
  b200ad_vae* h = new b200ad_vae();
  h->cfg = *cfg;
  h->norm_groups = cfg->norm_num_groups;
  h->norm_eps = cfg->norm_eps;
  vae_param_table(h);
  vae_packed_layout(h);
  h->pptr.assign(h->params.size(), nullptr);
  *out = h;
  return 0;
}
extern "C" void b200ad_vae_destroy(b200ad_vae* h) { delete h; }
extern "C" int b200ad_vae_num_params(const b200ad_vae* h) { return (int)h->params.size(); }
extern "C" const char* b200ad_vae_param_name(const b200ad_vae* h, int i) { return h->params[i].name.c_str(); }
extern "C" int b200ad_vae_param_shape(const b200ad_vae* h, int i, int64_t* dims) {
  const auto& s = h->params[i].shape;
  for (size_t k = 0; k < s.size(); ++k) dims[k] = s[k];
  return (int)s.size();
}
extern "C" size_t b200ad_vae_packed_bytes(const b200ad_vae* h) { return h->packed_bytes; }

extern "C" int b200ad_vae_set_params(b200ad_vae* h, const float* const* params, void* packed, size_t packed_bytes,
                                     void* stream) {
  if (packed_bytes < h->packed_bytes) return set_err("packed buffer too small: %zu < %zu", packed_bytes, h->packed_bytes);
  for (size_t i = 0; i < h->params.size(); ++i) h->pptr[i] = params[i];
  h->packed = (uint8_t*)packed;
  return pack_common(h, (cudaStream_t)stream);
}

extern "C" size_t b200ad_vae_workspace_bytes(const b200ad_vae* hc, int N, int H, int W) {
  b200ad_vae* h = const_cast<b200ad_vae*>(hc);
  auto saved_taps = h->taps;
  float* zq = h->zq;
  size_t bytes = 0;
  vae_build_plan(h, nullptr, N, H, W, &bytes);
  h->taps = saved_taps; h->zq = zq;
  return bytes;
}

extern "C" int b200ad_vae_bind_workspace(b200ad_vae* h, void* workspace, size_t bytes, int N, int H, int W, void* stream) {
  if (!h->packed) return set_err("set_params must be called before bind_workspace");
  const int f = 1 << (h->cfg.num_blocks - 1);
  if (H % f || W % f) return set_err("H and W must be multiples of %d", f);
  size_t need = 0;
  vae_build_plan(h, nullptr, N, H, W, &need);
  if (bytes < need) return set_err("workspace too small: %zu < %zu", bytes, need);
  CK(cudaMemsetAsync(workspace, 0, need, (cudaStream_t)stream));
  vae_build_plan(h, (uint8_t*)workspace, N, H, W, &need);
  h->N = N; h->H = H; h->W = W;
  h->ws = (uint8_t*)workspace; h->ws_bytes = need;
  int dev = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

extern "C" int b200ad_vae_encode(b200ad_vae* h, const float* x, const float* noise, float* z, float* moments, void* stream) {
  if (h->enc_plan.empty()) return set_err("bind_workspace must be called before encode");
  if (!x || !z) return set_err("x and z are required");
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemsetAsync(h->enc_stats, 0, h->enc_stats_bytes, st));
  return vae_run(h, h->enc_plan, x, noise, z, moments, st);
}

extern "C" int b200ad_vae_decode(b200ad_vae* h, const float* z, float* x_out, void* stream) {
  if (h->dec_plan.empty()) return set_err("bind_workspace must be called before decode");
  if (!z || !x_out) return set_err("z and x_out are required");
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemsetAsync(h->dec_stats, 0, h->dec_stats_bytes, st));
  return vae_run(h, h->dec_plan, z, nullptr, x_out, nullptr, st);
}

extern "C" int b200ad_vae_last_launch_count(const b200ad_vae* h) { return h->launches; }

extern "C" int b200ad_vae_debug_tensor(b200ad_vae* h, const char* name, float* dst, int* dims, void* stream) {
  auto it = h->taps.find(name);
  if (it == h->taps.end()) return set_err("unknown tap '%s'", name);
  const Act& a = it->second;
  if (dims) { dims[0] = a.C; dims[1] = a.H; dims[2] = a.W; }
  if (dst) CK(launch_pf8_to_nchw(a.p, dst, h->N, a.C, a.H, a.W, (cudaStream_t)stream));
  return a.C;
}
