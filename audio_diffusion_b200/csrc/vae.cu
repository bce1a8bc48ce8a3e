// Host side of the latent autoencoder: diffusers `AutoencoderKL` in the shape of config/ldm_autoencoder_kl.yaml:18-28
// (ch 128, ch_mult [1,2,4,4], 2 res blocks, z_channels 1), as the pipeline calls it:
//   audiodiffusion/pipeline_audio_diffusion.py:143-147   vqvae.encode(x).latent_dist.sample(generator) * scaling_factor
//   audiodiffusion/pipeline_audio_diffusion.py:187-190   vqvae.decode(1 / scaling_factor * z)["sample"]
// Parameter names are the diffusers state-dict keys that audiodiffusion/utils.py:156-303 (convert_ldm_to_hf_vae) emits.
// The resnets, attention and up/down-samplers run on the same wgmma implicit-GEMM kernel as the U-Net (net.cuh).
#include "vae.cuh"

using namespace b200ad;

namespace b200ad {

// AutoencoderKL as two block lists, h->parts[ENC] and h->parts[DEC].  Transient activations ping-pong between two pooled
// buffers per (C, H, W): every block reads its input from one and writes its output to the other (the shortcut K-segment
// re-reads the input while the output is being written).
static void vae_blocks(b200ad_vae* h) {
  const b200ad_vae_config& c = h->cfg;
  const int nb = c.num_blocks;
  const int* boc = c.block_out_channels;
  int flip = 0;
  auto pp = [&] { return (flip++ & 1) ? "pp1" : "pp0"; };
  auto mid = [&](std::vector<Block>& bl, const std::string& n) {
    const int ch = boc[nb - 1];
    add_block(bl, BK_RESNET, n + ".resnets.0", ch, ch, pp());
    add_block(bl, BK_ATTN, n + ".attentions.0", ch, ch, pp());
    add_block(bl, BK_RESNET, n + ".resnets.1", ch, ch, pp());
  };
  std::vector<Block>& e = h->parts[ENC];
  add_block(e, BK_CONV_IN, "encoder.", c.in_channels, boc[0], pp());
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < c.layers_per_block; ++j)
      add_block(e, BK_RESNET, S("encoder.down_blocks.%d.resnets.%d", i, j), e.back().cout, boc[i], pp());
    if (i != nb - 1) add_block(e, BK_DOWN_ASYM, S("encoder.down_blocks.%d.downsamplers.0.conv", i), boc[i], boc[i], pp());
  }
  mid(e, "encoder.mid_block");
  add_block(e, BK_LATENT_OUT, "encoder.", boc[nb - 1], 2 * c.latent_channels, "");
  std::vector<Block>& d = h->parts[DEC];
  add_block(d, BK_LATENT_IN, "decoder.", c.latent_channels, boc[nb - 1], pp());
  mid(d, "decoder.mid_block");
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < c.layers_per_block + 1; ++j)
      add_block(d, BK_RESNET, S("decoder.up_blocks.%d.resnets.%d", i, j), d.back().cout, boc[nb - 1 - i], pp());
    if (i != nb - 1) add_block(d, BK_UP, S("decoder.up_blocks.%d.upsamplers.0.conv", i), boc[nb - 1 - i], boc[nb - 1 - i], pp());
  }
  add_block(d, BK_CONV_OUT, "decoder.", boc[0], c.out_channels, "");
}

// Builds both plans (encoder, then decoder) into one workspace. Layout: [enc stats | dec stats | activations ...].
Plan vae_build_plan(const b200ad_vae* h, uint8_t* ws_base, int N, int H, int W) {
  const int f = 1 << (h->cfg.num_blocks - 1);
  Plan pl;
  pl.lists.resize(2);
  OpList& enc = pl.lists[ENC];
  OpList& dec = pl.lists[DEC];
  Builder B;
  B.h = h; B.built = &pl; B.N = N;
  B.ckpt = pl.checkpoint = h->training && h->checkpointing;
  B.nopool = debug_nopool() || (h->training && !B.ckpt);
  B.ws.base = ws_base;
  for (int pass = 0; pass < 2; ++pass) {
    enc.ops.clear(); dec.ops.clear();
    B.reset();
    B.st.off = 0;
    B.st.base = pass == 0 ? nullptr : ws_base;
    B.ws.off = pass == 0 ? 0 : ((enc.stats_bytes + dec.stats_bytes + 511) & ~(size_t)255);
    B.ops = &enc.ops; B.H = H; B.W = W;
    B.run(h->parts[ENC], &enc.recompute);
    if (pass == 0) enc.stats_bytes = (B.st.off + 255) & ~(size_t)255;
    B.st.base = (pass == 1 && ws_base) ? ws_base + enc.stats_bytes : nullptr;
    B.st.off = 0;
    B.ops = &dec.ops; B.H = H / f; B.W = W / f;
    B.run(h->parts[DEC], &dec.recompute);
    if (pass == 0) dec.stats_bytes = (B.st.off + 255) & ~(size_t)255;
  }
  enc.stats = (stat_t*)ws_base;
  dec.stats = ws_base ? (stat_t*)(ws_base + enc.stats_bytes) : nullptr;
  pl.ws_bytes = (B.ws.off + 255) & ~(size_t)255;
  return pl;
}

}  // namespace b200ad

// ================================================================================= C ABI: AutoencoderKL
extern "C" int b200ad_vae_create(const b200ad_vae_config* cfg, b200ad_vae** out) {
  if (!cfg || !out) return set_err("null argument");
  if (check_net_config(cfg->num_blocks, cfg->block_out_channels, cfg->out_channels, cfg->norm_num_groups)) return -1;
  if (cfg->latent_channels < 1 || cfg->latent_channels > 4) return set_err("latent_channels must be 1..4");
  b200ad_vae* h = new b200ad_vae();
  h->cfg = *cfg;
  h->nparts = 2;
  h->norm_groups = cfg->norm_num_groups;
  h->norm_eps = cfg->norm_eps;
  h->single_head = true;
  vae_blocks(h);
  Bump b;
  for (const std::vector<Block>& bl : h->parts)
    for (const Block& k : bl) p_block(h, k);
  for (std::vector<Block>& bl : h->parts)
    for (Block& k : bl) layout_block(h, b, k);
  h->packed_bytes = (b.off + 255) & ~(size_t)255;
  h->pptr.assign(h->params.size(), nullptr);
  *out = h;
  return 0;
}
extern "C" void b200ad_vae_destroy(b200ad_vae* h) {
  if (!h) return;
  release_backward(h);
  delete h;
}
extern "C" int b200ad_vae_num_params(const b200ad_vae* h) { return (int)h->params.size(); }
extern "C" const char* b200ad_vae_param_name(const b200ad_vae* h, int i) { return h->params[i].name.c_str(); }
extern "C" int b200ad_vae_param_shape(const b200ad_vae* h, int i, int64_t* dims) { return param_shape(h, i, dims); }
extern "C" size_t b200ad_vae_packed_bytes(const b200ad_vae* h) { return h->packed_bytes; }

extern "C" int b200ad_vae_set_params(b200ad_vae* h, const float* const* params, void* packed, size_t packed_bytes,
                                     void* stream) {
  if (packed_bytes < h->packed_bytes) return set_err("packed buffer too small: %zu < %zu", packed_bytes, h->packed_bytes);
  for (size_t i = 0; i < h->params.size(); ++i) h->pptr[i] = params[i];
  h->packed = (uint8_t*)packed;
  return pack_common(h, (cudaStream_t)stream);
}

extern "C" size_t b200ad_vae_workspace_bytes(const b200ad_vae* h, int N, int H, int W) {
  return vae_build_plan(h, nullptr, N, H, W).ws_bytes;
}

extern "C" int b200ad_vae_bind_workspace(b200ad_vae* h, void* workspace, size_t bytes, int N, int H, int W, void* stream) {
  return bind_workspace(h, vae_build_plan, workspace, bytes, N, H, W, (cudaStream_t)stream);
}

extern "C" int b200ad_vae_encode(b200ad_vae* h, const float* x, const float* noise, float* z, float* moments, void* stream) {
  if (h->plan.lists.empty()) return set_err("bind_workspace must be called before encode");
  if (!x || !z) return set_err("x and z are required");
  RunArgs a;
  a.in = x; a.noise = noise; a.out = z; a.moments = moments;
  return run_ops(h, h->plan.lists[ENC], a, (cudaStream_t)stream, &h->last_launches);
}

extern "C" int b200ad_vae_decode(b200ad_vae* h, const float* z, float* x_out, void* stream) {
  if (h->plan.lists.empty()) return set_err("bind_workspace must be called before decode");
  if (!z || !x_out) return set_err("z and x_out are required");
  RunArgs a;
  a.in = z; a.out = x_out;
  return run_ops(h, h->plan.lists[DEC], a, (cudaStream_t)stream, &h->last_launches);
}

extern "C" int b200ad_vae_last_launch_count(const b200ad_vae* h) { return h->last_launches; }

extern "C" int b200ad_vae_debug_tensor(b200ad_vae* h, const char* name, float* dst, int* dims, void* stream) {
  return debug_tensor(h, name, dst, dims, (cudaStream_t)stream);
}
