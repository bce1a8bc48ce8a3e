// Backward pass of the U-Net (scripts/train_unet.py:259, `accelerator.backward(loss)`): walks UNet2DModel.forward (or
// UNet2DConditionModel.forward) in reverse over the activations the training-mode forward kept (no buffer pooling), and
// fills one flat fp32 buffer with the gradients of all parameters.  The transformer blocks of the conditional model run
// their LayerNorm / GEGLU / cross-attention / multi-head attention backward kernels from cond_bwd.cu.
// The autoencoder (scripts/train_vae.py) walks its decoder and encoder block lists the same way, one backward plan per
// part; its single-head attention, encoder tail and decoder head run the kernels of vae_bwd_kernels.cu.
//   * data gradients of every convolution run on conv_tc_kernel with transposed / mirrored weight packing (stride-2 convs
//     as four scatter launches, the folded upsampling convs as one gather launch over the parity planes of the gradient);
//   * weight gradients run on wgrad_tc_kernel (wgmma, pixels as the reduction dimension, MN-major operands);
//   * GroupNorm(+SiLU), attention core, biases / time embedding, conv_in / conv_out are memory-bound kernels (bwd_kernels.cu).
// This first version materialises the normalised activations for the weight gradients (no fusion yet) — DESIGN.md §6.
#include "bwd_kernels.cuh"
#include "unet.cuh"
#include "vae.cuh"

using namespace b200ad;

namespace b200ad {

struct View {            // channel range of a PF8 tensor
  const __nv_bfloat16* p = nullptr;   // first plane of the view (image 0)
  int C = 0, img_planes = 0, H = 0, W = 0;
};

struct BOp {
  enum Kind { CONV, WGRAD, GNBWD, GNAPPLY, CHANSUM, REDUCE_N, SCATTER, PF8ADD, ATTNBWD, PARITY, UNFOLD, SCALAR_WGRAD, CONVIN,
              FLIP, SUMADD, LIN_IN, LIN_W, SILU_BWD, SILU_FWD, MEMSET,
              LNBWD, GEGLUBWD, XVECBWD, MHABWD, ATTN1BWD, QUANTBWD, LATENTINBWD, NKINDS } kind;
  ConvParams conv;
  WgradDesc wg;
  GnBwdParams gb;
  GnApplyParams ga;
  UnfoldMasks um;
  const __nv_bfloat16* src = nullptr;
  const __nv_bfloat16* src2 = nullptr;
  const __nv_bfloat16* src3 = nullptr;
  __nv_bfloat16* dst = nullptr;
  __nv_bfloat16* dst2 = nullptr;  // bf16 scratch
  const float* f0 = nullptr;
  const float* f1 = nullptr;
  const float* f2 = nullptr;
  float* o0 = nullptr;
  float* o1 = nullptr;
  float* o2 = nullptr;        // scratch (never a parameter gradient)
  int C = 0, H = 0, W = 0, a = 0, b = 0, c = 0, d = 0;
  long long n = 0;
  bool x_is_input = false;    // SCALAR_WGRAD: X = the forward input image passed to backward()
  bool x_is_geps = false;     // X / source = the output gradient passed to backward()
};

struct BwdArgs {              // the per-call inputs of a backward plan
  const float* x = nullptr;   // the forward's input image (SCALAR_WGRAD x_is_input)
  const float* g_eps = nullptr;   // the gradient of the model output (U-Net: eps; autoencoder decoder: the image)
  const float* g_mom = nullptr;   // autoencoder encoder: the gradient of the moments
  float* g_z = nullptr;           // autoencoder decoder: the gradient w.r.t. the latents (written)
};

}  // namespace b200ad

struct Backward {
  std::vector<BOp> ops;
  std::vector<PackJob> jobs;         // transposed weight packs, redone at every backward (the weights move every step)
  std::vector<size_t> goff;          // float offset of every parameter's gradient in the flat buffer
  size_t grad_floats = 0;
  size_t zero_off = 0, zero_floats = 0;   // the slots of the flat buffer this plan writes (zeroed unless accumulating)
  uint8_t* arena = nullptr;
  size_t arena_bytes = 0;
  float* grads = nullptr;
  int launches = 0;
  PackBatch pack_batch;              // one launch for all transposed packs
};

namespace b200ad {

struct BwdBuilder {
  NetBase* h;
  Backward* bw;
  Bump mem;                                   // arena allocator (base == nullptr: size pass)
  std::map<std::string, Act> grad;            // gradient w.r.t. a forward tensor (by tap name)
  std::map<std::string, Act> skipgrad;        // contribution of the skip connection to that gradient
  std::map<std::string, Act> pool;
  int N;
  float* cs = nullptr;                        // [N][maxC] channel sums scratch
  float* gsums = nullptr;                     // GroupNorm backward scratch [N][maxC][2]
  float* gproj = nullptr;                     // U-Net: [N][temb_rows]
  int heads = 8;                              // conditional U-Net: attention heads of the transformer blocks
  bool single_head = false;                   // attention with one head of dim C (the autoencoder) instead of head_dim 8
  // per-sample channel sums produced by the GroupNorm-backward apply pass for the gradient tensor it writes (keyed by that
  // tensor): the producer's bias gradient then is a reduction over N of a [N][C] array instead of a pass over the tensor
  float* csum_arena = nullptr;
  size_t csum_floats = 0, csum_used = 0;
  std::map<const __nv_bfloat16*, float*> csum_of;
  const float* last_cs = nullptr;             // [N][C] sums of the latest bias_grad (the time-embedding rows are read from it)

  Act act_alloc(int C, int H, int W) {
    Act a;
    a.C = C; a.H = H; a.W = W;
    const Geom g = make_geom(N, H, W);
    a.p = (__nv_bfloat16*)mem.take((size_t)N * (C / 8) * g.PL * 16);
    return a;
  }
  Act tmp(const std::string& tag, int C, int H, int W) {
    const std::string key = S("%s:%d:%d:%d", tag.c_str(), C, H, W);
    auto it = pool.find(key);
    if (it == pool.end()) it = pool.emplace(key, act_alloc(C, H, W)).first;
    return it->second;
  }
  const Act& fwd(const std::string& name) const { return h->plan.taps.at(name); }
  Act G(const std::string& name) {            // gradient tensor of a forward activation
    auto it = grad.find(name);
    if (it == grad.end()) {
      const Act& f = fwd(name);
      it = grad.emplace(name, act_alloc(f.C, f.H, f.W)).first;
    }
    return it->second;
  }
  float* PG(const std::string& pname) const {
    return bw->grads ? bw->grads + bw->goff[h->pidx.at(pname)] : nullptr;
  }
  const float* P(const std::string& name) const { return h->pptr[h->pidx.at(name)]; }
  static View view(const Act& a, int c0, int C) {
    View v;
    const Geom g = make_geom(1, a.H, a.W);
    v.p = a.p ? a.p + (long long)(c0 / 8) * g.PL * 8 : nullptr;
    v.C = C; v.img_planes = a.C / 8; v.H = a.H; v.W = a.W;
    return v;
  }
  static View whole(const Act& a) { return view(a, 0, a.C); }

  // ---- transposed weight packing jobs ----------------------------------------------------------------------------
  // GEMM out channels = the layer's input channels [i0, i0 + I) ... the kernel reads W[o][i][kh][kw] with i = co.
  // Returns the packed weights (null in the size pass).
  const __nv_bfloat16* tjob(const std::string& wname, int O, int I, int K, const TapSet& t) {
    PackJob j;
    j.w_param = h->pidx.at(wname);
    j.cout = I; j.cin_total = O; j.KH = K; j.KW = K; j.cin_off = 0; j.ksteps = O / 16;
    j.taps = t.pack;
    j.cout_real = I;
    j.off = take_off(mem, (size_t)(I / 128) * j.ksteps * t.pack.ntaps * CONV_B_TAP);
    bw->jobs.push_back(j);
    return bw->arena ? (const __nv_bfloat16*)(bw->arena + j.off) : nullptr;
  }

  // ---- op emitters ------------------------------------------------------------------------------------------------
  void conv_base(ConvParams& p, const Act& out) {
    const Geom g = make_geom(N, out.H, out.W);
    p = ConvParams{};
    p.N = N; p.H = out.H; p.W = out.W; p.Wp = g.Wp; p.lead = g.lead; p.PL = g.PL;
    p.cout = out.C; p.out = out.p;
  }
  static void seg(ConvSeg& s, const View& src, const __nv_bfloat16* wpack, const TapSet& t) {
    set_seg(s, src.p, src.img_planes, src.C, src.H, src.W, wpack, t);
  }
  // data gradient of a stride-1 KxK conv: out (I channels) = conv^T(gy (O channels))
  void dgrad(const std::string& wname, const View& gy, const Act& out, int K) {
    const TapSet t = taps_mirrored(K);
    BOp op{};
    op.kind = BOp::CONV;
    conv_base(op.conv, out);
    seg(op.conv.seg[0], gy, tjob(wname, gy.C, out.C, K, t), t);
    op.conv.nseg = 1;
    bw->ops.push_back(op);
  }
  // weight gradient of the forward K-segment with tap set t (of ntaps_total taps of the weight) that read `act`
  void wgrad(const View& gy, const View& act, float* dw, int cin_total, int ci_off, int ntaps_total, const TapSet& t) {
    BOp op{};
    op.kind = BOp::WGRAD;
    WgradDesc& d = op.wg;
    d.gy = gy.p; d.act = act.p; d.dw = dw; d.N = N; d.H = gy.H; d.W = gy.W; d.cout = gy.C; d.cin = act.C;
    d.gy_img_planes = gy.img_planes; d.act_img_planes = act.img_planes;
    d.cin_total = cin_total; d.ci_off = ci_off; d.ntaps_total = ntaps_total; d.ntaps = t.pack.ntaps;
    for (int k = 0; k < t.pack.ntaps; ++k) { d.dh[k] = t.dh[k]; d.dw_[k] = t.dw[k]; d.tapidx[k] = t.wtap[k]; }
    bw->ops.push_back(op);
  }
  void wgrad_conv(const View& gy, const View& act, const std::string& wname, int K) {   // plain stride-1 conv
    wgrad(gy, act, PG(wname), act.C, 0, K * K, taps_conv(K));
  }
  // per-channel sums of a gradient -> bias gradient(s); returns the [N][C] scratch (valid until the next chan_sum)
  void bias_grad(const View& g, const std::string& bname, const std::string& bname2 = "") {
    BOp op{};
    auto it = csum_of.find(g.p);
    if (it != csum_of.end() && g.img_planes * 8 == g.C) {     // whole tensor, sums already made by the pass that wrote it
      op.kind = BOp::REDUCE_N;
      op.f0 = it->second; op.o0 = PG(bname); op.o1 = bname2.empty() ? nullptr : PG(bname2); op.C = g.C;
      last_cs = it->second;
      bw->ops.push_back(op);
      return;
    }
    op.kind = BOp::CHANSUM;
    op.src = g.p; op.o0 = cs; op.C = g.C; op.a = g.img_planes; op.H = g.H; op.W = g.W;
    op.o1 = PG(bname);                                        // bias gradient(s) accumulated by the same kernel
    op.f1 = bname2.empty() ? nullptr : PG(bname2);
    last_cs = cs;
    bw->ops.push_back(op);
  }
  Act gn_apply(const std::string& tag, const Act& a, const Act* b, const std::string& norm, bool silu, float eps = -1.f) {
    const int Ct = a.C + (b ? b->C : 0);
    Act out = tmp(tag, Ct, a.H, a.W);
    BOp op{};
    op.kind = BOp::GNAPPLY;
    GnApplyParams& p = op.ga;
    p.src[0] = a.p; p.stats[0] = a.stats; p.C[0] = a.C;
    p.src[1] = b ? b->p : nullptr; p.stats[1] = b ? b->stats : nullptr; p.C[1] = b ? b->C : 0;
    p.gamma = P(norm + ".weight"); p.beta = P(norm + ".bias");
    p.dst = out.p; p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = eps < 0.f ? h->norm_eps : eps;
    p.silu = silu ? 1 : 0;
    bw->ops.push_back(op);
    return out;
  }
  void gn_bwd(const Act& ga, const Act& a, const Act* b, const std::string& norm, bool silu, const Act& d0, const Act* d1,
              const __nv_bfloat16* addS, const __nv_bfloat16* add0, float eps = -1.f) {
    BOp op{};
    op.kind = BOp::GNBWD;
    GnBwdParams& p = op.gb;
    p.ga = ga.p;
    p.src[0] = a.p; p.stats[0] = a.stats; p.C[0] = a.C;
    p.src[1] = b ? b->p : nullptr; p.stats[1] = b ? b->stats : nullptr; p.C[1] = b ? b->C : 0;
    p.gamma = P(norm + ".weight"); p.beta = P(norm + ".bias");
    p.dst[0] = d0.p; p.dst[1] = d1 ? d1->p : nullptr;
    p.addS = addS; p.add0 = add0;
    p.dgamma = PG(norm + ".weight"); p.dbeta = PG(norm + ".bias");
    p.sums = gsums;
    p.csum0 = nullptr;
    const size_t need = (size_t)N * a.C;
    if (csum_used + need <= csum_floats) {
      p.csum0 = csum_arena ? csum_arena + csum_used : nullptr;
      csum_of[d0.p] = p.csum0;
      csum_used += need;
      if (!csum_arena) csum_of[d0.p] = (float*)1;             // size pass: the plan must have the same shape as the real one
    }
    p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = eps < 0.f ? h->norm_eps : eps; p.silu = silu ? 1 : 0;
    bw->ops.push_back(op);
  }
  const __nv_bfloat16* skip_of(const std::string& name) const {
    auto it = skipgrad.find(name);
    return it == skipgrad.end() ? nullptr : it->second.p;
  }

  // ---- blocks -----------------------------------------------------------------------------------------------------
  // ResnetBlock2D n over cat(a, b): consumes G(n), produces G(a) and (if b) the skip contribution of b.
  void resnet_bwd(const Block& k, const std::string& an, const std::string& bn) {
    const std::string& n = k.name;
    const Act a = fwd(an);
    const bool has_b = !bn.empty();
    Act bsrc;
    if (has_b) bsrc = fwd(bn);
    const Act h1 = fwd(n + ".h1"), out = fwd(n);
    const int co = out.C, Ct = a.C + (has_b ? bsrc.C : 0), H = out.H, W = out.W;
    const Act Gout = G(n);
    // conv2
    Act T1 = tmp("T1", co, H, W);
    dgrad(n + ".conv2.weight", whole(Gout), T1, 3);
    Act A = gn_apply("A", h1, nullptr, n + ".norm2", true);
    wgrad_conv(whole(Gout), whole(A), n + ".conv2.weight", 3);
    const bool sc = Ct != co;
    bias_grad(whole(Gout), n + ".conv2.bias", sc ? n + ".conv_shortcut.bias" : "");
    // norm2 + SiLU
    Act Gh1 = tmp("Gh1", co, H, W);
    gn_bwd(T1, h1, nullptr, n + ".norm2", true, Gh1, nullptr, nullptr, nullptr);
    // conv1 bias + time embedding projection rows of this block
    bias_grad(whole(Gh1), n + ".conv1.bias");
    if (k.temb_row >= 0) {
      BOp op{};
      op.kind = BOp::SCATTER;
      op.f0 = last_cs; op.o0 = gproj; op.C = co; op.a = h->temb_rows; op.b = k.temb_row;
      bw->ops.push_back(op);
    }
    // conv1
    Act T2 = tmp("T2", Ct, H, W);
    dgrad(n + ".conv1.weight", whole(Gh1), T2, 3);
    Act A2 = gn_apply("A2", a, has_b ? &bsrc : nullptr, n + ".norm1", true);
    wgrad_conv(whole(Gh1), whole(A2), n + ".conv1.weight", 3);
    // shortcut
    const __nv_bfloat16* addS;
    if (sc) {
      Act T3 = tmp("T3", Ct, H, W);
      dgrad(n + ".conv_shortcut.weight", whole(Gout), T3, 1);
      wgrad(whole(Gout), whole(a), PG(n + ".conv_shortcut.weight"), Ct, 0, 1, taps_conv(1));
      if (has_b) wgrad(whole(Gout), whole(bsrc), PG(n + ".conv_shortcut.weight"), Ct, a.C, 1, taps_conv(1));
      addS = T3.p;
    } else {
      addS = Gout.p;
    }
    // norm1 + SiLU over the concatenation: gradient of a (plus its skip contribution, if it is a skip tensor) and of b
    Act Ga = G(an);
    Act Gb;
    if (has_b) {
      Gb = act_alloc(bsrc.C, H, W);
      skipgrad[bn] = Gb;
    }
    gn_bwd(T2, a, has_b ? &bsrc : nullptr, n + ".norm1", true, Ga, has_b ? &Gb : nullptr, addS, skip_of(an));
  }

  void attention_bwd(const std::string& n, const std::string& xn) {
    const Act x = fwd(xn), qkv = fwd(n + ".qkv"), ao = fwd(n + ".ao");
    const int C = x.C, H = x.H, W = x.W;
    const Act Gout = G(n);
    Act T1 = tmp("T1", C, H, W);
    dgrad(n + ".to_out.0.weight", whole(Gout), T1, 1);
    wgrad_conv(whole(Gout), whole(ao), n + ".to_out.0.weight", 1);
    bias_grad(whole(Gout), n + ".to_out.0.bias");
    Act Gqkv = tmp("Gqkv", 3 * C, H, W);
    if (single_head) {   // the forward's softmax P is kept: four GEMMs on the tensor cores
      const long long S = (long long)H * W;
      BOp op{};
      op.kind = BOp::ATTN1BWD;
      op.src = qkv.p; op.src2 = T1.p; op.src3 = ao.p; op.dst = Gqkv.p; op.f0 = h->plan.probs.at(n);
      op.o2 = (float*)mem.take((size_t)N * S * sizeof(float));
      op.dst2 = (__nv_bfloat16*)mem.take((size_t)N * S * S * sizeof(__nv_bfloat16));
      op.C = C; op.H = H; op.W = W;
      bw->ops.push_back(op);
    } else {
      BOp op{};
      op.kind = BOp::ATTNBWD;
      op.src = qkv.p; op.src2 = T1.p; op.dst = Gqkv.p; op.C = C; op.H = H; op.W = W;
      bw->ops.push_back(op);
    }
    Act XN = gn_apply("A", x, nullptr, n + ".group_norm", false);
    const char* names[3] = {"to_q", "to_k", "to_v"};
    for (int k = 0; k < 3; ++k) {
      const View gv = view(Gqkv, k * C, C);
      wgrad_conv(gv, whole(XN), n + "." + names[k] + ".weight", 1);
      bias_grad(gv, n + "." + names[k] + ".bias");
    }
    // g(norm(x)) = sum over q, k, v of W^T g: one launch, three K-segments
    Act T2 = tmp("T2", C, H, W);
    {
      BOp op{};
      op.kind = BOp::CONV;
      conv_base(op.conv, T2);
      const TapSet t = taps_mirrored(1);
      for (int k = 0; k < 3; ++k)
        seg(op.conv.seg[k], view(Gqkv, k * C, C), tjob(n + "." + names[k] + ".weight", C, C, 1, t), t);
      op.conv.nseg = 3;
      bw->ops.push_back(op);
    }
    gn_bwd(T2, x, nullptr, n + ".group_norm", false, G(xn), nullptr, Gout.p, skip_of(xn));
  }

  // LayerNorm over channels (eps 1e-5, as the forward): gx = LN-backward(gy; x) + add, gamma / beta gradients
  void layer_norm_bwd(const Act& gy, const Act& x, const std::string& norm, const Act& gx, const Act& add) {
    BOp op{};
    op.kind = BOp::LNBWD;
    op.src = x.p; op.src2 = gy.p; op.src3 = add.p; op.dst = gx.p;
    op.f0 = P(norm + ".weight"); op.o0 = PG(norm + ".weight"); op.o1 = PG(norm + ".bias");
    op.C = x.C; op.H = x.H; op.W = x.W;
    bw->ops.push_back(op);
  }

  // Transformer2DModel with one BasicTransformerBlock (Builder::transformer) in reverse, from G(out) to G(x):
  //   h0 = proj_in(GN(x));  h2 = h0 + attn1(LN1(h0)) + vec;  h3 = h2 + ff2(GEGLU(ff1(LN3(h2))));  out = proj_out(h3) + x
  // attn2 over ONE key is the per-sample vector vec = Wo (Wv enc) + bo: its gradient is the per-sample channel sum of G(h2)
  // (the sums the attn1.to_out bias gradient makes).  attn2.to_q, attn2.to_k and norm2 do not reach the output (softmax
  // over one key is 1), so their gradients stay exactly zero: nothing is launched for them.
  void transformer_bwd(const Block& k, const std::string& xn) {
    const std::string& n = k.name;
    const std::string t = n + ".transformer_blocks.0";
    const Act x = fwd(xn), h0 = fwd(n + ".h0"), n1 = fwd(n + ".n1"), qkv = fwd(n + ".qkv"), ao = fwd(n + ".ao"),
              h2 = fwd(n + ".attn2"), n3 = fwd(n + ".n3"), ff1 = fwd(n + ".ff1"), gg = fwd(n + ".gg"), h3 = fwd(n + ".h3");
    const int C = x.C, H = x.H, W = x.W;
    const Act Gout = G(n);
    // proj_out (its residual, G(x) += G(out), is added by the GroupNorm backward at the end)
    Act Gh3 = tmp("tf_Gh3", C, H, W);
    dgrad(n + ".proj_out.weight", whole(Gout), Gh3, 1);
    wgrad_conv(whole(Gout), whole(h3), n + ".proj_out.weight", 1);
    bias_grad(whole(Gout), n + ".proj_out.bias");
    // ff.net.2 (+ residual h2)
    Act Ggg = tmp("tf_Ggg", 4 * C, H, W);
    dgrad(t + ".ff.net.2.weight", whole(Gh3), Ggg, 1);
    wgrad_conv(whole(Gh3), whole(gg), t + ".ff.net.2.weight", 1);
    bias_grad(whole(Gh3), t + ".ff.net.2.bias");
    // GEGLU
    Act Gff1 = tmp("tf_Gff1", 8 * C, H, W);
    {
      BOp op{};
      op.kind = BOp::GEGLUBWD;
      op.src = ff1.p; op.src2 = Ggg.p; op.dst = Gff1.p; op.C = 4 * C; op.H = H; op.W = W;
      bw->ops.push_back(op);
    }
    // ff.net.0.proj
    Act Gn = tmp("tf_Gn", C, H, W);
    dgrad(t + ".ff.net.0.proj.weight", whole(Gff1), Gn, 1);
    wgrad_conv(whole(Gff1), whole(n3), t + ".ff.net.0.proj.weight", 1);
    bias_grad(whole(Gff1), t + ".ff.net.0.proj.bias");
    // norm3 (+ residual) -> G(h2)
    Act Gh2 = tmp("tf_Gh2", C, H, W);
    layer_norm_bwd(Gn, h2, t + ".norm3", Gh2, Gh3);
    // attn1.to_out and attn2.to_out both add their bias to every pixel of h2: one channel sum gives both bias gradients
    Act Gao = tmp("tf_Gao", C, H, W);
    dgrad(t + ".attn1.to_out.0.weight", whole(Gh2), Gao, 1);
    wgrad_conv(whole(Gh2), whole(ao), t + ".attn1.to_out.0.weight", 1);
    bias_grad(whole(Gh2), t + ".attn1.to_out.0.bias", t + ".attn2.to_out.0.bias");
    {
      BOp op{};
      op.kind = BOp::XVECBWD;   // dvec[n] = per-sample channel sums of G(h2) (last_cs, made just above)
      op.f0 = last_cs; op.f1 = P(t + ".attn2.to_v.weight"); op.f2 = P(t + ".attn2.to_out.0.weight");
      op.o0 = PG(t + ".attn2.to_out.0.weight"); op.o1 = PG(t + ".attn2.to_v.weight");
      op.o2 = (float*)mem.take((size_t)2 * N * C * sizeof(float));
      op.C = C; op.a = k.cross;
      bw->ops.push_back(op);
    }
    // attention core (P recomputed from the forward's row log-sum-exp)
    Act Gqkv = tmp("tf_Gqkv", 3 * C, H, W);
    {
      BOp op{};
      op.kind = BOp::MHABWD;
      op.src = qkv.p; op.src2 = Gao.p; op.src3 = ao.p; op.dst = Gqkv.p;
      op.f0 = h->plan.lse.at(n);
      op.o2 = (float*)mem.take((size_t)N * heads * H * W * sizeof(float));
      op.C = C; op.H = H; op.W = W; op.a = heads;
      bw->ops.push_back(op);
    }
    // q / k / v projections (no bias); g(n1) = sum over q, k, v of W^T g: one launch, three K-segments
    const char* names[3] = {"to_q", "to_k", "to_v"};
    for (int j = 0; j < 3; ++j) wgrad_conv(view(Gqkv, j * C, C), whole(n1), t + ".attn1." + names[j] + ".weight", 1);
    {
      BOp op{};
      op.kind = BOp::CONV;
      conv_base(op.conv, Gn);
      const TapSet ts = taps_mirrored(1);
      for (int j = 0; j < 3; ++j)
        seg(op.conv.seg[j], view(Gqkv, j * C, C), tjob(t + ".attn1." + names[j] + ".weight", C, C, 1, ts), ts);
      op.conv.nseg = 3;
      bw->ops.push_back(op);
    }
    // norm1 (+ residual) -> G(h0)
    Act Gh0 = tmp("tf_Gh0", C, H, W);
    layer_norm_bwd(Gn, h0, t + ".norm1", Gh0, Gh2);
    // proj_in over GroupNorm(x) (eps 1e-6, no SiLU), then the GroupNorm backward with the outer residual G(out)
    Act T = tmp("tf_T", C, H, W);
    dgrad(n + ".proj_in.weight", whole(Gh0), T, 1);
    Act XN = gn_apply("A", x, nullptr, n + ".norm", false, 1e-6f);
    wgrad_conv(whole(Gh0), whole(XN), n + ".proj_in.weight", 1);
    bias_grad(whole(Gh0), n + ".proj_in.bias");
    gn_bwd(T, x, nullptr, n + ".norm", false, G(xn), nullptr, Gout.p, skip_of(xn), 1e-6f);
  }

  // Downsample2D (BK_DOWN: padding 1; BK_DOWN_ASYM: padding (0, 1, 0, 1)): stride-2 3x3 conv on the raw tensor xn -> y
  void downsample_bwd(const Block& k, const std::string& xn) {
    const std::string& n = k.name;
    const Act x = fwd(xn), y = fwd(n), par = fwd(n + ".parity");
    const int C = x.C, Ho = y.H, Wo = y.W;
    const Act Gy = G(n);
    const Geom go = make_geom(N, Ho, Wo);
    const size_t tsz = (size_t)N * (C / 8) * go.PL * 8;
    bias_grad(whole(Gy), n + ".bias");
    // weight gradient: per parity plane (a, b) of x the taps that read it (forward: down_taps)
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        Act plane = par;
        plane.C = C; plane.H = Ho; plane.W = Wo;
        plane.p = par.p ? par.p + (size_t)(a * 2 + b) * tsz : nullptr;
        wgrad(whole(Gy), whole(plane), PG(n + ".weight"), C, 0, 9, down_taps(k, a, b));
      }
    // data gradient: input parity (a, b) <- taps with matching parity, scattered into the 2x tensor
    Act Gx = G(xn);
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const TapSet t = k.kind == BK_DOWN ? taps_scatter2(a, b) : taps_scatter2_asym(a, b);
        BOp op{};
        op.kind = BOp::CONV;
        Act lo = Gx;
        lo.H = Ho; lo.W = Wo;
        conv_base(op.conv, lo);
        op.conv.up2 = 1; op.conv.oy = a; op.conv.ox = b;
        seg(op.conv.seg[0], whole(Gy), tjob(n + ".weight", C, C, 3, t), t);
        op.conv.nseg = 1;
        bw->ops.push_back(op);
      }
    if (skipgrad.count(xn)) {
      BOp op{};
      op.kind = BOp::PF8ADD;
      op.dst = Gx.p; op.src = skip_of(xn); op.C = C; op.H = x.H; op.W = x.W;
      bw->ops.push_back(op);
    }
  }

  // Upsample2D folded into four 2x2 convs (forward taps_up2): x (low) -> y (2x)
  void upsample_bwd(const std::string& n, const std::string& xn) {
    const Act x = fwd(xn), y = fwd(n);
    const int C = x.C, H = x.H, W = x.W;
    const Act Gy = G(n);
    bias_grad(whole(Gy), n + ".bias");
    const Geom gl = make_geom(N, H, W);
    const size_t tsz = (size_t)N * (C / 8) * gl.PL * 8;
    Act gpar = tmp("gpar", 4 * C, H, W);          // parity planes of the gradient, 4 tensors back to back
    {
      BOp op{};
      op.kind = BOp::PARITY;
      op.src = Gy.p; op.dst = gpar.p; op.C = C; op.H = y.H; op.W = y.W;
      bw->ops.push_back(op);
    }
    float* dwf = (float*)mem.take((size_t)4 * C * C * 4 * sizeof(float));
    {
      BOp op{};
      op.kind = BOp::MEMSET;
      op.o0 = dwf; op.n = (long long)4 * C * C * 4 * sizeof(float);
      bw->ops.push_back(op);
    }
    BOp dg{};
    dg.kind = BOp::CONV;
    Act Gx = G(xn);
    conv_base(dg.conv, Gx);
    UnfoldMasks um{};
    for (int oy = 0; oy < 2; ++oy)
      for (int ox = 0; ox < 2; ++ox) {
        const int pidx = oy * 2 + ox;
        const TapSet fwd_taps = taps_up2(oy, ox), bwd_taps = taps_up2_neg(oy, ox);
        Act plane;
        plane.C = C; plane.H = H; plane.W = W;
        plane.p = gpar.p ? gpar.p + (size_t)pidx * tsz : nullptr;
        wgrad(whole(plane), whole(x), dwf ? dwf + (size_t)pidx * C * C * 4 : nullptr, C, 0, 4, fwd_taps);
        for (int t = 0; t < 4; ++t) um.mask[pidx][t] = fwd_taps.pack.fold_mask[t];
        seg(dg.conv.seg[pidx], whole(plane), tjob(n + ".weight", C, C, 3, bwd_taps), bwd_taps);
      }
    dg.conv.nseg = 4;
    {
      BOp op{};
      op.kind = BOp::UNFOLD;
      op.f0 = dwf; op.o0 = PG(n + ".weight"); op.n = (long long)C * C; op.um = um;
      bw->ops.push_back(op);
    }
    bw->ops.push_back(dg);
  }

  // conv_norm_out + SiLU + conv_out (C -> 1) on the last activation `in`, from the output gradient passed to backward()
  void conv_out_bwd(const Block& k, const std::string& in, float* wflip, const float* zbias) {
    const Act x = fwd(in);
    const int C = x.C;
    Act A = gn_apply("A", x, nullptr, k.name + "conv_norm_out", true);
    BOp w{};
    w.kind = BOp::SCALAR_WGRAD;
    w.src = A.p; w.x_is_geps = true; w.o0 = PG(k.name + "conv_out.weight"); w.C = C; w.H = x.H; w.W = x.W; w.a = 1;
    bw->ops.push_back(w);
    BOp sb{};
    sb.kind = BOp::SUMADD;
    sb.x_is_geps = true; sb.n = (long long)N * x.H * x.W; sb.o0 = PG(k.name + "conv_out.bias");
    bw->ops.push_back(sb);
    BOp f{};
    f.kind = BOp::FLIP;
    f.f0 = P(k.name + "conv_out.weight"); f.o0 = wflip; f.C = C;
    bw->ops.push_back(f);
    Act T1 = tmp("T1", C, x.H, x.W);
    BOp ci{};
    ci.kind = BOp::CONVIN;        // conv_in kernel: g_a[c] = sum_t g_eps[p + s_t] * wflip[c][t]
    ci.x_is_geps = true; ci.f0 = wflip; ci.f1 = zbias; ci.dst = T1.p; ci.C = C; ci.H = x.H; ci.W = x.W;
    bw->ops.push_back(ci);
    gn_bwd(T1, x, nullptr, k.name + "conv_norm_out", true, G(in), nullptr, nullptr, nullptr);
  }
};

static int build_backward(b200ad_unet* h, Backward* bw, uint8_t* arena, float* grads, size_t* bytes_out) {
  const b200ad_unet_config& c = h->cfg;
  if (!h->training || h->plan.lists.empty()) return set_err("backward needs set_training(1) before bind_workspace");
  bw->ops.clear();
  bw->jobs.clear();
  bw->arena = arena;
  bw->grads = grads;
  BwdBuilder B;
  B.h = h; B.bw = bw; B.N = h->N;
  B.heads = c.attention_head_dim;
  B.mem.base = arena;
  int maxC = c.block_out_channels[0];
  for (const auto& kv : h->plan.taps) maxC = kv.second.C > maxC ? kv.second.C : maxC;
  const int D = c.block_out_channels[0] * 4;
  B.cs = (float*)B.mem.take((size_t)h->N * 3 * maxC * sizeof(float));
  B.gsums = (float*)B.mem.take((size_t)h->N * 3 * maxC * 2 * sizeof(float));
  B.gproj = (float*)B.mem.take((size_t)h->N * h->temb_rows * sizeof(float));
  B.csum_floats = (size_t)h->N * 65536;       // all GroupNorm-backward outputs of the reference architecture: 16 K channels
  B.csum_arena = (float*)B.mem.take(B.csum_floats * sizeof(float));
  {
    BOp z{};
    z.kind = BOp::MEMSET;
    z.o0 = B.csum_arena; z.n = (long long)(B.csum_floats * sizeof(float));
    bw->ops.push_back(z);
  }
  float* g_act = (float*)B.mem.take((size_t)h->N * D * sizeof(float));   // gradient w.r.t. silu(linear_2)
  float* g_h1 = (float*)B.mem.take((size_t)h->N * D * sizeof(float));
  float* h1v = (float*)B.mem.take((size_t)h->N * D * sizeof(float));
  float* wflip = (float*)B.mem.take((size_t)c.block_out_channels[0] * 9 * sizeof(float));
  const float* zbias = (const float*)B.mem.take((size_t)c.block_out_channels[0] * sizeof(float));   // never written: zeros

  // the forward's blocks in reverse; a block's output is the forward tap of its name (the head's: conv_in)
  const std::vector<Block>& bl = h->blocks;
  auto tap = [&](int i) { return i < 0 ? std::string() : bl[i].kind == BK_UNET_HEAD ? bl[i].name + "conv_in" : bl[i].name; };
  for (int i = (int)bl.size() - 1; i >= 0; --i) {
    const Block& k = bl[i];
    const std::string in = tap(k.in);
    switch (k.kind) {
      case BK_CONV_OUT: {    // g_eps -> gradient of the last activation
        if (c.out_channels != 1) return set_err("backward: out_channels != 1 is not implemented");
        B.conv_out_bwd(k, in, wflip, zbias);
        BOp z{};
        z.kind = BOp::MEMSET;
        z.o0 = B.gproj; z.n = (long long)h->N * h->temb_rows * sizeof(float);
        bw->ops.push_back(z);
        break;
      }
      case BK_RESNET: B.resnet_bwd(k, in, tap(k.skip)); break;
      case BK_ATTN: B.attention_bwd(k.name, in); break;
      case BK_TRANSFORMER: B.transformer_bwd(k, in); break;
      case BK_DOWN: B.downsample_bwd(k, in); break;
      case BK_UP: B.upsample_bwd(k.name, in); break;
      case BK_UNET_HEAD: {   // conv_in, then the timestep embedding MLP and the per-resnet projections
        if (c.in_channels != 1) return set_err("backward: in_channels != 1 is not implemented");
        const std::string n = tap(i);
        const Act x = B.fwd(n);
        const Act Gx = B.G(n);
        if (!B.skipgrad.count(n)) return set_err("backward: conv_in skip gradient missing");
        // (the first resnet's GroupNorm backward already added the skip contribution)
        BOp w{};
        w.kind = BOp::SCALAR_WGRAD;
        w.src = Gx.p; w.x_is_input = true; w.o0 = B.PG(n + ".weight"); w.C = x.C; w.H = x.H; w.W = x.W; w.a = 0;
        bw->ops.push_back(w);
        B.bias_grad(BwdBuilder::whole(Gx), n + ".bias");
        const Plan& pl = h->plan;
        for (const Block& r : bl) {     // time_emb_proj of every resnet: dW = g_proj_rows^T temb_act
          if (r.temb_row < 0) continue;
          BOp op{};
          op.kind = BOp::LIN_W;
          op.f0 = B.gproj + r.temb_row; op.a = h->temb_rows; op.f1 = pl.temb_act; op.b = r.cout; op.c = D;
          op.o0 = B.PG(r.name + ".time_emb_proj.weight"); op.o1 = B.PG(r.name + ".time_emb_proj.bias");
          bw->ops.push_back(op);
        }
        BOp gi{};
        gi.kind = BOp::LIN_IN;   // g(temb_act) = g_proj Wcat
        gi.f0 = B.gproj; gi.a = h->temb_rows; gi.f1 = h->packed ? (const float*)(h->packed + h->off_wcat) : nullptr;
        gi.b = h->temb_rows; gi.c = D; gi.o0 = g_act;
        bw->ops.push_back(gi);
        BOp s2{};
        s2.kind = BOp::SILU_BWD;
        s2.o0 = g_act; s2.f0 = pl.temb_u2; s2.n = (long long)h->N * D;
        bw->ops.push_back(s2);
        BOp hf{};
        hf.kind = BOp::SILU_FWD;
        hf.f0 = pl.temb_u1; hf.o0 = h1v; hf.n = (long long)h->N * D;
        bw->ops.push_back(hf);
        BOp w2{};
        w2.kind = BOp::LIN_W;
        w2.f0 = g_act; w2.a = D; w2.f1 = h1v; w2.b = D; w2.c = D;
        w2.o0 = B.PG("time_embedding.linear_2.weight"); w2.o1 = B.PG("time_embedding.linear_2.bias");
        bw->ops.push_back(w2);
        BOp g1{};
        g1.kind = BOp::LIN_IN;
        g1.f0 = g_act; g1.a = D; g1.f1 = B.P("time_embedding.linear_2.weight"); g1.b = D; g1.c = D; g1.o0 = g_h1;
        bw->ops.push_back(g1);
        BOp s1{};
        s1.kind = BOp::SILU_BWD;
        s1.o0 = g_h1; s1.f0 = pl.temb_u1; s1.n = (long long)h->N * D;
        bw->ops.push_back(s1);
        BOp w1{};
        w1.kind = BOp::LIN_W;
        w1.f0 = g_h1; w1.a = D; w1.f1 = pl.temb_emb; w1.b = D; w1.c = k.cout;
        w1.o0 = B.PG("time_embedding.linear_1.weight"); w1.o1 = B.PG("time_embedding.linear_1.bias");
        bw->ops.push_back(w1);
        break;
      }
      default: return set_err("backward: block %s has no backward", k.name.c_str());
    }
  }
  if (bytes_out) *bytes_out = (B.mem.off + 255) & ~(size_t)255;
  return 0;
}

}  // namespace b200ad

namespace b200ad {
void release_backward(b200ad_unet* h) {
  delete h->bwd;
  h->bwd = nullptr;
}
}  // namespace b200ad

// ================================================================================= C ABI
extern "C" int b200ad_unet_set_training(b200ad_unet* h, int on) {
  if (!h) return set_err("null handle");
  if (h->training != (on != 0)) {
    h->training = on != 0;
    h->plan.lists.clear();    // the workspace layout changes: bind_workspace must be called again
  }
  return 0;
}

static void ensure_bwd(b200ad_unet* h) {
  if (h->bwd) return;
  Backward* bw = new Backward();
  size_t off = 0;
  for (const auto& p : h->params) {
    size_t n = 1;
    for (auto d : p.shape) n *= (size_t)d;
    bw->goff.push_back(off);
    off += (n + 63) & ~(size_t)63;
  }
  bw->grad_floats = off;
  bw->zero_floats = off;
  h->bwd = bw;
}

extern "C" size_t b200ad_unet_grad_floats(b200ad_unet* h) { ensure_bwd(h); return h->bwd->grad_floats; }
extern "C" size_t b200ad_unet_grad_offset(b200ad_unet* h, int i) { ensure_bwd(h); return h->bwd->goff[i]; }

extern "C" size_t b200ad_unet_backward_bytes(b200ad_unet* h) {
  ensure_bwd(h);
  Backward tmp;
  tmp.goff = h->bwd->goff;
  size_t bytes = 0;
  if (build_backward(h, &tmp, nullptr, nullptr, &bytes)) return 0;
  return bytes;
}

extern "C" int b200ad_unet_bind_backward(b200ad_unet* h, void* arena, size_t bytes, float* grads, void* stream) {
  ensure_bwd(h);
  size_t need = 0;
  {
    Backward tmp;
    tmp.goff = h->bwd->goff;
    if (build_backward(h, &tmp, nullptr, nullptr, &need)) return -1;
  }
  if (bytes < need) return set_err("backward arena too small: %zu < %zu", bytes, need);
  CK(cudaMemsetAsync(arena, 0, need, (cudaStream_t)stream));
  if (build_backward(h, h->bwd, (uint8_t*)arena, grads, &need)) return -1;
  h->bwd->arena_bytes = need;
  return 0;
}

// Runs a bound backward plan.
static int run_backward(NetBase* h, Backward* bw, const BwdArgs& a, int accumulate, cudaStream_t st) {
  const int N = h->N;
  const float* x = a.x;
  const float* g_eps = a.g_eps;
  int launches = 0;
  // B200AD_BWD_PROFILE=1: CUDA events around every op, per-kind totals printed to stderr (tools/train_bench.py)
  static const bool prof = [] { const char* e = getenv("B200AD_BWD_PROFILE"); return e && e[0] == '1'; }();
  std::vector<cudaEvent_t> ev;
  if (prof) {
    ev.resize(bw->ops.size() + 2);
    for (auto& e : ev) CK(cudaEventCreate(&e));
    CK(cudaEventRecord(ev[0], st));
  }
  if (!accumulate) CK(cudaMemsetAsync(bw->grads + bw->zero_off, 0, bw->zero_floats * sizeof(float), st));   // every kernel below ADDS
  {
    std::vector<PackItem> items;
    items.reserve(bw->jobs.size());
    for (const PackJob& j : bw->jobs) items.push_back(make_pack_item(h, j, bw->arena));
    CK(launch_pack_batch(bw->pack_batch, items, st));
  }
  launches += 1;
  if (prof) CK(cudaEventRecord(ev[1], st));
  size_t opi = 0;
  for (BOp& op : bw->ops) {
    switch (op.kind) {
      case BOp::CONV: CK(launch_conv_tc(op.conv, h->num_sms, st)); break;
      case BOp::WGRAD: CK(launch_wgrad_tc(op.wg, h->num_sms, st)); break;
      case BOp::GNBWD: CK(launch_gn_bwd(op.gb, st)); launches += 1; break;
      case BOp::GNAPPLY: CK(launch_gn_apply(op.ga, st)); break;
      case BOp::CHANSUM:
        CK(launch_chan_sum(op.src, op.o0, N, op.C, op.a, op.H, op.W, st, op.o1, const_cast<float*>(op.f1)));
        break;
      case BOp::REDUCE_N: CK(launch_reduce_n_add(op.f0, op.o0, op.o1, N, op.C, st)); break;
      case BOp::SCATTER: CK(launch_scatter_rows(op.f0, op.o0, N, op.C, op.a, op.b, st)); break;
      case BOp::PF8ADD: CK(launch_pf8_add(op.dst, op.src, N, op.C, op.H, op.W, st)); break;
      case BOp::ATTNBWD: CK(launch_attention_bwd(op.src, op.src2, op.dst, N, op.C, op.H, op.W, st)); break;
      case BOp::PARITY: CK(launch_parity_split(op.src, op.dst, N, op.C, op.H, op.W, st)); break;
      case BOp::UNFOLD: CK(launch_unfold_up2(op.f0, op.o0, op.n, op.um, st)); break;
      case BOp::SCALAR_WGRAD:     // X: f0, or an input of the call
        CK(launch_scalar_conv_wgrad(op.src, op.f0 ? op.f0 : op.x_is_geps ? g_eps : x, op.o0, N, op.C, op.H, op.W, op.a, st));
        break;
      case BOp::CONVIN:           // source: f2 (c channels), or the output gradient (1 channel)
        CK(launch_conv_in(op.f2 ? op.f2 : g_eps, op.f0, op.f1, N, op.c ? op.c : 1, op.H, op.W, op.C, op.dst, nullptr, st));
        break;
      case BOp::FLIP: CK(launch_flip_taps(op.f0, op.o0, op.C, st, op.a ? op.a : 1)); break;
      case BOp::SUMADD: CK(launch_sum_add(op.f0 ? op.f0 : g_eps, op.n, op.o0, st)); break;
      case BOp::LIN_IN: CK(launch_lin_bwd_input(op.f0, op.a, op.f1, op.b, op.c, op.o0, N, 0, st)); break;
      case BOp::LIN_W: CK(launch_lin_bwd_weight(op.f0, op.a, op.f1, op.b, op.c, op.o0, op.o1, N, st)); break;
      case BOp::SILU_BWD: CK(launch_silu_bwd(op.o0, op.f0, (int)op.n, st)); break;
      case BOp::SILU_FWD: CK(launch_silu_fwd(op.f0, op.o0, (int)op.n, st)); break;
      case BOp::MEMSET: CK(cudaMemsetAsync(op.o0, 0, (size_t)op.n, st)); break;
      case BOp::LNBWD:
        CK(launch_layernorm_bwd_pf8(op.src, op.src2, op.src3, op.dst, op.f0, op.o0, op.o1, N, op.C, op.H, op.W, 1e-5f, st));
        break;
      case BOp::GEGLUBWD: CK(launch_geglu_bwd_pf8(op.src, op.src2, op.dst, N, op.C, op.H, op.W, st)); break;
      case BOp::XVECBWD:
        if (!h->enc || h->enc_S != 1) return set_err("backward: the conditional U-Net needs the forward's encoding (S = 1) bound");
        CK(launch_cross_attn_vec_bwd(h->enc, op.f0, op.f1, op.f2, op.o0, op.o1, op.o2, N, op.C, op.a, st));
        launches += 1;
        break;
      case BOp::MHABWD:
        CK(launch_mha_bwd(op.src, op.src3, op.src2, op.f0, op.o2, op.dst, N, op.C, op.a, op.H, op.W, st));
        launches += 2;
        break;
      case BOp::ATTN1BWD:   // row dot products, then the dS, dV, dQ, dK GEMMs
        CK(launch_attention_1head_bwd(op.src, op.src3, op.src2, op.f0, op.o2, op.dst2, op.dst, N, op.C, op.H, op.W, st));
        launches += 4;
        break;
      case BOp::QUANTBWD:
        CK(launch_quant_conv_bwd(a.g_mom, op.src, op.f0, op.o2, op.o2 + (size_t)N * op.c * op.H * op.W, op.o0, op.o1, N,
                                 op.c, op.H, op.W, st));
        break;
      case BOp::LATENTINBWD:
        CK(launch_latent_in_bwd(op.src, op.f0, op.f1, op.f2, a.g_z, op.o0, op.o1, N, op.C, op.c, op.H, op.W, st));
        break;
      case BOp::NKINDS: break;
    }
    ++launches;
    if (prof) CK(cudaEventRecord(ev[2 + opi], st));
    ++opi;
  }
  bw->launches = launches;
  if (prof) {
    static const char* names[BOp::NKINDS] = {
        "conv_tc(dgrad)", "wgrad_tc", "gn_bwd", "gn_apply", "chan_sum", "reduce_n", "scatter", "pf8_add", "attention_bwd",
        "parity_split", "unfold_up2", "scalar_wgrad", "conv_in(dgrad)", "flip", "sum_add", "lin_in", "lin_w", "silu_bwd",
        "silu_fwd", "memset", "layernorm_bwd", "geglu_bwd", "cross_attn_vec_bwd", "mha_bwd", "attention_1head_bwd",
        "quant_conv_bwd", "latent_in_bwd"};
    CK(cudaStreamSynchronize(st));
    double tot[BOp::NKINDS] = {0};
    int cnt[BOp::NKINDS] = {0};
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    fprintf(stderr, "{\"backward_profile_ms\": {\"pack_transposed\": %.3f", ms);
    for (size_t i = 0; i < bw->ops.size(); ++i) {
      CK(cudaEventElapsedTime(&ms, ev[1 + i], ev[2 + i]));
      tot[bw->ops[i].kind] += ms;
      cnt[bw->ops[i].kind]++;
    }
    for (int k = 0; k < BOp::NKINDS; ++k)
      if (cnt[k]) fprintf(stderr, ", \"%s x%d\": %.3f", names[k], cnt[k], tot[k]);
    fprintf(stderr, "}}\n");
    for (auto& e : ev) cudaEventDestroy(e);
  }
  return 0;
}

extern "C" int b200ad_unet_backward(b200ad_unet* h, const float* x, const float* g_eps, int accumulate, void* stream) {
  if (!h || !h->bwd || h->bwd->ops.empty()) return set_err("bind_backward must be called before backward");
  if (!x || !g_eps) return set_err("backward: x and g_eps are required");
  BwdArgs a;
  a.x = x; a.g_eps = g_eps;
  return run_backward(h, h->bwd, a, accumulate, (cudaStream_t)stream);
}

extern "C" int b200ad_unet_backward_launch_count(const b200ad_unet* h) { return h && h->bwd ? h->bwd->launches : 0; }

// ================================================================================= autoencoder backward
namespace b200ad {

// Both parts' plans over one arena: the decoder first, then the encoder (the order of a training step's backward).
static int build_vae_backward(b200ad_vae* h, Backward* const* bws, uint8_t* arena, float* grads, size_t* bytes_out) {
  const b200ad_vae_config& c = h->cfg;
  if (!h->training || h->plan.lists.empty()) return set_err("backward needs set_training(1) before bind_workspace");
  if (c.in_channels != 1 || c.out_channels != 1 || c.latent_channels != 1)
    return set_err("autoencoder backward: only in_channels = out_channels = latent_channels = 1 is implemented");
  const int f = 1 << (c.num_blocks - 1), hl = h->H / f, wl = h->W / f, L2 = 2 * c.latent_channels;
  const int Cmax = c.block_out_channels[c.num_blocks - 1] > c.block_out_channels[0] ? c.block_out_channels[c.num_blocks - 1]
                                                                                    : c.block_out_channels[0];
  if ((hl * wl) % 64) return set_err("autoencoder backward: the latent must have a multiple of 64 pixels");
  BwdBuilder B;
  B.h = h; B.N = h->N;
  B.single_head = true;
  B.mem.base = arena;
  int maxC = Cmax;
  for (const auto& kv : h->plan.taps) maxC = kv.second.C > maxC ? kv.second.C : maxC;
  B.cs = (float*)B.mem.take((size_t)h->N * 3 * maxC * sizeof(float));
  B.gsums = (float*)B.mem.take((size_t)h->N * 3 * maxC * 2 * sizeof(float));
  B.csum_floats = (size_t)h->N * 65536;
  B.csum_arena = (float*)B.mem.take(B.csum_floats * sizeof(float));
  float* wflip = (float*)B.mem.take((size_t)Cmax * L2 * 9 * sizeof(float));
  const float* zbias = (const float*)B.mem.take((size_t)Cmax * sizeof(float));   // never written: zeros
  float* gh = (float*)B.mem.take((size_t)2 * h->N * L2 * hl * wl * sizeof(float));  // encoder tail: [N][2L] | [2L][N]
  const Plan& pl = h->plan;
  for (int part : {DEC, ENC}) {
    Backward* bw = bws[part];
    bw->ops.clear();
    bw->jobs.clear();
    bw->arena = arena;
    bw->grads = grads;
    B.bw = bw;
    B.grad.clear(); B.skipgrad.clear(); B.csum_of.clear();
    B.csum_used = 0;
    BOp z{};
    z.kind = BOp::MEMSET;
    z.o0 = B.csum_arena; z.n = (long long)(B.csum_floats * sizeof(float));
    bw->ops.push_back(z);
    const std::vector<Block>& bl = part == ENC ? h->enc : h->dec;
    auto tap = [&](int i) {
      return i < 0 ? std::string() : (bl[i].kind == BK_CONV_IN || bl[i].kind == BK_LATENT_IN) ? bl[i].name + "conv_in" : bl[i].name;
    };
    for (int i = (int)bl.size() - 1; i >= 0; --i) {
      const Block& k = bl[i];
      const std::string in = tap(k.in);
      switch (k.kind) {
        case BK_CONV_OUT: B.conv_out_bwd(k, in, wflip, zbias); break;
        case BK_LATENT_OUT: {   // g_moments -> quant_conv -> conv_out (C -> 2L, per output channel) -> conv_norm_out + SiLU
          const Act x = B.fwd(in), eo = B.fwd(k.name + "conv_out");
          const int C = x.C, H = x.H, W = x.W;
          const size_t plane = (size_t)h->N * H * W;
          float* gh_cn = gh ? gh + L2 * plane : nullptr;
          BOp q{};
          q.kind = BOp::QUANTBWD;
          q.src = eo.p; q.f0 = B.P("quant_conv.weight"); q.o0 = B.PG("quant_conv.weight"); q.o1 = B.PG("quant_conv.bias");
          q.o2 = gh; q.c = L2; q.H = H; q.W = W;
          bw->ops.push_back(q);
          Act A = B.gn_apply("A", x, nullptr, k.name + "conv_norm_out", true);
          float* dw = B.PG(k.name + "conv_out.weight");
          float* db = B.PG(k.name + "conv_out.bias");
          for (int o = 0; o < L2; ++o) {
            BOp w{};
            w.kind = BOp::SCALAR_WGRAD;
            w.src = A.p; w.f0 = gh_cn ? gh_cn + o * plane : nullptr; w.o0 = dw ? dw + (size_t)o * C * 9 : nullptr;
            w.C = C; w.H = H; w.W = W; w.a = 1;
            bw->ops.push_back(w);
            BOp sb{};
            sb.kind = BOp::SUMADD;
            sb.f0 = w.f0; sb.n = (long long)plane; sb.o0 = db ? db + o : nullptr;
            bw->ops.push_back(sb);
          }
          BOp fl{};
          fl.kind = BOp::FLIP;
          fl.f0 = B.P(k.name + "conv_out.weight"); fl.o0 = wflip; fl.C = C; fl.a = L2;
          bw->ops.push_back(fl);
          Act T1 = B.tmp("T1", C, H, W);
          BOp ci{};
          ci.kind = BOp::CONVIN;        // g_a[c] = sum_o sum_t g_h[o][p + s_t] * wflip[c][o][t]
          ci.f2 = gh; ci.c = L2; ci.f0 = wflip; ci.f1 = zbias; ci.dst = T1.p; ci.C = C; ci.H = H; ci.W = W;
          bw->ops.push_back(ci);
          B.gn_bwd(T1, x, nullptr, k.name + "conv_norm_out", true, B.G(in), nullptr, nullptr, nullptr);
          break;
        }
        case BK_RESNET: B.resnet_bwd(k, in, tap(k.skip)); break;
        case BK_ATTN: B.attention_bwd(k.name, in); break;
        case BK_DOWN_ASYM: B.downsample_bwd(k, in); break;
        case BK_UP: B.upsample_bwd(k.name, in); break;
        case BK_CONV_IN:        // encoder head: weight gradients only (no gradient w.r.t. the image)
        case BK_LATENT_IN: {    // decoder head: conv_in on post_quant_conv(z), then the gradient w.r.t. z
          const std::string n = tap(i);
          const Act x = B.fwd(n);
          const Act Gx = B.G(n);
          BOp w{};
          w.kind = BOp::SCALAR_WGRAD;
          w.src = Gx.p; w.o0 = B.PG(n + ".weight"); w.C = x.C; w.H = x.H; w.W = x.W; w.a = 0;
          if (k.kind == BK_CONV_IN) w.x_is_input = true;
          else w.f0 = pl.zq;
          bw->ops.push_back(w);
          B.bias_grad(BwdBuilder::whole(Gx), n + ".bias");
          if (k.kind == BK_LATENT_IN) {
            BOp li{};
            li.kind = BOp::LATENTINBWD;
            li.src = Gx.p; li.f0 = B.P(n + ".weight"); li.f1 = B.P("post_quant_conv.weight"); li.f2 = pl.z_in;
            li.o0 = B.PG("post_quant_conv.weight"); li.o1 = B.PG("post_quant_conv.bias");
            li.C = x.C; li.c = k.cin; li.H = x.H; li.W = x.W;
            bw->ops.push_back(li);
          }
          break;
        }
        default: return set_err("autoencoder backward: block %s has no backward", k.name.c_str());
      }
    }
  }
  if (bytes_out) *bytes_out = (B.mem.off + 255) & ~(size_t)255;
  return 0;
}

void release_backward(b200ad_vae* h) {
  for (Backward*& b : h->bwd) {
    delete b;
    b = nullptr;
  }
}

}  // namespace b200ad

extern "C" int b200ad_vae_set_training(b200ad_vae* h, int on) {
  if (!h) return set_err("null handle");
  if (h->training != (on != 0)) {
    h->training = on != 0;
    h->plan.lists.clear();    // the workspace layout changes: bind_workspace must be called again
  }
  return 0;
}

// The flat gradient buffer: encoder parameters (with quant_conv) first, then the decoder's (with post_quant_conv); each
// part's plan zeroes only its own range.
static void ensure_bwd(b200ad_vae* h) {
  if (h->bwd[0]) return;
  std::vector<size_t> goff;
  size_t off = 0, dec_off = 0;
  for (const auto& p : h->params) {
    if (!dec_off && (p.name.rfind("decoder.", 0) == 0 || p.name.rfind("post_quant_conv.", 0) == 0)) dec_off = off;
    size_t n = 1;
    for (auto d : p.shape) n *= (size_t)d;
    goff.push_back(off);
    off += (n + 63) & ~(size_t)63;
  }
  for (int part : {ENC, DEC}) {
    Backward* bw = new Backward();
    bw->goff = goff;
    bw->grad_floats = off;
    bw->zero_off = part == ENC ? 0 : dec_off;
    bw->zero_floats = part == ENC ? dec_off : off - dec_off;
    h->bwd[part] = bw;
  }
}

extern "C" size_t b200ad_vae_grad_floats(b200ad_vae* h) { ensure_bwd(h); return h->bwd[0]->grad_floats; }
extern "C" size_t b200ad_vae_grad_offset(b200ad_vae* h, int i) { ensure_bwd(h); return h->bwd[0]->goff[i]; }

static size_t vae_backward_size(b200ad_vae* h) {
  ensure_bwd(h);
  Backward t0, t1;
  t0.goff = t1.goff = h->bwd[0]->goff;
  Backward* tb[2] = {&t0, &t1};
  size_t bytes = 0;
  if (build_vae_backward(h, tb, nullptr, nullptr, &bytes)) return 0;
  return bytes;
}

extern "C" size_t b200ad_vae_backward_bytes(b200ad_vae* h) { return vae_backward_size(h); }

extern "C" int b200ad_vae_bind_backward(b200ad_vae* h, void* arena, size_t bytes, float* grads, void* stream) {
  const size_t need = vae_backward_size(h);
  if (!need) return -1;
  if (bytes < need) return set_err("backward arena too small: %zu < %zu", bytes, need);
  CK(cudaMemsetAsync(arena, 0, need, (cudaStream_t)stream));
  size_t got = 0;
  if (build_vae_backward(h, h->bwd, (uint8_t*)arena, grads, &got)) return -1;
  for (Backward* b : h->bwd) b->arena_bytes = got;
  return 0;
}

static int vae_backward(b200ad_vae* h, int part, const BwdArgs& a, int accumulate, cudaStream_t st) {
  if (!h || !h->bwd[part] || h->bwd[part]->ops.empty()) return set_err("bind_backward must be called before backward");
  return run_backward(h, h->bwd[part], a, accumulate, st);
}

extern "C" int b200ad_vae_decoder_backward(b200ad_vae* h, const float* g_x, float* g_z_out, int accumulate, void* stream) {
  if (!g_x || !g_z_out) return set_err("decoder_backward: g_x and g_z_out are required");
  BwdArgs a;
  a.g_eps = g_x; a.g_z = g_z_out;
  return vae_backward(h, DEC, a, accumulate, (cudaStream_t)stream);
}

extern "C" int b200ad_vae_encoder_backward(b200ad_vae* h, const float* x, const float* g_moments, int accumulate,
                                           void* stream) {
  if (!x || !g_moments) return set_err("encoder_backward: x and g_moments are required");
  BwdArgs a;
  a.x = x; a.g_mom = g_moments;
  return vae_backward(h, ENC, a, accumulate, (cudaStream_t)stream);
}

extern "C" int b200ad_vae_backward_launch_count(const b200ad_vae* h) {
  return h && h->bwd[0] ? h->bwd[0]->launches + h->bwd[1]->launches : 0;
}
