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
// The normalised activations the weight gradients read are materialised (no fusion yet).
// A backward plan is an OpList of net.cuh, run by the forward's executor (run_ops).
#include "bwd_kernels.cuh"
#include "unet.cuh"
#include "vae.cuh"

using namespace b200ad;

namespace b200ad {

struct View {            // channel range of a PF8 tensor
  const __nv_bfloat16* p = nullptr;   // first plane of the view (image 0)
  int C = 0, img_planes = 0, H = 0, W = 0;
  size_t off = 0;                     // byte offset of p in its arena (Act::off)
};

struct Backward {
  OpList list;                       // the ops (no GroupNorm statistics)
  std::vector<PackJob> jobs;         // transposed weight packs, redone at every backward (the weights move every step)
  std::vector<size_t> goff;          // float offset of every parameter's gradient in the flat buffer
  size_t grad_floats = 0;
  size_t zero_off = 0, zero_floats = 0;   // the slots of the flat buffer this plan writes (zeroed unless accumulating)
  uint8_t* arena = nullptr;
  size_t arena_bytes = 0;
  float* grads = nullptr;
  int launches = 0;
  PackBatch pack_batch;              // one launch for all transposed packs
  int enc_len = 1;                   // conditional U-Net: the encoder sequence length the plan was built for
  // the builder's gradient tensors by forward tap name (arena tensors of their own, final once the plan has run):
  // the whole gradient, and the share of it a skip connection brought (debug_grad)
  std::map<std::string, Act> grad, skipgrad;
};

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
  // tensor's arena offset, the same in the size pass): the producer's bias gradient then is a reduction over N of a [N][C]
  // array instead of a pass over the tensor
  float* csum_arena = nullptr;
  size_t csum_floats = 0, csum_used = 0;
  std::map<size_t, float*> csum_of;
  const float* last_cs = nullptr;             // [N][C] sums of the latest bias_grad (the time-embedding rows are read from it)

  Act act_alloc(int C, int H, int W) { return take_act(mem, N, C, H, W); }
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
    v.off = a.off + (size_t)(c0 / 8) * g.PL * 16;
    return v;
  }
  static View whole(const Act& a) { return view(a, 0, a.C); }

  void emit(OpKind kind, OpFn run, int launches = 1) { bw->list.ops.push_back(Op{kind, launches, {}, std::move(run)}); }
  void zero(void* p, size_t bytes) {
    emit(OP_MEMSET, [p, bytes](const RunArgs&, cudaStream_t s) { return cudaMemsetAsync(p, 0, bytes, s); });
  }

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
  // the plan's first op: all of its transposed packs in one launch
  void pack_op() {
    emit(OP_PACK_T, [h = h, bw = bw](const RunArgs&, cudaStream_t s) {
      std::vector<PackItem> items;
      items.reserve(bw->jobs.size());
      for (const PackJob& j : bw->jobs) items.push_back(make_pack_item(h, j, bw->arena));
      return launch_pack_batch(bw->pack_batch, items, s);
    });
  }

  // ---- op emitters ------------------------------------------------------------------------------------------------
  void conv(const ConvParams& p) {
    Op op{OP_DGRAD};
    op.conv = p;
    bw->list.ops.push_back(op);
  }
  static void seg(ConvSeg& s, const View& src, const __nv_bfloat16* wpack, const TapSet& t) {
    set_seg(s, src.p, src.img_planes, src.C, src.H, src.W, wpack, t);
  }
  // data gradient of a stride-1 KxK conv: out (I channels) = conv^T(gy (O channels))
  void dgrad(const std::string& wname, const View& gy, const Act& out, int K) {
    const TapSet t = taps_mirrored(K);
    ConvParams p = conv_geom(N, out);
    seg(p.seg[0], gy, tjob(wname, gy.C, out.C, K, t), t);
    p.nseg = 1;
    conv(p);
  }
  // weight gradient of the forward K-segment with tap set t (of ntaps_total taps of the weight) that read `act`
  void wgrad(const View& gy, const View& act, float* dw, int cin_total, int ci_off, int ntaps_total, const TapSet& t) {
    WgradDesc d{};
    d.gy = gy.p; d.act = act.p; d.dw = dw; d.N = N; d.H = gy.H; d.W = gy.W; d.cout = gy.C; d.cin = act.C;
    d.gy_img_planes = gy.img_planes; d.act_img_planes = act.img_planes;
    d.cin_total = cin_total; d.ci_off = ci_off; d.ntaps_total = ntaps_total; d.ntaps = t.pack.ntaps;
    for (int k = 0; k < t.pack.ntaps; ++k) { d.dh[k] = t.dh[k]; d.dw_[k] = t.dw[k]; d.tapidx[k] = t.wtap[k]; }
    emit(OP_WGRAD, [h = h, d](const RunArgs&, cudaStream_t s) { return launch_wgrad_tc(d, h->num_sms, s); });
  }
  void wgrad_conv(const View& gy, const View& act, const std::string& wname, int K) {   // plain stride-1 conv
    wgrad(gy, act, PG(wname), act.C, 0, K * K, taps_conv(K));
  }
  // per-channel sums of a gradient -> bias gradient(s); last_cs: the [N][C] sums (valid until the next chan_sum)
  void bias_grad(const View& g, const std::string& bname, const std::string& bname2 = "") {
    float* db = PG(bname);
    float* db2 = bname2.empty() ? nullptr : PG(bname2);
    auto it = csum_of.find(g.off);
    if (it != csum_of.end() && g.img_planes * 8 == g.C) {     // whole tensor, sums already made by the pass that wrote it
      last_cs = it->second;
      emit(OP_REDUCE_N, [sums = it->second, db, db2, N = N, C = g.C](const RunArgs&, cudaStream_t s) {
        return launch_reduce_n_add(sums, db, db2, N, C, s);
      });
      return;
    }
    last_cs = cs;
    emit(OP_CHANSUM, [g, sums = cs, db, db2, N = N](const RunArgs&, cudaStream_t s) {   // bias gradients by the same kernel
      return launch_chan_sum(g.p, sums, N, g.C, g.img_planes, g.H, g.W, s, db, db2);
    });
  }
  Act gn_apply(const std::string& tag, const Act& a, const Act* b, const std::string& norm, bool silu, float eps = -1.f) {
    Act out = tmp(tag, a.C + (b ? b->C : 0), a.H, a.W);
    const GnApplyParams p = gn_params(h, N, a, b, norm, out.p, silu, eps);
    emit(OP_GNAPPLY, [p](const RunArgs&, cudaStream_t s) { return launch_gn_apply(p, s); });
    return out;
  }
  void gn_bwd(const Act& ga, const Act& a, const Act* b, const std::string& norm, bool silu, const Act& d0, const Act* d1,
              const __nv_bfloat16* addS, const __nv_bfloat16* add0, float eps = -1.f) {
    GnBwdParams p{};
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
      csum_of[d0.off] = p.csum0;
      csum_used += need;
    }
    p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = eps < 0.f ? h->norm_eps : eps; p.silu = silu ? 1 : 0;
    emit(OP_GN_BWD, [p](const RunArgs&, cudaStream_t s) { return launch_gn_bwd(p, s); }, 2);
  }
  const __nv_bfloat16* skip_of(const std::string& name) const {
    auto it = skipgrad.find(name);
    return it == skipgrad.end() ? nullptr : it->second.p;
  }
  // conv_out's data gradient (3x3, O -> C channels) as the conv_in kernel over the fp32 output gradient gy (null: the
  // gradient passed to backward()): g_a[c] = sum_o sum_t gy[o][p + s_t] * wflip[c][o][t]
  void conv_out_dgrad(const std::string& wname, const float* gy, int O, float* wflip, const float* zbias, const Act& out) {
    emit(OP_FLIP, [w = P(wname), wflip, C = out.C, O](const RunArgs&, cudaStream_t s) {
      return launch_flip_taps(w, wflip, C, s, O);
    });
    emit(OP_CONV_IN_BWD, [gy, wflip, zbias, out, N = N, O](const RunArgs& a, cudaStream_t s) {
      return launch_conv_in(gy ? gy : a.g_eps, wflip, zbias, N, O, out.H, out.W, out.C, out.p, nullptr, s);
    });
  }
  // weight gradient of a 3x3 conv with one fp32 output channel x (null: the gradient passed to backward(); flip: x is
  // that output's gradient, `g` the conv's input) or one fp32 input channel x (the conv's output gradient is `g`)
  void scalar_wgrad(const Act& g, const float* x, bool x_is_input, float* dw, int flip) {
    emit(OP_SCALAR_WGRAD, [g, x, x_is_input, dw, flip, N = N](const RunArgs& a, cudaStream_t s) {
      return launch_scalar_conv_wgrad(g.p, x ? x : x_is_input ? a.in : a.g_eps, dw, N, g.C, g.H, g.W, flip, s);
    });
  }
  void sum_add(const float* x, long long n, float* dst) {   // x null: the gradient passed to backward()
    emit(OP_SUMADD, [x, n, dst](const RunArgs& a, cudaStream_t s) { return launch_sum_add(x ? x : a.g_eps, n, dst, s); });
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
    if (k.temb_row >= 0)
      emit(OP_SCATTER, [sums = last_cs, gproj = gproj, N = N, co, rows = h->temb_rows, row = k.temb_row](const RunArgs&,
                                                                                                         cudaStream_t s) {
        return launch_scatter_rows(sums, gproj, N, co, rows, row, s);
      });
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
    if (single_head) {   // the forward's softmax P is kept: dP GEMM for the row sums of P o dP, then dS, dV, dQ, dK
      const long long S = (long long)H * W;
      float* D = (float*)mem.take((size_t)N * S * sizeof(float));
      __nv_bfloat16* dS = (__nv_bfloat16*)mem.take((size_t)N * S * S * sizeof(__nv_bfloat16));
      emit(OP_ATTN1_BWD, [q = qkv.p, go = T1.p, probs = h->plan.probs.at(n), D, dS, gq = Gqkv.p, N = N, C, H,
                          W](const RunArgs&, cudaStream_t s) {
        return launch_attention_1head_bwd(q, go, probs, D, dS, gq, N, C, H, W, s);
      }, 6);
    } else {
      emit(OP_ATTN_BWD, [q = qkv.p, go = T1.p, gq = Gqkv.p, N = N, C, H, W](const RunArgs&, cudaStream_t s) {
        return launch_attention_bwd(q, go, gq, N, C, H, W, s);
      });
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
      ConvParams p = conv_geom(N, T2);
      const TapSet t = taps_mirrored(1);
      for (int k = 0; k < 3; ++k)
        seg(p.seg[k], view(Gqkv, k * C, C), tjob(n + "." + names[k] + ".weight", C, C, 1, t), t);
      p.nseg = 3;
      conv(p);
    }
    gn_bwd(T2, x, nullptr, n + ".group_norm", false, G(xn), nullptr, Gout.p, skip_of(xn));
  }

  // LayerNorm over channels (eps 1e-5, as the forward): gx = LN-backward(gy; x) + add, gamma / beta gradients
  void layer_norm_bwd(const Act& gy, const Act& x, const std::string& norm, const Act& gx, const Act& add) {
    emit(OP_LN_BWD, [x, gy = gy.p, add = add.p, gx = gx.p, gamma = P(norm + ".weight"), dgamma = PG(norm + ".weight"),
                     dbeta = PG(norm + ".bias"), N = N](const RunArgs&, cudaStream_t s) {
      return launch_layernorm_bwd_pf8(x.p, gy, add, gx, gamma, dgamma, dbeta, N, x.C, x.H, x.W, 1e-5f, s);
    });
  }

  // Transformer2DModel with one BasicTransformerBlock (Builder::transformer) in reverse, from G(out) to G(x):
  //   h0 = proj_in(GN(x));  h2 = h0 + attn1(LN1(h0)) + vec;  h3 = h2 + ff2(GEGLU(ff1(LN3(h2))));  out = proj_out(h3) + x
  // Encoder sequence length S = 1: attn2 over ONE key is the per-sample vector vec = Wo (Wv enc) + bo: its gradient is the
  // per-sample channel sum of G(h2) (the sums the attn1.to_out bias gradient makes).  attn2.to_q, attn2.to_k and norm2 do
  // not reach the output (softmax over one key is 1), so their gradients stay exactly zero: nothing is launched for them.
  // S > 1: h1 = h0 + attn1(LN1(h0)), h2 = h1 + attn2(LN2(h1), enc), walked back by cross_attention_bwd.
  void transformer_bwd(const Block& k, const std::string& xn, int S) {
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
    emit(OP_GEGLU_BWD, [src = ff1.p, gy = Ggg.p, gx = Gff1.p, N = N, C, H, W](const RunArgs&, cudaStream_t s) {
      return launch_geglu_bwd_pf8(src, gy, gx, N, 4 * C, H, W, s);
    });
    // ff.net.0.proj
    Act Gn = tmp("tf_Gn", C, H, W);
    dgrad(t + ".ff.net.0.proj.weight", whole(Gff1), Gn, 1);
    wgrad_conv(whole(Gff1), whole(n3), t + ".ff.net.0.proj.weight", 1);
    bias_grad(whole(Gff1), t + ".ff.net.0.proj.bias");
    // norm3 (+ residual) -> G(h2)
    Act Gh2 = tmp("tf_Gh2", C, H, W);
    layer_norm_bwd(Gn, h2, t + ".norm3", Gh2, Gh3);
    Act Gao = tmp("tf_Gao", C, H, W);
    Act Gh1 = Gh2;   // the gradient of attn1's output projection, with its residual h0
    if (S == 1) {
      // attn1.to_out and attn2.to_out both add their bias to every pixel of h2: one channel sum gives both bias gradients
      dgrad(t + ".attn1.to_out.0.weight", whole(Gh2), Gao, 1);
      wgrad_conv(whole(Gh2), whole(ao), t + ".attn1.to_out.0.weight", 1);
      bias_grad(whole(Gh2), t + ".attn1.to_out.0.bias", t + ".attn2.to_out.0.bias");
      // dvec[n] = per-sample channel sums of G(h2) (last_cs, made just above)
      emit(OP_XVEC_BWD, [h = h, dvec = last_cs, wv = P(t + ".attn2.to_v.weight"), wo = P(t + ".attn2.to_out.0.weight"),
                         dwo = PG(t + ".attn2.to_out.0.weight"), dwv = PG(t + ".attn2.to_v.weight"),
                         scratch = (float*)mem.take((size_t)2 * N * C * sizeof(float)), N = N, C,
                         X = k.cross](const RunArgs&, cudaStream_t s) {
        return launch_cross_attn_vec_bwd(h->enc, dvec, wv, wo, dwo, dwv, scratch, N, C, X, s);
      }, 2);
    } else {
      Gh1 = cross_attention_bwd(k, Gh2, Gao, Gn, S);
      dgrad(t + ".attn1.to_out.0.weight", whole(Gh1), Gao, 1);
      wgrad_conv(whole(Gh1), whole(ao), t + ".attn1.to_out.0.weight", 1);
      bias_grad(whole(Gh1), t + ".attn1.to_out.0.bias");
    }
    // attention core (P recomputed from the forward's row log-sum-exp)
    Act Gqkv = tmp("tf_Gqkv", 3 * C, H, W);
    emit(OP_MHA_BWD, [q = qkv.p, o = ao.p, go = Gao.p, lse = h->plan.lse.at(n),
                      dsum = (float*)mem.take((size_t)N * heads * H * W * sizeof(float)), gq = Gqkv.p, N = N, C,
                      heads = heads, H, W](const RunArgs&, cudaStream_t s) {
      return launch_mha_bwd(q, o, go, lse, dsum, gq, N, C, heads, H, W, s);
    }, 3);
    // q / k / v projections (no bias); g(n1) = sum over q, k, v of W^T g: one launch, three K-segments
    const char* names[3] = {"to_q", "to_k", "to_v"};
    for (int j = 0; j < 3; ++j) wgrad_conv(view(Gqkv, j * C, C), whole(n1), t + ".attn1." + names[j] + ".weight", 1);
    {
      ConvParams p = conv_geom(N, Gn);
      const TapSet ts = taps_mirrored(1);
      for (int j = 0; j < 3; ++j)
        seg(p.seg[j], view(Gqkv, j * C, C), tjob(t + ".attn1." + names[j] + ".weight", C, C, 1, ts), ts);
      p.nseg = 3;
      conv(p);
    }
    // norm1 (+ residual) -> G(h0)
    Act Gh0 = tmp("tf_Gh0", C, H, W);
    layer_norm_bwd(Gn, h0, t + ".norm1", Gh0, Gh1);
    // proj_in over GroupNorm(x) (eps 1e-6, no SiLU), then the GroupNorm backward with the outer residual G(out)
    Act T = tmp("tf_T", C, H, W);
    dgrad(n + ".proj_in.weight", whole(Gh0), T, 1);
    Act XN = gn_apply("A", x, nullptr, n + ".norm", false, 1e-6f);
    wgrad_conv(whole(Gh0), whole(XN), n + ".proj_in.weight", 1);
    bias_grad(whole(Gh0), n + ".proj_in.bias");
    gn_bwd(T, x, nullptr, n + ".norm", false, G(xn), nullptr, Gout.p, skip_of(xn), 1e-6f);
  }

  // attn2 against S > 1 encoder tokens (Builder::cross_attention) in reverse, from G(h2) to G(h1) (returned):
  //   h2 = h1 + to_out(ao2),  ao2 = xattn(q2, K, V),  q2 = to_q(n2),  n2 = LN2(h1),  K = enc Wk^T,  V = enc Wv^T
  // Gao2 and Gn are scratch tensors of C channels (the caller's, free at this point of the walk).
  Act cross_attention_bwd(const Block& k, const Act& Gh2, const Act& Gao2, const Act& Gn, int S) {
    const std::string& n = k.name;
    const std::string t = n + ".transformer_blocks.0";
    const Act h1 = fwd(n + ".attn1"), n2 = fwd(n + ".n2"), q2 = fwd(n + ".q2"), ao2 = fwd(n + ".ao2");
    const int C = h1.C, H = h1.H, W = h1.W;
    // to_out (its residual is h1: G(h1) += G(h2) in the LayerNorm backward below)
    dgrad(t + ".attn2.to_out.0.weight", whole(Gh2), Gao2, 1);
    wgrad_conv(whole(Gh2), whole(ao2), t + ".attn2.to_out.0.weight", 1);
    bias_grad(whole(Gh2), t + ".attn2.to_out.0.bias");
    // attention core -> G(q2) and dK, dV (fp32 [N][S][C]), then the K / V projections' weight gradients
    Act Gq2 = tmp("tf_Gq2", C, H, W);
    const size_t kv = (size_t)N * S * C;
    float* dkv = (float*)mem.take(2 * kv * sizeof(float));
    emit(OP_XATTN_BWD, [q = q2.p, kvp = h->plan.xkv.at(n), o = ao2.p, go = Gao2.p, lse = h->plan.lse.at(n + ".attn2"),
                        dsum = (float*)mem.take((size_t)N * heads * H * W * sizeof(float)),
                        part = (float*)mem.take(xattn_part_floats(N, C, heads, H, W, S) * sizeof(float)), gq = Gq2.p, dkv,
                        kv, N = N, C, heads = heads, H, W, S](const RunArgs&, cudaStream_t s) {
      return launch_xattn_bwd(q, kvp, kvp + kv, o, go, lse, dsum, part, gq, dkv, dkv + kv, N, C, heads, H, W, S, s);
    }, 4);
    emit(OP_XKV_BWD, [h = h, dkv, kv, dwk = PG(t + ".attn2.to_k.weight"), dwv = PG(t + ".attn2.to_v.weight"), M = N * S, C,
                      X = k.cross](const RunArgs&, cudaStream_t s) {
      return launch_xattn_kv_wgrad(dkv, dkv + kv, h->enc, dwk, dwv, M, C, X, s);
    });
    // to_q (no bias)
    wgrad_conv(whole(Gq2), whole(n2), t + ".attn2.to_q.weight", 1);
    dgrad(t + ".attn2.to_q.weight", whole(Gq2), Gn, 1);
    // norm2 (+ residual) -> G(h1)
    Act Gh1 = tmp("tf_Gh1", C, H, W);
    layer_norm_bwd(Gn, h1, t + ".norm2", Gh1, Gh2);
    return Gh1;
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
        Act lo = Gx;
        lo.H = Ho; lo.W = Wo;
        ConvParams p = conv_geom(N, lo);
        p.up2 = 1; p.oy = a; p.ox = b;
        seg(p.seg[0], whole(Gy), tjob(n + ".weight", C, C, 3, t), t);
        p.nseg = 1;
        conv(p);
      }
    if (skipgrad.count(xn))
      emit(OP_PF8ADD, [gx = Gx.p, add = skip_of(xn), N = N, C, H = x.H, W = x.W](const RunArgs&, cudaStream_t s) {
        return launch_pf8_add(gx, add, N, C, H, W, s);
      });
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
    emit(OP_PARITY, [gy = Gy.p, gpar = gpar.p, N = N, C, H = y.H, W = y.W](const RunArgs&, cudaStream_t s) {
      return launch_parity_split(gy, gpar, N, C, H, W, s);
    });
    float* dwf = (float*)mem.take((size_t)4 * C * C * 4 * sizeof(float));
    zero(dwf, (size_t)4 * C * C * 4 * sizeof(float));
    Act Gx = G(xn);
    ConvParams dg = conv_geom(N, Gx);
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
        seg(dg.seg[pidx], whole(plane), tjob(n + ".weight", C, C, 3, bwd_taps), bwd_taps);
      }
    dg.nseg = 4;
    emit(OP_UNFOLD, [dwf, dw = PG(n + ".weight"), nco_ci = (long long)C * C, um](const RunArgs&, cudaStream_t s) {
      return launch_unfold_up2(dwf, dw, nco_ci, um, s);
    });
    conv(dg);
  }

  // conv_norm_out + SiLU + conv_out (C -> 1) on the last activation `in`, from the output gradient passed to backward()
  void conv_out_bwd(const Block& k, const std::string& in, float* wflip, const float* zbias) {
    const Act x = fwd(in);
    Act A = gn_apply("A", x, nullptr, k.name + "conv_norm_out", true);
    scalar_wgrad(A, nullptr, false, PG(k.name + "conv_out.weight"), 1);
    sum_add(nullptr, (long long)N * x.H * x.W, PG(k.name + "conv_out.bias"));
    Act T1 = tmp("T1", x.C, x.H, x.W);
    conv_out_dgrad(k.name + "conv_out.weight", nullptr, 1, wflip, zbias, T1);
    gn_bwd(T1, x, nullptr, k.name + "conv_norm_out", true, G(in), nullptr, nullptr, nullptr);
  }
};

static int build_unet_backward(b200ad_unet* h, Backward* const* bws, uint8_t* arena, float* grads, size_t* bytes_out) {
  const b200ad_unet_config& c = h->cfg;
  if (!h->training || h->plan.lists.empty()) return set_err("backward needs set_training(1) before bind_workspace");
  if (h->enc_len != h->plan_enc_len)
    return set_err("backward: the encoder sequence length is set to %d but the workspace is planned for %d (bind the "
                   "workspace again)", h->enc_len, h->plan_enc_len);
  Backward* bw = bws[0];
  bw->enc_len = h->plan_enc_len;
  bw->list.ops.clear();
  bw->jobs.clear();
  bw->arena = arena;
  bw->grads = grads;
  BwdBuilder B;
  B.h = h; B.bw = bw; B.N = h->N;
  B.heads = c.attention_head_dim;
  B.mem.base = arena;
  B.pack_op();
  int maxC = c.block_out_channels[0];
  for (const auto& kv : h->plan.taps) maxC = kv.second.C > maxC ? kv.second.C : maxC;
  const int D = c.block_out_channels[0] * 4;
  B.cs = (float*)B.mem.take((size_t)h->N * 3 * maxC * sizeof(float));
  B.gsums = (float*)B.mem.take((size_t)h->N * 3 * maxC * 2 * sizeof(float));
  B.gproj = (float*)B.mem.take((size_t)h->N * h->temb_rows * sizeof(float));
  B.csum_floats = (size_t)h->N * 65536;       // all GroupNorm-backward outputs of the reference architecture: 16 K channels
  B.csum_arena = (float*)B.mem.take(B.csum_floats * sizeof(float));
  B.zero(B.csum_arena, B.csum_floats * sizeof(float));
  float* g_act = (float*)B.mem.take((size_t)h->N * D * sizeof(float));   // gradient w.r.t. silu(linear_2)
  float* g_h1 = (float*)B.mem.take((size_t)h->N * D * sizeof(float));
  float* h1v = (float*)B.mem.take((size_t)h->N * D * sizeof(float));
  float* wflip = (float*)B.mem.take((size_t)c.block_out_channels[0] * 9 * sizeof(float));
  const float* zbias = (const float*)B.mem.take((size_t)c.block_out_channels[0] * sizeof(float));   // never written: zeros

  // linear layers of the timestep embedding: dW, db from the output gradient g (row stride gs) and the input x;
  // gin = g W; u: SiLU pre-activation
  const int N = h->N;
  auto lin_w = [&](const float* g, int gs, const float* x, int O, int I, const std::string& name) {
    B.emit(OP_LIN_W, [g, gs, x, O, I, dw = B.PG(name + ".weight"), db = B.PG(name + ".bias"), N](const RunArgs&,
                                                                                                 cudaStream_t s) {
      return launch_lin_bwd_weight(g, gs, x, O, I, dw, db, N, s);
    });
  };
  auto lin_in = [&](const float* g, int gs, const float* w, int O, int I, float* gin) {
    B.emit(OP_LIN_IN, [g, gs, w, O, I, gin, N](const RunArgs&, cudaStream_t s) {
      return launch_lin_bwd_input(g, gs, w, O, I, gin, N, 0, s);
    });
  };
  auto silu_bwd = [&](float* g, const float* u) {
    B.emit(OP_SILU_BWD, [g, u, n = N * D](const RunArgs&, cudaStream_t s) { return launch_silu_bwd(g, u, n, s); });
  };

  // the forward's blocks in reverse; a block's output is the forward tap of its name (the head's: conv_in)
  const std::vector<Block>& bl = h->blocks;
  auto tap = [&](int i) { return i < 0 ? std::string() : bl[i].kind == BK_UNET_HEAD ? bl[i].name + "conv_in" : bl[i].name; };
  for (int i = (int)bl.size() - 1; i >= 0; --i) {
    const Block& k = bl[i];
    const std::string in = tap(k.in);
    switch (k.kind) {
      case BK_CONV_OUT:      // g_eps -> gradient of the last activation
        if (c.out_channels != 1) return set_err("backward: out_channels != 1 is not implemented");
        B.conv_out_bwd(k, in, wflip, zbias);
        B.zero(B.gproj, (size_t)h->N * h->temb_rows * sizeof(float));
        break;
      case BK_RESNET: B.resnet_bwd(k, in, tap(k.skip)); break;
      case BK_ATTN: B.attention_bwd(k.name, in); break;
      case BK_TRANSFORMER: B.transformer_bwd(k, in, h->plan_enc_len); break;
      case BK_DOWN: B.downsample_bwd(k, in); break;
      case BK_UP: B.upsample_bwd(k.name, in); break;
      case BK_UNET_HEAD: {   // conv_in, then the timestep embedding MLP and the per-resnet projections
        if (c.in_channels != 1) return set_err("backward: in_channels != 1 is not implemented");
        const std::string n = tap(i);
        const Act Gx = B.G(n);
        if (!B.skipgrad.count(n)) return set_err("backward: conv_in skip gradient missing");
        // (the first resnet's GroupNorm backward already added the skip contribution)
        B.scalar_wgrad(Gx, nullptr, true, B.PG(n + ".weight"), 0);
        B.bias_grad(BwdBuilder::whole(Gx), n + ".bias");
        const Plan& pl = h->plan;
        for (const Block& r : bl)        // time_emb_proj of every resnet: dW = g_proj_rows^T temb_act
          if (r.temb_row >= 0) lin_w(B.gproj + r.temb_row, h->temb_rows, pl.temb_act, r.cout, D, r.name + ".time_emb_proj");
        // g(temb_act) = g_proj Wcat
        lin_in(B.gproj, h->temb_rows, h->packed ? (const float*)(h->packed + h->off_wcat) : nullptr, h->temb_rows, D, g_act);
        silu_bwd(g_act, pl.temb_u2);
        B.emit(OP_SILU_FWD, [u = pl.temb_u1, h1v, n = N * D](const RunArgs&, cudaStream_t s) {
          return launch_silu_fwd(u, h1v, n, s);
        });
        lin_w(g_act, D, h1v, D, D, "time_embedding.linear_2");
        lin_in(g_act, D, B.P("time_embedding.linear_2.weight"), D, D, g_h1);
        silu_bwd(g_h1, pl.temb_u1);
        lin_w(g_h1, D, pl.temb_emb, D, k.cout, "time_embedding.linear_1");
        break;
      }
      default: return set_err("backward: block %s has no backward", k.name.c_str());
    }
  }
  bw->grad = B.grad;
  bw->skipgrad = B.skipgrad;
  if (bytes_out) *bytes_out = (B.mem.off + 255) & ~(size_t)255;
  return 0;
}

// ================================================================================= autoencoder backward

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
    bw->list.ops.clear();
    bw->jobs.clear();
    bw->arena = arena;
    bw->grads = grads;
    B.bw = bw;
    B.grad.clear(); B.skipgrad.clear(); B.csum_of.clear();
    B.csum_used = 0;
    B.pack_op();
    B.zero(B.csum_arena, B.csum_floats * sizeof(float));
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
          B.emit(OP_QUANT_BWD, [eo = eo.p, w = B.P("quant_conv.weight"), gh, gh_cn, dw = B.PG("quant_conv.weight"),
                                db = B.PG("quant_conv.bias"), N = h->N, L2, H, W](const RunArgs& a, cudaStream_t s) {
            return launch_quant_conv_bwd(a.g_mom, eo, w, gh, gh_cn, dw, db, N, L2, H, W, s);
          });
          Act A = B.gn_apply("A", x, nullptr, k.name + "conv_norm_out", true);
          float* dw = B.PG(k.name + "conv_out.weight");
          float* db = B.PG(k.name + "conv_out.bias");
          for (int o = 0; o < L2; ++o) {
            const float* g = gh_cn ? gh_cn + o * plane : nullptr;
            B.scalar_wgrad(A, g, false, dw ? dw + (size_t)o * C * 9 : nullptr, 1);
            B.sum_add(g, (long long)plane, db ? db + o : nullptr);
          }
          Act T1 = B.tmp("T1", C, H, W);
          B.conv_out_dgrad(k.name + "conv_out.weight", gh, L2, wflip, zbias, T1);
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
          B.scalar_wgrad(Gx, k.kind == BK_CONV_IN ? nullptr : pl.zq, true, B.PG(n + ".weight"), 0);
          B.bias_grad(BwdBuilder::whole(Gx), n + ".bias");
          if (k.kind == BK_LATENT_IN)
            B.emit(OP_LATENT_IN_BWD, [gy = Gx.p, win = B.P(n + ".weight"), wpq = B.P("post_quant_conv.weight"), z = pl.z_in,
                                      dw = B.PG("post_quant_conv.weight"), db = B.PG("post_quant_conv.bias"), N = h->N,
                                      C = x.C, L = k.cin, H = x.H, W = x.W](const RunArgs& a, cudaStream_t s) {
              return launch_latent_in_bwd(gy, win, wpq, z, a.g_z, dw, db, N, C, L, H, W, s);
            });
          break;
        }
        default: return set_err("autoencoder backward: block %s has no backward", k.name.c_str());
      }
    }
    bw->grad = B.grad;         // the maps are cleared for the next part
    bw->skipgrad = B.skipgrad;
  }
  if (bytes_out) *bytes_out = (B.mem.off + 255) & ~(size_t)255;
  return 0;
}

// ================================================================================= the handle protocol of both models
// fp32 NCHW copy of a gradient tensor of a bound backward plan (skip: the skip connection's share); as debug_tensor.  The
// parts are searched in order: the autoencoder's tap names all start with "encoder." or "decoder.", so a name is found in
// one part only.
static int debug_grad(const NetBase* h, const char* name, int skip, float* dst, int* dims, cudaStream_t st) {
  if (!h || !name) return set_err("null argument");
  for (int i = 0; i < h->nparts; ++i) {
    const Backward* bw = h->bwd[i];
    if (!bw || bw->list.ops.empty()) return set_err("debug_grad: bind_backward must be called first");
    const std::map<std::string, Act>& m = skip ? bw->skipgrad : bw->grad;
    auto it = m.find(name);
    if (it == m.end()) continue;
    const Act& a = it->second;
    if (dims) { dims[0] = a.C; dims[1] = a.H; dims[2] = a.W; }
    if (dst) CK(launch_pf8_to_nchw(a.p, dst, h->N, a.C, a.H, a.W, st));
    return a.C;
  }
  return set_err("debug_grad: no %sgradient for '%s'", skip ? "skip " : "", name);
}

// The size pass (null arena) must plan the ops the bound pass plans, or the arena size it found may be wrong.
static int check_same_plan(const Backward& sized, Backward* bound) {
  bool same = sized.list.ops.size() == bound->list.ops.size();
  for (size_t i = 0; same && i < sized.list.ops.size(); ++i) same = sized.list.ops[i].kind == bound->list.ops[i].kind;
  if (same) return 0;
  bound->list.ops.clear();
  return set_err("bind_backward: the size pass and the bound pass planned different ops");
}

// Runs the bound backward plan of `part`: zeroes its gradient slots (unless accumulating), then its ops.
static int run_backward(NetBase* h, int part, const RunArgs& a, int accumulate, cudaStream_t st) {
  if (!h || !h->bwd[part] || h->bwd[part]->list.ops.empty()) return set_err("bind_backward must be called before backward");
  Backward* bw = h->bwd[part];
  // B200AD_BWD_PROFILE=1: CUDA events around every op, per-kind totals printed to stderr (tools/train_bench.py)
  static const bool prof = [] { const char* e = getenv("B200AD_BWD_PROFILE"); return e && e[0] == '1'; }();
  if (!accumulate) CK(cudaMemsetAsync(bw->grads + bw->zero_off, 0, bw->zero_floats * sizeof(float), st));   // every kernel below ADDS
  OpEvents ev;
  if (run_ops(h, bw->list, a, st, &bw->launches, prof ? &ev : nullptr)) return -1;
  if (prof) {
    CK(cudaStreamSynchronize(st));
    double tot[OP_NKINDS] = {0};
    int cnt[OP_NKINDS] = {0};
    for (size_t i = 0; i < bw->list.ops.size(); ++i) {
      float ms = 0.f;
      if (ev.ms(i, &ms)) return -1;
      tot[bw->list.ops[i].kind] += ms;
      cnt[bw->list.ops[i].kind]++;
    }
    fprintf(stderr, "{\"backward_profile_ms\": {");
    const char* sep = "";
    for (int k = 0; k < OP_NKINDS; ++k) {
      if (!cnt[k]) continue;
      if (k == OP_PACK_T) fprintf(stderr, "%s\"%s\": %.3f", sep, op_names[k], tot[k]);   // one per plan
      else fprintf(stderr, "%s\"%s x%d\": %.3f", sep, op_names[k], cnt[k], tot[k]);
      sep = ", ";
    }
    fprintf(stderr, "}}\n");
  }
  return 0;
}

void release_backward(NetBase* h) {
  for (Backward*& b : h->bwd) {
    delete b;
    b = nullptr;
  }
}

// The flat gradient buffer: every parameter's gradient at a 64-float-aligned offset, in table order.  Each part's plan
// zeroes only its own range: the autoencoder's decoder part starts at its first decoder. / post_quant_conv. parameter.
static void ensure_bwd(NetBase* h) {
  if (h->bwd[0]) return;
  std::vector<size_t> goff;
  size_t off = 0, split = 0;
  for (const auto& p : h->params) {
    if (!split && (p.name.rfind("decoder.", 0) == 0 || p.name.rfind("post_quant_conv.", 0) == 0)) split = off;
    size_t n = 1;
    for (auto d : p.shape) n *= (size_t)d;
    goff.push_back(off);
    off += (n + 63) & ~(size_t)63;
  }
  for (int part = 0; part < h->nparts; ++part) {
    Backward* bw = new Backward();
    bw->goff = goff;
    bw->grad_floats = off;
    bw->zero_off = part == 0 ? 0 : split;
    bw->zero_floats = (part == h->nparts - 1 ? off : split) - bw->zero_off;
    h->bwd[part] = bw;
  }
}

// A model's backward plan builder: the plans of all its parts over one arena (null: size pass), into bws[0..nparts).
template <class Net> using BuildBackward = int (*)(Net*, Backward* const*, uint8_t*, float*, size_t*);

// Size pass of every part into sized[]; returns the arena bytes (0: error).
template <class Net> static size_t backward_size(Net* h, BuildBackward<Net> build, Backward* sized) {
  ensure_bwd(h);
  Backward* parts[2] = {&sized[0], &sized[1]};
  for (Backward* b : parts) b->goff = h->bwd[0]->goff;
  size_t bytes = 0;
  return build(h, parts, nullptr, nullptr, &bytes) ? 0 : bytes;
}

template <class Net> static size_t backward_bytes(Net* h, BuildBackward<Net> build) {
  Backward sized[2];
  return backward_size(h, build, sized);
}

template <class Net>
static int bind_backward(Net* h, BuildBackward<Net> build, void* arena, size_t bytes, float* grads, cudaStream_t st) {
  Backward sized[2];
  const size_t need = backward_size(h, build, sized);
  if (!need) return -1;
  if (bytes < need) return set_err("backward arena too small: %zu < %zu", bytes, need);
  CK(cudaMemsetAsync(arena, 0, need, st));
  size_t got = 0;
  if (build(h, h->bwd, (uint8_t*)arena, grads, &got)) return -1;
  for (int part = 0; part < h->nparts; ++part)
    if (check_same_plan(sized[part], h->bwd[part])) return -1;
  for (int part = 0; part < h->nparts; ++part) h->bwd[part]->arena_bytes = got;
  return 0;
}

static int backward_launch_count(const NetBase* h) {   // the last backward of every part
  int n = 0;
  for (int part = 0; h && part < h->nparts; ++part) n += h->bwd[part] ? h->bwd[part]->launches : 0;
  return n;
}

}  // namespace b200ad

// ================================================================================= C ABI: the handle protocol
extern "C" int b200ad_unet_set_training(b200ad_unet* h, int on) { return set_training(h, on); }
extern "C" size_t b200ad_unet_grad_floats(b200ad_unet* h) { ensure_bwd(h); return h->bwd[0]->grad_floats; }
extern "C" size_t b200ad_unet_grad_offset(b200ad_unet* h, int i) { ensure_bwd(h); return h->bwd[0]->goff[i]; }
extern "C" size_t b200ad_unet_backward_bytes(b200ad_unet* h) { return backward_bytes(h, build_unet_backward); }
extern "C" int b200ad_unet_bind_backward(b200ad_unet* h, void* arena, size_t bytes, float* grads, void* stream) {
  return bind_backward(h, build_unet_backward, arena, bytes, grads, (cudaStream_t)stream);
}
extern "C" int b200ad_unet_backward_launch_count(const b200ad_unet* h) { return backward_launch_count(h); }
extern "C" int b200ad_unet_debug_grad(b200ad_unet* h, const char* name, int skip, float* dst, int* dims, void* stream) {
  return debug_grad(h, name, skip, dst, dims, (cudaStream_t)stream);
}

extern "C" int b200ad_vae_set_training(b200ad_vae* h, int on) { return set_training(h, on); }
extern "C" size_t b200ad_vae_grad_floats(b200ad_vae* h) { ensure_bwd(h); return h->bwd[0]->grad_floats; }
extern "C" size_t b200ad_vae_grad_offset(b200ad_vae* h, int i) { ensure_bwd(h); return h->bwd[0]->goff[i]; }
extern "C" size_t b200ad_vae_backward_bytes(b200ad_vae* h) { return backward_bytes(h, build_vae_backward); }
extern "C" int b200ad_vae_bind_backward(b200ad_vae* h, void* arena, size_t bytes, float* grads, void* stream) {
  return bind_backward(h, build_vae_backward, arena, bytes, grads, (cudaStream_t)stream);
}
extern "C" int b200ad_vae_backward_launch_count(const b200ad_vae* h) { return backward_launch_count(h); }
extern "C" int b200ad_vae_debug_grad(b200ad_vae* h, const char* name, int skip, float* dst, int* dims, void* stream) {
  return debug_grad(h, name, skip, dst, dims, (cudaStream_t)stream);
}

extern "C" int b200ad_vae_decoder_backward(b200ad_vae* h, const float* g_x, float* g_z_out, int accumulate, void* stream) {
  if (!g_x || !g_z_out) return set_err("decoder_backward: g_x and g_z_out are required");
  RunArgs a;
  a.g_eps = g_x; a.g_z = g_z_out;
  return run_backward(h, DEC, a, accumulate, (cudaStream_t)stream);
}

extern "C" int b200ad_vae_encoder_backward(b200ad_vae* h, const float* x, const float* g_moments, int accumulate,
                                           void* stream) {
  if (!x || !g_moments) return set_err("encoder_backward: x and g_moments are required");
  RunArgs a;
  a.in = x; a.g_mom = g_moments;
  return run_backward(h, ENC, a, accumulate, (cudaStream_t)stream);
}

extern "C" int b200ad_unet_backward(b200ad_unet* h, const float* x, const float* g_eps, int accumulate, void* stream) {
  if (!x || !g_eps) return set_err("backward: x and g_eps are required");
  if (h && h->cfg.cross_attention_dim && !h->enc) return set_err("backward: the conditional U-Net needs the forward's encoding bound");
  if (h && h->cfg.cross_attention_dim && h->bwd[0] && !h->bwd[0]->list.ops.empty()) {
    const int planned = h->bwd[0]->enc_len;
    if (planned != h->plan_enc_len)
      return set_err("backward: the backward plan was built for %d encoder tokens but the workspace is planned for %d "
                     "(call bind_backward again)", planned, h->plan_enc_len);
    if (h->enc_S != planned)
      return set_err("backward: the bound encoding has %d tokens but the plan was built for %d", h->enc_S, planned);
  }
  RunArgs a;
  a.in = x; a.g_eps = g_eps;
  return run_backward(h, 0, a, accumulate, (cudaStream_t)stream);
}
