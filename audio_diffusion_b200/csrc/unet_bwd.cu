// Backward pass of the U-Net (scripts/train_unet.py:259, `accelerator.backward(loss)`): walks UNet2DModel.forward in
// reverse over the activations the training-mode forward kept (no buffer pooling), and fills one flat fp32 buffer with
// the gradients of all parameters.
//   * data gradients of every convolution run on conv_tc_kernel with transposed / mirrored weight packing (stride-2 convs
//     as four scatter launches, the folded upsampling convs as one gather launch over the parity planes of the gradient);
//   * weight gradients run on wgrad_tc_kernel (wgmma, pixels as the reduction dimension, MN-major operands);
//   * GroupNorm(+SiLU), attention core, biases / time embedding, conv_in / conv_out are memory-bound kernels (bwd_kernels.cu).
// This first version materialises the normalised activations for the weight gradients (no fusion yet) — DESIGN.md §6.
#include "bwd_kernels.cuh"
#include "unet.cuh"

using namespace b200ad;

namespace b200ad {

struct View {            // channel range of a PF8 tensor
  const __nv_bfloat16* p = nullptr;   // first plane of the view (image 0)
  int C = 0, img_planes = 0, H = 0, W = 0;
};

struct BOp {
  enum Kind { CONV, WGRAD, GNBWD, GNAPPLY, CHANSUM, REDUCE_N, SCATTER, PF8ADD, ATTNBWD, PARITY, UNFOLD, SCALAR_WGRAD, CONVIN,
              FLIP, SUMADD, LIN_IN, LIN_W, SILU_BWD, SILU_FWD, MEMSET } kind;
  ConvParams conv;
  WgradDesc wg;
  GnBwdParams gb;
  GnApplyParams ga;
  UnfoldMasks um;
  const __nv_bfloat16* src = nullptr;
  const __nv_bfloat16* src2 = nullptr;
  __nv_bfloat16* dst = nullptr;
  const float* f0 = nullptr;
  const float* f1 = nullptr;
  float* o0 = nullptr;
  float* o1 = nullptr;
  int C = 0, H = 0, W = 0, a = 0, b = 0, c = 0, d = 0;
  long long n = 0;
  bool x_is_input = false;    // SCALAR_WGRAD: X = the forward input image passed to backward()
  bool x_is_geps = false;     // X / source = the output gradient passed to backward()
};

}  // namespace b200ad

struct Backward {
  std::vector<BOp> ops;
  std::vector<PackJob> jobs;         // transposed weight packs, redone at every backward (the weights move every step)
  std::vector<size_t> goff;          // float offset of every parameter's gradient in the flat buffer
  size_t grad_floats = 0;
  uint8_t* arena = nullptr;
  size_t arena_bytes = 0;
  float* grads = nullptr;
  int launches = 0;
  PackBatch pack_batch;              // one launch for all transposed packs
  // gradient buckets (data-parallel all-reduce overlapped with the rest of the backward pass): bucket k = floats
  // [bucket_lo[k], bucket_lo[k+1]); its event is recorded right after the last launch that adds into it
  std::vector<size_t> bucket_lo;
  std::vector<cudaEvent_t> bucket_ev;
  std::vector<int> bucket_last_op;   // index into ops (-1: nothing writes it -> recorded before the first op)
};

static void free_bucket_events(Backward* bw) {
  for (cudaEvent_t e : bw->bucket_ev) cudaEventDestroy(e);
  bw->bucket_ev.clear();
  bw->bucket_lo.clear();
  bw->bucket_last_op.clear();
}


namespace b200ad {

struct BwdBuilder {
  b200ad_unet* h;
  Backward* bw;
  Bump mem;                                   // arena allocator (base == nullptr: size pass)
  std::map<std::string, Act> grad;            // gradient w.r.t. a forward tensor (by tap name)
  std::map<std::string, Act> skipgrad;        // contribution of the skip connection to that gradient
  std::map<std::string, Act> pool;
  std::map<std::string, size_t> toff;         // transposed packed weights
  int N;
  float* cs = nullptr;                        // [N][maxC] channel sums scratch
  float* gsums = nullptr;                     // GroupNorm backward scratch [N][maxC][2]
  float* gproj = nullptr;                     // [N][temb_rows]
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
  const Act& fwd(const std::string& name) const { return h->taps.at(name); }
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
  const __nv_bfloat16* WT(const std::string& key) const {
    return bw->arena ? (const __nv_bfloat16*)(bw->arena + toff.at(key)) : nullptr;
  }
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
  void tjob(const std::string& key, const std::string& wname, int O, int I, int K, const PackTaps& taps_in) {
    PackJob j;
    j.w_param = h->pidx.at(wname);
    j.cout = I; j.cin_total = O; j.KH = K; j.KW = K; j.cin_off = 0; j.ksteps = O / 16;
    j.taps = taps_in;
    j.taps.transpose = 1;
    j.cout_real = I;
    j.off = take_off(mem, (size_t)(I / 128) * j.ksteps * taps_in.ntaps * CONV_B_TAP);
    toff[key] = j.off;
    bw->jobs.push_back(j);
  }
  static PackTaps mirrored(int K) {
    PackTaps t{};
    t.ntaps = K * K;
    for (int k = 0; k < K * K; ++k) { t.kh[k] = K - 1 - k / K; t.kw[k] = K - 1 - k % K; }
    return t;
  }

  // ---- op emitters ------------------------------------------------------------------------------------------------
  void conv_base(ConvParams& p, const Act& out) {
    const Geom g = make_geom(N, out.H, out.W);
    p = ConvParams{};
    p.N = N; p.H = out.H; p.W = out.W; p.Wp = g.Wp; p.lead = g.lead; p.PL = g.PL;
    p.cout = out.C; p.out = out.p;
  }
  static void seg(ConvSeg& s, const View& src, const __nv_bfloat16* wpack, int ntaps, const signed char* dh,
                  const signed char* dw) {
    const Geom g = make_geom(1, src.H, src.W);
    s.src = src.p; s.wpack = wpack;
    s.img_stride = (long long)src.img_planes * g.PL * 8;
    s.ksteps = src.C / 16;
    s.ntaps = ntaps;
    s.ht = s.hb = s.hl = s.hr = 0;
    for (int t = 0; t < ntaps; ++t) {
      s.dh[t] = dh[t]; s.dw[t] = dw[t];
      if (dh[t] < 0) s.ht = 1;
      if (dh[t] > 0) s.hb = 1;
      if (dw[t] < 0) s.hl = 1;
      if (dw[t] > 0) s.hr = 1;
    }
    s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
  }
  // data gradient of a stride-1 KxK conv: out (I channels) = conv^T(gy (O channels))
  void dgrad(const std::string& key, const std::string& wname, const View& gy, const Act& out, int K) {
    tjob(key, wname, gy.C, out.C, K, mirrored(K));
    BOp op{};
    op.kind = BOp::CONV;
    conv_base(op.conv, out);
    signed char dh[9], dw[9];
    for (int k = 0; k < K * K; ++k) { dh[k] = (signed char)(k / K - K / 2); dw[k] = (signed char)(k % K - K / 2); }
    seg(op.conv.seg[0], gy, WT(key), K * K, dh, dw);
    op.conv.nseg = 1;
    bw->ops.push_back(op);
  }
  void wgrad(const View& gy, const View& act, float* dw, int cin_total, int ci_off, int ntaps_total, int ntaps,
             const signed char* dh, const signed char* dwv, const int* tapidx) {
    BOp op{};
    op.kind = BOp::WGRAD;
    WgradDesc& d = op.wg;
    d.gy = gy.p; d.act = act.p; d.dw = dw; d.N = N; d.H = gy.H; d.W = gy.W; d.cout = gy.C; d.cin = act.C;
    d.gy_img_planes = gy.img_planes; d.act_img_planes = act.img_planes;
    d.cin_total = cin_total; d.ci_off = ci_off; d.ntaps_total = ntaps_total; d.ntaps = ntaps;
    for (int t = 0; t < ntaps; ++t) { d.dh[t] = dh[t]; d.dw_[t] = dwv[t]; d.tapidx[t] = tapidx[t]; }
    bw->ops.push_back(op);
  }
  void wgrad_conv(const View& gy, const View& act, const std::string& wname, int K) {   // plain stride-1 conv
    signed char dh[9], dw[9];
    int ti[9];
    for (int k = 0; k < K * K; ++k) { dh[k] = (signed char)(k / K - K / 2); dw[k] = (signed char)(k % K - K / 2); ti[k] = k; }
    wgrad(gy, act, PG(wname), act.C, 0, K * K, K * K, dh, dw, ti);
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
  Act gn_apply(const std::string& tag, const Act& a, const Act* b, const std::string& norm, bool silu) {
    const int Ct = a.C + (b ? b->C : 0);
    Act out = tmp(tag, Ct, a.H, a.W);
    BOp op{};
    op.kind = BOp::GNAPPLY;
    GnApplyParams& p = op.ga;
    p.src[0] = a.p; p.stats[0] = a.stats; p.C[0] = a.C;
    p.src[1] = b ? b->p : nullptr; p.stats[1] = b ? b->stats : nullptr; p.C[1] = b ? b->C : 0;
    p.gamma = P(norm + ".weight"); p.beta = P(norm + ".bias");
    p.dst = out.p; p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = h->norm_eps; p.silu = silu ? 1 : 0;
    bw->ops.push_back(op);
    return out;
  }
  void gn_bwd(const Act& ga, const Act& a, const Act* b, const std::string& norm, bool silu, const Act& d0, const Act* d1,
              const __nv_bfloat16* addS, const __nv_bfloat16* add0) {
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
    {
      static const bool off = [] { const char* e = getenv("B200AD_NO_CSUM_FUSE"); return e && e[0] == '1'; }();   // A/B switch
      const size_t need = (size_t)N * a.C;
      if (!off && csum_used + need <= csum_floats) {
        p.csum0 = csum_arena ? csum_arena + csum_used : nullptr;
        csum_of[d0.p] = p.csum0;
        csum_used += need;
        if (!csum_arena) csum_of[d0.p] = (float*)1;           // size pass: the plan must have the same shape as the real one
      }
    }
    p.N = N; p.H = a.H; p.W = a.W; p.groups = h->norm_groups; p.eps = h->norm_eps; p.silu = silu ? 1 : 0;
    bw->ops.push_back(op);
  }
  const __nv_bfloat16* skip_of(const std::string& name) const {
    auto it = skipgrad.find(name);
    return it == skipgrad.end() ? nullptr : it->second.p;
  }

  // ---- blocks -----------------------------------------------------------------------------------------------------
  // ResnetBlock2D n over cat(a, b): consumes G(n), produces G(a) and (if b) the skip contribution of b.
  void resnet_bwd(const std::string& n, const std::string& an, const std::string& bn) {
    const Act a = fwd(an);
    const bool has_b = !bn.empty();
    Act bsrc;
    if (has_b) bsrc = fwd(bn);
    const Act h1 = fwd(n + ".h1"), out = fwd(n);
    const int co = out.C, Ct = a.C + (has_b ? bsrc.C : 0), H = out.H, W = out.W;
    const Act Gout = G(n);
    // conv2
    Act T1 = tmp("T1", co, H, W);
    dgrad(n + ".conv2.T", n + ".conv2.weight", whole(Gout), T1, 3);
    Act A = gn_apply("A", h1, nullptr, n + ".norm2", true);
    wgrad_conv(whole(Gout), whole(A), n + ".conv2.weight", 3);
    const bool sc = Ct != co;
    bias_grad(whole(Gout), n + ".conv2.bias", sc ? n + ".conv_shortcut.bias" : "");
    // norm2 + SiLU
    Act Gh1 = tmp("Gh1", co, H, W);
    gn_bwd(T1, h1, nullptr, n + ".norm2", true, Gh1, nullptr, nullptr, nullptr);
    // conv1 bias + time embedding projection rows of this block
    bias_grad(whole(Gh1), n + ".conv1.bias");
    {
      BOp op{};
      op.kind = BOp::SCATTER;
      op.f0 = last_cs; op.o0 = gproj; op.C = co; op.a = h->temb_rows; op.b = h->temb_row_off.at(n);
      bw->ops.push_back(op);
    }
    // conv1
    Act T2 = tmp("T2", Ct, H, W);
    dgrad(n + ".conv1.T", n + ".conv1.weight", whole(Gh1), T2, 3);
    Act A2 = gn_apply("A2", a, has_b ? &bsrc : nullptr, n + ".norm1", true);
    wgrad_conv(whole(Gh1), whole(A2), n + ".conv1.weight", 3);
    // shortcut
    const __nv_bfloat16* addS;
    if (sc) {
      Act T3 = tmp("T3", Ct, H, W);
      dgrad(n + ".conv_shortcut.T", n + ".conv_shortcut.weight", whole(Gout), T3, 1);
      const signed char z = 0;
      const int zi = 0;
      wgrad(whole(Gout), whole(a), PG(n + ".conv_shortcut.weight"), Ct, 0, 1, 1, &z, &z, &zi);
      if (has_b) wgrad(whole(Gout), whole(bsrc), PG(n + ".conv_shortcut.weight"), Ct, a.C, 1, 1, &z, &z, &zi);
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
    dgrad(n + ".to_out.T", n + ".to_out.0.weight", whole(Gout), T1, 1);
    wgrad_conv(whole(Gout), whole(ao), n + ".to_out.0.weight", 1);
    bias_grad(whole(Gout), n + ".to_out.0.bias");
    Act Gqkv = tmp("Gqkv", 3 * C, H, W);
    {
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
      const signed char z = 0;
      for (int k = 0; k < 3; ++k) {
        const std::string key = n + "." + names[k] + ".T";
        tjob(key, n + "." + names[k] + ".weight", C, C, 1, mirrored(1));
        seg(op.conv.seg[k], view(Gqkv, k * C, C), WT(key), 1, &z, &z);
      }
      op.conv.nseg = 3;
      bw->ops.push_back(op);
    }
    gn_bwd(T2, x, nullptr, n + ".group_norm", false, G(xn), nullptr, Gout.p, skip_of(xn));
  }

  // Downsample2D: stride-2 3x3 conv on the raw tensor xn -> y (tap n)
  void downsample_bwd(const std::string& n, const std::string& xn) {
    const Act x = fwd(xn), y = fwd(n), par = fwd(n + ".parity");
    const int C = x.C, Ho = y.H, Wo = y.W;
    const Act Gy = G(n);
    const Geom go = make_geom(N, Ho, Wo);
    const size_t tsz = (size_t)N * (C / 8) * go.PL * 8;
    bias_grad(whole(Gy), n + ".bias");
    // weight gradient: per parity plane (a, b) of x the taps that read it (forward: taps_parity)
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const PackTaps pt = taps_parity(a, b);
        signed char dh[9], dw[9];
        int ti[9];
        for (int t = 0; t < pt.ntaps; ++t) {
          dh[t] = (pt.kh[t] == 0) ? -1 : 0; dw[t] = (pt.kw[t] == 0) ? -1 : 0; ti[t] = pt.kh[t] * 3 + pt.kw[t];
        }
        Act plane = par;
        plane.C = C; plane.H = Ho; plane.W = Wo;
        plane.p = par.p ? par.p + (size_t)(a * 2 + b) * tsz : nullptr;
        wgrad(whole(Gy), whole(plane), PG(n + ".weight"), C, 0, 9, pt.ntaps, dh, dw, ti);
      }
    // data gradient: input parity (a, b) <- taps with matching parity, scattered into the 2x tensor
    Act Gx = G(xn);
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        PackTaps pt{};
        signed char dh[9], dw[9];
        const int khs[2][2] = {{1, -1}, {0, 2}};      // a = 0: kh 1;  a = 1: kh 0 (dh +1), kh 2 (dh 0)
        for (int i = 0; i < 2; ++i)
          for (int j = 0; j < 2; ++j) {
            const int kh = khs[a][i], kw = khs[b][j];
            if (kh < 0 || kw < 0) continue;
            pt.kh[pt.ntaps] = kh; pt.kw[pt.ntaps] = kw;
            dh[pt.ntaps] = (kh == 0) ? 1 : 0; dw[pt.ntaps] = (kw == 0) ? 1 : 0;
            ++pt.ntaps;
          }
        const std::string key = n + S(".T%d", a * 2 + b);
        tjob(key, n + ".weight", C, C, 3, pt);
        BOp op{};
        op.kind = BOp::CONV;
        Act lo = Gx;
        lo.H = Ho; lo.W = Wo;
        conv_base(op.conv, lo);
        op.conv.up2 = 1; op.conv.oy = a; op.conv.ox = b;
        seg(op.conv.seg[0], whole(Gy), WT(key), pt.ntaps, dh, dw);
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
        const UpTaps ut = taps_up2(oy, ox);
        Act plane;
        plane.C = C; plane.H = H; plane.W = W;
        plane.p = gpar.p ? gpar.p + (size_t)pidx * tsz : nullptr;
        int ti[4] = {0, 1, 2, 3};
        wgrad(whole(plane), whole(x), dwf ? dwf + (size_t)pidx * C * C * 4 : nullptr, C, 0, 4, 4, ut.dh, ut.dw, ti);
        for (int t = 0; t < 4; ++t) um.mask[pidx][t] = ut.pack.fold_mask[t];
        const std::string key = n + S(".T%d", pidx);
        tjob(key, n + ".weight", C, C, 3, ut.pack);
        signed char ndh[4], ndw[4];
        for (int t = 0; t < 4; ++t) { ndh[t] = (signed char)-ut.dh[t]; ndw[t] = (signed char)-ut.dw[t]; }
        seg(dg.conv.seg[pidx], whole(plane), WT(key), 4, ndh, ndw);
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
};

struct Rec {
  int kind;  // 0 resnet, 1 attention, 2 down, 3 up
  std::string n, a, b;
};

static int build_backward(b200ad_unet* h, Backward* bw, uint8_t* arena, float* grads, size_t* bytes_out) {
  const b200ad_unet_config& c = h->cfg;
  const int nb = c.num_blocks;
  if (!h->training || h->plan.empty()) return set_err("backward needs set_training(1) before bind_workspace");
  bw->ops.clear();
  bw->jobs.clear();
  bw->arena = arena;
  bw->grads = grads;
  BwdBuilder B;
  B.h = h; B.bw = bw; B.N = h->N;
  B.mem.base = arena;
  // forward structure, by tensor name (mirrors build_plan in unet.cu)
  std::vector<Rec> recs;
  std::string cur = "conv_in";
  std::vector<std::string> skips{cur};
  int maxC = c.block_out_channels[0];
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < c.layers_per_block; ++j) {
      const std::string rn = S("down_blocks.%d.resnets.%d", i, j);
      recs.push_back({0, rn, cur, ""});
      cur = rn;
      if (c.down_attn[i]) {
        const std::string an = S("down_blocks.%d.attentions.%d", i, j);
        recs.push_back({1, an, cur, ""});
        cur = an;
      }
      skips.push_back(cur);
    }
    if (i != nb - 1) {
      const std::string dn = S("down_blocks.%d.downsamplers.0.conv", i);
      recs.push_back({2, dn, cur, ""});
      cur = dn;
      skips.push_back(cur);
    }
  }
  recs.push_back({0, "mid_block.resnets.0", cur, ""});
  recs.push_back({1, "mid_block.attentions.0", "mid_block.resnets.0", ""});
  recs.push_back({0, "mid_block.resnets.1", "mid_block.attentions.0", ""});
  cur = "mid_block.resnets.1";
  for (int i = 0; i < nb; ++i) {
    for (int j = 0; j < c.layers_per_block + 1; ++j) {
      const std::string sk = skips.back();
      skips.pop_back();
      const std::string rn = S("up_blocks.%d.resnets.%d", i, j);
      recs.push_back({0, rn, cur, sk});
      cur = rn;
      if (c.up_attn[i]) {
        const std::string an = S("up_blocks.%d.attentions.%d", i, j);
        recs.push_back({1, an, cur, ""});
        cur = an;
      }
    }
    if (i != nb - 1) {
      const std::string un = S("up_blocks.%d.upsamplers.0.conv", i);
      recs.push_back({3, un, cur, ""});
      cur = un;
    }
  }
  for (const auto& kv : h->taps) maxC = kv.second.C > maxC ? kv.second.C : maxC;
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

  // ---- conv_out: g_eps -> gradient of the last activation ---------------------------------------------------------
  {
    const Act x = h->taps.at("pre_out");
    const int C = x.C;
    if (c.out_channels != 1) return set_err("backward: out_channels != 1 is not implemented");
    Act A = B.gn_apply("A", x, nullptr, "conv_norm_out", true);
    BOp w{};
    w.kind = BOp::SCALAR_WGRAD;
    w.src = A.p; w.x_is_geps = true; w.o0 = B.PG("conv_out.weight"); w.C = C; w.H = x.H; w.W = x.W; w.a = 1;
    bw->ops.push_back(w);
    BOp sb{};
    sb.kind = BOp::SUMADD;
    sb.x_is_geps = true; sb.n = (long long)h->N * x.H * x.W; sb.o0 = B.PG("conv_out.bias");
    bw->ops.push_back(sb);
    BOp f{};
    f.kind = BOp::FLIP;
    f.f0 = B.P("conv_out.weight"); f.o0 = wflip; f.C = C;
    bw->ops.push_back(f);
    Act T1 = B.tmp("T1", C, x.H, x.W);
    BOp ci{};
    ci.kind = BOp::CONVIN;        // conv_in kernel: g_a[c] = sum_t g_eps[p + s_t] * wflip[c][t]
    ci.x_is_geps = true; ci.f0 = wflip; ci.f1 = zbias; ci.dst = T1.p; ci.C = C; ci.H = x.H; ci.W = x.W;
    bw->ops.push_back(ci);
    B.gn_bwd(T1, x, nullptr, "conv_norm_out", true, B.G(cur), nullptr, nullptr, nullptr);
  }
  // ---- blocks in reverse ------------------------------------------------------------------------------------------
  {
    BOp z{};
    z.kind = BOp::MEMSET;
    z.o0 = B.gproj; z.n = (long long)h->N * h->temb_rows * sizeof(float);
    bw->ops.push_back(z);
  }
  for (int r = (int)recs.size() - 1; r >= 0; --r) {
    const Rec& rc = recs[r];
    if (rc.kind == 0) B.resnet_bwd(rc.n, rc.a, rc.b);
    else if (rc.kind == 1) B.attention_bwd(rc.n, rc.a);
    else if (rc.kind == 2) B.downsample_bwd(rc.n, rc.a);
    else B.upsample_bwd(rc.n, rc.a);
  }
  // ---- conv_in ----------------------------------------------------------------------------------------------------
  {
    if (c.in_channels != 1) return set_err("backward: in_channels != 1 is not implemented");
    const Act x = h->taps.at("conv_in");
    const Act Gx = B.G("conv_in");
    if (!B.skipgrad.count("conv_in")) return set_err("backward: conv_in skip gradient missing");
    // (the first resnet's GroupNorm backward already added the skip contribution)
    BOp w{};
    w.kind = BOp::SCALAR_WGRAD;
    w.src = Gx.p; w.x_is_input = true; w.o0 = B.PG("conv_in.weight"); w.C = x.C; w.H = x.H; w.W = x.W; w.a = 0;
    bw->ops.push_back(w);
    B.bias_grad(BwdBuilder::whole(Gx), "conv_in.bias");
  }
  // ---- timestep embedding MLP and the per-resnet projections ------------------------------------------------------
  {
    const int d0 = c.block_out_channels[0];
    for (const auto& kv : h->temb_row_off) {     // time_emb_proj of every resnet: dW = g_proj_rows^T temb_act
      const int co = (int)h->params[h->pidx.at(kv.first + ".time_emb_proj.bias")].shape[0];
      BOp op{};
      op.kind = BOp::LIN_W;
      op.f0 = B.gproj + kv.second; op.a = h->temb_rows; op.f1 = h->temb_act; op.b = co; op.c = D;
      op.o0 = B.PG(kv.first + ".time_emb_proj.weight"); op.o1 = B.PG(kv.first + ".time_emb_proj.bias");
      bw->ops.push_back(op);
    }
    BOp gi{};
    gi.kind = BOp::LIN_IN;   // g(temb_act) = g_proj Wcat
    gi.f0 = B.gproj; gi.a = h->temb_rows; gi.f1 = h->packed ? (const float*)(h->packed + h->off_wcat) : nullptr;
    gi.b = h->temb_rows; gi.c = D; gi.o0 = g_act;
    bw->ops.push_back(gi);
    BOp s2{};
    s2.kind = BOp::SILU_BWD;
    s2.o0 = g_act; s2.f0 = h->temb_u2; s2.n = (long long)h->N * D;
    bw->ops.push_back(s2);
    BOp hf{};
    hf.kind = BOp::SILU_FWD;
    hf.f0 = h->temb_u1; hf.o0 = h1v; hf.n = (long long)h->N * D;
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
    s1.o0 = g_h1; s1.f0 = h->temb_u1; s1.n = (long long)h->N * D;
    bw->ops.push_back(s1);
    BOp w1{};
    w1.kind = BOp::LIN_W;
    w1.f0 = g_h1; w1.a = D; w1.f1 = h->temb_emb; w1.b = D; w1.c = d0;
    w1.o0 = B.PG("time_embedding.linear_1.weight"); w1.o1 = B.PG("time_embedding.linear_1.bias");
    bw->ops.push_back(w1);
  }
  if (bytes_out) *bytes_out = (B.mem.off + 255) & ~(size_t)255;
  return 0;
}

}  // namespace b200ad

namespace b200ad {
void release_backward(b200ad_unet* h) {
  if (h->bwd) free_bucket_events(h->bwd);
  delete h->bwd;
  h->bwd = nullptr;
}
}  // namespace b200ad

// ================================================================================= C ABI
extern "C" int b200ad_unet_set_training(b200ad_unet* h, int on) {
  if (!h) return set_err("null handle");
  if (on && h->cfg.cross_attention_dim) return set_err("training of the conditional U-Net is not implemented (inference only)");
  if (h->training != (on != 0)) {
    h->training = on != 0;
    h->plan.clear();          // the workspace layout changes: bind_workspace must be called again
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
  free_bucket_events(h->bwd);          // the op list is rebuilt: buckets must be set again
  if (build_backward(h, h->bwd, (uint8_t*)arena, grads, &need)) return -1;
  h->bwd->arena_bytes = need;
  return 0;
}

extern "C" int b200ad_unet_backward(b200ad_unet* h, const float* x, const float* g_eps, int accumulate, void* stream) {
  if (!h || !h->bwd || h->bwd->ops.empty()) return set_err("bind_backward must be called before backward");
  if (!x || !g_eps) return set_err("backward: x and g_eps are required");
  Backward* bw = h->bwd;
  cudaStream_t st = (cudaStream_t)stream;
  const int N = h->N;
  int launches = 0;
  // B200AD_BWD_PROFILE=1: CUDA events around every op, per-kind totals printed to stderr (tools/train_bench.py)
  static const bool prof = [] { const char* e = getenv("B200AD_BWD_PROFILE"); return e && e[0] == '1'; }();
  std::vector<cudaEvent_t> ev;
  if (prof) {
    ev.resize(bw->ops.size() + 2);
    for (auto& e : ev) CK(cudaEventCreate(&e));
    CK(cudaEventRecord(ev[0], st));
  }
  if (!accumulate) CK(cudaMemsetAsync(bw->grads, 0, bw->grad_floats * sizeof(float), st));   // every kernel below ADDS
  {
    std::vector<PackItem> items;
    items.reserve(bw->jobs.size());
    for (const PackJob& j : bw->jobs) items.push_back(make_pack_item(h, j, bw->arena));
    CK(launch_pack_batch(bw->pack_batch, items, st));
  }
  launches += 1;
  if (prof) CK(cudaEventRecord(ev[1], st));
  size_t opi = 0;
  for (size_t k = 0; k < bw->bucket_ev.size(); ++k)
    if (bw->bucket_last_op[k] < 0) CK(cudaEventRecord(bw->bucket_ev[k], st));
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
      case BOp::SCALAR_WGRAD:
        CK(launch_scalar_conv_wgrad(op.src, op.x_is_geps ? g_eps : x, op.o0, N, op.C, op.H, op.W, op.a, st));
        break;
      case BOp::CONVIN:
        CK(launch_conv_in(g_eps, op.f0, op.f1, N, 1, op.H, op.W, op.C, op.dst, nullptr, st));
        break;
      case BOp::FLIP: CK(launch_flip_taps(op.f0, op.o0, op.C, st)); break;
      case BOp::SUMADD: CK(launch_sum_add(g_eps, op.n, op.o0, st)); break;
      case BOp::LIN_IN: CK(launch_lin_bwd_input(op.f0, op.a, op.f1, op.b, op.c, op.o0, N, 0, st)); break;
      case BOp::LIN_W: CK(launch_lin_bwd_weight(op.f0, op.a, op.f1, op.b, op.c, op.o0, op.o1, N, st)); break;
      case BOp::SILU_BWD: CK(launch_silu_bwd(op.o0, op.f0, (int)op.n, st)); break;
      case BOp::SILU_FWD: CK(launch_silu_fwd(op.f0, op.o0, (int)op.n, st)); break;
      case BOp::MEMSET: CK(cudaMemsetAsync(op.o0, 0, (size_t)op.n, st)); break;
    }
    ++launches;
    if (prof) CK(cudaEventRecord(ev[2 + opi], st));
    for (size_t k = 0; k < bw->bucket_ev.size(); ++k)
      if (bw->bucket_last_op[k] == (int)opi) CK(cudaEventRecord(bw->bucket_ev[k], st));
    ++opi;
  }
  bw->launches = launches;
  if (prof) {
    static const char* names[] = {"conv_tc(dgrad)", "wgrad_tc", "gn_bwd", "gn_apply", "chan_sum", "reduce_n", "scatter",
                                  "pf8_add", "attention_bwd", "parity_split", "unfold_up2", "scalar_wgrad", "conv_in(dgrad)",
                                  "flip", "sum_add", "lin_in", "lin_w", "silu_bwd", "silu_fwd", "memset"};
    CK(cudaStreamSynchronize(st));
    double tot[20] = {0};
    int cnt[20] = {0};
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    fprintf(stderr, "{\"backward_profile_ms\": {\"pack_transposed\": %.3f", ms);
    for (size_t i = 0; i < bw->ops.size(); ++i) {
      CK(cudaEventElapsedTime(&ms, ev[1 + i], ev[2 + i]));
      tot[bw->ops[i].kind] += ms;
      cnt[bw->ops[i].kind]++;
    }
    for (int k = 0; k < 20; ++k)
      if (cnt[k]) fprintf(stderr, ", \"%s x%d\": %.3f", names[k], cnt[k], tot[k]);
    fprintf(stderr, "}}\n");
    for (auto& e : ev) cudaEventDestroy(e);
  }
  return 0;
}

extern "C" int b200ad_unet_backward_launch_count(const b200ad_unet* h) { return h && h->bwd ? h->bwd->launches : 0; }

extern "C" int b200ad_unet_set_grad_buckets(b200ad_unet* h, int n, const size_t* lo) {
  if (!h || !h->bwd || !h->bwd->grads) return set_err("set_grad_buckets: bind_backward first");
  Backward* bw = h->bwd;
  free_bucket_events(bw);
  if (n <= 0) return 0;
  if (n > 64 || !lo || lo[0] != 0 || lo[n] != bw->grad_floats) return set_err("set_grad_buckets: bad bucket table");
  for (int k = 0; k < n; ++k)
    if (lo[k + 1] <= lo[k]) return set_err("set_grad_buckets: boundaries must ascend");
  bw->bucket_lo.assign(lo, lo + n + 1);
  bw->bucket_last_op.assign(n, -1);
  // every float* an op may ADD parameter gradients through (an over-approximation only delays an event)
  for (size_t i = 0; i < bw->ops.size(); ++i) {
    const BOp& op = bw->ops[i];
    const float* outs[6] = {op.wg.dw, op.gb.dgamma, op.gb.dbeta, op.o0, op.o1, op.f1};
    for (const float* q : outs) {
      if (!q || q < bw->grads || q >= bw->grads + bw->grad_floats) continue;
      const size_t off = (size_t)(q - bw->grads);
      for (int k = 0; k < n; ++k)
        if (off >= lo[k] && off < lo[k + 1]) bw->bucket_last_op[k] = (int)i;
    }
  }
  bw->bucket_ev.resize(n);
  for (int k = 0; k < n; ++k) CK(cudaEventCreateWithFlags(&bw->bucket_ev[k], cudaEventDisableTiming));
  return 0;
}

extern "C" int b200ad_unet_grad_bucket_wait(b200ad_unet* h, int k, void* stream) {
  if (!h || !h->bwd || k < 0 || k >= (int)h->bwd->bucket_ev.size()) return set_err("grad_bucket_wait: no such bucket");
  CK(cudaStreamWaitEvent((cudaStream_t)stream, h->bwd->bucket_ev[k], 0));
  return 0;
}
