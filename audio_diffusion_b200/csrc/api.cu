// Op-level C-ABI entry points (parity tests drive single kernels through these) and small utilities.
#include <cstdio>
#include <cstring>

#include "../../include/b200ad.h"
#include "conv_tc.cuh"
#include "bwd_kernels.cuh"
#include "kernels.cuh"

namespace b200ad {
int set_err(const char* fmt, ...);
}
using namespace b200ad;

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (call);                                                         \
    if (e__ != cudaSuccess) return set_err("%s: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

static size_t al(size_t x) { return (x + 255) & ~(size_t)255; }

struct ConvScratch {
  size_t x, par, res, out, wpack, ident, stats, instats, ss, total;
};
static ConvScratch conv_scratch_layout(int N, int cin, int cout, int H, int W, int K, int stride) {
  ConvScratch s{};
  const Geom gi = make_geom(N, H, W);
  const int Ho = stride > 0 ? H / stride : 2 * H, Wo = stride > 0 ? W / stride : 2 * W;
  const Geom go = make_geom(N, Ho, Wo);
  size_t off = 0;
  s.x = off; off = al(off + (size_t)N * (cin / 8) * gi.PL * 16);
  s.par = off; if (stride == 2) off = al(off + (size_t)4 * N * (cin / 8) * go.PL * 16);
  s.res = off; off = al(off + (size_t)N * (cout / 8) * go.PL * 16);
  s.out = off; off = al(off + (size_t)N * (cout / 8) * go.PL * 16);
  s.wpack = off; off = al(off + (size_t)(cout / 128) * (cin / 16) * (K * K > 16 ? K * K : 16) * CONV_B_TAP);
  s.ident = off; off = al(off + (size_t)(cout / 128) * (cout / 16) * CONV_B_TAP);
  s.stats = off; off = al(off + (size_t)N * (cout / 4) * 2 * sizeof(stat_t));
  s.instats = off; off = al(off + (size_t)N * (cin / 4) * 2 * sizeof(stat_t));
  s.ss = off; off = al(off + (size_t)N * cin * sizeof(float2));
  s.total = off;
  return s;
}

extern "C" size_t b200ad_conv2d_scratch_bytes(int N, int cin, int cout, int H, int W, int K, int stride) {
  return conv_scratch_layout(N, cin, cout, H, W, K, stride).total;
}

static int conv2d_impl(const float* x, const float* w, const float* bias, const float* temb, const float* residual,
                       float* y, float* stats_out, int N, int cin, int cout, int H, int W, int K, int stride,
                       const float* gn_gamma, const float* gn_beta, int gn_groups, float gn_eps, int gn_silu,
                       void* scratch, size_t scratch_bytes, void* stream) {
  if (cin % 16 || cout % 128) return set_err("conv2d: cin %% 16 and cout %% 128 must be 0");
  if (!((K == 3 || K == 1) && (stride == 1 || ((stride == 2 || stride == -2) && K == 3)))) return set_err("conv2d: unsupported K/stride");
  if (stride == -2 && (residual || gn_gamma || temb)) return set_err("conv2d: upsample form takes no residual / GroupNorm / temb");
  if (stride == 2 && (H % 2 || W % 2)) return set_err("conv2d: stride 2 needs even H, W");
  if (stride == 2 && (residual || gn_gamma)) return set_err("conv2d: residual / fused GroupNorm need stride 1");
  const ConvScratch L = conv_scratch_layout(N, cin, cout, H, W, K, stride);
  if (scratch_bytes < L.total) return set_err("conv2d: scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sb = (uint8_t*)scratch;
  CK(cudaMemsetAsync(sb, 0, L.total, st));
  const int Ho = stride > 0 ? H / stride : 2 * H, Wo = stride > 0 ? W / stride : 2 * W;
  const Geom go = make_geom(N, Ho, Wo);
  __nv_bfloat16* xp = (__nv_bfloat16*)(sb + L.x);
  __nv_bfloat16* par = (__nv_bfloat16*)(sb + L.par);
  __nv_bfloat16* rp = (__nv_bfloat16*)(sb + L.res);
  __nv_bfloat16* op = (__nv_bfloat16*)(sb + L.out);
  __nv_bfloat16* wp = (__nv_bfloat16*)(sb + L.wpack);
  stat_t* stp = (stat_t*)(sb + L.stats);
  CK(launch_nchw_to_pf8(x, xp, N, cin, H, W, st));
  if (residual) CK(launch_nchw_to_pf8(residual, rp, N, cout, Ho, Wo, st));

  ConvParams p{};
  p.N = N; p.H = Ho; p.W = Wo; p.Wp = go.Wp; p.lead = go.lead; p.PL = go.PL;
  p.cout = cout;
  p.out = op; p.bias = bias; p.temb = temb; p.temb_stride = cout;
  p.stats = stats_out ? stp : nullptr;
  const long long img_stride = (long long)(cin / 8) * go.PL * 8;
  if (stride == -2) {
    // segments are built per output parity below
  } else if (stride == 1) {
    PackTaps t{};
    t.ntaps = K * K;
    for (int k = 0; k < K * K; ++k) { t.kh[k] = k / K; t.kw[k] = k % K; }
    CK(launch_pack_weights(w, cout, cin, K, K, 0, cin / 16, t, wp, st));
    ConvSeg& s = p.seg[0];
    s.src = xp; s.wpack = wp; s.img_stride = img_stride; s.ksteps = cin / 16; s.ntaps = K * K;
    s.ht = s.hb = s.hl = s.hr = (K == 3) ? 1 : 0;
    for (int k = 0; k < K * K; ++k) { s.dh[k] = (signed char)(k / K - K / 2); s.dw[k] = (signed char)(k % K - K / 2); }
    s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
    p.nseg = 1;
    if (gn_gamma) {  // GroupNorm(+SiLU) of x fused into the conv's A staging
      stat_t* ist = (stat_t*)(sb + L.instats);
      float2* ss = (float2*)(sb + L.ss);
      CK(launch_quad_stats(xp, ist, N, cin, H, W, st));
      GnApplyParams g{};
      g.src[0] = xp; g.stats[0] = ist; g.C[0] = cin; g.C[1] = 0; g.gamma = gn_gamma; g.beta = gn_beta;
      g.N = N; g.H = H; g.W = W; g.groups = gn_groups; g.eps = gn_eps;
      CK(launch_gn_finalize(g, ss, st));
      s.ss = ss; s.ss_stride = cin; s.silu = gn_silu;
    }
    if (residual) {  // residual add = 1-tap identity-weight segment over the raw residual tensor
      __nv_bfloat16* ident = (__nv_bfloat16*)(sb + L.ident);
      CK(launch_pack_identity(cout, ident, st));
      ConvSeg& r = p.seg[1];
      r.src = rp; r.wpack = ident; r.img_stride = (long long)(cout / 8) * go.PL * 8; r.ksteps = cout / 16; r.ntaps = 1;
      r.ht = r.hb = r.hl = r.hr = 0; r.dh[0] = 0; r.dw[0] = 0; r.ss = nullptr; r.ss_stride = 0; r.silu = 0;
      p.nseg = 2;
    }
  } else {
    CK(launch_parity_split(xp, par, N, cin, H, W, st));
    const size_t tsz = (size_t)N * (cin / 8) * go.PL * 8;
    size_t woff = 0;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        PackTaps t{};
        for (int kh = 0; kh < 3; ++kh)
          for (int kw = 0; kw < 3; ++kw)
            if (((kh == 1) ? 0 : 1) == a && ((kw == 1) ? 0 : 1) == b) { t.kh[t.ntaps] = kh; t.kw[t.ntaps] = kw; ++t.ntaps; }
        __nv_bfloat16* wseg = wp + woff / 2;
        CK(launch_pack_weights(w, cout, cin, 3, 3, 0, cin / 16, t, wseg, st));
        woff += (size_t)(cout / 128) * (cin / 16) * t.ntaps * CONV_B_TAP;
        ConvSeg& s = p.seg[a * 2 + b];
        s.src = par + (size_t)(a * 2 + b) * tsz; s.wpack = wseg; s.img_stride = img_stride; s.ksteps = cin / 16;
        s.ntaps = t.ntaps;
        s.ht = a; s.hb = 0; s.hl = b; s.hr = 0; s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
        for (int k = 0; k < t.ntaps; ++k) { s.dh[k] = (t.kh[k] == 0) ? -1 : 0; s.dw[k] = (t.kw[k] == 0) ? -1 : 0; }
      }
    p.nseg = 4;
  }
  int dev = 0, sms = 132;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (stride == -2) {  // nearest-2x upsample + 3x3 conv as four folded 2x2 convs on the low-res input
    const Geom gi = make_geom(N, H, W);
    p.H = H; p.W = W; p.Wp = gi.Wp; p.lead = gi.lead; p.PL = gi.PL;
    p.up2 = 1;
    p.nseg = 1;
    size_t woff = 0;
    for (int pa = 0; pa < 2; ++pa)
      for (int pb = 0; pb < 2; ++pb) {
        const UpTaps ut = taps_up2(pa, pb);
        __nv_bfloat16* wseg = wp + woff / 2;
        CK(launch_pack_weights(w, cout, cin, 3, 3, 0, cin / 16, ut.pack, wseg, st));
        woff += (size_t)(cout / 128) * (cin / 16) * 4 * CONV_B_TAP;
        ConvSeg& s = p.seg[0];
        s.src = xp; s.wpack = wseg; s.img_stride = (long long)(cin / 8) * gi.PL * 8; s.ksteps = cin / 16; s.ntaps = 4;
        s.ht = s.hb = s.hl = s.hr = 0; s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
        for (int t = 0; t < 4; ++t) {
          s.dh[t] = ut.dh[t]; s.dw[t] = ut.dw[t];
          if (ut.dh[t] < 0) s.ht = 1;
          if (ut.dh[t] > 0) s.hb = 1;
          if (ut.dw[t] < 0) s.hl = 1;
          if (ut.dw[t] > 0) s.hr = 1;
        }
        p.oy = pa; p.ox = pb;
        CK(launch_conv_tc(p, sms, st));
      }
  } else {
    CK(launch_conv_tc(p, sms, st));
  }
  CK(launch_pf8_to_nchw(op, y, N, cout, Ho, Wo, st));
  if (stats_out) CK(launch_stats_to_float(stp, stats_out, N * (cout / 4) * 2, st));
  return 0;
}

extern "C" int b200ad_conv2d(const float* x, const float* w, const float* bias, const float* temb, const float* residual,
                             float* y, float* stats_out, int N, int cin, int cout, int H, int W, int K, int stride,
                             void* scratch, size_t scratch_bytes, void* stream) {
  return conv2d_impl(x, w, bias, temb, residual, y, stats_out, N, cin, cout, H, W, K, stride, nullptr, nullptr, 0, 0.f, 0,
                     scratch, scratch_bytes, stream);
}

// Data gradient of a stride-1 conv: gx[n][i] = sum_o sum_taps W[o][i][kh][kw] * gy[n][o][y - (kh - K/2)][x - (kw - K/2)] — the
// same implicit GEMM with the roles of the channel dimensions swapped and the taps mirrored, so it runs on conv_tc_kernel
// with a transposed weight packing (this is how the backward pass will reuse the forward kernel; DESIGN.md §6).
extern "C" int b200ad_conv2d_dgrad(const float* gy, const float* w, float* gx, int N, int cin, int cout, int H, int W, int K,
                                   void* scratch, size_t scratch_bytes, void* stream) {
  if (cout % 16 || cin % 128) return set_err("conv2d_dgrad: cout %% 16 and cin %% 128 must be 0");
  if (K != 3 && K != 1) return set_err("conv2d_dgrad: K must be 1 or 3");
  const ConvScratch L = conv_scratch_layout(N, cout, cin, H, W, K, 1);   // GEMM view: cout -> cin channels
  if (scratch_bytes < L.total) return set_err("conv2d_dgrad: scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sb = (uint8_t*)scratch;
  CK(cudaMemsetAsync(sb, 0, L.total, st));
  const Geom g = make_geom(N, H, W);
  __nv_bfloat16* gyp = (__nv_bfloat16*)(sb + L.x);
  __nv_bfloat16* gxp = (__nv_bfloat16*)(sb + L.out);
  __nv_bfloat16* wp = (__nv_bfloat16*)(sb + L.wpack);
  CK(launch_nchw_to_pf8(gy, gyp, N, cout, H, W, st));
  PackTaps t{};
  t.ntaps = K * K;
  t.transpose = 1;
  for (int k = 0; k < K * K; ++k) { t.kh[k] = K - 1 - k / K; t.kw[k] = K - 1 - k % K; }   // mirrored taps
  CK(launch_pack_weights(w, cin, cin, K, K, 0, cout / 16, t, wp, st, cin));
  ConvParams p{};
  p.N = N; p.H = H; p.W = W; p.Wp = g.Wp; p.lead = g.lead; p.PL = g.PL;
  p.cout = cin;
  p.out = gxp; p.bias = nullptr; p.temb = nullptr; p.temb_stride = 0; p.stats = nullptr;
  ConvSeg& s = p.seg[0];
  s.src = gyp; s.wpack = wp; s.img_stride = (long long)(cout / 8) * g.PL * 8; s.ksteps = cout / 16; s.ntaps = K * K;
  s.ht = s.hb = s.hl = s.hr = (K == 3) ? 1 : 0;
  for (int k = 0; k < K * K; ++k) { s.dh[k] = (signed char)(k / K - K / 2); s.dw[k] = (signed char)(k % K - K / 2); }
  s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
  p.nseg = 1;
  int dev = 0, sms = 132;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CK(launch_conv_tc(p, sms, st));
  CK(launch_pf8_to_nchw(gxp, gx, N, cin, H, W, st));
  return 0;
}

// Weight gradient of the stride-1 conv: dw[o][i][kh][kw] = sum_{n,y,x} gy[n][o][y][x] * a[n][i][y + kh - K/2][x + kw - K/2].
extern "C" int b200ad_conv2d_wgrad(const float* gy, const float* a, float* dw, int N, int cin, int cout, int H, int W, int K,
                                   void* scratch, size_t scratch_bytes, void* stream) {
  if (cout % 128 || cin % 32) return set_err("conv2d_wgrad: cout %% 128 and cin %% 32 must be 0");
  if (K != 3 && K != 1) return set_err("conv2d_wgrad: K must be 1 or 3");
  const Geom g = make_geom(N, H, W);
  const size_t gyb = al((size_t)N * (cout / 8) * g.PL * 16), ab = al((size_t)N * (cin / 8) * g.PL * 16);
  if (scratch_bytes < gyb + ab) return set_err("conv2d_wgrad: scratch too small (%zu < %zu)", scratch_bytes, gyb + ab);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sb = (uint8_t*)scratch;
  CK(cudaMemsetAsync(sb, 0, gyb + ab, st));
  __nv_bfloat16* gyp = (__nv_bfloat16*)sb;
  __nv_bfloat16* ap = (__nv_bfloat16*)(sb + gyb);
  CK(launch_nchw_to_pf8(gy, gyp, N, cout, H, W, st));
  CK(launch_nchw_to_pf8(a, ap, N, cin, H, W, st));
  CK(cudaMemsetAsync(dw, 0, (size_t)cout * cin * K * K * sizeof(float), st));
  int dev = 0, sms = 132;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  WgradDesc d{};
  d.gy = gyp; d.act = ap; d.dw = dw; d.N = N; d.H = H; d.W = W; d.cout = cout; d.cin = cin;
  d.gy_img_planes = cout / 8; d.act_img_planes = cin / 8; d.cin_total = cin; d.ci_off = 0; d.ntaps_total = K * K;
  d.ntaps = K * K;
  for (int t = 0; t < K * K; ++t) { d.dh[t] = t / K - K / 2; d.dw_[t] = t % K - K / 2; d.tapidx[t] = t; }
  CK(launch_wgrad_tc(d, sms, st));
  return 0;
}
extern "C" size_t b200ad_conv2d_wgrad_scratch_bytes(int N, int cin, int cout, int H, int W) {
  const Geom g = make_geom(N, H, W);
  return al((size_t)N * (cout / 8) * g.PL * 16) + al((size_t)N * (cin / 8) * g.PL * 16);
}

extern "C" int b200ad_gn_conv2d(const float* x, const float* gamma, const float* beta, int groups, float eps, int silu,
                                const float* w, const float* bias, float* y, int N, int cin, int cout, int H, int W, int K,
                                void* scratch, size_t scratch_bytes, void* stream) {
  if (!gamma || !beta) return set_err("gn_conv2d: gamma and beta are required");
  return conv2d_impl(x, w, bias, nullptr, nullptr, y, nullptr, N, cin, cout, H, W, K, 1, gamma, beta, groups, eps, silu,
                     scratch, scratch_bytes, stream);
}

extern "C" int b200ad_group_norm(const float* x, const float* gamma, const float* beta, float* y, int N, int C, int H,
                                 int W, int groups, float eps, int silu, void* scratch, size_t scratch_bytes, void* stream) {
  if (C % 32) return set_err("group_norm: C %% 32 != 0");
  const Geom g = make_geom(N, H, W);
  const size_t tb = al((size_t)N * (C / 8) * g.PL * 16);
  const size_t need = 2 * tb + al((size_t)N * (C / 4) * 2 * sizeof(stat_t));
  if (scratch_bytes < need) return set_err("group_norm: scratch too small (%zu < %zu)", scratch_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sb = (uint8_t*)scratch;
  CK(cudaMemsetAsync(sb, 0, need, st));
  __nv_bfloat16* xp = (__nv_bfloat16*)sb;
  __nv_bfloat16* yp = (__nv_bfloat16*)(sb + tb);
  stat_t* stats = (stat_t*)(sb + 2 * tb);
  CK(launch_nchw_to_pf8(x, xp, N, C, H, W, st));
  CK(launch_quad_stats(xp, stats, N, C, H, W, st));
  GnApplyParams p{};
  p.src[0] = xp; p.stats[0] = stats; p.C[0] = C; p.src[1] = nullptr; p.stats[1] = nullptr; p.C[1] = 0;
  p.gamma = gamma; p.beta = beta; p.dst = yp; p.N = N; p.H = H; p.W = W; p.groups = groups; p.eps = eps; p.silu = silu;
  CK(launch_gn_apply(p, st));
  CK(launch_pf8_to_nchw(yp, y, N, C, H, W, st));
  return 0;
}

extern "C" int b200ad_sample_to_u8(const float* x, uint8_t* img, size_t n, void* stream) {
  CK(launch_sample_to_u8(x, img, n, (cudaStream_t)stream));
  return 0;
}
