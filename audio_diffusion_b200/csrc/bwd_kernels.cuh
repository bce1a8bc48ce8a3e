// Launchers of the backward-pass kernels (bwd_kernels.cu, wgrad_tc.cu).
#pragma once
#include "kernels.cuh"

namespace b200ad {

struct GnBwdParams {
  const __nv_bfloat16* ga;        // gradient w.r.t. the normalised (+SiLU) tensor, PF8, C0 + C1 channels
  const __nv_bfloat16* src[2];    // the raw forward sources
  const stat_t* stats[2];         // their (sum, sumsq) quads
  int C[2];
  const float* gamma;
  const float* beta;
  __nv_bfloat16* dst[2];          // gradients w.r.t. the raw sources (C0 / C1 channels)
  const __nv_bfloat16* addS;      // optional, C0 + C1 channels: added to both halves (the shortcut path's gradient)
  const __nv_bfloat16* add0;      // optional, C0 channels: added to dst[0] (e.g. the skip connection's gradient)
  float* dgamma;                  // [C0 + C1], accumulated
  float* dbeta;
  float* sums;                    // scratch [N][C0 + C1][2]
  float* csum0;                   // optional [N][C0]: per-sample channel sums of dst[0] are ADDED here (zeroed by the caller):
                                  // the bias / time-embedding gradients of the layer that produced src[0] (no chan_sum pass)
  int N, H, W, groups;
  float eps;
  int silu;
};
cudaError_t launch_gn_bwd(const GnBwdParams& p, cudaStream_t s);

// out[n][c] = sum_pix src[n][c] for a C-channel view of a tensor with img_planes planes per image
// bias0 / bias1 (optional): the sample-summed channel sums are also added there (bias gradients)
cudaError_t launch_chan_sum(const __nv_bfloat16* src, float* out, int N, int C, int img_planes, int H, int W, cudaStream_t s,
                            float* bias0 = nullptr, float* bias1 = nullptr);
cudaError_t launch_reduce_n_add(const float* src, float* dst, float* dst2, int N, int C, cudaStream_t s);
cudaError_t launch_scatter_rows(const float* src, float* dst, int N, int C, int dstride, int doff, cudaStream_t s);
cudaError_t launch_pf8_add(__nv_bfloat16* dst, const __nv_bfloat16* src, int N, int C, int H, int W, cudaStream_t s);
cudaError_t launch_attention_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* go, __nv_bfloat16* gqkv, int N, int C, int H,
                                 int W, cudaStream_t s);
cudaError_t launch_scalar_conv_wgrad(const __nv_bfloat16* G, const float* X, float* dW, int N, int C, int H, int W, int flip,
                                     cudaStream_t s);
cudaError_t launch_flip_taps(const float* w, float* wf, int C, cudaStream_t s, int O = 1);
cudaError_t launch_sum_add(const float* x, long long n, float* dst, cudaStream_t s);
struct UnfoldMasks { unsigned mask[4][4]; };
cudaError_t launch_unfold_up2(const float* dwf, float* dw3, long long nco_ci, const UnfoldMasks& m, cudaStream_t s);
cudaError_t launch_lin_bwd_input(const float* g, int gstride, const float* W, int O, int I, float* gin, int N, int accumulate,
                                 cudaStream_t s);
cudaError_t launch_lin_bwd_weight(const float* g, int gstride, const float* x, int O, int I, float* dW, float* db, int N,
                                  cudaStream_t s);
cudaError_t launch_silu_bwd(float* g, const float* u, int n, cudaStream_t s);
cudaError_t launch_silu_fwd(const float* u, float* y, int n, cudaStream_t s);

// Transformer blocks of the conditional U-Net (cond_bwd.cu).
// LayerNorm over channels: gx = LN-backward(gy; x) (+ add, optional, same shape); dgamma / dbeta [C] accumulated. C <= 512.
cudaError_t launch_layernorm_bwd_pf8(const __nv_bfloat16* x, const __nv_bfloat16* gy, const __nv_bfloat16* add,
                                     __nv_bfloat16* gx, const float* gamma, float* dgamma, float* dbeta, int N, int C, int H,
                                     int W, float eps, cudaStream_t s);
// GEGLU: src = the forward input (2*Ch channels: hidden | gate), gy: Ch channels -> dst: 2*Ch channels
cudaError_t launch_geglu_bwd_pf8(const __nv_bfloat16* src, const __nv_bfloat16* gy, __nv_bfloat16* dst, int N, int Ch, int H,
                                 int W, cudaStream_t s);
// cross-attention against one encoder token: dvec [N][C] = gradient of the per-sample vector Wo (Wv enc) + bo ->
// dWo [C][C], dWv [C][X] accumulated.  scratch: 2 * N * C floats.
cudaError_t launch_cross_attn_vec_bwd(const float* enc, const float* dvec, const float* wv, const float* wo, float* dwo,
                                      float* dwv, float* scratch, int N, int C, int X, cudaStream_t s);
// multi-head self-attention (head_dim C / heads in {16, 32, 64}): qkv and o as the forward read / wrote them, go = dL/do
// (PF8, C channels), lse from launch_mha_flash -> gqkv (PF8, 3C channels).  dsum: N * heads * H * W floats of scratch.
cudaError_t launch_mha_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* o, const __nv_bfloat16* go, const float* lse,
                           float* dsum, __nv_bfloat16* gqkv, int N, int C, int heads, int H, int W, cudaStream_t s);
// cross-attention against S > 1 encoder tokens: q, o as the forward read / wrote them (PF8, C channels), k, v bf16
// [N][S][C], go = dL/do (PF8, C channels), lse from launch_xattn -> gq (PF8, C channels) and dk, dv fp32 [N][S][C]
// (overwritten).  Scratch: dsum (N * heads * H * W floats) and part (xattn_part_floats floats): per query split fp32
// partial sums of dK and dV, added in split order (no atomics: the result is deterministic).
size_t xattn_part_floats(int N, int C, int heads, int H, int W, int S);
cudaError_t launch_xattn_bwd(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v, const __nv_bfloat16* o,
                             const __nv_bfloat16* go, const float* lse, float* dsum, float* part, __nv_bfloat16* gq, float* dk,
                             float* dv, int N, int C, int heads, int H, int W, int S, cudaStream_t s);
// the K / V projections' weight gradients: dwk[c][x] += sum over the M = N * S tokens of dk[m][c] enc[m][x], dwv the same
cudaError_t launch_xattn_kv_wgrad(const float* dk, const float* dv, const float* enc, float* dwk, float* dwv, int M, int C,
                                  int X, cudaStream_t s);

// Autoencoder layers (vae_bwd_kernels.cu).
// single-head attention (one head of dim C, S = H * W tokens, S % 64 == 0, C % 64 == 0): qkv as the forward read it,
// go = dL/do (PF8, C channels), P the forward's softmax (fp32 [N][S][S]) -> gqkv (PF8, 3C channels).
// Scratch: D (N * S floats), dS (N * S * S bf16).
cudaError_t launch_attention_1head_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* go, const float* P, float* D,
                                       __nv_bfloat16* dS, __nv_bfloat16* gqkv, int N, int C, int H, int W, cudaStream_t s);
// quant_conv (1x1, L2 -> L2) on the first L2 channels of h (PF8, 128 channels), from gm (fp32 [N][L2][H][W]) -> g_h as
// fp32 [N][L2][H][W] (gh_nc) and [L2][N][H][W] (gh_cn); dwq / dbq accumulated.  L2 <= 8.
cudaError_t launch_quant_conv_bwd(const float* gm, const __nv_bfloat16* h, const float* wq, float* gh_nc, float* gh_cn,
                                  float* dwq, float* dbq, int N, int L2, int H, int W, cudaStream_t s);
// conv_in (3x3, L -> C) on post_quant_conv(z) (1x1, L -> L): gy (PF8, C channels) -> gz (fp32 [N][L][H][W]);
// dwpq / dbpq accumulated (z: the forward's input latents).  L <= 4.
cudaError_t launch_latent_in_bwd(const __nv_bfloat16* gy, const float* win, const float* wpq, const float* z, float* gz,
                                 float* dwpq, float* dbpq, int N, int C, int L, int H, int W, cudaStream_t s);

// Weight gradient on wgmma (wgrad_tc.cu):  dw[(co * cin_total + ci_off + ci) * ntaps_total + tapidx[t]] +=
//   sum_{n, p} gy[n][co][p] * act[n][ci][p + shift[t]].   gy / act are channel views: `*_img_planes` planes per image in the
// underlying tensors, the pointers already offset to the view's first plane.
struct WgradDesc {
  const __nv_bfloat16* gy;
  const __nv_bfloat16* act;
  float* dw;
  int N, H, W;            // geometry of both tensors
  int cout, cin;          // channels of the two views (cout % 128 == 0, cin % 32 == 0)
  int gy_img_planes, act_img_planes;
  int cin_total, ci_off, ntaps_total;
  int ntaps;
  int dh[9], dw_[9], tapidx[9];
};
cudaError_t launch_wgrad_tc(const WgradDesc& d, int num_sms, cudaStream_t s);

}  // namespace b200ad
