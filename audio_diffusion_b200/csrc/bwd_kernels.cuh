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
cudaError_t launch_flip_taps(const float* w, float* wf, int C, cudaStream_t s);
cudaError_t launch_sum_add(const float* x, long long n, float* dst, cudaStream_t s);
struct UnfoldMasks { unsigned mask[4][4]; };
cudaError_t launch_unfold_up2(const float* dwf, float* dw3, long long nco_ci, const UnfoldMasks& m, cudaStream_t s);
cudaError_t launch_lin_bwd_input(const float* g, int gstride, const float* W, int O, int I, float* gin, int N, int accumulate,
                                 cudaStream_t s);
cudaError_t launch_lin_bwd_weight(const float* g, int gstride, const float* x, int O, int I, float* dW, float* db, int N,
                                  cudaStream_t s);
cudaError_t launch_silu_bwd(float* g, const float* u, int n, cudaStream_t s);
cudaError_t launch_silu_fwd(const float* u, float* y, int n, cudaStream_t s);

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
