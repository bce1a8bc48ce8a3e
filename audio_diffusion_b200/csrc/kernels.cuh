// Launchers of the non-tensor-core kernels of the U-Net path (elementwise.cu, attention.cu, temb.cu).
#pragma once
#include <vector>
#include "common.cuh"

namespace b200ad {

// weights fp32 [cout][cin_total][KH][KW]  ->  packed bf16 blocks [cout/128][ksteps][ntaps][2][16][8][8]
// for input channels [cin_off, cin_off + 16*ksteps) and the listed (kh, kw) taps.
// If fold != 0 the tap list is interpreted as groups: tap t sums the source taps whose bit is set in
// fold_mask[t] (bit kh*KW+kw) — used to fold nearest-2x upsampling into the conv weights.
// transpose != 0 packs the weights of the data-gradient conv: GEMM output channel = the layer's INPUT channel, GEMM input
// channel = the layer's output channel, i.e. element W[ci][co][kh][kw] of the fp32 tensor [O][I][KH][KW] with I = cout_real.
struct PackTaps {
  int ntaps;
  int kh[9], kw[9];
  unsigned fold_mask[9];
  int fold;
  int transpose;
};
cudaError_t launch_pack_weights(const float* w, int cout, int cin_total, int KH, int KW, int cin_off, int ksteps,
                                const PackTaps& taps, __nv_bfloat16* dst, cudaStream_t s, int cout_real = -1);

// Batched form: all K-segments of a model in ONE launch. `PackBatch` owns a small device-side job table, rebuilt only when
// a source / destination pointer changes.
struct PackItem {
  const float* w;
  __nv_bfloat16* dst;
  int cout, cin_total, KH, KW, cin_off, ksteps, cout_real;
  PackTaps taps;
  long long nvec;
};
struct PackBatch {
  std::vector<PackItem> host;      // last uploaded table
  void* d_items = nullptr;         // PackItem[njobs]
  void* d_blk = nullptr;           // int2 {job, first vector of the block / 256} per block
  int nblocks = 0;
  PackBatch() = default;
  PackBatch(const PackBatch&) = delete;
  PackBatch& operator=(const PackBatch&) = delete;
  ~PackBatch();
};
cudaError_t launch_pack_batch(PackBatch& pb, const std::vector<PackItem>& items, cudaStream_t s);

// GroupNorm (+ optional SiLU) apply over the channel concatenation of up to two raw PF8 sources.
// stats: running (sum, sumsq) per (n, 4-channel quad) written by the producers' epilogues.
struct GnApplyParams {
  const __nv_bfloat16* src[2];
  const stat_t* stats[2];     // [N][C_i/4][2]
  int C[2];                   // channels of each source (C[1] = 0 if single)
  const float* gamma;         // [C0 + C1]
  const float* beta;
  __nv_bfloat16* dst;         // PF8 with C0 + C1 channels
  int N, H, W, groups;
  float eps;
  int silu;
};
cudaError_t launch_gn_apply(const GnApplyParams& p, cudaStream_t s);
// statistics -> per-(sample, channel) (scale, shift) [N][C0 + C1] for the GroupNorm fused into conv_tc_kernel
// (src / dst / silu of `p` are ignored)
cudaError_t launch_gn_finalize(const GnApplyParams& p, float2* ss, cudaStream_t s);

// conv_in: fp32 NCHW (N, cin, H, W), 3x3 pad 1 -> raw bf16 PF8 (cout channels) + quad stats.
cudaError_t launch_conv_in(const float* x, const float* w, const float* b, int N, int cin, int H, int W, int cout,
                           __nv_bfloat16* out, stat_t* stats, cudaStream_t s);

// conv_norm_out + SiLU + conv_out (3x3, C -> cout small) fused with the scheduler update.
// eps_out (optional): model output, fp32 NCHW.  If x_out != null:
//   x0 = clamp((x - sqrt_1m_at * eps) * inv_sqrt_at, -clip, clip);  x_out = c_x0 * x0 + c_xt * x + c_eps * eps + c_z * z
// which covers DDPM (c_eps = 0) and DDIM (c_xt = 0).  Multistep (DPM-Solver++, hist1 != null): x_out also gets
// c_h1 * hist1 + c_h2 * hist2 (the x0 of the previous two steps), then hist2 <- hist1 (if hist2) and hist1 <- x0.
struct StepCoef {
  float sqrt_1m_at, inv_sqrt_at, clip, c_x0, c_xt, c_eps, c_z;
  int do_clip;
};
struct MultistepCoef {
  StepCoef s;
  float c_h1, c_h2;
};
struct ConvOutParams {
  const __nv_bfloat16* src;   // raw PF8, C channels
  const stat_t* stats;        // [N][C/4][2]
  const float2* ss;           // [N][C] GroupNorm (scale, shift), finalised by the producer's last CTA; null: use stats here
  const float* gamma;
  const float* beta;
  const float* w;             // fp32 [cout][C][3][3]
  const float* b;             // [cout]
  int N, C, H, W, cout, groups;
  float eps;
  float* eps_out;             // fp32 NCHW or null
  const float* x;             // fp32 NCHW current sample (scheduler input) or null
  const float* z;             // fp32 NCHW noise or null
  float* x_out;               // fp32 NCHW or null
  MultistepCoef coef;
  const MultistepCoef* coef_dev;  // optional: the coefficients live on the device (CUDA-graph replay: nothing per-step is
                                  // baked into the launch); overrides `coef`.  Without history only its `s` is read, so
                                  // it may point at a plain StepCoef.
  float* hist1;               // fp32 NCHW x0 of the previous step, or null (then c_h1 / c_h2 and hist2 are unused)
  float* hist2;               // fp32 NCHW x0 of the step before that, or null
};
cudaError_t launch_conv_out(const ConvOutParams& p, cudaStream_t s);

// stride-2 parity split PF8 (H, W) -> 4 x PF8 (H/2, W/2)
cudaError_t launch_parity_split(const __nv_bfloat16* src, __nv_bfloat16* dst4, int N, int C, int H, int W, cudaStream_t s);

cudaError_t launch_quad_stats(const __nv_bfloat16* src, stat_t* stats, int N, int C, int H, int W, cudaStream_t s);
cudaError_t launch_stats_to_float(const stat_t* s, float* d, int n, cudaStream_t st);
cudaError_t launch_sample_to_u8(const float* x, uint8_t* img, size_t n, cudaStream_t s);

// layout conversion for tests / debugging
cudaError_t launch_nchw_to_pf8(const float* src, __nv_bfloat16* dst, int N, int C, int H, int W, cudaStream_t s);
cudaError_t launch_pf8_to_nchw(const __nv_bfloat16* src, float* dst, int N, int C, int H, int W, cudaStream_t s);

// timestep embedding: t[N] -> sinusoid(dim0) -> linear1 -> SiLU -> linear2 -> SiLU = temb_act [N][4*dim0];
// then all resnet projections at once: proj [N][rows] = Wcat [rows][4*dim0] * temb_act + bcat.
cudaError_t launch_temb(const float* t, int N, int dim0, const float* w1, const float* b1, const float* w2,
                        const float* b2, float* temb_act, const float* wcat, const float* bcat, int rows,
                        float* proj, cudaStream_t s, float* save_emb = nullptr, float* save_u1 = nullptr,
                        float* save_u2 = nullptr, int* lead = nullptr);   // lead [N] scratch: share the work of equal timesteps

// self-attention core on the fused qkv tensor (PF8, 3*C channels: q | k | v; head_dim 8 = one plane per head).
cudaError_t launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int N, int C, int H, int W, cudaStream_t s);

// transformer blocks of the conditional U-Net (cond_ops.cu)
cudaError_t launch_layernorm_pf8(const __nv_bfloat16* src, __nv_bfloat16* dst, const float* gamma, const float* beta, int N,
                                 int C, int H, int W, float eps, cudaStream_t s);
cudaError_t launch_geglu_pf8(const __nv_bfloat16* src, __nv_bfloat16* dst, int N, int Ch, int H, int W, cudaStream_t s);
cudaError_t launch_cross_attn_vec(const float* enc, const float* wv, const float* wo, const float* bo, float* vec, int N, int C,
                                  int X, cudaStream_t s);
// lse (optional, training): row log-sum-exp fp32 [N][heads][H*W] for the backward (log2 domain of the scaled scores)
cudaError_t launch_mha_flash(const __nv_bfloat16* qkv, __nv_bfloat16* out, int N, int C, int heads, int H, int W, cudaStream_t s,
                             float* lse = nullptr);
// cross-attention against an encoding of S > 1 tokens (1 <= S <= XATTN_MAX_S).  K / V: bf16 [N][S][C] (token-major).
constexpr int XATTN_MAX_S = 256;
// enc fp32 [N][S][X] -> K = enc Wk^T, V = enc Wv^T (wk, wv fp32 [C][X])
cudaError_t launch_xattn_kv(const float* enc, const float* wk, const float* wv, __nv_bfloat16* k, __nv_bfloat16* v, int N, int S,
                            int C, int X, cudaStream_t s);
// fp32 -> bf16, n elements (the parity entry point's K / V)
cudaError_t launch_f32_to_bf16(const float* src, __nv_bfloat16* dst, long long n, cudaStream_t s);
// q, out: PF8 with C channels; 8 heads of dim C / heads in {16, 32, 64}; lse (optional, training) as launch_mha_flash's
cudaError_t launch_xattn(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v, __nv_bfloat16* out, int N,
                         int C, int heads, int H, int W, int S, cudaStream_t s, float* lse = nullptr);

// generic single-head attention over the fused qkv tensor (AutoencoderKL mid block); scores: N * seq * seq floats of scratch
cudaError_t launch_attention_1head(const __nv_bfloat16* qkv, __nv_bfloat16* out, float* scores, int N, int C, int H, int W,
                                   cudaStream_t s);
// quant_conv + DiagonalGaussianDistribution.sample on the encoder output; post_quant_conv (1x1 on fp32 NCHW latents)
cudaError_t launch_vae_sample(const __nv_bfloat16* enc, const float* wq, const float* bq, const float* noise, float* z,
                              float* moments, int N, int C, int L, int H, int W, cudaStream_t s);
cudaError_t launch_mix1x1(const float* x, const float* w, const float* b, float* y, int N, int L, int HW, cudaStream_t s);

// Stages the K and V of one (sample, head) in shared memory as [plane][key] rows of 8 channels, keys S..SP-1 zero
// (the layout mha_flash_kernel streams its key tiles in).  The forward (cond_ops.cu) and the
// backward (cond_bwd.cu) kernels of the cross-attention share it.
template <int D>
__device__ __forceinline__ void xattn_stage_kv(uint4* ks, uint4* vs, const __nv_bfloat16* k, const __nv_bfloat16* v, int n,
                                               int head, int C, int S, int SP) {
  constexpr int DP = D / 8;
  const __nv_bfloat16* kg = k + (long long)n * S * C + head * D;
  const __nv_bfloat16* vg = v + (long long)n * S * C + head * D;
  for (int i = threadIdx.x; i < DP * SP; i += blockDim.x) {
    const int key = i / DP, pl = i - key * DP;
    uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
    if (key < S) {
      a = *reinterpret_cast<const uint4*>(kg + (long long)key * C + pl * 8);
      b = *reinterpret_cast<const uint4*>(vg + (long long)key * C + pl * 8);
    }
    ks[pl * SP + key] = a;
    vs[pl * SP + key] = b;
  }
}

}  // namespace b200ad
