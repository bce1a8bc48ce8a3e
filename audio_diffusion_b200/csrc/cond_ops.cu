// Kernels of the conditional U-Net's transformer blocks (UNet2DConditionModel as built at scripts/train_unet.py:139-159;
// called at audiodiffusion/pipeline_audio_diffusion.py:160-161): LayerNorm over channels, multi-head self-attention with
// head_dim 16 / 32 / 64 (flash-style, warp-level tensor cores), GEGLU, and the cross-attention against the audio encoding.
// All 1x1 projections / linears run on conv_tc_kernel; these are the memory-bound or attention-shaped rest.
// Reference semantics: diffusers 0.24 BasicTransformerBlock / Attention / FeedForward(GEGLU) - oracle/unet_cond_oracle.py.
#include "kernels.cuh"

namespace b200ad {

// ------------------------------------------------------------------------------------ LayerNorm over channels (per token)
// y[n][c][p] = (x - mean_p) * rstd_p * gamma[c] + beta[c];  one warp per pixel, lanes stride over the 8-channel planes.
__global__ void __launch_bounds__(256) layernorm_pf8_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                                            int N, int C, int H, int W, float eps) {
  const Geom g = make_geom(N, H, W);
  const int planes = C >> 3;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = blockIdx.x * 8 + warp, n = blockIdx.y;
  if (p >= H * W) return;
  const long long off = pf8_pixel(g, p, W);
  const __nv_bfloat16* sp = src + (long long)n * planes * g.PL * 8 + off;
  __nv_bfloat16* dp = dst + (long long)n * planes * g.PL * 8 + off;
  float s = 0.f, q = 0.f;
  for (int pl = lane; pl < planes; pl += 32) {
    const uint4 v = *reinterpret_cast<const uint4*>(sp + (long long)pl * g.PL * 8);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = unpack_bf16x2(u[e]); s += f.x + f.y; q += f.x * f.x + f.y * f.y; }
  }
#pragma unroll
  for (int sh = 16; sh >= 1; sh >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, sh); q += __shfl_xor_sync(0xffffffffu, q, sh); }
  const float mean = s / (float)C;
  const float rstd = rsqrtf(fmaxf(q / (float)C - mean * mean, 0.f) + eps);
  for (int pl = lane; pl < planes; pl += 32) {
    const uint4 v = *reinterpret_cast<const uint4*>(sp + (long long)pl * g.PL * 8);
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_bf16x2(u[e]);
      const int c = pl * 8 + 2 * e;
      o[e] = pack_bf16x2((f.x - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c),
                         (f.y - mean) * rstd * __ldg(gamma + c + 1) + __ldg(beta + c + 1));
    }
    *reinterpret_cast<uint4*>(dp + (long long)pl * g.PL * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
cudaError_t launch_layernorm_pf8(const __nv_bfloat16* src, __nv_bfloat16* dst, const float* gamma, const float* beta, int N,
                                 int C, int H, int W, float eps, cudaStream_t s) {
  layernorm_pf8_kernel<<<dim3((H * W + 7) / 8, N), 256, 0, s>>>(src, dst, gamma, beta, N, C, H, W, eps);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ GEGLU
// src: PF8 with 2*Ch channels (hidden | gate), dst: PF8 with Ch channels: hidden * gelu(gate), exact (erf) GELU.
__global__ void __launch_bounds__(256) geglu_pf8_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                                        int N, int Ch, int H, int W) {
  const Geom g = make_geom(N, H, W);
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= H * W) return;
  const int pl = blockIdx.y, n = blockIdx.z, planes = Ch >> 3;
  const long long off = pf8_pixel(g, p, W);
  const __nv_bfloat16* sp = src + (long long)n * 2 * planes * g.PL * 8 + off;
  const uint4 hv = *reinterpret_cast<const uint4*>(sp + (long long)pl * g.PL * 8);
  const uint4 gv = *reinterpret_cast<const uint4*>(sp + (long long)(planes + pl) * g.PL * 8);
  const uint32_t hu[4] = {hv.x, hv.y, hv.z, hv.w}, gu[4] = {gv.x, gv.y, gv.z, gv.w};
  uint32_t o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 h = unpack_bf16x2(hu[e]), t = unpack_bf16x2(gu[e]);
    o[e] = pack_bf16x2(h.x * 0.5f * t.x * (1.0f + erff(t.x * 0.70710678118654752f)),
                       h.y * 0.5f * t.y * (1.0f + erff(t.y * 0.70710678118654752f)));
  }
  *reinterpret_cast<uint4*>(dst + ((long long)n * planes + pl) * g.PL * 8 + off) = make_uint4(o[0], o[1], o[2], o[3]);
}
cudaError_t launch_geglu_pf8(const __nv_bfloat16* src, __nv_bfloat16* dst, int N, int Ch, int H, int W, cudaStream_t s) {
  geglu_pf8_kernel<<<dim3((H * W + 255) / 256, Ch >> 3, N), 256, 0, s>>>(src, dst, N, Ch, H, W);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ cross-attention, one key
// With ONE encoder token per sample (the reference's audio encodings are (B, 1, 100)) the softmax over keys is 1 for every
// query, so attn2(x, enc) = to_out(to_v(enc)) for every pixel: a per-sample vector.  vec[n][c] = Wo (Wv enc_n) + bo.
// It is added by the epilogue of the attn1 output projection (the conv kernel's per-sample additive term).
__global__ void __launch_bounds__(256) cross_attn_vec_kernel(const float* __restrict__ enc, const float* __restrict__ wv,
                                                             const float* __restrict__ wo, const float* __restrict__ bo,
                                                             float* __restrict__ vec, int C, int X) {
  extern __shared__ float csm[];   // enc[X], v[C]
  float* es = csm;
  float* vs = csm + X;
  const int n = blockIdx.x;
  for (int i = threadIdx.x; i < X; i += blockDim.x) es[i] = enc[(long long)n * X + i];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f;
    for (int i = 0; i < X; ++i) a = fmaf(__ldg(wv + (long long)c * X + i), es[i], a);
    vs[c] = a;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int c = warp; c < C; c += 8) {
    float a = 0.f;
    for (int i = lane; i < C; i += 32) a = fmaf(__ldg(wo + (long long)c * C + i), vs[i], a);
#pragma unroll
    for (int sh = 16; sh >= 1; sh >>= 1) a += __shfl_xor_sync(0xffffffffu, a, sh);
    if (lane == 0) vec[(long long)n * C + c] = a + __ldg(bo + c);
  }
}
cudaError_t launch_cross_attn_vec(const float* enc, const float* wv, const float* wo, const float* bo, float* vec, int N, int C,
                                  int X, cudaStream_t s) {
  cross_attn_vec_kernel<<<N, 256, (size_t)(X + C) * sizeof(float), s>>>(enc, wv, wo, bo, vec, C, X);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ multi-head self-attention
// qkv: PF8 with 3C channels (q | k | v), head h = channels [h D, (h+1) D) of each third.  One CTA = 64 queries of one
// (sample, head): 4 warps x 16 query rows; K / V stream through shared memory in tiles of 64 keys; online softmax in
// the exp2 domain; Q K^T and P V on mma.sync.m16n8k16 (bf16 in, fp32 accumulate), V fragments by transposing ldmatrix.
// lse (training, may be null): the row log-sum-exp of the scaled scores in the log2 domain, fp32 [N][heads][seq], which
// the backward (cond_bwd.cu) recomputes P from.
template <int D, bool LSE>
__global__ void __launch_bounds__(128) mha_flash_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out,
                                                        int N, int C, int H, int W, float scale_log2, float* __restrict__ lse) {
  constexpr int DP = D / 8;    // planes per head
  constexpr int KS = D / 16;   // k-steps of Q K^T
  __shared__ __align__(16) uint4 ks[DP][64];   // [plane][key] 8 channels
  __shared__ __align__(16) uint4 vs[DP][64];
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3;
  const int head = blockIdx.y, n = blockIdx.z, q0 = blockIdx.x * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* qb = base + (long long)(head * DP) * g.PL * 8;
  const __nv_bfloat16* kb = base + (long long)(planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* vb = base + (long long)(2 * planes + head * DP) * g.PL * 8;
  // Q fragments of this warp's 16 rows (rows beyond seq read row seq-1: their results are never stored)
  const int r0 = min(q0 + warp * 16 + gq, seq - 1), r1 = min(q0 + warp * 16 + gq + 8, seq - 1);
  const long long o0 = pf8_pixel(g, r0, W), o1 = pf8_pixel(g, r1, W);
  uint32_t qa[KS][4];
#pragma unroll
  for (int j = 0; j < KS; ++j) {
    qa[j][0] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j) * g.PL * 8 + o0 + 2 * tq);
    qa[j][1] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j) * g.PL * 8 + o1 + 2 * tq);
    qa[j][2] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j + 1) * g.PL * 8 + o0 + 2 * tq);
    qa[j][3] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j + 1) * g.PL * 8 + o1 + 2 * tq);
  }
  float oacc[DP][4];
#pragma unroll
  for (int i = 0; i < DP; ++i) { oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const uint32_t* ks32 = reinterpret_cast<const uint32_t*>(ks);
  const uint32_t vs_addr = smem_u32(vs);

  for (int k0 = 0; k0 < seq; k0 += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < DP * 64; i += 128) {
      const int pl = i >> 6, kk = i & 63, key = k0 + kk;
      uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
      if (key < seq) {
        const long long off = pf8_pixel(g, key, W);
        kv = *reinterpret_cast<const uint4*>(kb + (long long)pl * g.PL * 8 + off);
        vv = *reinterpret_cast<const uint4*>(vb + (long long)pl * g.PL * 8 + off);
      }
      ks[pl][kk] = kv;
      vs[pl][kk] = vv;
    }
    __syncthreads();
    // S = Q K^T for 64 keys: 8 n-tiles of 8 keys
    float sc[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      sc[t][0] = sc[t][1] = sc[t][2] = sc[t][3] = 0.f;
#pragma unroll
      for (int j = 0; j < KS; ++j) {
        const uint32_t b0 = ks32[((2 * j) * 64 + t * 8 + gq) * 4 + tq], b1 = ks32[((2 * j + 1) * 64 + t * 8 + gq) * 4 + tq];
        mma_bf16_16x8x16(sc[t], qa[j][0], qa[j][1], qa[j][2], qa[j][3], b0, b1);
      }
    }
    // scale (log2 domain), mask keys beyond seq, running maxima
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int key = k0 + t * 8 + 2 * tq;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float v = (key + (e & 1) < seq) ? sc[t][e] * scale_log2 : -INFINITY;
        sc[t][e] = v;
        if (e < 2) mx0 = fmaxf(mx0, v); else mx1 = fmaxf(mx1, v);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float c0 = exp2f(m0 - mx0), c1 = exp2f(m1 - mx1);
    m0 = mx0; m1 = mx1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int i = 0; i < DP; ++i) { oacc[i][0] *= c0; oacc[i][1] *= c0; oacc[i][2] *= c1; oacc[i][3] *= c1; }
    // P = exp2(S - m); O += P V, 16 keys at a time
#pragma unroll
    for (int kb16 = 0; kb16 < 4; ++kb16) {
      float* s0 = sc[2 * kb16];
      float* s1 = sc[2 * kb16 + 1];
      const float e00 = exp2f(s0[0] - m0), e01 = exp2f(s0[1] - m0), e02 = exp2f(s0[2] - m1), e03 = exp2f(s0[3] - m1);
      const float e10 = exp2f(s1[0] - m0), e11 = exp2f(s1[1] - m0), e12 = exp2f(s1[2] - m1), e13 = exp2f(s1[3] - m1);
      l0 += (e00 + e01) + (e10 + e11);
      l1 += (e02 + e03) + (e12 + e13);
      const uint32_t pa0 = pack_bf16x2(e00, e01), pa1 = pack_bf16x2(e02, e03), pa2 = pack_bf16x2(e10, e11), pa3 = pack_bf16x2(e12, e13);
#pragma unroll
      for (int i = 0; i < DP; ++i) {
        uint32_t vb0, vb1;  // V[keys 16][8 ch of plane i] as the col-major B fragment: transposing ldmatrix of two 8x8 tiles
        const uint32_t va = vs_addr + (uint32_t)((i * 64 + kb16 * 16 + (lane & 15)) * 16);
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(vb0), "=r"(vb1) : "r"(va));
        mma_bf16_16x8x16(oacc[i], pa0, pa1, pa2, pa3, vb0, vb1);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  __nv_bfloat16* ob = out + ((long long)n * planes + head * DP) * g.PL * 8;
  const int q_a = q0 + warp * 16 + gq, q_b = q_a + 8;
#pragma unroll
  for (int i = 0; i < DP; ++i) {   // accumulator (c0, c1) = (row gq, channels 8i + 2tq, +1), (c2, c3) = row gq + 8
    if (q_a < seq) *reinterpret_cast<uint32_t*>(ob + (long long)i * g.PL * 8 + o0 + 2 * tq) = pack_bf16x2(oacc[i][0] * i0, oacc[i][1] * i0);
    if (q_b < seq) *reinterpret_cast<uint32_t*>(ob + (long long)i * g.PL * 8 + o1 + 2 * tq) = pack_bf16x2(oacc[i][2] * i1, oacc[i][3] * i1);
  }
  if (LSE && tq == 0) {
    float* lr = lse + ((long long)n * gridDim.y + head) * seq;
    if (q_a < seq) lr[q_a] = m0 + __log2f(l0);   // l >= 1 (the row maximum contributes 1)
    if (q_b < seq) lr[q_b] = m1 + __log2f(l1);
  }
}

cudaError_t launch_mha_flash(const __nv_bfloat16* qkv, __nv_bfloat16* out, int N, int C, int heads, int H, int W, cudaStream_t s,
                             float* lse) {
  const int D = C / heads, seq = H * W;
  const float sl2 = 1.4426950408889634f / sqrtf((float)D);
  dim3 grid((seq + 63) / 64, heads, N);
  // inference (lse null) runs an instantiation without the log-sum-exp store
  if (D == 16) lse ? mha_flash_kernel<16, true><<<grid, 128, 0, s>>>(qkv, out, N, C, H, W, sl2, lse)
                   : mha_flash_kernel<16, false><<<grid, 128, 0, s>>>(qkv, out, N, C, H, W, sl2, nullptr);
  else if (D == 32) lse ? mha_flash_kernel<32, true><<<grid, 128, 0, s>>>(qkv, out, N, C, H, W, sl2, lse)
                        : mha_flash_kernel<32, false><<<grid, 128, 0, s>>>(qkv, out, N, C, H, W, sl2, nullptr);
  else if (D == 64) lse ? mha_flash_kernel<64, true><<<grid, 128, 0, s>>>(qkv, out, N, C, H, W, sl2, lse)
                        : mha_flash_kernel<64, false><<<grid, 128, 0, s>>>(qkv, out, N, C, H, W, sl2, nullptr);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ cross-attention, S > 1 keys
// attn2(x, enc) = to_out(softmax(q K^T / sqrt(D)) V) with q = to_q(LN2(x)) (a 1x1 conv of the plan), K = enc Wk^T and
// V = enc Wv^T over the S tokens of the same sample.

// K / V projections: one CTA = XKV_ROWS tokens (their encodings in shared memory), one thread per output channel of K | V;
// each weight element is read once per CTA.  bf16 [N][S][C] out.
constexpr int XKV_ROWS = 8;
__global__ void __launch_bounds__(256) xattn_kv_kernel(const float* __restrict__ enc, const float* __restrict__ wk,
                                                       const float* __restrict__ wv, __nv_bfloat16* __restrict__ k,
                                                       __nv_bfloat16* __restrict__ v, int M, int C, int X) {
  extern __shared__ float es[];   // [XKV_ROWS][X]
  const int m0 = blockIdx.x * XKV_ROWS, rows = min(XKV_ROWS, M - m0);
  for (int i = threadIdx.x; i < XKV_ROWS * X; i += blockDim.x) es[i] = i < rows * X ? enc[(long long)m0 * X + i] : 0.f;
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) {
    const float* w = c < C ? wk + (long long)c * X : wv + (long long)(c - C) * X;
    float a[XKV_ROWS];
#pragma unroll
    for (int r = 0; r < XKV_ROWS; ++r) a[r] = 0.f;
    for (int x = 0; x < X; ++x) {
      const float wx = __ldg(w + x);
#pragma unroll
      for (int r = 0; r < XKV_ROWS; ++r) a[r] = fmaf(wx, es[r * X + x], a[r]);
    }
    __nv_bfloat16* dst = c < C ? k + c : v + (c - C);
#pragma unroll
    for (int r = 0; r < XKV_ROWS; ++r)
      if (r < rows) dst[(long long)(m0 + r) * C] = __float2bfloat16(a[r]);
  }
}
cudaError_t launch_xattn_kv(const float* enc, const float* wk, const float* wv, __nv_bfloat16* k, __nv_bfloat16* v, int N, int S,
                            int C, int X, cudaStream_t s) {
  const int M = N * S;
  xattn_kv_kernel<<<(M + XKV_ROWS - 1) / XKV_ROWS, 256, (size_t)XKV_ROWS * X * sizeof(float), s>>>(enc, wk, wv, k, v, M, C, X);
  return cudaGetLastError();
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __float2bfloat16(src[i]);
}
cudaError_t launch_f32_to_bf16(const float* src, __nv_bfloat16* dst, long long n, cudaStream_t s) {
  f32_to_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, dst, n);
  return cudaGetLastError();
}

// Forward: one CTA = one (sample, head), K and V staged once, then XATTN_QT tiles of 64 queries (4 warps x 16 rows); keys
// in tiles of 64 with the online softmax of mha_flash_kernel (exp2 domain, P V by transposing ldmatrix).  Keys S..SP-1
// are masked; 8-key column tiles and 16-key P V steps wholly beyond S are skipped (warp-uniform).
constexpr int XATTN_QT = 4;
template <int D, bool LSE>
__global__ void __launch_bounds__(128) xattn_fwd_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                        const __nv_bfloat16* __restrict__ v, __nv_bfloat16* __restrict__ out,
                                                        int N, int C, int H, int W, int S, float scale_log2,
                                                        float* __restrict__ lse) {
  constexpr int DP = D / 8, KS = D / 16;
  extern __shared__ __align__(16) uint4 xsm[];
  const int SP = (S + 63) & ~63;
  uint4* ks = xsm;
  uint4* vs = xsm + DP * SP;
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3, heads = gridDim.y;
  const int head = blockIdx.y, n = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
  xattn_stage_kv<D>(ks, vs, k, v, n, head, C, S, SP);
  __syncthreads();
  const uint32_t* ks32 = reinterpret_cast<const uint32_t*>(ks);
  const uint32_t vs_addr = smem_u32(vs);
  const __nv_bfloat16* qb = q + ((long long)n * planes + head * DP) * g.PL * 8;
  __nv_bfloat16* ob = out + ((long long)n * planes + head * DP) * g.PL * 8;
  const int ntiles = (seq + 63) / 64;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int q0 = tile * 64;
    const int r0 = min(q0 + warp * 16 + gq, seq - 1), r1 = min(q0 + warp * 16 + gq + 8, seq - 1);
    const long long o0 = pf8_pixel(g, r0, W), o1 = pf8_pixel(g, r1, W);
    uint32_t qa[KS][4];
#pragma unroll
    for (int j = 0; j < KS; ++j) {
      qa[j][0] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j) * g.PL * 8 + o0 + 2 * tq);
      qa[j][1] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j) * g.PL * 8 + o1 + 2 * tq);
      qa[j][2] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j + 1) * g.PL * 8 + o0 + 2 * tq);
      qa[j][3] = *reinterpret_cast<const uint32_t*>(qb + (long long)(2 * j + 1) * g.PL * 8 + o1 + 2 * tq);
    }
    float oacc[DP][4];
#pragma unroll
    for (int i = 0; i < DP; ++i) { oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    for (int k0 = 0; k0 < S; k0 += 64) {
      float sc[8][4];
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        sc[t][0] = sc[t][1] = sc[t][2] = sc[t][3] = 0.f;
        if (k0 + t * 8 < S) {
#pragma unroll
          for (int j = 0; j < KS; ++j) {
            const uint32_t b0 = ks32[((2 * j) * SP + k0 + t * 8 + gq) * 4 + tq];
            const uint32_t b1 = ks32[((2 * j + 1) * SP + k0 + t * 8 + gq) * 4 + tq];
            mma_bf16_16x8x16(sc[t], qa[j][0], qa[j][1], qa[j][2], qa[j][3], b0, b1);
          }
        }
      }
      float mx0 = m0, mx1 = m1;
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int key = k0 + t * 8 + 2 * tq;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float x = (key + (e & 1) < S) ? sc[t][e] * scale_log2 : -INFINITY;
          sc[t][e] = x;
          if (e < 2) mx0 = fmaxf(mx0, x); else mx1 = fmaxf(mx1, x);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float c0 = exp2f(m0 - mx0), c1 = exp2f(m1 - mx1);
      m0 = mx0; m1 = mx1;
      l0 *= c0; l1 *= c1;
#pragma unroll
      for (int i = 0; i < DP; ++i) { oacc[i][0] *= c0; oacc[i][1] *= c0; oacc[i][2] *= c1; oacc[i][3] *= c1; }
#pragma unroll
      for (int kb16 = 0; kb16 < 4; ++kb16) {
        if (k0 + kb16 * 16 >= S) continue;
        float* s0 = sc[2 * kb16];
        float* s1 = sc[2 * kb16 + 1];
        const float e00 = exp2f(s0[0] - m0), e01 = exp2f(s0[1] - m0), e02 = exp2f(s0[2] - m1), e03 = exp2f(s0[3] - m1);
        const float e10 = exp2f(s1[0] - m0), e11 = exp2f(s1[1] - m0), e12 = exp2f(s1[2] - m1), e13 = exp2f(s1[3] - m1);
        l0 += (e00 + e01) + (e10 + e11);
        l1 += (e02 + e03) + (e12 + e13);
        const uint32_t pa0 = pack_bf16x2(e00, e01), pa1 = pack_bf16x2(e02, e03), pa2 = pack_bf16x2(e10, e11),
                       pa3 = pack_bf16x2(e12, e13);
#pragma unroll
        for (int i = 0; i < DP; ++i) {
          uint32_t vb0, vb1;
          const uint32_t va = vs_addr + (uint32_t)((i * SP + k0 + kb16 * 16 + (lane & 15)) * 16);
          asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(vb0), "=r"(vb1) : "r"(va));
          mma_bf16_16x8x16(oacc[i], pa0, pa1, pa2, pa3, vb0, vb1);
        }
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    const int q_a = q0 + warp * 16 + gq, q_b = q_a + 8;
#pragma unroll
    for (int i = 0; i < DP; ++i) {
      if (q_a < seq) *reinterpret_cast<uint32_t*>(ob + (long long)i * g.PL * 8 + o0 + 2 * tq) = pack_bf16x2(oacc[i][0] * i0, oacc[i][1] * i0);
      if (q_b < seq) *reinterpret_cast<uint32_t*>(ob + (long long)i * g.PL * 8 + o1 + 2 * tq) = pack_bf16x2(oacc[i][2] * i1, oacc[i][3] * i1);
    }
    if (LSE && tq == 0) {
      float* lr = lse + ((long long)n * heads + head) * seq;
      if (q_a < seq) lr[q_a] = m0 + __log2f(l0);
      if (q_b < seq) lr[q_b] = m1 + __log2f(l1);
    }
  }
}

template <int D, bool LSE>
static cudaError_t xattn_launch(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v, __nv_bfloat16* out, int N,
                                int C, int heads, int H, int W, int S, cudaStream_t s, float* lse) {
  const size_t smem = (size_t)2 * (D / 8) * ((S + 63) & ~63) * sizeof(uint4);
  static const cudaError_t attr = cudaFuncSetAttribute(xattn_fwd_kernel<D, LSE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       2 * (D / 8) * XATTN_MAX_S * (int)sizeof(uint4));
  if (attr != cudaSuccess) return attr;
  const int ntiles = (H * W + 63) / 64;
  const dim3 grid((ntiles + XATTN_QT - 1) / XATTN_QT, heads, N);
  xattn_fwd_kernel<D, LSE><<<grid, 128, smem, s>>>(q, k, v, out, N, C, H, W, S, 1.4426950408889634f / sqrtf((float)D), lse);
  return cudaGetLastError();
}
cudaError_t launch_xattn(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v, __nv_bfloat16* out, int N,
                         int C, int heads, int H, int W, int S, cudaStream_t s, float* lse) {
  if (S < 1 || S > XATTN_MAX_S || C % heads) return cudaErrorInvalidValue;
  const int D = C / heads;
  // inference (lse null) runs an instantiation without the log-sum-exp store
  if (D == 16) return lse ? xattn_launch<16, true>(q, k, v, out, N, C, heads, H, W, S, s, lse)
                          : xattn_launch<16, false>(q, k, v, out, N, C, heads, H, W, S, s, nullptr);
  if (D == 32) return lse ? xattn_launch<32, true>(q, k, v, out, N, C, heads, H, W, S, s, lse)
                          : xattn_launch<32, false>(q, k, v, out, N, C, heads, H, W, S, s, nullptr);
  if (D == 64) return lse ? xattn_launch<64, true>(q, k, v, out, N, C, heads, H, W, S, s, lse)
                          : xattn_launch<64, false>(q, k, v, out, N, C, heads, H, W, S, s, nullptr);
  return cudaErrorInvalidValue;
}

}  // namespace b200ad
