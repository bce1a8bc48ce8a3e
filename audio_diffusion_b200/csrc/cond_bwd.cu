// Backward kernels of the conditional U-Net's transformer blocks (the forward is cond_ops.cu; the walk is
// BwdBuilder::transformer_bwd in backward.cu): LayerNorm and GEGLU backward, the cross-attention vector's weight
// gradients, and the multi-head self-attention backward on tensor cores (FlashAttention-2 style: P is recomputed from Q, K
// and the row log-sum-exp the training forward saved, never materialised).
// Oracle: torch autograd over oracle/unet_cond_oracle.py.
#include "bwd_kernels.cuh"

namespace b200ad {

__device__ __forceinline__ void unpack8_f(const uint4& v, float (&f)[8]) {
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) { const float2 t = unpack_bf16x2(u[e]); f[2 * e] = t.x; f[2 * e + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8_f(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}
__device__ __forceinline__ float warp_allsum(float v) {
#pragma unroll
  for (int sh = 16; sh >= 1; sh >>= 1) v += __shfl_xor_sync(0xffffffffu, v, sh);
  return v;
}

// ------------------------------------------------------------------------------------ LayerNorm over channels, backward
// y = xhat * gamma + beta, xhat = (x - mean) * rstd (mean / rstd recomputed from the kept input exactly as the forward does):
//   gx = rstd * (gy gamma - mean_c(gy gamma) - xhat * mean_c(gy gamma xhat)) + add;  dgamma += sum gy xhat, dbeta += sum gy.
// One warp per pixel (lane l holds planes l and l + 32: C <= 512), LNB_PIX pixels per warp; the CTA's dgamma / dbeta partial
// sums meet in shared memory and are added to the fp32 gradients once per CTA.
constexpr int LNB_PIX = 32;
__global__ void __launch_bounds__(256) layernorm_bwd_pf8_kernel(const __nv_bfloat16* __restrict__ x,
                                                                const __nv_bfloat16* __restrict__ gy,
                                                                const __nv_bfloat16* __restrict__ add,
                                                                __nv_bfloat16* __restrict__ gx, const float* __restrict__ gamma,
                                                                float* __restrict__ dgamma, float* __restrict__ dbeta, int N,
                                                                int C, int H, int W, float eps) {
  __shared__ float red[2][512];
  const Geom g = make_geom(N, H, W);
  const int planes = C >> 3, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n = blockIdx.y;
  for (int i = threadIdx.x; i < C; i += blockDim.x) { red[0][i] = 0.f; red[1][i] = 0.f; }
  float gam[2][8], ag[2][8], ab[2][8];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int pl = lane + 32 * j;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      gam[j][e] = pl < planes ? __ldg(gamma + pl * 8 + e) : 0.f;
      ag[j][e] = 0.f;
      ab[j][e] = 0.f;
    }
  }
  __syncthreads();
  const long long img = (long long)n * planes * g.PL * 8;
  const float invC = 1.0f / (float)C;
  for (int k = 0; k < LNB_PIX; ++k) {
    const int p = (blockIdx.x * LNB_PIX + k) * 8 + warp;
    if (p >= H * W) break;
    const long long off = img + (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
    float xv[2][8], gv[2][8];
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int pl = lane + 32 * j;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (pl < planes) {
        a = *reinterpret_cast<const uint4*>(x + off + (long long)pl * g.PL * 8);
        b = *reinterpret_cast<const uint4*>(gy + off + (long long)pl * g.PL * 8);
      }
      unpack8_f(a, xv[j]);
      unpack8_f(b, gv[j]);
#pragma unroll
      for (int e = 0; e < 8; ++e) { s += xv[j][e]; q += xv[j][e] * xv[j][e]; }
    }
    s = warp_allsum(s);
    q = warp_allsum(q);
    const float mean = s * invC;
    const float rstd = rsqrtf(fmaxf(q * invC - mean * mean, 0.f) + eps);
    float a1 = 0.f, a2 = 0.f;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        xv[j][e] = (xv[j][e] - mean) * rstd;            // xhat
        const float gg = gv[j][e] * gam[j][e];
        a1 += gg;
        a2 = fmaf(gg, xv[j][e], a2);
        ag[j][e] = fmaf(gv[j][e], xv[j][e], ag[j][e]);
        ab[j][e] += gv[j][e];
      }
    a1 = warp_allsum(a1) * invC;
    a2 = warp_allsum(a2) * invC;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int pl = lane + 32 * j;
      if (pl >= planes) continue;
      float r[8], o[8];
      if (add) unpack8_f(*reinterpret_cast<const uint4*>(add + off + (long long)pl * g.PL * 8), r);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rstd * (gv[j][e] * gam[j][e] - a1 - xv[j][e] * a2) + (add ? r[e] : 0.f);
      *reinterpret_cast<uint4*>(gx + off + (long long)pl * g.PL * 8) = pack8_f(o);
    }
  }
  if (!dgamma) return;   // no parameter gradients (uniform over the CTA)
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int pl = lane + 32 * j;
    if (pl >= planes) continue;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      atomicAdd(&red[0][pl * 8 + e], ag[j][e]);
      atomicAdd(&red[1][pl * 8 + e], ab[j][e]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    atomicAdd(dgamma + i, red[0][i]);
    atomicAdd(dbeta + i, red[1][i]);
  }
}
cudaError_t launch_layernorm_bwd_pf8(const __nv_bfloat16* x, const __nv_bfloat16* gy, const __nv_bfloat16* add,
                                     __nv_bfloat16* gx, const float* gamma, float* dgamma, float* dbeta, int N, int C, int H,
                                     int W, float eps, cudaStream_t s) {
  if (C > 512 || C % 8) return cudaErrorInvalidValue;
  const int per_cta = LNB_PIX * 8;
  layernorm_bwd_pf8_kernel<<<dim3((H * W + per_cta - 1) / per_cta, N), 256, 0, s>>>(x, gy, add, gx, gamma, dgamma, dbeta, N, C,
                                                                                      H, W, eps);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ GEGLU backward
// src: the forward's PF8 input with 2*Ch channels (hidden | gate), gy: gradient of hidden * gelu(gate) (Ch channels),
// dst: 2*Ch channels:  d hidden = gy gelu(gate),  d gate = gy hidden gelu'(gate),  exact (erf) GELU.
__global__ void __launch_bounds__(256) geglu_bwd_pf8_kernel(const __nv_bfloat16* __restrict__ src,
                                                            const __nv_bfloat16* __restrict__ gy,
                                                            __nv_bfloat16* __restrict__ dst, int N, int Ch, int H, int W) {
  const Geom g = make_geom(N, H, W);
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= H * W) return;
  const int pl = blockIdx.y, n = blockIdx.z, planes = Ch >> 3;
  const long long off = (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
  const long long img2 = (long long)n * 2 * planes * g.PL * 8;
  float hv[8], tv[8], dy[8], dh[8], dg[8];
  unpack8_f(*reinterpret_cast<const uint4*>(src + img2 + (long long)pl * g.PL * 8 + off), hv);
  unpack8_f(*reinterpret_cast<const uint4*>(src + img2 + (long long)(planes + pl) * g.PL * 8 + off), tv);
  unpack8_f(*reinterpret_cast<const uint4*>(gy + ((long long)n * planes + pl) * g.PL * 8 + off), dy);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float t = tv[e];
    const float cdf = 0.5f * (1.0f + erff(t * 0.70710678118654752f));
    const float pdf = 0.39894228040143268f * __expf(-0.5f * t * t);
    dh[e] = dy[e] * t * cdf;
    dg[e] = dy[e] * hv[e] * fmaf(t, pdf, cdf);
  }
  *reinterpret_cast<uint4*>(dst + img2 + (long long)pl * g.PL * 8 + off) = pack8_f(dh);
  *reinterpret_cast<uint4*>(dst + img2 + (long long)(planes + pl) * g.PL * 8 + off) = pack8_f(dg);
}
cudaError_t launch_geglu_bwd_pf8(const __nv_bfloat16* src, const __nv_bfloat16* gy, __nv_bfloat16* dst, int N, int Ch, int H,
                                 int W, cudaStream_t s) {
  geglu_bwd_pf8_kernel<<<dim3((H * W + 255) / 256, Ch >> 3, N), 256, 0, s>>>(src, gy, dst, N, Ch, H, W);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ cross-attention vector, backward
// Forward (cross_attn_vec_kernel): v[n] = Wv enc[n], vec[n] = Wo v[n] + bo, added to every pixel of h2. With dvec[n][c] =
// sum over the pixels of G(h2) (the per-sample channel sums the attn1.to_out bias gradient already makes):
//   dv[n] = Wo^T dvec[n];  dWo[c][i] += sum_n dvec[n][c] v[n][i];  dWv[i][x] += sum_n dv[n][i] enc[n][x].
// (The bias gradient, sum_n dvec[n], is written by that bias-gradient launch.)  Pass 1: grid N, v and dv into scratch.
__global__ void __launch_bounds__(256) cross_attn_vec_bwd_kernel(const float* __restrict__ enc, const float* __restrict__ dvec,
                                                                 const float* __restrict__ wv, const float* __restrict__ wo,
                                                                 float* __restrict__ vdv, int N, int C, int X) {
  extern __shared__ float csm[];   // enc[X], dvec[C]
  float* es = csm;
  float* ds = csm + X;
  const int n = blockIdx.x;
  for (int i = threadIdx.x; i < X; i += blockDim.x) es[i] = enc[(long long)n * X + i];
  for (int i = threadIdx.x; i < C; i += blockDim.x) ds[i] = dvec[(long long)n * C + i];
  __syncthreads();
  float* v = vdv + (long long)n * C;
  float* dv = vdv + (long long)(N + n) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f;
    for (int i = 0; i < X; ++i) a = fmaf(__ldg(wv + (long long)c * X + i), es[i], a);
    v[c] = a;
    float b = 0.f;   // column c of Wo: consecutive threads read consecutive addresses
    for (int o = 0; o < C; ++o) b = fmaf(__ldg(wo + (long long)o * C + c), ds[o], b);
    dv[c] = b;
  }
}
// pass 2: one thread per weight-gradient element (Wo: C x C, then Wv: C x X)
__global__ void __launch_bounds__(256) cross_attn_vec_wgrad_kernel(const float* __restrict__ enc, const float* __restrict__ dvec,
                                                                   const float* __restrict__ vdv, float* __restrict__ dwo,
                                                                   float* __restrict__ dwv, int N, int C, int X) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nwo = (long long)C * C;
  if (idx < nwo) {
    const int c = (int)(idx / C), i = (int)(idx - (long long)c * C);
    float a = 0.f;
    for (int n = 0; n < N; ++n) a = fmaf(dvec[(long long)n * C + c], vdv[(long long)n * C + i], a);
    dwo[idx] += a;
  } else if (idx < nwo + (long long)C * X) {
    const long long j = idx - nwo;
    const int c = (int)(j / X), xi = (int)(j - (long long)c * X);
    float a = 0.f;
    for (int n = 0; n < N; ++n) a = fmaf(vdv[(long long)(N + n) * C + c], enc[(long long)n * X + xi], a);
    dwv[j] += a;
  }
}
cudaError_t launch_cross_attn_vec_bwd(const float* enc, const float* dvec, const float* wv, const float* wo, float* dwo,
                                      float* dwv, float* scratch, int N, int C, int X, cudaStream_t s) {
  cross_attn_vec_bwd_kernel<<<N, 256, (size_t)(X + C) * sizeof(float), s>>>(enc, dvec, wv, wo, scratch, N, C, X);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const long long tot = (long long)C * C + (long long)C * X;
  cross_attn_vec_wgrad_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(enc, dvec, scratch, dwo, dwv, N, C, X);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ multi-head self-attention, backward
// Same PF8 q | k | v layout and head split as mha_flash_kernel. With S = Q K^T / sqrt(D), P = softmax(S) (rows = queries),
// dP = dO V^T, D_i = rowsum(dO o O)_i = sum_j P_ij dP_ij:   dS = P o (dP - D),  dV = P^T dO,  dK = dS^T Q / sqrt(D),
// dQ = dS K / sqrt(D).  P is recomputed from Q, K and the forward's row log-sum-exp (log2 domain of the scaled scores).
// Three launches: D; dK and dV (key-block parallel, accumulators in registers); dQ (query-block parallel, accumulators in
// registers).  The separate dQ kernel recomputes S and dP once more (7 instead of 5 seq^2 D matrix products) but needs no
// fp32 scratch and no atomics: every element of dQ is written once, so the result is deterministic.

// D[n][head][i] = sum_d dO[i][d] O[i][d]
template <int D>
__global__ void __launch_bounds__(256) mha_bwd_dot_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ go,
                                                          float* __restrict__ dsum, int N, int C, int H, int W) {
  constexpr int DP = D / 8;
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= seq) return;
  const int head = blockIdx.y, n = blockIdx.z, heads = gridDim.y;
  const long long base = ((long long)n * (C >> 3) + head * DP) * g.PL * 8 + pf8_pixel(g, p, W);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < DP; ++i) {
    float a[8], b[8];
    unpack8_f(*reinterpret_cast<const uint4*>(o + base + (long long)i * g.PL * 8), a);
    unpack8_f(*reinterpret_cast<const uint4*>(go + base + (long long)i * g.PL * 8), b);
#pragma unroll
    for (int e = 0; e < 8; ++e) s = fmaf(a[e], b[e], s);
  }
  dsum[((long long)n * heads + head) * seq + p] = s;
}

// A fragments (m16 x k16, row-major) of 16 rows r0 / r1 = r0 + 8 of one head of a PF8 tensor: a[j] covers channels 16j..16j+15
template <int KS>
__device__ __forceinline__ void load_rows_a(uint32_t (&a)[KS][4], const __nv_bfloat16* b, const Geom& g, long long o0,
                                            long long o1, int tq) {
#pragma unroll
  for (int j = 0; j < KS; ++j) {
    a[j][0] = *reinterpret_cast<const uint32_t*>(b + (long long)(2 * j) * g.PL * 8 + o0 + 2 * tq);
    a[j][1] = *reinterpret_cast<const uint32_t*>(b + (long long)(2 * j) * g.PL * 8 + o1 + 2 * tq);
    a[j][2] = *reinterpret_cast<const uint32_t*>(b + (long long)(2 * j + 1) * g.PL * 8 + o0 + 2 * tq);
    a[j][3] = *reinterpret_cast<const uint32_t*>(b + (long long)(2 * j + 1) * g.PL * 8 + o1 + 2 * tq);
  }
}
// B fragment (k16 x n8, "col") from a [plane][64 rows] tile whose rows run along k: transposing ldmatrix of two 8x8 tiles
__device__ __forceinline__ void ldsm_b_trans(uint32_t& b0, uint32_t& b1, uint32_t tile_addr, int plane, int k16, int lane) {
  const uint32_t a = tile_addr + (uint32_t)((plane * 64 + k16 * 16 + (lane & 15)) * 16);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(a));
}

// dK, dV: one CTA = 64 keys of one (sample, head), 4 warps x 16 keys; queries stream through shared memory in tiles of 64.
// Per tile and warp: S^T = K Q^T and dP^T = V dO^T (16 keys x 64 queries), P^T and dS^T elementwise, then dV += P^T dO and
// dK += dS^T Q with P^T / dS^T re-used from the accumulators as A fragments.
template <int D>
__global__ void __launch_bounds__(128) mha_bwd_kv_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ go,
                                                         const float* __restrict__ lse, const float* __restrict__ dsum,
                                                         __nv_bfloat16* __restrict__ gqkv, int N, int C, int H, int W,
                                                         float scale_log2, float scale) {
  constexpr int DP = D / 8, KS = D / 16;
  __shared__ __align__(16) uint4 qs[DP][64];    // [plane][query] 8 channels
  __shared__ __align__(16) uint4 dos[DP][64];
  __shared__ float ls[64], dd[64];
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3, heads = gridDim.y;
  const int head = blockIdx.y, n = blockIdx.z, k0 = blockIdx.x * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* qb = base + (long long)(head * DP) * g.PL * 8;
  const __nv_bfloat16* kb = base + (long long)(planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* vb = base + (long long)(2 * planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* gob = go + ((long long)n * planes + head * DP) * g.PL * 8;
  const float* lrow = lse + ((long long)n * heads + head) * seq;
  const float* drow = dsum + ((long long)n * heads + head) * seq;
  // this warp's 16 keys (keys beyond seq read key seq-1: their gradients are never stored)
  const int r0 = min(k0 + warp * 16 + gq, seq - 1), r1 = min(k0 + warp * 16 + gq + 8, seq - 1);
  const long long o0 = pf8_pixel(g, r0, W), o1 = pf8_pixel(g, r1, W);
  uint32_t ka[KS][4], va[KS][4];
  load_rows_a<KS>(ka, kb, g, o0, o1, tq);
  load_rows_a<KS>(va, vb, g, o0, o1, tq);
  float dk[DP][4], dv[DP][4];
#pragma unroll
  for (int i = 0; i < DP; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) { dk[i][e] = 0.f; dv[i][e] = 0.f; }
  const uint32_t* qs32 = reinterpret_cast<const uint32_t*>(qs);
  const uint32_t* do32 = reinterpret_cast<const uint32_t*>(dos);
  const uint32_t qs_addr = smem_u32(qs), do_addr = smem_u32(dos);

  for (int q0 = 0; q0 < seq; q0 += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < DP * 64; i += 128) {
      const int pl = i >> 6, qq = i & 63, q = q0 + qq;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (q < seq) {
        const long long off = pf8_pixel(g, q, W);
        a = *reinterpret_cast<const uint4*>(qb + (long long)pl * g.PL * 8 + off);
        b = *reinterpret_cast<const uint4*>(gob + (long long)pl * g.PL * 8 + off);
      }
      qs[pl][qq] = a;
      dos[pl][qq] = b;
    }
    if (threadIdx.x < 64) {   // queries beyond seq: lse = +inf -> P = 0
      const int q = q0 + threadIdx.x;
      ls[threadIdx.x] = q < seq ? lrow[q] : INFINITY;
      dd[threadIdx.x] = q < seq ? drow[q] : 0.f;
    }
    __syncthreads();
    float st[8][4], dpt[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
#pragma unroll
      for (int e = 0; e < 4; ++e) { st[t][e] = 0.f; dpt[t][e] = 0.f; }
#pragma unroll
      for (int j = 0; j < KS; ++j) {
        const int w0 = ((2 * j) * 64 + t * 8 + gq) * 4 + tq, w1 = ((2 * j + 1) * 64 + t * 8 + gq) * 4 + tq;
        mma_bf16_16x8x16(st[t], ka[j][0], ka[j][1], ka[j][2], ka[j][3], qs32[w0], qs32[w1]);
        mma_bf16_16x8x16(dpt[t], va[j][0], va[j][1], va[j][2], va[j][3], do32[w0], do32[w1]);
      }
    }
    // accumulator (e0, e1) = key row gq, queries t*8 + 2tq, +1;  (e2, e3) = key row gq + 8
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = t * 8 + 2 * tq + (e & 1);
        const float p = exp2f(st[t][e] * scale_log2 - ls[col]);
        st[t][e] = p;
        dpt[t][e] = p * (dpt[t][e] - dd[col]);
      }
#pragma unroll
    for (int k16 = 0; k16 < 4; ++k16) {
      const float* p0 = st[2 * k16];
      const float* p1 = st[2 * k16 + 1];
      const float* s0 = dpt[2 * k16];
      const float* s1 = dpt[2 * k16 + 1];
      const uint32_t pa0 = pack_bf16x2(p0[0], p0[1]), pa1 = pack_bf16x2(p0[2], p0[3]), pa2 = pack_bf16x2(p1[0], p1[1]),
                     pa3 = pack_bf16x2(p1[2], p1[3]);
      const uint32_t sa0 = pack_bf16x2(s0[0], s0[1]), sa1 = pack_bf16x2(s0[2], s0[3]), sa2 = pack_bf16x2(s1[0], s1[1]),
                     sa3 = pack_bf16x2(s1[2], s1[3]);
#pragma unroll
      for (int i = 0; i < DP; ++i) {
        uint32_t b0, b1;
        ldsm_b_trans(b0, b1, do_addr, i, k16, lane);
        mma_bf16_16x8x16(dv[i], pa0, pa1, pa2, pa3, b0, b1);
        ldsm_b_trans(b0, b1, qs_addr, i, k16, lane);
        mma_bf16_16x8x16(dk[i], sa0, sa1, sa2, sa3, b0, b1);
      }
    }
  }
  __nv_bfloat16* gb = gqkv + (long long)n * 3 * planes * g.PL * 8;
  const int ka_row = k0 + warp * 16 + gq, kb_row = ka_row + 8;
#pragma unroll
  for (int i = 0; i < DP; ++i) {   // accumulator (c0, c1) = (row gq, channels 8i + 2tq, +1), (c2, c3) = row gq + 8
    __nv_bfloat16* kd = gb + (long long)(planes + head * DP + i) * g.PL * 8;
    __nv_bfloat16* vd = gb + (long long)(2 * planes + head * DP + i) * g.PL * 8;
    if (ka_row < seq) {
      *reinterpret_cast<uint32_t*>(kd + o0 + 2 * tq) = pack_bf16x2(dk[i][0] * scale, dk[i][1] * scale);
      *reinterpret_cast<uint32_t*>(vd + o0 + 2 * tq) = pack_bf16x2(dv[i][0], dv[i][1]);
    }
    if (kb_row < seq) {
      *reinterpret_cast<uint32_t*>(kd + o1 + 2 * tq) = pack_bf16x2(dk[i][2] * scale, dk[i][3] * scale);
      *reinterpret_cast<uint32_t*>(vd + o1 + 2 * tq) = pack_bf16x2(dv[i][2], dv[i][3]);
    }
  }
}

// dQ: one CTA = 64 queries of one (sample, head), 4 warps x 16 queries; keys stream through shared memory in tiles of 64.
// Per tile and warp: S = Q K^T and dP = dO V^T, dS = P o (dP - D) (keys beyond seq masked), dQ += dS K.
template <int D>
__global__ void __launch_bounds__(128) mha_bwd_dq_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ go,
                                                         const float* __restrict__ lse, const float* __restrict__ dsum,
                                                         __nv_bfloat16* __restrict__ gqkv, int N, int C, int H, int W,
                                                         float scale_log2, float scale) {
  constexpr int DP = D / 8, KS = D / 16;
  __shared__ __align__(16) uint4 ks[DP][64];    // [plane][key] 8 channels
  __shared__ __align__(16) uint4 vs[DP][64];
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3, heads = gridDim.y;
  const int head = blockIdx.y, n = blockIdx.z, q0 = blockIdx.x * 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* qb = base + (long long)(head * DP) * g.PL * 8;
  const __nv_bfloat16* kb = base + (long long)(planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* vb = base + (long long)(2 * planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* gob = go + ((long long)n * planes + head * DP) * g.PL * 8;
  const int r0 = min(q0 + warp * 16 + gq, seq - 1), r1 = min(q0 + warp * 16 + gq + 8, seq - 1);
  const long long o0 = pf8_pixel(g, r0, W), o1 = pf8_pixel(g, r1, W);
  uint32_t qa[KS][4], oa[KS][4];
  load_rows_a<KS>(qa, qb, g, o0, o1, tq);
  load_rows_a<KS>(oa, gob, g, o0, o1, tq);
  const long long rowb = ((long long)n * heads + head) * seq;
  const float l0 = lse[rowb + r0], l1 = lse[rowb + r1], d0 = dsum[rowb + r0], d1 = dsum[rowb + r1];
  float dq[DP][4];
#pragma unroll
  for (int i = 0; i < DP; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }
  const uint32_t* ks32 = reinterpret_cast<const uint32_t*>(ks);
  const uint32_t* vs32 = reinterpret_cast<const uint32_t*>(vs);
  const uint32_t ks_addr = smem_u32(ks);

  for (int k0 = 0; k0 < seq; k0 += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < DP * 64; i += 128) {
      const int pl = i >> 6, kk = i & 63, key = k0 + kk;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (key < seq) {
        const long long off = pf8_pixel(g, key, W);
        a = *reinterpret_cast<const uint4*>(kb + (long long)pl * g.PL * 8 + off);
        b = *reinterpret_cast<const uint4*>(vb + (long long)pl * g.PL * 8 + off);
      }
      ks[pl][kk] = a;
      vs[pl][kk] = b;
    }
    __syncthreads();
    float sc[8][4], dp[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
#pragma unroll
      for (int e = 0; e < 4; ++e) { sc[t][e] = 0.f; dp[t][e] = 0.f; }
#pragma unroll
      for (int j = 0; j < KS; ++j) {
        const int w0 = ((2 * j) * 64 + t * 8 + gq) * 4 + tq, w1 = ((2 * j + 1) * 64 + t * 8 + gq) * 4 + tq;
        mma_bf16_16x8x16(sc[t], qa[j][0], qa[j][1], qa[j][2], qa[j][3], ks32[w0], ks32[w1]);
        mma_bf16_16x8x16(dp[t], oa[j][0], oa[j][1], oa[j][2], oa[j][3], vs32[w0], vs32[w1]);
      }
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int key = k0 + t * 8 + 2 * tq;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = (key + (e & 1) < seq) ? exp2f(sc[t][e] * scale_log2 - (e < 2 ? l0 : l1)) : 0.f;
        dp[t][e] = p * (dp[t][e] - (e < 2 ? d0 : d1));
      }
    }
#pragma unroll
    for (int k16 = 0; k16 < 4; ++k16) {
      const float* s0 = dp[2 * k16];
      const float* s1 = dp[2 * k16 + 1];
      const uint32_t sa0 = pack_bf16x2(s0[0], s0[1]), sa1 = pack_bf16x2(s0[2], s0[3]), sa2 = pack_bf16x2(s1[0], s1[1]),
                     sa3 = pack_bf16x2(s1[2], s1[3]);
#pragma unroll
      for (int i = 0; i < DP; ++i) {
        uint32_t b0, b1;
        ldsm_b_trans(b0, b1, ks_addr, i, k16, lane);
        mma_bf16_16x8x16(dq[i], sa0, sa1, sa2, sa3, b0, b1);
      }
    }
  }
  __nv_bfloat16* qd = gqkv + (long long)n * 3 * planes * g.PL * 8 + (long long)(head * DP) * g.PL * 8;
  const int qa_row = q0 + warp * 16 + gq, qb_row = qa_row + 8;
#pragma unroll
  for (int i = 0; i < DP; ++i) {
    if (qa_row < seq) *reinterpret_cast<uint32_t*>(qd + (long long)i * g.PL * 8 + o0 + 2 * tq) = pack_bf16x2(dq[i][0] * scale, dq[i][1] * scale);
    if (qb_row < seq) *reinterpret_cast<uint32_t*>(qd + (long long)i * g.PL * 8 + o1 + 2 * tq) = pack_bf16x2(dq[i][2] * scale, dq[i][3] * scale);
  }
}

template <int D>
static cudaError_t mha_bwd_launch(const __nv_bfloat16* qkv, const __nv_bfloat16* o, const __nv_bfloat16* go, const float* lse,
                                  float* dsum, __nv_bfloat16* gqkv, int N, int C, int heads, int H, int W, cudaStream_t s) {
  const int seq = H * W;
  const float scale = 1.0f / sqrtf((float)D), sl2 = 1.4426950408889634f * scale;
  mha_bwd_dot_kernel<D><<<dim3((seq + 255) / 256, heads, N), 256, 0, s>>>(o, go, dsum, N, C, H, W);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const dim3 grid((seq + 63) / 64, heads, N);
  mha_bwd_kv_kernel<D><<<grid, 128, 0, s>>>(qkv, go, lse, dsum, gqkv, N, C, H, W, sl2, scale);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  mha_bwd_dq_kernel<D><<<grid, 128, 0, s>>>(qkv, go, lse, dsum, gqkv, N, C, H, W, sl2, scale);
  return cudaGetLastError();
}
cudaError_t launch_mha_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* o, const __nv_bfloat16* go, const float* lse,
                           float* dsum, __nv_bfloat16* gqkv, int N, int C, int heads, int H, int W, cudaStream_t s) {
  const int D = C / heads;
  if (D * heads != C) return cudaErrorInvalidValue;
  if (D == 16) return mha_bwd_launch<16>(qkv, o, go, lse, dsum, gqkv, N, C, heads, H, W, s);
  if (D == 32) return mha_bwd_launch<32>(qkv, o, go, lse, dsum, gqkv, N, C, heads, H, W, s);
  if (D == 64) return mha_bwd_launch<64>(qkv, o, go, lse, dsum, gqkv, N, C, heads, H, W, s);
  return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------ cross-attention, S > 1 keys, backward
// The forward is xattn_fwd_kernel (cond_ops.cu): q and O are PF8 tensors of C channels, K and V bf16 [N][S][C].  The same
// identities as the self-attention backward above, in four launches: D = rowsum(dO o O) (mha_bwd_dot_kernel); dQ
// (query-parallel, K and V staged once per CTA); dK and dV as fp32 partial sums per split of the queries (65 536 queries
// of one sample meet at most 256 keys, so the key-parallel form alone would leave most SMs idle); the partials added in
// split order.

// B fragment (k16 x n8, "col") by transposing ldmatrix from a [plane][SP rows] tile whose rows run along k
__device__ __forceinline__ void ldsm_b_trans_sp(uint32_t& b0, uint32_t& b1, uint32_t tile_addr, int plane, int SP, int row0,
                                                int lane) {
  const uint32_t a = tile_addr + (uint32_t)((plane * SP + row0 + (lane & 15)) * 16);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(a));
}

// dQ: one CTA = one (sample, head), K / V staged once, XATTN_BWD_QT tiles of 64 queries; per 64-key tile and warp:
// S = Q K^T, dP = dO V^T, dS = P o (dP - D) (keys beyond S masked), dQ += dS K.
constexpr int XATTN_BWD_QT = 4;
template <int D>
// (minimum 1 CTA per SM: without it ptxas caps the D = 16 / 32 instantiations below their needs and spills)
__global__ void __launch_bounds__(128, 1) xattn_bwd_dq_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                           const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ go,
                                                           const float* __restrict__ lse, const float* __restrict__ dsum,
                                                           __nv_bfloat16* __restrict__ gq, int N, int C, int H, int W, int S,
                                                           float scale_log2, float scale) {
  constexpr int DP = D / 8, KS = D / 16;
  extern __shared__ __align__(16) uint4 xsm[];
  const int SP = (S + 63) & ~63;
  uint4* ks = xsm;
  uint4* vs = xsm + DP * SP;
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3, heads = gridDim.y;
  const int head = blockIdx.y, n = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq8 = lane >> 2, tq = lane & 3;
  xattn_stage_kv<D>(ks, vs, k, v, n, head, C, S, SP);
  __syncthreads();
  const uint32_t* ks32 = reinterpret_cast<const uint32_t*>(ks);
  const uint32_t* vs32 = reinterpret_cast<const uint32_t*>(vs);
  const uint32_t ks_addr = smem_u32(ks);
  const long long hoff = ((long long)n * planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* qb = q + hoff;
  const __nv_bfloat16* gob = go + hoff;
  __nv_bfloat16* qd = gq + hoff;
  const long long rowb = ((long long)n * heads + head) * seq;
  const int ntiles = (seq + 63) / 64;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int q0 = tile * 64;
    const int r0 = min(q0 + warp * 16 + gq8, seq - 1), r1 = min(q0 + warp * 16 + gq8 + 8, seq - 1);
    const long long o0 = pf8_pixel(g, r0, W), o1 = pf8_pixel(g, r1, W);
    uint32_t qa[KS][4], oa[KS][4];
    load_rows_a<KS>(qa, qb, g, o0, o1, tq);
    load_rows_a<KS>(oa, gob, g, o0, o1, tq);
    const float l0 = lse[rowb + r0], l1 = lse[rowb + r1], d0 = dsum[rowb + r0], d1 = dsum[rowb + r1];
    float dq[DP][4];
#pragma unroll
    for (int i = 0; i < DP; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }
    for (int k0 = 0; k0 < S; k0 += 64) {
      float sc[8][4], dp[8][4];
#pragma unroll
      for (int t = 0; t < 8; ++t) {
#pragma unroll
        for (int e = 0; e < 4; ++e) { sc[t][e] = 0.f; dp[t][e] = 0.f; }
        if (k0 + t * 8 < S) {
#pragma unroll
          for (int j = 0; j < KS; ++j) {
            const int w0 = ((2 * j) * SP + k0 + t * 8 + gq8) * 4 + tq, w1 = ((2 * j + 1) * SP + k0 + t * 8 + gq8) * 4 + tq;
            mma_bf16_16x8x16(sc[t], qa[j][0], qa[j][1], qa[j][2], qa[j][3], ks32[w0], ks32[w1]);
            mma_bf16_16x8x16(dp[t], oa[j][0], oa[j][1], oa[j][2], oa[j][3], vs32[w0], vs32[w1]);
          }
        }
      }
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int key = k0 + t * 8 + 2 * tq;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float p = (key + (e & 1) < S) ? exp2f(sc[t][e] * scale_log2 - (e < 2 ? l0 : l1)) : 0.f;
          dp[t][e] = p * (dp[t][e] - (e < 2 ? d0 : d1));
        }
      }
#pragma unroll
      for (int k16 = 0; k16 < 4; ++k16) {
        if (k0 + k16 * 16 < S) {
          const float* s0 = dp[2 * k16];
          const float* s1 = dp[2 * k16 + 1];
          const uint32_t sa0 = pack_bf16x2(s0[0], s0[1]), sa1 = pack_bf16x2(s0[2], s0[3]), sa2 = pack_bf16x2(s1[0], s1[1]),
                         sa3 = pack_bf16x2(s1[2], s1[3]);
#pragma unroll
          for (int i = 0; i < DP; ++i) {
            uint32_t b0, b1;
            ldsm_b_trans_sp(b0, b1, ks_addr, i, SP, k0 + k16 * 16, lane);
            mma_bf16_16x8x16(dq[i], sa0, sa1, sa2, sa3, b0, b1);
          }
        }
      }
    }
    const int qa_row = q0 + warp * 16 + gq8, qb_row = qa_row + 8;
#pragma unroll
    for (int i = 0; i < DP; ++i) {
      if (qa_row < seq) *reinterpret_cast<uint32_t*>(qd + (long long)i * g.PL * 8 + o0 + 2 * tq) = pack_bf16x2(dq[i][0] * scale, dq[i][1] * scale);
      if (qb_row < seq) *reinterpret_cast<uint32_t*>(qd + (long long)i * g.PL * 8 + o1 + 2 * tq) = pack_bf16x2(dq[i][2] * scale, dq[i][3] * scale);
    }
  }
}

// How the queries of one (sample, head) are split for the dK / dV partial sums: a function of the shapes only (not of
// the GPU), so the summation order, and with it every bit of the result, is the same on any device.
struct XattnSplit {
  int SP, ntiles, per_split, nsplit;
};
static XattnSplit xattn_split(int N, int heads, int H, int W, int S) {
  XattnSplit x;
  x.SP = (S + 63) & ~63;
  x.ntiles = (H * W + 63) / 64;
  const int base = (x.SP / 64) * heads * N;                 // CTAs without splitting
  int want = (1024 + base - 1) / base;                      // about 8 CTAs per SM of an H100
  want = want < 1 ? 1 : want > x.ntiles ? x.ntiles : want;
  x.per_split = (x.ntiles + want - 1) / want;
  x.nsplit = (x.ntiles + x.per_split - 1) / x.per_split;
  return x;
}
size_t xattn_part_floats(int N, int C, int heads, int H, int W, int S) {
  const XattnSplit x = xattn_split(N, heads, H, W, S);
  return (size_t)2 * x.nsplit * N * x.SP * C;               // dK | dV, [split][n][head][key][D]
}

// dK, dV partials: one CTA = 64 keys of one (sample, head) (4 warps x 16 keys, K / V rows as A fragments) and the query
// tiles of one split, streamed through shared memory as in mha_bwd_kv_kernel.  Writes every one of its SP key rows (rows
// beyond S read key S - 1 and are never summed).
template <int D>
__global__ void __launch_bounds__(128) xattn_bwd_kv_kernel(const __nv_bfloat16* __restrict__ q, const __nv_bfloat16* __restrict__ k,
                                                           const __nv_bfloat16* __restrict__ v, const __nv_bfloat16* __restrict__ go,
                                                           const float* __restrict__ lse, const float* __restrict__ dsum,
                                                           float* __restrict__ part, int N, int C, int heads, int H, int W, int S,
                                                           int per_split, float scale_log2) {
  constexpr int DP = D / 8, KS = D / 16;
  __shared__ __align__(16) uint4 qs[DP][64];
  __shared__ __align__(16) uint4 dos[DP][64];
  __shared__ float ls[64], dd[64];
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3, SP = (S + 63) & ~63, nsplit = gridDim.y;
  const int k0 = blockIdx.x * 64, split = blockIdx.y, n = blockIdx.z / heads, head = blockIdx.z - n * heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq8 = lane >> 2, tq = lane & 3;
  const long long hoff = ((long long)n * planes + head * DP) * g.PL * 8;
  const __nv_bfloat16* qb = q + hoff;
  const __nv_bfloat16* gob = go + hoff;
  const float* lrow = lse + ((long long)n * heads + head) * seq;
  const float* drow = dsum + ((long long)n * heads + head) * seq;
  const int r0 = min(k0 + warp * 16 + gq8, S - 1), r1 = min(k0 + warp * 16 + gq8 + 8, S - 1);
  const __nv_bfloat16* kr0 = k + ((long long)n * S + r0) * C + head * D;
  const __nv_bfloat16* kr1 = k + ((long long)n * S + r1) * C + head * D;
  const __nv_bfloat16* vr0 = v + ((long long)n * S + r0) * C + head * D;
  const __nv_bfloat16* vr1 = v + ((long long)n * S + r1) * C + head * D;
  uint32_t ka[KS][4], va[KS][4];
#pragma unroll
  for (int j = 0; j < KS; ++j) {
    ka[j][0] = *reinterpret_cast<const uint32_t*>(kr0 + 16 * j + 2 * tq);
    ka[j][1] = *reinterpret_cast<const uint32_t*>(kr1 + 16 * j + 2 * tq);
    ka[j][2] = *reinterpret_cast<const uint32_t*>(kr0 + 16 * j + 8 + 2 * tq);
    ka[j][3] = *reinterpret_cast<const uint32_t*>(kr1 + 16 * j + 8 + 2 * tq);
    va[j][0] = *reinterpret_cast<const uint32_t*>(vr0 + 16 * j + 2 * tq);
    va[j][1] = *reinterpret_cast<const uint32_t*>(vr1 + 16 * j + 2 * tq);
    va[j][2] = *reinterpret_cast<const uint32_t*>(vr0 + 16 * j + 8 + 2 * tq);
    va[j][3] = *reinterpret_cast<const uint32_t*>(vr1 + 16 * j + 8 + 2 * tq);
  }
  float dk[DP][4], dv[DP][4];
#pragma unroll
  for (int i = 0; i < DP; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) { dk[i][e] = 0.f; dv[i][e] = 0.f; }
  const uint32_t* qs32 = reinterpret_cast<const uint32_t*>(qs);
  const uint32_t* do32 = reinterpret_cast<const uint32_t*>(dos);
  const uint32_t qs_addr = smem_u32(qs), do_addr = smem_u32(dos);
  const int t_end = min((split + 1) * per_split, (seq + 63) / 64);
  for (int tile = split * per_split; tile < t_end; ++tile) {
    const int q0 = tile * 64;
    __syncthreads();
    for (int i = threadIdx.x; i < DP * 64; i += 128) {
      const int pl = i >> 6, qq = i & 63, qi = q0 + qq;
      uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
      if (qi < seq) {
        const long long off = pf8_pixel(g, qi, W);
        a = *reinterpret_cast<const uint4*>(qb + (long long)pl * g.PL * 8 + off);
        b = *reinterpret_cast<const uint4*>(gob + (long long)pl * g.PL * 8 + off);
      }
      qs[pl][qq] = a;
      dos[pl][qq] = b;
    }
    if (threadIdx.x < 64) {   // queries beyond seq: lse = +inf -> P = 0
      const int qi = q0 + threadIdx.x;
      ls[threadIdx.x] = qi < seq ? lrow[qi] : INFINITY;
      dd[threadIdx.x] = qi < seq ? drow[qi] : 0.f;
    }
    __syncthreads();
    float st[8][4], dpt[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
#pragma unroll
      for (int e = 0; e < 4; ++e) { st[t][e] = 0.f; dpt[t][e] = 0.f; }
#pragma unroll
      for (int j = 0; j < KS; ++j) {
        const int w0 = ((2 * j) * 64 + t * 8 + gq8) * 4 + tq, w1 = ((2 * j + 1) * 64 + t * 8 + gq8) * 4 + tq;
        mma_bf16_16x8x16(st[t], ka[j][0], ka[j][1], ka[j][2], ka[j][3], qs32[w0], qs32[w1]);
        mma_bf16_16x8x16(dpt[t], va[j][0], va[j][1], va[j][2], va[j][3], do32[w0], do32[w1]);
      }
    }
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = t * 8 + 2 * tq + (e & 1);
        const float p = exp2f(st[t][e] * scale_log2 - ls[col]);
        st[t][e] = p;
        dpt[t][e] = p * (dpt[t][e] - dd[col]);
      }
#pragma unroll
    for (int k16 = 0; k16 < 4; ++k16) {
      const float* p0 = st[2 * k16];
      const float* p1 = st[2 * k16 + 1];
      const float* s0 = dpt[2 * k16];
      const float* s1 = dpt[2 * k16 + 1];
      const uint32_t pa0 = pack_bf16x2(p0[0], p0[1]), pa1 = pack_bf16x2(p0[2], p0[3]), pa2 = pack_bf16x2(p1[0], p1[1]),
                     pa3 = pack_bf16x2(p1[2], p1[3]);
      const uint32_t sa0 = pack_bf16x2(s0[0], s0[1]), sa1 = pack_bf16x2(s0[2], s0[3]), sa2 = pack_bf16x2(s1[0], s1[1]),
                     sa3 = pack_bf16x2(s1[2], s1[3]);
#pragma unroll
      for (int i = 0; i < DP; ++i) {
        uint32_t b0, b1;
        ldsm_b_trans(b0, b1, do_addr, i, k16, lane);
        mma_bf16_16x8x16(dv[i], pa0, pa1, pa2, pa3, b0, b1);
        ldsm_b_trans(b0, b1, qs_addr, i, k16, lane);
        mma_bf16_16x8x16(dk[i], sa0, sa1, sa2, sa3, b0, b1);
      }
    }
  }
  // accumulator (c0, c1) = (key row gq8, channels 8i + 2tq, +1), (c2, c3) = key row gq8 + 8
  const size_t half = (size_t)nsplit * N * SP * C;
  float* pk = part + (((size_t)split * N + n) * heads + head) * SP * D;
  float* pv = pk + half;
  const int ra = k0 + warp * 16 + gq8, rb = ra + 8;
#pragma unroll
  for (int i = 0; i < DP; ++i) {
    *reinterpret_cast<float2*>(pk + (size_t)ra * D + 8 * i + 2 * tq) = make_float2(dk[i][0], dk[i][1]);
    *reinterpret_cast<float2*>(pk + (size_t)rb * D + 8 * i + 2 * tq) = make_float2(dk[i][2], dk[i][3]);
    *reinterpret_cast<float2*>(pv + (size_t)ra * D + 8 * i + 2 * tq) = make_float2(dv[i][0], dv[i][1]);
    *reinterpret_cast<float2*>(pv + (size_t)rb * D + 8 * i + 2 * tq) = make_float2(dv[i][2], dv[i][3]);
  }
}

// dk[n][s][c] = scale * sum over the splits (in order) of the dK partials; dv the same without the scale
__global__ void __launch_bounds__(256) xattn_kv_reduce_kernel(const float* __restrict__ part, float* __restrict__ dk,
                                                              float* __restrict__ dv, int N, int C, int heads, int S, int SP,
                                                              int nsplit, float scale) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)N * S * C) return;
  const int D = C / heads;
  const int c = (int)(idx % C), s = (int)((idx / C) % S), n = (int)(idx / ((long long)C * S));
  const int head = c / D, d = c - head * D;
  const size_t half = (size_t)nsplit * N * SP * C;
  const size_t stride = (size_t)N * SP * C;   // one split
  const float* pk = part + (((size_t)n * heads + head) * SP + s) * D + d;
  float a = 0.f, b = 0.f;
  for (int j = 0; j < nsplit; ++j) {
    a += pk[j * stride];
    b += pk[half + j * stride];
  }
  dk[idx] = a * scale;
  dv[idx] = b;
}

template <int D>
static cudaError_t xattn_bwd_launch(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v, const __nv_bfloat16* o,
                                    const __nv_bfloat16* go, const float* lse, float* dsum, float* part, __nv_bfloat16* gq,
                                    float* dk, float* dv, int N, int C, int heads, int H, int W, int S, cudaStream_t s) {
  const int seq = H * W;
  const float scale = 1.0f / sqrtf((float)D), sl2 = 1.4426950408889634f * scale;
  const XattnSplit x = xattn_split(N, heads, H, W, S);
  static const cudaError_t attr = cudaFuncSetAttribute(xattn_bwd_dq_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       2 * (D / 8) * XATTN_MAX_S * (int)sizeof(uint4));
  if (attr != cudaSuccess) return attr;
  mha_bwd_dot_kernel<D><<<dim3((seq + 255) / 256, heads, N), 256, 0, s>>>(o, go, dsum, N, C, H, W);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const size_t smem = (size_t)2 * (D / 8) * x.SP * sizeof(uint4);
  xattn_bwd_dq_kernel<D><<<dim3((x.ntiles + XATTN_BWD_QT - 1) / XATTN_BWD_QT, heads, N), 128, smem, s>>>(
      q, k, v, go, lse, dsum, gq, N, C, H, W, S, sl2, scale);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  xattn_bwd_kv_kernel<D><<<dim3(x.SP / 64, x.nsplit, N * heads), 128, 0, s>>>(q, k, v, go, lse, dsum, part, N, C, heads, H, W,
                                                                               S, x.per_split, sl2);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  const long long tot = (long long)N * S * C;
  xattn_kv_reduce_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(part, dk, dv, N, C, heads, S, x.SP, x.nsplit, scale);
  return cudaGetLastError();
}
cudaError_t launch_xattn_bwd(const __nv_bfloat16* q, const __nv_bfloat16* k, const __nv_bfloat16* v, const __nv_bfloat16* o,
                             const __nv_bfloat16* go, const float* lse, float* dsum, float* part, __nv_bfloat16* gq, float* dk,
                             float* dv, int N, int C, int heads, int H, int W, int S, cudaStream_t s) {
  if (S < 1 || S > XATTN_MAX_S || C % heads) return cudaErrorInvalidValue;
  const int D = C / heads;
  if (D == 16) return xattn_bwd_launch<16>(q, k, v, o, go, lse, dsum, part, gq, dk, dv, N, C, heads, H, W, S, s);
  if (D == 32) return xattn_bwd_launch<32>(q, k, v, o, go, lse, dsum, part, gq, dk, dv, N, C, heads, H, W, S, s);
  if (D == 64) return xattn_bwd_launch<64>(q, k, v, o, go, lse, dsum, part, gq, dk, dv, N, C, heads, H, W, S, s);
  return cudaErrorInvalidValue;
}

// dW[c][x] += sum_m G[m][c] E[m][x] for the K (blockIdx.z = 0) and V (1) projections: 64 x 64 output tiles, 256 threads
// of 4 x 4 outputs, the token dimension in steps of 16 through shared memory (fixed order: deterministic).
__global__ void __launch_bounds__(256) xattn_kv_wgrad_kernel(const float* __restrict__ dk, const float* __restrict__ dv,
                                                             const float* __restrict__ enc, float* __restrict__ dwk,
                                                             float* __restrict__ dwv, int M, int C, int X) {
  __shared__ float gs[16][64], es[16][64];
  const float* G = blockIdx.z ? dv : dk;
  float* dw = blockIdx.z ? dwv : dwk;
  const int c0 = blockIdx.y * 64, x0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int m0 = 0; m0 < M; m0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      const int r = i >> 6, col = i & 63, m = m0 + r;
      gs[r][col] = (m < M && c0 + col < C) ? G[(long long)m * C + c0 + col] : 0.f;
      es[r][col] = (m < M && x0 + col < X) ? enc[(long long)m * X + x0 + col] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float a[4], b[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { a[u] = gs[r][ty * 4 + u]; b[u] = es[r][tx * 4 + u]; }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int w = 0; w < 4; ++w) acc[u][w] = fmaf(a[u], b[w], acc[u][w]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int c = c0 + ty * 4 + u, x = x0 + tx * 4 + w;
      if (c < C && x < X) dw[(long long)c * X + x] += acc[u][w];
    }
}
cudaError_t launch_xattn_kv_wgrad(const float* dk, const float* dv, const float* enc, float* dwk, float* dwv, int M, int C,
                                  int X, cudaStream_t s) {
  xattn_kv_wgrad_kernel<<<dim3((X + 63) / 64, (C + 63) / 64, 2), 256, 0, s>>>(dk, dv, enc, dwk, dwv, M, C, X);
  return cudaGetLastError();
}

}  // namespace b200ad
