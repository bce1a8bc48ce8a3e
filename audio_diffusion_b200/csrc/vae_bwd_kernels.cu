// Backward kernels of the autoencoder's own layers (AutoencoderKL training, scripts/train_vae.py): the single-head
// attention of the mid blocks on the tensor cores, the encoder tail (quant_conv on the moments) and conv_in's data gradient
// (the decoder head's, through post_quant_conv to the latents; the U-Net's and the encoder's, to their inputs).  Everything
// else of the autoencoder backward reuses the U-Net's kernels.
// Oracle: torch autograd over oracle/vae_oracle.py.
#include "bwd_kernels.cuh"

namespace b200ad {

namespace {
__device__ __forceinline__ float warp_sum_v(float v) {
#pragma unroll
  for (int sh = 16; sh >= 1; sh >>= 1) v += __shfl_xor_sync(0xffffffffu, v, sh);
  return v;
}
}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// Single-head attention backward (one head of dim C over S = H*W tokens).  The forward kept P = softmax(scale Q K^T)
// (fp32 [N][S][S]).  With dO the gradient of the attention output O and dP = dO V^T:
//   D[q] = sum_k P[q][k] dP[q][k]
//   dS   = P o (dP - D) * scale           (bf16 [N][S][S] scratch)
//   dV   = P^T dO,  dQ = dS K,  dK = dS^T Q   -> PF8 gqkv (q | k | v), the layout the q/k/v projections' backward reads.
// D equals sum_c dO[q][c] O[q][c] in exact arithmetic, but formed from the stored bf16 O it does not match the fp32 P and
// dP that dS is made of: over S = 1024 tokens with a near-uniform P, dP - D cancels to a few percent of dP and O's
// rounding alone put 1.5 % into the to_q / to_k weight gradients.  So D is summed from P and dP themselves: a first dP
// GEMM writes each 64-key tile's partial row sums, one pass adds them in a fixed order, and the dS GEMM recomputes dP.
// The five GEMMs run on one kernel: CTA tile 64 x 64, K step 32, four warps of 32 x 32 on mma.sync m16n8k16 (bf16
// operands, fp32 accumulation).  Every operand tile is staged in shared memory as [row][k] with k contiguous, so the A
// and B fragments are plain 32-bit loads; the loaders transpose where the global layout runs the other way.
enum { A1_DV = 0, A1_DS = 1, A1_DQ = 2, A1_DK = 3, A1_DP = 4 };
struct Attn1Bwd {
  const __nv_bfloat16* qkv;   // PF8, 3C channels
  const __nv_bfloat16* go;    // PF8, C channels
  const float* P;
  const float* D;             // [N][S]
  float* Dp;                  // [N][S][S / 64] partial row sums of P o dP, in the dS scratch until the dS GEMM runs
  __nv_bfloat16* dS;
  __nv_bfloat16* gqkv;        // PF8, 3C channels
  int C, H, W, S;
  float scale;
};
constexpr int A1_BK = 32, A1_LD = A1_BK + 8;   // row pitch 80 B: the fragment loads of a warp hit 32 distinct banks

// D[token] = the A1_DP partials of its S / 64 key tiles, added in tile order
__global__ void __launch_bounds__(256) attn1_rowdot_kernel(const float* __restrict__ Dp, float* __restrict__ D, int NS,
                                                           int tiles) {
  const int tok = blockIdx.x * 256 + threadIdx.x;
  if (tok >= NS) return;
  float s = 0.f;
  for (int t = 0; t < tiles; ++t) s += Dp[(long long)tok * tiles + t];
  D[tok] = s;
}

// X[r][0..7 of vector v] <- 8 channels of token `tok` (rows = tokens, k = channels)
__device__ __forceinline__ void a1_rows_pf8(__nv_bfloat16 (*X)[A1_LD], const __nv_bfloat16* img, const Geom& g, int W,
                                            int tok0, int ch0) {
  for (int i = threadIdx.x; i < 64 * (A1_BK / 8); i += 128) {
    const int r = i >> 2, v = i & 3;
    *reinterpret_cast<uint4*>(&X[r][v * 8]) =
        *reinterpret_cast<const uint4*>(img + (long long)((ch0 >> 3) + v) * g.PL * 8 + pf8_pixel(g, tok0 + r, W));
  }
}
// X[channel][token] (rows = 64 channels from ch0, k = 32 tokens from tok0)
__device__ __forceinline__ void a1_cols_pf8(__nv_bfloat16 (*X)[A1_LD], const __nv_bfloat16* img, const Geom& g, int W,
                                            int tok0, int ch0) {
  for (int i = threadIdx.x; i < A1_BK * 8; i += 128) {
    const int t = i & (A1_BK - 1), v = i / A1_BK;
    const uint4 u =
        *reinterpret_cast<const uint4*>(img + (long long)((ch0 >> 3) + v) * g.PL * 8 + pf8_pixel(g, tok0 + t, W));
    const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
    for (int k = 0; k < 8; ++k) X[v * 8 + k][t] = e[k];
  }
}

template <int MODE>
__global__ void __launch_bounds__(128) attn1_gemm_kernel(const Attn1Bwd a, int N) {
  __shared__ __align__(16) __nv_bfloat16 As[64][A1_LD];
  __shared__ __align__(16) __nv_bfloat16 Bs[64][A1_LD];
  const Geom g = make_geom(N, a.H, a.W);
  const int S = a.S, C = a.C, W = a.W, planes = C >> 3;
  const int n = blockIdx.z, m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const __nv_bfloat16* qkv = a.qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* go = a.go + (long long)n * planes * g.PL * 8;
  const float* P = a.P + (long long)n * S * S;
  __nv_bfloat16* dS = a.dS + (long long)n * S * S;
  const int K = MODE == A1_DS || MODE == A1_DP ? C : S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gr = lane >> 2, tq = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  float acc[2][4][4] = {};
  for (int k0 = 0; k0 < K; k0 += A1_BK) {
    if (MODE == A1_DV) {          // A[key][q] = P[q][key];  B[c][q] = dO[q][c]
      for (int i = threadIdx.x; i < A1_BK * 16; i += 128) {
        const int q = i >> 4, j = i & 15;
        const float4 f = *reinterpret_cast<const float4*>(P + (long long)(k0 + q) * S + m0 + 4 * j);
        As[4 * j + 0][q] = __float2bfloat16_rn(f.x);
        As[4 * j + 1][q] = __float2bfloat16_rn(f.y);
        As[4 * j + 2][q] = __float2bfloat16_rn(f.z);
        As[4 * j + 3][q] = __float2bfloat16_rn(f.w);
      }
      a1_cols_pf8(Bs, go, g, W, k0, n0);
    } else if (MODE == A1_DS || MODE == A1_DP) {   // A[q][c] = dO[q][c];  B[key][c] = V[key][c]
      a1_rows_pf8(As, go, g, W, m0, k0);
      a1_rows_pf8(Bs, qkv + (long long)2 * planes * g.PL * 8, g, W, n0, k0);
    } else if (MODE == A1_DQ) {   // A[q][key] = dS[q][key];  B[c][key] = K[key][c]
      for (int i = threadIdx.x; i < 64 * (A1_BK / 8); i += 128) {
        const int r = i >> 2, v = i & 3;
        *reinterpret_cast<uint4*>(&As[r][v * 8]) = *reinterpret_cast<const uint4*>(dS + (long long)(m0 + r) * S + k0 + v * 8);
      }
      a1_cols_pf8(Bs, qkv + (long long)planes * g.PL * 8, g, W, k0, n0);
    } else {                      // A[key][q] = dS[q][key];  B[c][q] = Q[q][c]
      for (int i = threadIdx.x; i < A1_BK * 8; i += 128) {
        const int q = i >> 3, v = i & 7;
        const uint4 u = *reinterpret_cast<const uint4*>(dS + (long long)(k0 + q) * S + m0 + v * 8);
        const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
        for (int k = 0; k < 8; ++k) As[v * 8 + k][q] = e[k];
      }
      a1_cols_pf8(Bs, qkv, g, W, k0, n0);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < A1_BK; kk += 16) {
      uint32_t af[2][4], bf[4][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = wm + i * 16 + gr;
        af[i][0] = *reinterpret_cast<const uint32_t*>(&As[r][kk + 2 * tq]);
        af[i][1] = *reinterpret_cast<const uint32_t*>(&As[r + 8][kk + 2 * tq]);
        af[i][2] = *reinterpret_cast<const uint32_t*>(&As[r][kk + 2 * tq + 8]);
        af[i][3] = *reinterpret_cast<const uint32_t*>(&As[r + 8][kk + 2 * tq + 8]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = wn + j * 8 + gr;
        bf[j][0] = *reinterpret_cast<const uint32_t*>(&Bs[c][kk + 2 * tq]);
        bf[j][1] = *reinterpret_cast<const uint32_t*>(&Bs[c][kk + 2 * tq + 8]);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_bf16_16x8x16(acc[i][j], af[i][0], af[i][1], af[i][2], af[i][3], bf[j][0], bf[j][1]);
    }
    __syncthreads();
  }
  // epilogue: lane holds rows (gr, gr + 8) x columns (2 tq, 2 tq + 1) of every 16 x 8 tile
  if (MODE == A1_DP) {   // sum over this tile's 64 keys of P dP per row: lanes of one row, then the two column warps
    __shared__ float red[2][64];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wm + i * 16 + gr + 8 * h;
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 p = *reinterpret_cast<const float2*>(P + (long long)(m0 + r) * S + n0 + wn + j * 8 + 2 * tq);
          s += p.x * acc[i][j][2 * h] + p.y * acc[i][j][2 * h + 1];
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        if (tq == 0) red[warp & 1][r] = s;
      }
    __syncthreads();
    if (threadIdx.x < 64)
      a.Dp[((long long)n * S + m0 + threadIdx.x) * (S / 64) + blockIdx.x] = red[0][threadIdx.x] + red[1][threadIdx.x];
    return;
  }
  const float* D = a.D + (long long)n * S;
  __nv_bfloat16* gout = a.gqkv + ((long long)n * 3 * planes + (MODE == A1_DV ? 2 * planes : MODE == A1_DK ? planes : 0)) *
                                     g.PL * 8;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = m0 + wm + i * 16 + gr + 8 * h, c = n0 + wn + j * 8 + 2 * tq;
        float v0 = acc[i][j][2 * h], v1 = acc[i][j][2 * h + 1];
        if (MODE == A1_DS) {
          const float2 p = *reinterpret_cast<const float2*>(P + (long long)r * S + c);
          const float d = D[r];
          v0 = p.x * (v0 - d) * a.scale;
          v1 = p.y * (v1 - d) * a.scale;
          *reinterpret_cast<uint32_t*>(dS + (long long)r * S + c) = pack_bf16x2(v0, v1);
        } else {
          *reinterpret_cast<uint32_t*>(gout + (long long)(c >> 3) * g.PL * 8 + pf8_pixel(g, r, W) + (c & 7)) =
              pack_bf16x2(v0, v1);
        }
      }
}

cudaError_t launch_attention_1head_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* go, const float* P, float* D,
                                       __nv_bfloat16* dS, __nv_bfloat16* gqkv, int N, int C, int H, int W, cudaStream_t s) {
  const int S = H * W;
  if (S % 64 || C % 64) return cudaErrorInvalidValue;
  Attn1Bwd a{qkv, go, P, D, reinterpret_cast<float*>(dS), dS, gqkv, C, H, W, S, rsqrtf((float)C)};
  attn1_gemm_kernel<A1_DP><<<dim3(S / 64, S / 64, N), 128, 0, s>>>(a, N);   // partial row sums of P o dP
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  attn1_rowdot_kernel<<<(N * S + 255) / 256, 256, 0, s>>>(a.Dp, D, N * S, S / 64);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  attn1_gemm_kernel<A1_DS><<<dim3(S / 64, S / 64, N), 128, 0, s>>>(a, N);   // dS first: dQ and dK read it
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  attn1_gemm_kernel<A1_DV><<<dim3(C / 64, S / 64, N), 128, 0, s>>>(a, N);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  attn1_gemm_kernel<A1_DQ><<<dim3(C / 64, S / 64, N), 128, 0, s>>>(a, N);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  attn1_gemm_kernel<A1_DK><<<dim3(C / 64, S / 64, N), 128, 0, s>>>(a, N);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Encoder tail: moments = quant_conv(h) (1x1, 2L -> 2L) on the first 2L channels of the conv_out output h (PF8, 128
// channels).  From g_moments (fp32 [N][2L][H][W]):  g_h = Wq^T g_m, written twice (fp32, [N][2L][HW] for the data gradient
// of conv_out and [2L][N][HW] for its per-channel weight gradient);  dWq += g_m h^T, dbq += sum g_m.  One thread per pixel.
__global__ void __launch_bounds__(256) quant_conv_bwd_kernel(const float* __restrict__ gm, const __nv_bfloat16* __restrict__ h,
                                                             const float* __restrict__ wq, float* __restrict__ gh_nc,
                                                             float* __restrict__ gh_cn, float* __restrict__ dwq,
                                                             float* __restrict__ dbq, int N, int L2, int H, int W) {
  const Geom g = make_geom(N, H, W);
  const int HW = H * W, n = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
  const bool ok = p < HW;
  float hv[8] = {}, gv[8] = {};
  if (ok) {
    const uint4 u = *reinterpret_cast<const uint4*>(h + (long long)n * 16 * g.PL * 8 + pf8_pixel(g, p, W));
    const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float2 f = unpack_bf16x2(uu[e]); hv[2 * e] = f.x; hv[2 * e + 1] = f.y; }
    for (int o = 0; o < L2; ++o) gv[o] = gm[((long long)n * L2 + o) * HW + p];
    for (int i = 0; i < L2; ++i) {
      float s = 0.f;
      for (int o = 0; o < L2; ++o) s = fmaf(wq[o * L2 + i], gv[o], s);
      gh_nc[((long long)n * L2 + i) * HW + p] = s;
      gh_cn[((long long)i * N + n) * HW + p] = s;
    }
  }
  if (!dwq) return;   // no parameter gradients (uniform over the CTA)
  for (int o = 0; o < L2; ++o) {
    float b = warp_sum_v(gv[o]);
    if ((threadIdx.x & 31) == 0) atomicAdd(dbq + o, b);
    for (int i = 0; i < L2; ++i) {
      const float w = warp_sum_v(gv[o] * hv[i]);
      if ((threadIdx.x & 31) == 0) atomicAdd(dwq + o * L2 + i, w);
    }
  }
}
cudaError_t launch_quant_conv_bwd(const float* gm, const __nv_bfloat16* h, const float* wq, float* gh_nc, float* gh_cn,
                                  float* dwq, float* dbq, int N, int L2, int H, int W, cudaStream_t s) {
  if (L2 > 8) return cudaErrorInvalidValue;
  quant_conv_bwd_kernel<<<dim3((H * W + 255) / 256, N), 256, 0, s>>>(gm, h, wq, gh_nc, gh_cn, dwq, dbq, N, L2, H, W);
  return cudaGetLastError();
}

// conv_in's data gradient down to its one input channel (the U-Net's sample, the encoder's image, the decoder's
// post_quant_conv(z)).  From g_y (PF8, C channels, the gradient of conv_in's output):
//   g[n][p] = sum_c sum_t Win[c][t] g_y[n][c][p - shift(t)]
// One thread per pixel: the 32 threads of a warp read 32 neighbouring pixels of one 8-channel plane per tap, so g_y is
// read from DRAM once and the taps' re-reads hit L1; the weights sit in shared memory as [plane][tap][8].  The sum is
// fixed-order fp32: plane pl goes into partial pl % 32 (its planes, taps and channels in order), and the 32 partials
// are added pairwise at distances 16, 8, 4, 2, 1 (as a binary tree: partial i + partial i + 16 first).  That is the order of the earlier one-warp-per-pixel decoder kernel
// (lanes over planes, then an xor-shuffle sum), so the decoder's g_z is bitwise what it was.
// wpq null: gx = g (fp32 [N][H][W], overwritten, no atomics).  Otherwise the decoder head, zq = post_quant_conv(z) (1x1,
// 1 -> 1): gx = Wpq g, and with dwpq given, dWpq += sum g z, dbpq += sum g.
constexpr int CIN_DG_THREADS = 256;
__global__ void __launch_bounds__(CIN_DG_THREADS) conv_in_dgrad_kernel(const __nv_bfloat16* __restrict__ gy,
                                                                       const float* __restrict__ win,
                                                                       const float* __restrict__ wpq,
                                                                       const float* __restrict__ z, float* __restrict__ gx,
                                                                       float* __restrict__ dwpq, float* __restrict__ dbpq,
                                                                       int N, int C, int H, int W) {
  extern __shared__ float4 sw4[];   // [C/8][9][8] floats
  float* sw = reinterpret_cast<float*>(sw4);
  for (int i = threadIdx.x; i < C * 9; i += blockDim.x) {
    const int c = i / 9, t = i - c * 9;
    sw[((c >> 3) * 9 + t) * 8 + (c & 7)] = win[i];
  }
  __syncthreads();
  const Geom g = make_geom(N, H, W);
  const int HW = H * W, np = C / 8;
  const int tok = blockIdx.x * CIN_DG_THREADS + threadIdx.x;
  if (tok >= N * HW) return;
  const int n = tok / HW, p = tok - n * HW, y = p / W, x = p - y * W;
  const __nv_bfloat16* img = gy + (long long)n * np * g.PL * 8;
  // the partials in bit-reversed order j(k), so that each pairwise sum is made as soon as both halves exist: after leaf
  // k, the subtrees of levels 0 .. (trailing ones of k) are complete; stk[l] holds the pending left half of level l
  float stk[5], gs = 0.f;
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const int j = ((k & 1) << 4) | ((k & 2) << 2) | (k & 4) | ((k & 8) >> 2) | ((k & 16) >> 4);
    float acc = 0.f;
    for (int pl = j; pl < np; pl += 32) {
      const __nv_bfloat16* plane = img + (long long)pl * g.PL * 8;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int yy = y - (t / 3 - 1), xx = x - (t % 3 - 1);
        if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(plane + (long long)(g.lead + yy * g.Wp + xx) * 8));
        const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
        const float4 w0 = sw4[(pl * 9 + t) * 2], w1 = sw4[(pl * 9 + t) * 2 + 1];
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = unpack_bf16x2(uu[e]);
          acc = fmaf(wv[2 * e], f.x, acc);
          acc = fmaf(wv[2 * e + 1], f.y, acc);
        }
      }
    }
    bool open = true;
#pragma unroll
    for (int l = 0; l < 5; ++l)
      if (open) {
        if (k & (1 << l)) acc = stk[l] + acc;
        else { stk[l] = acc; open = false; }
      }
    if (open) gs = acc;   // k = 31: the whole tree
  }
  const long long at = (long long)n * HW + p;
  if (!wpq) {
    gx[at] = gs;
    return;
  }
  gx[at] = fmaf(wpq[0], gs, 0.f);
  if (dwpq) {
    atomicAdd(dbpq, gs);
    atomicAdd(dwpq, gs * z[at]);
  }
}
cudaError_t launch_conv_in_dgrad(const __nv_bfloat16* gy, const float* win, float* gx, int N, int C, int H, int W,
                                 cudaStream_t s, const float* wpq, const float* z, float* dwpq, float* dbpq) {
  if (C % 8 || C > 1024) return cudaErrorInvalidValue;
  conv_in_dgrad_kernel<<<(N * H * W + CIN_DG_THREADS - 1) / CIN_DG_THREADS, CIN_DG_THREADS, (size_t)C * 9 * sizeof(float), s>>>(
      gy, win, wpq, z, gx, dwpq, dbpq, N, C, H, W);
  return cudaGetLastError();
}

}  // namespace b200ad
