// Memory-bound pieces of the U-Net backward pass (scripts/train_unet.py:259 `accelerator.backward(loss)`): GroupNorm(+SiLU)
// backward, per-channel gradient sums (bias / time-embedding gradients), head_dim-8 attention backward, the cin = 1 /
// cout = 1 convolution weight gradients, the timestep-MLP linears, and small helpers. Gradients of activations are PF8
// bf16 (what autocast gives the reference); parameter gradients are accumulated in fp32.
// Oracle: torch autograd over oracle/unet_oracle.py (oracle/train_oracle.py::loss_and_grads).
#include "bwd_kernels.cuh"

namespace b200ad {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int sh = 16; sh >= 1; sh >>= 1) v += __shfl_xor_sync(0xffffffffu, v, sh);
  return v;
}
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) { const float2 t = unpack_bf16x2(u[e]); f[2 * e] = t.x; f[2 * e + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

// ---------------------------------------------------------------------------------------------------------------------
// GroupNorm (+SiLU) backward over the channel concatenation of up to two raw sources.
//   y = gamma * xhat + beta, a = silu(y) (or y);  gy = ga * silu'(y)
//   S1[n][c] = sum_pix gy, S2[n][c] = sum_pix gy * xhat;  dbeta = sum_n S1, dgamma = sum_n S2
//   gx = rstd * (gamma * gy - (A + xhat * B) / M),  A = sum_{c in group} gamma_c S1_c, B = sum gamma_c S2_c, M = cpg*H*W
constexpr int GB_THREADS = 256;
constexpr int GB_PIX = 4096;     // pixels per CTA of the scalar-conv weight gradient
constexpr int GB_CHUNK = 8192;   // flat PF8 positions per CTA of the GroupNorm passes (32 vectors per thread, 4 in flight)

// Both passes walk the FLAT position range [0, H * Wp) of one 8-channel plane (coalesced 16-byte vectors, no div / mod per
// pixel).  The pad column of every row is zero in the raw tensors AND in the incoming gradient (buffers are zeroed at bind
// time and every writer, conv_tc_kernel included, leaves the layout's guards zero), so it contributes nothing to the sums; the apply pass writes zeros there.
// A CTA only needs the statistics of the (at most two) groups its plane touches: eight threads derive them.
struct PlaneCoef {
  float mean[8], rstd[8], gam[8], bet[8];
};
__device__ __forceinline__ void plane_coef(const GnBwdParams& p, int n, int pl, float (*sm)[8], PlaneCoef& k) {
  const int Ct = p.C[0] + p.C[1];
  const int cpg = Ct / p.groups;
  if (threadIdx.x < 8) {
    const int c = pl * 8 + threadIdx.x, gi = c / cpg;
    double s = 0., q = 0.;
    for (int cc = gi * cpg; cc < (gi + 1) * cpg; cc += 4) {
      const stat_t* st = (cc < p.C[0]) ? p.stats[0] + ((long long)n * (p.C[0] >> 2) + (cc >> 2)) * 2
                                      : p.stats[1] + ((long long)n * (p.C[1] >> 2) + ((cc - p.C[0]) >> 2)) * 2;
      s += st[0];
      q += st[1];
    }
    const double cnt = (double)cpg * (double)p.H * (double)p.W;
    const double mean = s / cnt;
    sm[0][threadIdx.x] = (float)mean;
    sm[1][threadIdx.x] = (float)(1.0 / sqrt(fmax(q / cnt - mean * mean, 0.) + (double)p.eps));
    sm[2][threadIdx.x] = p.gamma[c];
    sm[3][threadIdx.x] = p.beta[c];
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < 8; ++e) { k.mean[e] = sm[0][e]; k.rstd[e] = sm[1][e]; k.gam[e] = sm[2][e]; k.bet[e] = sm[3][e]; }
}

// silu'(y) = s (1 + y (1 - s)), s = sigmoid(y) = 0.5 + 0.5 tanh(y / 2): one MUFU per element
__device__ __forceinline__ float silu_grad(float y) {
  const float sig = fmaf(0.5f, tanh_approx(0.5f * y), 0.5f);
  return sig * fmaf(y, 1.0f - sig, 1.0f);
}

// pass 1: grid (position chunks, planes, N). Thread-local sums over the CTA's positions of one 8-channel plane.
__global__ void __launch_bounds__(GB_THREADS, 2) gn_bwd_reduce_kernel(const GnBwdParams p) {
  __shared__ float coef[4][8];
  __shared__ float red[GB_THREADS / 32][16];
  const int Ct = p.C[0] + p.C[1];
  const int n = blockIdx.z, pl = blockIdx.y;
  const Geom g = make_geom(p.N, p.H, p.W);
  PlaneCoef k;
  plane_coef(p, n, pl, coef, k);
  const int planes0 = p.C[0] >> 3;
  const __nv_bfloat16* xs = (pl < planes0) ? p.src[0] + ((long long)n * planes0 + pl) * g.PL * 8
                                          : p.src[1] + ((long long)n * (p.C[1] >> 3) + (pl - planes0)) * g.PL * 8;
  const __nv_bfloat16* gs = p.ga + ((long long)n * (Ct >> 3) + pl) * g.PL * 8;
  const uint4* xv4 = reinterpret_cast<const uint4*>(xs) + g.lead;
  const uint4* gv4 = reinterpret_cast<const uint4*>(gs) + g.lead;
  float s1[8] = {0, 0, 0, 0, 0, 0, 0, 0}, s2[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int mend = min(p.H * g.Wp, (int)(blockIdx.x + 1) * GB_CHUNK);
  for (int m0 = blockIdx.x * GB_CHUNK + threadIdx.x; m0 < mend; m0 += 4 * GB_THREADS) {
    uint4 xr[4], gr[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + u * GB_THREADS;
      if (m < mend) { xr[u] = xv4[m]; gr[u] = gv4[m]; }
      else { xr[u] = make_uint4(0, 0, 0, 0); gr[u] = make_uint4(0, 0, 0, 0); }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float xv[8], gv[8];
      unpack8(xr[u], xv);
      unpack8(gr[u], gv);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float xh = (xv[e] - k.mean[e]) * k.rstd[e];
        float gy = gv[e];
        if (p.silu) gy *= silu_grad(fmaf(k.gam[e], xh, k.bet[e]));
        s1[e] += gy;
        s2[e] = fmaf(gy, xh, s2[e]);
      }
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float a = warp_sum_f(s1[e]), b = warp_sum_f(s2[e]);
    if (lane == 0) { red[warp][e] = a; red[warp][8 + e] = b; }
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    float t = 0.f;
    for (int w = 0; w < GB_THREADS / 32; ++w) t += red[w][threadIdx.x];
    const int e = threadIdx.x & 7, which = threadIdx.x >> 3;
    atomicAdd(p.sums + ((long long)n * Ct + pl * 8 + e) * 2 + which, t);
    if (p.dgamma) atomicAdd((which ? p.dgamma : p.dbeta) + pl * 8 + e, t);   // dbeta = sum S1, dgamma = sum S2 over n
  }
}

// pass 2: grid (position chunks, planes, N): gx (+ optional addends) of one plane
__global__ void __launch_bounds__(GB_THREADS, 2) gn_bwd_apply_kernel(const GnBwdParams p) {
  __shared__ float coef[4][8];
  __shared__ float gAB[2][8];
  __shared__ float cred[GB_THREADS / 32][8];
  const int Ct = p.C[0] + p.C[1];
  const int n = blockIdx.z, pl = blockIdx.y;
  const int cpg = Ct / p.groups;
  const Geom g = make_geom(p.N, p.H, p.W);
  if (threadIdx.x >= 32 && threadIdx.x < 40) {   // (A, B) / M of this channel's group (a second warp, next to plane_coef's)
    const int e = threadIdx.x - 32, c = pl * 8 + e, gi = c / cpg;
    float a = 0.f, b = 0.f;
    for (int cc = gi * cpg; cc < (gi + 1) * cpg; ++cc) {
      const float gm = p.gamma[cc];
      a = fmaf(gm, p.sums[((long long)n * Ct + cc) * 2], a);
      b = fmaf(gm, p.sums[((long long)n * Ct + cc) * 2 + 1], b);
    }
    const float invM = 1.0f / ((float)cpg * (float)p.H * (float)p.W);
    gAB[0][e] = a * invM;
    gAB[1][e] = b * invM;
  }
  PlaneCoef k;
  plane_coef(p, n, pl, coef, k);
  float gA[8], gB[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { gA[e] = gAB[0][e]; gB[e] = gAB[1][e]; }
  const int planes0 = p.C[0] >> 3;
  const bool first = pl < planes0;
  const int lp = first ? pl : pl - planes0;                 // plane inside its own source / destination
  const int lplanes = first ? planes0 : (p.C[1] >> 3);
  const uint4* xv4 = reinterpret_cast<const uint4*>((first ? p.src[0] : p.src[1]) + ((long long)n * lplanes + lp) * g.PL * 8) + g.lead;
  const uint4* gv4 = reinterpret_cast<const uint4*>(p.ga + ((long long)n * (Ct >> 3) + pl) * g.PL * 8) + g.lead;
  const uint4* as4 = p.addS ? reinterpret_cast<const uint4*>(p.addS + ((long long)n * (Ct >> 3) + pl) * g.PL * 8) + g.lead : nullptr;
  const uint4* a04 = (p.add0 && first) ? reinterpret_cast<const uint4*>(p.add0 + ((long long)n * planes0 + pl) * g.PL * 8) + g.lead : nullptr;
  uint4* dv4 = reinterpret_cast<uint4*>((first ? p.dst[0] : p.dst[1]) + ((long long)n * lplanes + lp) * g.PL * 8) + g.lead;
  const int mend = min(p.H * g.Wp, (int)(blockIdx.x + 1) * GB_CHUNK);
  int m0 = blockIdx.x * GB_CHUNK + threadIdx.x;
  int col = m0 % g.Wp;
  const int dcol = GB_THREADS % g.Wp;
  const bool want_cs = p.csum0 && first;
  float cs[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (; m0 < mend; m0 += 4 * GB_THREADS) {
    uint4 xr[4], gr[4], ar[4], br[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + u * GB_THREADS;
      const bool in = m < mend;
      xr[u] = in ? xv4[m] : make_uint4(0, 0, 0, 0);
      gr[u] = in ? gv4[m] : make_uint4(0, 0, 0, 0);
      ar[u] = (in && as4) ? as4[m] : make_uint4(0, 0, 0, 0);
      br[u] = (in && a04) ? a04[m] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + u * GB_THREADS;
      const bool pad = col == p.W;
      col += dcol;
      if (col >= g.Wp) col -= g.Wp;
      if (m >= mend) continue;
      float xv[8], gv[8], av[8], bv[8], o[8];
      unpack8(xr[u], xv);
      unpack8(gr[u], gv);
      unpack8(ar[u], av);
      unpack8(br[u], bv);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float xh = (xv[e] - k.mean[e]) * k.rstd[e];
        float gy = gv[e];
        if (p.silu) gy *= silu_grad(fmaf(k.gam[e], xh, k.bet[e]));
        o[e] = k.rstd[e] * (k.gam[e] * gy - (gA[e] + xh * gB[e])) + av[e] + bv[e];
      }
      dv4[m] = pad ? make_uint4(0, 0, 0, 0) : pack8(o);
      if (want_cs && !pad) {
#pragma unroll
        for (int e = 0; e < 8; ++e) cs[e] += o[e];
      }
    }
  }
  if (want_cs) {   // per-sample channel sums of the gradient just written (uniform per CTA: `first` depends on blockIdx.y)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float a = warp_sum_f(cs[e]);
      if (lane == 0) cred[warp][e] = a;
    }
    __syncthreads();
    if (threadIdx.x < 8) {
      float t = 0.f;
      for (int w = 0; w < GB_THREADS / 32; ++w) t += cred[w][threadIdx.x];
      atomicAdd(p.csum0 + (long long)n * p.C[0] + pl * 8 + threadIdx.x, t);
    }
  }
}

cudaError_t launch_gn_bwd(const GnBwdParams& p, cudaStream_t s) {
  const int Ct = p.C[0] + p.C[1];
  if (p.groups > 64 || (Ct % p.groups)) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(p.sums, 0, (size_t)p.N * Ct * 2 * sizeof(float), s);
  if (e != cudaSuccess) return e;
  const int npos = p.H * (p.W + 1);
  const dim3 grid((npos + GB_CHUNK - 1) / GB_CHUNK, Ct >> 3, p.N);
  gn_bwd_reduce_kernel<<<grid, GB_THREADS, 0, s>>>(p);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  gn_bwd_apply_kernel<<<grid, GB_THREADS, 0, s>>>(p);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// out[n][c] = sum over pixels of src[n][c][.] (PF8 bf16 -> fp32).  `out` must be zeroed by the caller (launcher does).
__global__ void __launch_bounds__(GB_THREADS) chan_sum_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ out,
                                                              int N, int C, int img_planes, int H, int W,
                                                              float* __restrict__ bias0, float* __restrict__ bias1) {
  __shared__ float red[GB_THREADS / 32][8];
  const int n = blockIdx.z, pl = blockIdx.y;
  const Geom g = make_geom(N, H, W);
  // flat positions of the plane: the pad column of every row holds zeros and adds nothing
  const uint4* sv4 = reinterpret_cast<const uint4*>(src + ((long long)n * img_planes + pl) * g.PL * 8) + g.lead;
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const int mend = min(H * g.Wp, (int)(blockIdx.x + 1) * GB_CHUNK);
  for (int m0 = blockIdx.x * GB_CHUNK + threadIdx.x; m0 < mend; m0 += 4 * GB_THREADS) {
    uint4 r[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + u * GB_THREADS;
      r[u] = (m < mend) ? sv4[m] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      float v[8];
      unpack8(r[u], v);
#pragma unroll
      for (int e = 0; e < 8; ++e) s[e] += v[e];
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float a = warp_sum_f(s[e]);
    if (lane == 0) red[warp][e] = a;
  }
  __syncthreads();
  if (threadIdx.x < 8) {
    float t = 0.f;
    for (int k = 0; k < GB_THREADS / 32; ++k) t += red[k][threadIdx.x];
    atomicAdd(out + (long long)n * C + pl * 8 + threadIdx.x, t);
    if (bias0) atomicAdd(bias0 + pl * 8 + threadIdx.x, t);     // bias gradient = sum over samples and pixels
    if (bias1) atomicAdd(bias1 + pl * 8 + threadIdx.x, t);
  }
}
cudaError_t launch_chan_sum(const __nv_bfloat16* src, float* out, int N, int C, int img_planes, int H, int W, cudaStream_t s,
                            float* bias0, float* bias1) {
  cudaError_t e = cudaMemsetAsync(out, 0, (size_t)N * C * sizeof(float), s);
  if (e != cudaSuccess) return e;
  chan_sum_kernel<<<dim3((H * (W + 1) + GB_CHUNK - 1) / GB_CHUNK, C >> 3, N), GB_THREADS, 0, s>>>(src, out, N, C, img_planes, H, W,
                                                                                          bias0, bias1);
  return cudaGetLastError();
}

// dst[c] += sum_n src[n][c]   (bias gradients);  dst2 (optional) receives the same sum
__global__ void reduce_n_add_kernel(const float* __restrict__ src, float* __restrict__ dst, float* __restrict__ dst2, int N,
                                    int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f;
  for (int n = 0; n < N; ++n) a += src[(long long)n * C + c];
  dst[c] += a;
  if (dst2) dst2[c] += a;
}
cudaError_t launch_reduce_n_add(const float* src, float* dst, float* dst2, int N, int C, cudaStream_t s) {
  reduce_n_add_kernel<<<(C + 127) / 128, 128, 0, s>>>(src, dst, dst2, N, C);
  return cudaGetLastError();
}

// copy rows: dst[n][doff + c] = src[n][c]  (time-embedding gradient rows of one resnet into g_proj[N][rows])
__global__ void scatter_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int C, int dstride, int doff) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i - n * C;
  dst[(long long)n * dstride + doff + c] = src[i];
}
cudaError_t launch_scatter_rows(const float* src, float* dst, int N, int C, int dstride, int doff, cudaStream_t s) {
  scatter_rows_kernel<<<(N * C + 255) / 256, 256, 0, s>>>(src, dst, N, C, dstride, doff);
  return cudaGetLastError();
}

// dst += src over whole PF8 buffers (pads are zero on both sides)
__global__ void pf8_add_kernel(__nv_bfloat16* __restrict__ dst, const __nv_bfloat16* __restrict__ src, long long nvec) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nvec) return;
  float a[8], b[8];
  unpack8(reinterpret_cast<const uint4*>(dst)[i], a);
  unpack8(reinterpret_cast<const uint4*>(src)[i], b);
#pragma unroll
  for (int e = 0; e < 8; ++e) a[e] += b[e];
  reinterpret_cast<uint4*>(dst)[i] = pack8(a);
}
cudaError_t launch_pf8_add(__nv_bfloat16* dst, const __nv_bfloat16* src, int N, int C, int H, int W, cudaStream_t s) {
  const Geom g = make_geom(N, H, W);
  const long long nvec = (long long)N * (C >> 3) * g.PL;
  pf8_add_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, s>>>(dst, src, nvec);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Attention backward, heads of dim 8 (one plane each).  grid (heads, N).  qkv: PF8 3C; go: gradient of the attention output
// (PF8 C); gqkv: PF8 3C.  Phase 1 (thread per query): row max / sum, D_i = sum_j P_ij dP_ij, dQ_i.  Phase 2 (thread per
// key): dK_j, dV_j with P recomputed from the saved row statistics.
__global__ void __launch_bounds__(256) attention_bwd_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                            const __nv_bfloat16* __restrict__ go,
                                                            __nv_bfloat16* __restrict__ gqkv, int N, int C, int H, int W) {
  extern __shared__ float ab[];
  const int seq = H * W;
  float* qs = ab;                  // [seq][8]
  float* ks = qs + seq * 8;
  float* vs = ks + seq * 8;
  float* ds = vs + seq * 8;        // dO
  float* rm = ds + seq * 8;        // row max
  float* rl = rm + seq;            // 1 / row sum
  float* rd = rl + seq;            // D_i
  const Geom g = make_geom(N, H, W);
  const int head = blockIdx.x, n = blockIdx.y, planes = C >> 3;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* gop = go + ((long long)n * planes + head) * g.PL * 8;
  for (int p = threadIdx.x; p < seq; p += blockDim.x) {
    const long long pix = (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
    float t[8];
    unpack8(*reinterpret_cast<const uint4*>(base + (long long)head * g.PL * 8 + pix), t);
#pragma unroll
    for (int e = 0; e < 8; ++e) qs[p * 8 + e] = t[e];
    unpack8(*reinterpret_cast<const uint4*>(base + (long long)(planes + head) * g.PL * 8 + pix), t);
#pragma unroll
    for (int e = 0; e < 8; ++e) ks[p * 8 + e] = t[e];
    unpack8(*reinterpret_cast<const uint4*>(base + (long long)(2 * planes + head) * g.PL * 8 + pix), t);
#pragma unroll
    for (int e = 0; e < 8; ++e) vs[p * 8 + e] = t[e];
    unpack8(*reinterpret_cast<const uint4*>(gop + pix), t);
#pragma unroll
    for (int e = 0; e < 8; ++e) ds[p * 8 + e] = t[e];
  }
  __syncthreads();
  const float sc = 0.35355339059327373f;  // 8^-0.5
  __nv_bfloat16* gbase = gqkv + (long long)n * 3 * planes * g.PL * 8;
  for (int i = threadIdx.x; i < seq; i += blockDim.x) {
    float q[8], dO[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { q[e] = qs[i * 8 + e] * sc; dO[e] = ds[i * 8 + e]; }
    float mx = -INFINITY;
    for (int j = 0; j < seq; ++j) {
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(q[e], ks[j * 8 + e], s);
      mx = fmaxf(mx, s);
    }
    float l = 0.f, dsum = 0.f;
    for (int j = 0; j < seq; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { s = fmaf(q[e], ks[j * 8 + e], s); dp = fmaf(dO[e], vs[j * 8 + e], dp); }
      const float ex = __expf(s - mx);
      l += ex;
      dsum = fmaf(ex, dp, dsum);
    }
    const float il = 1.0f / l, D = dsum * il;
    float dq[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < seq; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { s = fmaf(q[e], ks[j * 8 + e], s); dp = fmaf(dO[e], vs[j * 8 + e], dp); }
      const float dS = __expf(s - mx) * il * (dp - D);
#pragma unroll
      for (int e = 0; e < 8; ++e) dq[e] = fmaf(dS, ks[j * 8 + e], dq[e]);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) dq[e] *= sc;
    rm[i] = mx; rl[i] = il; rd[i] = D;
    const long long pix = (long long)(g.lead + (i / W) * g.Wp + (i % W)) * 8;
    *reinterpret_cast<uint4*>(gbase + (long long)head * g.PL * 8 + pix) = pack8(dq);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < seq; j += blockDim.x) {
    float k[8], v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { k[e] = ks[j * 8 + e]; v[e] = vs[j * 8 + e]; }
    float dk[8] = {0, 0, 0, 0, 0, 0, 0, 0}, dv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < seq; ++i) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { s = fmaf(qs[i * 8 + e], k[e], s); dp = fmaf(ds[i * 8 + e], v[e], dp); }
      const float P = __expf(s * sc - rm[i]) * rl[i];
      const float dS = P * (dp - rd[i]) * sc;
#pragma unroll
      for (int e = 0; e < 8; ++e) { dv[e] = fmaf(P, ds[i * 8 + e], dv[e]); dk[e] = fmaf(dS, qs[i * 8 + e], dk[e]); }
    }
    const long long pix = (long long)(g.lead + (j / W) * g.Wp + (j % W)) * 8;
    *reinterpret_cast<uint4*>(gbase + (long long)(planes + head) * g.PL * 8 + pix) = pack8(dk);
    *reinterpret_cast<uint4*>(gbase + (long long)(2 * planes + head) * g.PL * 8 + pix) = pack8(dv);
  }
}
cudaError_t launch_attention_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* go, __nv_bfloat16* gqkv, int N, int C, int H,
                                 int W, cudaStream_t s) {
  const int seq = H * W;
  const size_t smem = (size_t)seq * 35 * sizeof(float);
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  static size_t smem_set = 48 * 1024;
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    smem_set = smem;
  }
  const int threads = seq >= 256 ? 256 : ((seq + 31) / 32) * 32;
  attention_bwd_kernel<<<dim3(C >> 3, N), threads, smem, s>>>(qkv, go, gqkv, N, C, H, W);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient of a conv with ONE scalar-side channel:  dW[c][tap] += sum_{n,p} G[n][c][p] * X[n][p + shift(tap)]
// G: PF8 bf16 (C channels), X: fp32 [N][H][W] (zero outside the image).  flip: write tap 8 - t (the cout = 1 conv_out, whose
// weight gradient is sum_p a[c][p + shift] * g_eps[p]).  grid (pixel chunks, planes, N).
__global__ void __launch_bounds__(GB_THREADS) scalar_conv_wgrad_kernel(const __nv_bfloat16* __restrict__ G,
                                                                       const float* __restrict__ X, float* __restrict__ dW,
                                                                       int N, int C, int H, int W, int flip) {
  __shared__ float red[GB_THREADS / 32][72];
  const int n = blockIdx.z, pl = blockIdx.y;
  const Geom g = make_geom(N, H, W);
  const __nv_bfloat16* gp = G + ((long long)n * (C >> 3) + pl) * g.PL * 8;
  const float* xi = X + (long long)n * H * W;
  float acc[8][9];
#pragma unroll
  for (int e = 0; e < 8; ++e)
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[e][t] = 0.f;
  const int hw = H * W;
  const int pend = min(hw, (int)(blockIdx.x + 1) * GB_PIX);
  for (int pidx = blockIdx.x * GB_PIX + threadIdx.x; pidx < pend; pidx += GB_THREADS) {
    const int h = pidx / W, w = pidx - h * W;
    float gv[8], xv[9];
    unpack8(*reinterpret_cast<const uint4*>(gp + (long long)(g.lead + h * g.Wp + w) * 8), gv);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hh = h + t / 3 - 1, ww = w + t % 3 - 1;
      xv[t] = (hh >= 0 && hh < H && ww >= 0 && ww < W) ? __ldg(xi + hh * W + ww) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e)
#pragma unroll
      for (int t = 0; t < 9; ++t) acc[e][t] = fmaf(gv[e], xv[t], acc[e][t]);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int e = 0; e < 8; ++e)
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float a = warp_sum_f(acc[e][t]);
      if (lane == 0) red[warp][e * 9 + t] = a;
    }
  __syncthreads();
  if (threadIdx.x < 72) {
    float s = 0.f;
    for (int k = 0; k < GB_THREADS / 32; ++k) s += red[k][threadIdx.x];
    const int e = threadIdx.x / 9, t = threadIdx.x - e * 9;
    atomicAdd(dW + (long long)(pl * 8 + e) * 9 + (flip ? 8 - t : t), s);
  }
}
cudaError_t launch_scalar_conv_wgrad(const __nv_bfloat16* G, const float* X, float* dW, int N, int C, int H, int W, int flip,
                                     cudaStream_t s) {
  scalar_conv_wgrad_kernel<<<dim3((H * W + GB_PIX - 1) / GB_PIX, C >> 3, N), GB_THREADS, 0, s>>>(G, X, dW, N, C, H, W, flip);
  return cudaGetLastError();
}

// conv_out's data gradient is a cin = O convolution of its output gradient with the transposed, mirrored weights:
// w'[c][o][t] = w[o][c][8 - t]
__global__ void flip_taps_kernel(const float* __restrict__ w, float* __restrict__ wf, int C, int O) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C * O * 9) return;
  const int co = i / 9, t = i - co * 9, c = co / O, o = co - c * O;
  wf[i] = w[((long long)o * C + c) * 9 + 8 - t];
}
cudaError_t launch_flip_taps(const float* w, float* wf, int C, cudaStream_t s, int O) {
  flip_taps_kernel<<<(C * O * 9 + 255) / 256, 256, 0, s>>>(w, wf, C, O);
  return cudaGetLastError();
}

// sum of a fp32 array into dst[0] (+=): conv_out bias gradient
__global__ void __launch_bounds__(256) sum_add_kernel(const float* __restrict__ x, long long n, float* __restrict__ dst) {
  __shared__ float red[8];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) s += x[i];
  s = warp_sum_f(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k];
    atomicAdd(dst, t);
  }
}
cudaError_t launch_sum_add(const float* x, long long n, float* dst, cudaStream_t s) {
  const int grid = (int)((n + 2047) / 2048 < 296 ? (n + 2047) / 2048 : 296);
  sum_add_kernel<<<grid, 256, 0, s>>>(x, n, dst);
  return cudaGetLastError();
}

// folded-upsample weight gradient back to the 3x3 taps: dW3[co][ci][k] += sum over (parity p, folded tap t) whose fold mask
// contains k of dWf[p][co][ci][t]
__global__ void unfold_up2_kernel(const float* __restrict__ dwf, float* __restrict__ dw3, long long nco_ci, UnfoldMasks m) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nco_ci) return;
  float a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int p = 0; p < 4; ++p)
    for (int t = 0; t < 4; ++t) {
      const float v = dwf[((long long)p * nco_ci + i) * 4 + t];
      const unsigned mask = m.mask[p][t];
#pragma unroll
      for (int k = 0; k < 9; ++k)
        if (mask & (1u << k)) a[k] += v;
    }
#pragma unroll
  for (int k = 0; k < 9; ++k) dw3[i * 9 + k] += a[k];
}
cudaError_t launch_unfold_up2(const float* dwf, float* dw3, long long nco_ci, const UnfoldMasks& m, cudaStream_t s) {
  unfold_up2_kernel<<<(unsigned)((nco_ci + 255) / 256), 256, 0, s>>>(dwf, dw3, nco_ci, m);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// Small dense layers of the timestep path.  y[n][o] = sum_i W[o][i] x[n][i] + b[o]
//   g_in[n][i] (+)= sum_o g[n][o] W[o][i];   dW[o][i] += sum_n g[n][o] x[n][i];   db[o] += sum_n g[n][o]
constexpr int LIN_OCHUNK = 128;   // output rows per CTA along grid.y (partial sums combined with atomics)
__global__ void lin_bwd_input_kernel(const float* __restrict__ g, int gstride, const float* __restrict__ Wt, int O, int I,
                                     float* __restrict__ gin, int N) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * I) return;
  const int n = idx / I, i = idx - n * I;
  const int o1 = min(O, (int)(blockIdx.y + 1) * LIN_OCHUNK);
  float a = 0.f;
  for (int o = blockIdx.y * LIN_OCHUNK; o < o1; ++o) a = fmaf(g[(long long)n * gstride + o], Wt[(long long)o * I + i], a);
  atomicAdd(gin + idx, a);
}
__global__ void lin_bwd_weight_kernel(const float* __restrict__ g, int gstride, const float* __restrict__ x, int O, int I,
                                      float* __restrict__ dW, float* __restrict__ db, int N) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= O * I) return;
  const int o = idx / I, i = idx - o * I;
  float a = 0.f, b = 0.f;
  for (int n = 0; n < N; ++n) {
    const float gv = g[(long long)n * gstride + o];
    a = fmaf(gv, x[(long long)n * I + i], a);
    b += gv;
  }
  dW[idx] += a;
  if (i == 0 && db) db[o] += b;
}
__global__ void silu_bwd_kernel(float* __restrict__ g, const float* __restrict__ u, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float y = u[i];
  const float sig = 1.0f / (1.0f + expf(-y));
  g[i] *= sig * (1.0f + y * (1.0f - sig));
}
cudaError_t launch_lin_bwd_input(const float* g, int gstride, const float* W, int O, int I, float* gin, int N, int accumulate,
                                 cudaStream_t s) {
  if (!accumulate) {
    cudaError_t e = cudaMemsetAsync(gin, 0, (size_t)N * I * sizeof(float), s);
    if (e != cudaSuccess) return e;
  }
  lin_bwd_input_kernel<<<dim3((N * I + 127) / 128, (O + LIN_OCHUNK - 1) / LIN_OCHUNK), 128, 0, s>>>(g, gstride, W, O, I, gin, N);
  return cudaGetLastError();
}
cudaError_t launch_lin_bwd_weight(const float* g, int gstride, const float* x, int O, int I, float* dW, float* db, int N,
                                  cudaStream_t s) {
  lin_bwd_weight_kernel<<<(O * I + 127) / 128, 128, 0, s>>>(g, gstride, x, O, I, dW, db, N);
  return cudaGetLastError();
}
cudaError_t launch_silu_bwd(float* g, const float* u, int n, cudaStream_t s) {
  silu_bwd_kernel<<<(n + 255) / 256, 256, 0, s>>>(g, u, n);
  return cudaGetLastError();
}
__global__ void silu_fwd_kernel(const float* __restrict__ u, float* __restrict__ y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = silu_f(u[i]);
}
cudaError_t launch_silu_fwd(const float* u, float* y, int n, cudaStream_t s) {
  silu_fwd_kernel<<<(n + 255) / 256, 256, 0, s>>>(u, y, n);
  return cudaGetLastError();
}

}  // namespace b200ad
