// Timestep embedding (sinusoid -> MLP -> all 32 resnet projections) and the head_dim-8 self-attention core.
// Reference semantics: diffusers get_timestep_embedding(flip_sin_to_cos=True, freq_shift=0), TimestepEmbedding,
// ResnetBlock2D.time_emb_proj(silu(emb)) and Attention/AttnProcessor2_0 (oracle/unet_oracle.py restates them;
// reached from audiodiffusion/pipeline_audio_diffusion.py:163).
#include "kernels.cuh"

namespace b200ad {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int sh = 16; sh >= 1; sh >>= 1) v += __shfl_xor_sync(0xffffffffu, v, sh);
  return v;
}

// one CTA per sample: emb[dim0] -> h1[4 dim0] -> temb_act[4 dim0]
__global__ void __launch_bounds__(256) temb_mlp_kernel(const float* __restrict__ t, int dim0, const float* __restrict__ w1,
                                                       const float* __restrict__ b1, const float* __restrict__ w2,
                                                       const float* __restrict__ b2, float* __restrict__ temb_act,
                                                       float* __restrict__ save_emb, float* __restrict__ save_u1,
                                                       float* __restrict__ save_u2, int* __restrict__ lead) {
  extern __shared__ float tsm[];
  float* emb = tsm;          // dim0
  float* h1 = tsm + dim0;    // 4*dim0
  const int n = blockIdx.x, D = 4 * dim0, half = dim0 / 2;
  const float tv = t[n];
  if (lead) {
    // Samples that share a timestep share the whole embedding (the sampling loop passes ONE t for the batch,
    // pipeline_audio_diffusion.py:163): only the first sample of each class ("leader") is computed, the projection kernel
    // copies its rows to the others.  lead == nullptr (training: per-sample t, activations saved for backward): no sharing.
    __shared__ int s_lead;
    if (threadIdx.x == 0) {
      int m = 0;
      while (m < n && t[m] != tv) ++m;
      s_lead = m;
      lead[n] = m;
    }
    __syncthreads();
    if (s_lead != n) return;
  }
  for (int i = threadIdx.x; i < half; i += blockDim.x) {
    const float freq = expf(-logf(10000.0f) * (float)i / (float)half);
    const float a = tv * freq;
    emb[i] = cosf(a);          // flip_sin_to_cos: [cos | sin]
    emb[half + i] = sinf(a);
    if (save_emb) { save_emb[(long long)n * dim0 + i] = emb[i]; save_emb[(long long)n * dim0 + half + i] = emb[half + i]; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int r = warp; r < D; r += nw) {
    float s = 0.f;
    for (int k = lane; k < dim0; k += 32) s += w1[(long long)r * dim0 + k] * emb[k];
    s = warp_sum(s);
    if (lane == 0) {
      h1[r] = silu_f(s + b1[r]);
      if (save_u1) save_u1[(long long)n * D + r] = s + b1[r];
    }
  }
  __syncthreads();
  for (int r = warp; r < D; r += nw) {
    float s = 0.f;
    for (int k = lane; k < D; k += 32) s += w2[(long long)r * D + k] * h1[k];
    s = warp_sum(s);
    if (lane == 0) {
      temb_act[(long long)n * D + r] = silu_f(s + b2[r]);
      if (save_u2) save_u2[(long long)n * D + r] = s + b2[r];
    }
  }
}

// one warp per projection row, all samples
__global__ void __launch_bounds__(256) temb_proj_kernel(const float* __restrict__ temb_act, int N, int D,
                                                        const float* __restrict__ wcat, const float* __restrict__ bcat,
                                                        int rows, float* __restrict__ proj, const int* __restrict__ lead) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + warp;
  if (r >= rows) return;
  float wv[32];  // D <= 1024
  const int per = D / 32;
  for (int k = 0; k < per; ++k) wv[k] = wcat[(long long)r * D + k * 32 + lane];
  const float bias = bcat[r];
  for (int n = 0; n < N; ++n) {
    const int ld = lead ? lead[n] : n;
    if (ld == n) {
      float s = 0.f;
      for (int k = 0; k < per; ++k) s += wv[k] * temb_act[(long long)n * D + k * 32 + lane];
      s = warp_sum(s);
      if (lane == 0) proj[(long long)n * rows + r] = s + bias;
    } else if (lane == 0) {      // same timestep as an earlier sample: its row was written by this very lane
      proj[(long long)n * rows + r] = proj[(long long)ld * rows + r];
    }
  }
}

cudaError_t launch_temb(const float* t, int N, int dim0, const float* w1, const float* b1, const float* w2,
                        const float* b2, float* temb_act, const float* wcat, const float* bcat, int rows,
                        float* proj, cudaStream_t s, float* save_emb, float* save_u1, float* save_u2, int* lead) {
  const int D = 4 * dim0;
  if (D > 1024 || (D % 32) != 0) return cudaErrorInvalidValue;
  temb_mlp_kernel<<<N, 256, (dim0 + D) * sizeof(float), s>>>(t, dim0, w1, b1, w2, b2, temb_act, save_emb, save_u1, save_u2, lead);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  temb_proj_kernel<<<(rows + 7) / 8, 256, 0, s>>>(temb_act, N, D, wcat, bcat, rows, proj, lead);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ attention
// grid (heads, N). K and V of one (sample, head) are staged in shared memory as fp32; one thread per query.
__global__ void __launch_bounds__(256) attention_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                        __nv_bfloat16* __restrict__ out, int N, int C, int H, int W) {
  extern __shared__ float asm_[];
  const int seq = H * W;
  float* ks = asm_;            // [seq][8]
  float* vs = asm_ + seq * 8;  // [seq][8]
  const Geom g = make_geom(N, H, W);
  const int head = blockIdx.x, n = blockIdx.y;
  const int planes = C >> 3;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* qp = base + (long long)head * g.PL * 8;
  const __nv_bfloat16* kp = base + (long long)(planes + head) * g.PL * 8;
  const __nv_bfloat16* vp = base + (long long)(2 * planes + head) * g.PL * 8;
  for (int p = threadIdx.x; p < seq; p += blockDim.x) {
    const long long pix = (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
    const uint4 kv = *reinterpret_cast<const uint4*>(kp + pix);
    const uint4 vv = *reinterpret_cast<const uint4*>(vp + pix);
    const uint32_t ku[4] = {kv.x, kv.y, kv.z, kv.w}, vu[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = unpack_bf16x2(ku[e]);
      ks[p * 8 + 2 * e] = f.x; ks[p * 8 + 2 * e + 1] = f.y;
      f = unpack_bf16x2(vu[e]);
      vs[p * 8 + 2 * e] = f.x; vs[p * 8 + 2 * e + 1] = f.y;
    }
  }
  __syncthreads();
  const float sc = 0.35355339059327373f * 1.4426950408889634f;  // 8^-0.5 * log2(e)
  for (int p = threadIdx.x; p < seq; p += blockDim.x) {
    const long long pix = (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
    const uint4 qv = *reinterpret_cast<const uint4*>(qp + pix);
    const uint32_t qu[4] = {qv.x, qv.y, qv.z, qv.w};
    float q[8];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = unpack_bf16x2(qu[e]);
      q[2 * e] = f.x * sc; q[2 * e + 1] = f.y * sc;
    }
    float mx = -INFINITY;
    for (int j = 0; j < seq; ++j) {
      const float4 k0 = *reinterpret_cast<const float4*>(ks + j * 8), k1 = *reinterpret_cast<const float4*>(ks + j * 8 + 4);
      const float s = q[0] * k0.x + q[1] * k0.y + q[2] * k0.z + q[3] * k0.w + q[4] * k1.x + q[5] * k1.y + q[6] * k1.z + q[7] * k1.w;
      mx = fmaxf(mx, s);
    }
    float den = 0.f, o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < seq; ++j) {
      const float4 k0 = *reinterpret_cast<const float4*>(ks + j * 8), k1 = *reinterpret_cast<const float4*>(ks + j * 8 + 4);
      const float s = q[0] * k0.x + q[1] * k0.y + q[2] * k0.z + q[3] * k0.w + q[4] * k1.x + q[5] * k1.y + q[6] * k1.z + q[7] * k1.w;
      const float pj = exp2f(s - mx);
      den += pj;
      const float4 v0 = *reinterpret_cast<const float4*>(vs + j * 8), v1 = *reinterpret_cast<const float4*>(vs + j * 8 + 4);
      o[0] += pj * v0.x; o[1] += pj * v0.y; o[2] += pj * v0.z; o[3] += pj * v0.w;
      o[4] += pj * v1.x; o[5] += pj * v1.y; o[6] += pj * v1.z; o[7] += pj * v1.w;
    }
    const float inv = 1.0f / den;
    uint4 ov;
    ov.x = pack_bf16x2(o[0] * inv, o[1] * inv); ov.y = pack_bf16x2(o[2] * inv, o[3] * inv);
    ov.z = pack_bf16x2(o[4] * inv, o[5] * inv); ov.w = pack_bf16x2(o[6] * inv, o[7] * inv);
    *reinterpret_cast<uint4*>(out + ((long long)n * planes + head) * g.PL * 8 + pix) = ov;
  }
}

// ---- tensor-core variant (seq % 16 == 0): warp-level mma.sync, one warp per 16 queries -----------------------------
// head_dim 8 is exactly one k-step of m16n8k8 for Q.K^T, and the P.V product is one m16n8k16 per 16 keys with n = the 8
// output dims.  Two passes over the keys (exact row max first, then exp / sum / P.V), no online rescaling.
__device__ __forceinline__ void mma_16x8x8_bf16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(b0));
}
__device__ __forceinline__ void mma_16x8x16_bf16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(128) attention_mma_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                            __nv_bfloat16* __restrict__ out, int N, int C, int H, int W) {
  extern __shared__ __align__(16) uint8_t amem[];
  const int seq = H * W;
  uint4* ks = reinterpret_cast<uint4*>(amem);  // [seq] rows of 8 bf16
  uint4* vs = ks + seq;
  const Geom g = make_geom(N, H, W);
  const int head = blockIdx.x, n = blockIdx.y;
  const int planes = C >> 3;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const __nv_bfloat16* qp = base + (long long)head * g.PL * 8;
  const __nv_bfloat16* kp = base + (long long)(planes + head) * g.PL * 8;
  const __nv_bfloat16* vp = base + (long long)(2 * planes + head) * g.PL * 8;
  for (int p = threadIdx.x; p < seq; p += blockDim.x) {
    const long long pix = (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
    ks[p] = *reinterpret_cast<const uint4*>(kp + pix);
    vs[p] = *reinterpret_cast<const uint4*>(vp + pix);
  }
  __syncthreads();
  const uint32_t* ks32 = reinterpret_cast<const uint32_t*>(ks);
  const uint32_t vs_addr = (uint32_t)__cvta_generic_to_shared(vs);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
  const float sc = 0.35355339059327373f * 1.4426950408889634f;  // 8^-0.5 * log2(e)
  __nv_bfloat16* op = out + ((long long)n * planes + head) * g.PL * 8;
  for (int q0 = warp * 16; q0 < seq; q0 += 64) {
    const int qa = q0 + gq, qb = qa + 8;
    const long long pa = (long long)(g.lead + (qa / W) * g.Wp + (qa % W)) * 8;
    const long long pb = (long long)(g.lead + (qb / W) * g.Wp + (qb % W)) * 8;
    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(qp + pa + 2 * t);
    const uint32_t a1 = *reinterpret_cast<const uint32_t*>(qp + pb + 2 * t);
    float m0 = -INFINITY, m1 = -INFINITY;
    for (int k0 = 0; k0 < seq; k0 += 8) {
      float c[4] = {0.f, 0.f, 0.f, 0.f};
      mma_16x8x8_bf16(c, a0, a1, ks32[(k0 + gq) * 4 + t]);
      m0 = fmaxf(m0, fmaxf(c[0], c[1]));
      m1 = fmaxf(m1, fmaxf(c[2], c[3]));
    }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    m0 *= sc; m1 *= sc;
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    float l0 = 0.f, l1 = 0.f;
    for (int k0 = 0; k0 < seq; k0 += 16) {
      float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
      mma_16x8x8_bf16(s0, a0, a1, ks32[(k0 + gq) * 4 + t]);
      mma_16x8x8_bf16(s1, a0, a1, ks32[(k0 + 8 + gq) * 4 + t]);
      const float e00 = exp2f(fmaf(s0[0], sc, -m0)), e01 = exp2f(fmaf(s0[1], sc, -m0));
      const float e02 = exp2f(fmaf(s0[2], sc, -m1)), e03 = exp2f(fmaf(s0[3], sc, -m1));
      const float e10 = exp2f(fmaf(s1[0], sc, -m0)), e11 = exp2f(fmaf(s1[1], sc, -m0));
      const float e12 = exp2f(fmaf(s1[2], sc, -m1)), e13 = exp2f(fmaf(s1[3], sc, -m1));
      l0 += (e00 + e01) + (e10 + e11);
      l1 += (e02 + e03) + (e12 + e13);
      uint32_t vb0, vb1;  // V[k0 .. k0+15][0..7] as the col-major B fragment: transposing ldmatrix of two 8x8 tiles
      const uint32_t va = vs_addr + (uint32_t)(k0 + (lane & 15)) * 16u;
      asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(vb0), "=r"(vb1) : "r"(va));
      mma_16x8x16_bf16(o, pack_bf16x2(e00, e01), pack_bf16x2(e02, e03), pack_bf16x2(e10, e11), pack_bf16x2(e12, e13),
                       vb0, vb1);
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    *reinterpret_cast<uint32_t*>(op + pa + 2 * t) = pack_bf16x2(o[0] * i0, o[1] * i0);
    *reinterpret_cast<uint32_t*>(op + pb + 2 * t) = pack_bf16x2(o[2] * i1, o[3] * i1);
  }
}

cudaError_t launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int N, int C, int H, int W, cudaStream_t s) {
  const int seq = H * W;
  dim3 grid(C >> 3, N);
  if ((seq % 16) == 0 && (size_t)seq * 32 <= 48 * 1024) {
    attention_mma_kernel<<<grid, 128, (size_t)seq * 32, s>>>(qkv, out, N, C, H, W);
    return cudaGetLastError();
  }
  const size_t smem = (size_t)seq * 16 * sizeof(float);
  if (smem > 200 * 1024) return cudaErrorInvalidValue;
  static size_t smem_set = 48 * 1024;
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    smem_set = smem;
  }
  const int threads = seq >= 256 ? 256 : ((seq + 31) / 32) * 32;
  attention_kernel<<<grid, threads, smem, s>>>(qkv, out, N, C, H, W);
  return cudaGetLastError();
}

}  // namespace b200ad

// =====================================================================================================================
// Generic single-head attention (AutoencoderKL mid block: one head of dim C = 512 over seq = H*W up to 1024+).
// Runs once per sample (not per denoising step), so three plain tiled SIMT kernels: scores, row softmax, P*V.
// Reference semantics: diffusers Attention (AttnProcessor2_0) with heads = 1 — oracle/vae_oracle.py::_attn.
namespace b200ad {

__device__ __forceinline__ long long pf8_pix(const Geom& g, int p, int W) {
  return (long long)(g.lead + (p / W) * g.Wp + (p % W)) * 8;
}

// S[n][q][k] = scale * sum_c Q[q][c] K[k][c];  qkv: PF8 with 3C channels (q | k | v).  grid (seq/64, seq/64, N), 256 thr
__global__ void __launch_bounds__(256) attn_scores_kernel(const __nv_bfloat16* __restrict__ qkv, float* __restrict__ S,
                                                          int N, int C, int H, int W, float scale) {
  __shared__ float qs[16][65], ks[16][65];
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3;
  const int n = blockIdx.z, q0 = blockIdx.x * 64, k0 = blockIdx.y * 64;
  const __nv_bfloat16* base = qkv + (long long)n * 3 * planes * g.PL * 8;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int c0 = 0; c0 < C; c0 += 16) {
    // 64 pixels x 16 channels each for Q and K: 128 (pixel, plane) vectors apiece
    for (int i = threadIdx.x; i < 256; i += 256) {
      const int which = i >> 7, r = i & 127, px = r & 63, pl = r >> 6;
      const int p = (which ? k0 : q0) + px;
      float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (p < seq) {
        const int plane = (which ? planes : 0) + (c0 >> 3) + pl;
        const uint4 u = *reinterpret_cast<const uint4*>(base + (long long)plane * g.PL * 8 + pf8_pix(g, p, W));
        const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) { const float2 f = unpack_bf16x2(uu[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
      }
      float (*dst)[65] = which ? ks : qs;
#pragma unroll
      for (int e = 0; e < 8; ++e) dst[pl * 8 + e][px] = v[e];
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = qs[c][ty + 16 * i]; b[i] = ks[c][tx + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = q0 + ty + 16 * i, k = k0 + tx + 16 * j;
      if (q < seq && k < seq) S[((long long)n * seq + q) * seq + k] = acc[i][j] * scale;
    }
}

// in-place softmax over rows of length seq. grid (seq, N), 256 threads
__global__ void __launch_bounds__(256) softmax_rows_kernel(float* __restrict__ S, int seq) {
  __shared__ float red[8];
  float* row = S + ((long long)blockIdx.y * seq + blockIdx.x) * seq;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < seq; i += blockDim.x) mx = fmaxf(mx, row[i]);
  for (int sh = 16; sh >= 1; sh >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, sh));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < seq; i += blockDim.x) { const float e = __expf(row[i] - mx); row[i] = e; s += e; }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
  for (int i = 0; i < 8; ++i) s += red[i];
  const float inv = 1.0f / s;
  for (int i = threadIdx.x; i < seq; i += blockDim.x) row[i] *= inv;
}

// O[q][c] = sum_k P[q][k] V[k][c] -> PF8 bf16 (C channels). grid (seq/64, C/64, N), 256 threads
__global__ void __launch_bounds__(256) attn_pv_kernel(const float* __restrict__ P, const __nv_bfloat16* __restrict__ qkv,
                                                      __nv_bfloat16* __restrict__ out, int N, int C, int H, int W) {
  __shared__ float ps[16][65], vs[16][65];
  const Geom g = make_geom(N, H, W);
  const int seq = H * W, planes = C >> 3;
  const int n = blockIdx.z, q0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const __nv_bfloat16* vbase = qkv + ((long long)n * 3 * planes + 2 * planes) * g.PL * 8;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // tx -> channel, ty -> query
  float acc[4][4] = {};
  for (int k0 = 0; k0 < seq; k0 += 16) {
    for (int i = threadIdx.x; i < 1024; i += 256) {   // P tile: 64 q x 16 k
      const int kk = i & 15, qq = i >> 4;
      const int q = q0 + qq, k = k0 + kk;
      ps[kk][qq] = (q < seq && k < seq) ? P[((long long)n * seq + q) * seq + k] : 0.f;
    }
    if (threadIdx.x < 128) {                            // V tile: 16 k x 64 c = 16 x 8 vectors
      const int kk = threadIdx.x & 15, pl = threadIdx.x >> 4;
      const int k = k0 + kk;
      float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (k < seq) {
        const uint4 u = *reinterpret_cast<const uint4*>(vbase + (long long)((c0 >> 3) + pl) * g.PL * 8 + pf8_pix(g, k, W));
        const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) { const float2 f = unpack_bf16x2(uu[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) vs[kk][pl * 8 + e] = v[e];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = ps[k][ty * 4 + i]; b[i] = vs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  // thread holds queries ty*4..+3, channels c0 + tx*4..+3 (half of an 8-channel vector)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + ty * 4 + i;
    if (q >= seq) continue;
    const int c = c0 + tx * 4;
    __nv_bfloat16* dp = out + ((long long)n * planes + (c >> 3)) * g.PL * 8 + pf8_pix(g, q, W) + (c & 7);
    uint2 o;
    o.x = pack_bf16x2(acc[i][0], acc[i][1]);
    o.y = pack_bf16x2(acc[i][2], acc[i][3]);
    *reinterpret_cast<uint2*>(dp) = o;
  }
}

cudaError_t launch_attention_1head(const __nv_bfloat16* qkv, __nv_bfloat16* out, float* scores, int N, int C, int H, int W,
                                   cudaStream_t s) {
  const int seq = H * W;
  const int t = (seq + 63) / 64;
  attn_scores_kernel<<<dim3(t, t, N), 256, 0, s>>>(qkv, scores, N, C, H, W, rsqrtf((float)C));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  softmax_rows_kernel<<<dim3(seq, N), 256, 0, s>>>(scores, seq);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  attn_pv_kernel<<<dim3(t, C / 64, N), 256, 0, s>>>(scores, qkv, out, N, C, H, W);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// AutoencoderKL.encode tail: quant_conv (1x1, 2L -> 2L) on the encoder output (PF8, first 2L channels of plane 0) and
// DiagonalGaussianDistribution.sample(): z = mean + exp(0.5 * clamp(logvar, -30, 20)) * noise  -> fp32 NCHW (N, L, H, W).
__global__ void vae_sample_kernel(const __nv_bfloat16* __restrict__ enc, const float* __restrict__ wq, const float* __restrict__ bq,
                                  const float* __restrict__ noise, float* __restrict__ z, float* __restrict__ moments,
                                  int N, int C, int L, int H, int W) {
  const Geom g = make_geom(N, H, W);
  const int p = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
  if (p >= H * W) return;
  const uint4 u = *reinterpret_cast<const uint4*>(enc + (long long)n * (C >> 3) * g.PL * 8 + pf8_pix(g, p, W));
  const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
  float h[8];
#pragma unroll
  for (int e = 0; e < 4; ++e) { const float2 f = unpack_bf16x2(uu[e]); h[2 * e] = f.x; h[2 * e + 1] = f.y; }
  float m[8];
  for (int o = 0; o < 2 * L; ++o) {
    float a = bq[o];
    for (int i = 0; i < 2 * L; ++i) a = fmaf(wq[o * 2 * L + i], h[i], a);
    m[o] = a;
    if (moments) moments[((long long)n * 2 * L + o) * H * W + p] = a;
  }
  for (int l = 0; l < L; ++l) {
    const float lv = fminf(fmaxf(m[L + l], -30.f), 20.f);
    const long long idx = ((long long)n * L + l) * H * W + p;
    z[idx] = m[l] + expf(0.5f * lv) * (noise ? noise[idx] : 0.f);
  }
}
cudaError_t launch_vae_sample(const __nv_bfloat16* enc, const float* wq, const float* bq, const float* noise, float* z,
                              float* moments, int N, int C, int L, int H, int W, cudaStream_t s) {
  if (2 * L > 8) return cudaErrorInvalidValue;
  vae_sample_kernel<<<dim3((H * W + 255) / 256, N), 256, 0, s>>>(enc, wq, bq, noise, z, moments, N, C, L, H, W);
  return cudaGetLastError();
}

// post_quant_conv: 1x1 conv L -> L on fp32 NCHW (L <= 4)
__global__ void mix1x1_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                              float* __restrict__ y, int N, int L, int HW) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
  if (p >= HW) return;
  for (int o = 0; o < L; ++o) {
    float a = b[o];
    for (int i = 0; i < L; ++i) a = fmaf(w[o * L + i], x[((long long)n * L + i) * HW + p], a);
    y[((long long)n * L + o) * HW + p] = a;
  }
}
cudaError_t launch_mix1x1(const float* x, const float* w, const float* b, float* y, int N, int L, int HW, cudaStream_t s) {
  mix1x1_kernel<<<dim3((HW + 255) / 256, N), 256, 0, s>>>(x, w, b, y, N, L, HW);
  return cudaGetLastError();
}

}  // namespace b200ad
