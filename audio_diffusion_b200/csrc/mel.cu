// Mel codec kernels: batched STFT -> power -> mel -> dB -> uint8 (Mel.audio_slice_to_image, audiodiffusion/mel.py:135-151)
// and uint8 -> dB -> power -> inverse mel -> 32-iteration Griffin-Lim (Mel.image_to_audio, audiodiffusion/mel.py:153-168).
// The librosa 0.10.2 arithmetic these follow is restated in oracle/mel_oracle.py.
//
// All FFTs run in fp64 (H100 has the fp64 rate to spare; the reference mixes fp64 FFTs with fp32 storage), one frame per
// CTA.  A real n_fft-point transform is ONE complex transform of n_fft / 2 points (even samples = real parts, odd samples =
// imaginary parts) plus an O(n_fft) split / merge step, and the complex transform is a Stockham autosort with radix-4
// passes in shared memory (one radix-2 pass first when log2 is odd): 5 passes over 1024 points for n_fft = 2048 where the
// first version made 11 radix-2 passes over 2048.  Window, twiddles and the overlap-add normaliser come from tables built
// once per call.  Spectra are kept frame-major so every load is coalesced.
#include <math_constants.h>

#include "../../include/b200ad.h"
#include "common.cuh"

namespace b200ad {
int set_err(const char* fmt, ...);

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double hann(int i, int N) {  // periodic Hann, scipy get_window("hann", N, fftbins=True)
  return 0.5 - 0.5 * cospi(2.0 * (double)i / (double)N);
}

// Tables of one call: tw[i] = exp(-2 pi i / N) for i < N (the full circle), win[i] = periodic Hann(N), and (decode only,
// `wss` may be null) wss[p] = sum over the frames f covering padded position p of win[p - f hop]^2, as librosa.istft's
// window_sumsquare, rounded to float32.
__global__ void mel_tables_kernel(double2* tw, double* win, float* wss, int N, int T, int hop) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) {
    double sn, cs;
    sincospi(-2.0 * (double)i / (double)N, &sn, &cs);
    tw[i] = make_double2(cs, sn);
    win[i] = hann(i, N);
  }
  if (wss && i < N + (T - 1) * hop) {
    int f_hi = i / hop;
    if (f_hi > T - 1) f_hi = T - 1;
    int f_lo = (i - N + hop) / hop;
    if (i - N + 1 <= 0) f_lo = 0;
    double acc = 0.0;
    for (int f = f_lo; f <= f_hi; ++f) {
      const int k = i - f * hop;
      if (k < 0 || k >= N) continue;
      const double w = hann(k, N);
      acc += w * w;
    }
    wss[i] = (float)acc;
  }
}

// Complex FFT of M = N / 2 points in shared memory (Stockham autosort, ping-pong a <-> b); returns the buffer holding the
// result.  `tw` is the N-entry table above: exp(-2 pi i q k / (4 p)) = tw[q k N / (4 p)] (< 3 N / 4).  All threads call it.
template <bool INVERSE>
__device__ double2* cfft(double2* a, double2* b, const double2* __restrict__ tw, int M, int logM) {
  const int N = 2 * M;
  int p = 1;
  if (logM & 1) {   // one radix-2 pass (p = 1: unit twiddles)
    const int half = M >> 1;
    for (int j = threadIdx.x; j < half; j += blockDim.x) {
      const double2 v0 = a[j], v1 = a[j + half];
      b[2 * j] = cadd(v0, v1);
      b[2 * j + 1] = csub(v0, v1);
    }
    __syncthreads();
    double2* t = a; a = b; b = t;
    p = 2;
  }
  const int t4 = M >> 2;
  for (; p < M; p <<= 2) {
    const int tstep = N / (4 * p);
    for (int j = threadIdx.x; j < t4; j += blockDim.x) {
      const int k = j & (p - 1);
      double2 w1 = __ldg(tw + k * tstep), w2 = __ldg(tw + 2 * k * tstep), w3 = __ldg(tw + 3 * k * tstep);
      if (INVERSE) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
      const double2 u0 = a[j];
      const double2 u1 = cmul(a[j + t4], w1);
      const double2 u2 = cmul(a[j + 2 * t4], w2);
      const double2 u3 = cmul(a[j + 3 * t4], w3);
      const double2 v0 = cadd(u0, u2), v1 = csub(u0, u2), v2 = cadd(u1, u3);
      const double2 d = csub(u1, u3);
      const double2 v3 = INVERSE ? make_double2(-d.y, d.x) : make_double2(d.y, -d.x);   // +-i (u1 - u3)
      const int j0 = ((j - k) << 2) + k;
      b[j0] = cadd(v0, v2);
      b[j0 + p] = cadd(v1, v3);
      b[j0 + 2 * p] = csub(v0, v2);
      b[j0 + 3 * p] = csub(v1, v3);
    }
    __syncthreads();
    double2* t = a; a = b; b = t;
  }
  return a;
}

// Real transform from the half-size complex one.  z = cfft(x[2j] + i x[2j+1]); with E / O the spectra of the even / odd
// samples, Z[k] = E[k] + i O[k], E[k] = (Z[k] + conj Z[M-k]) / 2, O[k] = (Z[k] - conj Z[M-k]) / 2i and
//   X[k] = E[k] + W^k O[k],   X[M-k] = conj(E[k] - W^k O[k]),   W = exp(-2 pi i / N),   k = 0 .. M/2  (Z[M] = Z[0]).
__device__ __forceinline__ void rfft_pair(const double2* z, const double2* __restrict__ tw, int M, int k, double2& xk, double2& xmk) {
  const double2 zk = z[k], zm = z[(M - k) & (M - 1)];
  const double2 e = make_double2(0.5 * (zk.x + zm.x), 0.5 * (zk.y - zm.y));
  const double2 o = make_double2(0.5 * (zk.y + zm.y), -0.5 * (zk.x - zm.x));
  const double2 wo = cmul(__ldg(tw + k), o);
  xk = cadd(e, wo);
  const double2 dm = csub(e, wo);
  xmk = make_double2(dm.x, -dm.y);
}
// Inverse: Z[k] = E[k] + i O[k] with E = (X[k] + conj X[M-k]) / 2, O = (X[k] - conj X[M-k]) / 2 * conj(W^k), and
// Z[M-k] = conj(E) + i conj(O); the imaginary parts of X[0] and X[M] are ignored (numpy.fft.irfft).
__device__ __forceinline__ void irfft_pair(double2 xk, double2 xm, const double2* __restrict__ tw, int k, double2& zk, double2& zmk) {
  const double2 e = make_double2(0.5 * (xk.x + xm.x), 0.5 * (xk.y - xm.y));
  const double2 dd = make_double2(0.5 * (xk.x - xm.x), 0.5 * (xk.y + xm.y));
  double2 w = __ldg(tw + k);
  w.y = -w.y;
  const double2 o = cmul(dd, w);
  zk = make_double2(e.x - o.y, e.y + o.x);
  zmk = make_double2(e.x + o.y, o.x - e.y);     // conj(E) + i conj(O)
}

struct MelDims {
  int T, M, F, N, logN, hop, L;  // frames (x_res), mels (y_res), bins, n_fft, log2 n_fft, hop, slice length
};

// ------------------------------------------------------------------------------------------ encode
// grid (T, n): one frame. STFT (fp64, rounded to complex64 like librosa), |X|^2 (fp32), mel = M * S (fp32).
__global__ void __launch_bounds__(256) enc_frame_kernel(const float* __restrict__ audio, const float* __restrict__ basis_t,
                                                        const double2* __restrict__ tw, const double* __restrict__ win,
                                                        float* __restrict__ mel, unsigned* __restrict__ smax, MelDims d) {
  extern __shared__ __align__(16) uint8_t msm[];
  const int M = d.N >> 1;
  double2* a = reinterpret_cast<double2*>(msm);
  double2* b = a + M;
  float* pw = reinterpret_cast<float*>(b + M);
  const int t = blockIdx.x, n = blockIdx.y;
  const float* y = audio + (size_t)n * d.L;
  for (int j = threadIdx.x; j < M; j += blockDim.x) {
    const int p0 = t * d.hop + 2 * j - d.N / 2;     // center=True, zero padding (librosa 0.10 pad_mode="constant")
    const double v0 = (p0 >= 0 && p0 < d.L) ? (double)y[p0] : 0.0;
    const double v1 = (p0 + 1 >= 0 && p0 + 1 < d.L) ? (double)y[p0 + 1] : 0.0;
    a[j] = make_double2(v0 * win[2 * j], v1 * win[2 * j + 1]);
  }
  __syncthreads();
  const double2* Z = cfft<false>(a, b, tw, M, d.logN - 1);
  for (int k = threadIdx.x; k <= M / 2; k += blockDim.x) {
    double2 xk, xm;
    rfft_pair(Z, tw, M, k, xk, xm);
    {
      const float re = (float)xk.x, im = (float)xk.y;    // stft_matrix is complex64
      const float mag = hypotf(re, im);                  // np.abs(complex64)
      pw[k] = mag * mag;                                 // ** 2 in float32
    }
    {
      const float re = (float)xm.x, im = (float)xm.y;
      const float mag = hypotf(re, im);
      pw[M - k] = mag * mag;
    }
  }
  __syncthreads();
  float lmax = 0.f;
  for (int m = threadIdx.x; m < d.M; m += blockDim.x) {
    float acc = 0.f;
    for (int f = 0; f < d.F; ++f) acc = fmaf(basis_t[(size_t)f * d.M + m], pw[f], acc);
    mel[((size_t)n * d.M + m) * d.T + t] = acc;
    lmax = fmaxf(lmax, acc);
  }
  // ref = np.max(S): non-negative floats order like their bit patterns
  for (int sh = 16; sh >= 1; sh >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, sh));
  if ((threadIdx.x & 31) == 0) atomicMax(smax + n, __float_as_uint(lmax));
}

// power_to_db(ref, amin=1e-10, top_db) followed by mel.py:149 (float32 arithmetic, truncating cast).  ref = np.max(S) (the
// reference default: `refs` == nullptr) or a caller-supplied value per slice (mel.py:135 accepts any scalar / callable).
__global__ void enc_db_kernel(const float* __restrict__ mel, const unsigned* __restrict__ smax, const float* __restrict__ refs,
                              uint8_t* __restrict__ img, int per, float top_db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = blockIdx.y;
  if (i >= per) return;
  const float amin = 1e-10f;
  const float vmax = __uint_as_float(smax[n]);
  const float ref = refs ? fabsf(refs[n]) : vmax;        // librosa: ref_value = np.abs(ref)
  const float lref = __fmul_rn(10.0f, (float)log10((double)fmaxf(amin, ref)));
  const float s = mel[(size_t)n * per + i];
  float ls = __fsub_rn(__fmul_rn(10.0f, (float)log10((double)fmaxf(amin, s))), lref);
  // log_spec.max() - top_db: exactly -top_db when ref is the maximum of S
  const float lmax = __fsub_rn(__fmul_rn(10.0f, (float)log10((double)fmaxf(amin, vmax))), lref);
  ls = fmaxf(ls, __fsub_rn(lmax, top_db));
  float v = __fdiv_rn(__fmul_rn(__fadd_rn(ls, top_db), 255.0f), top_db);
  v = fminf(fmaxf(v, 0.0f), 255.0f);
  img[(size_t)n * per + i] = (uint8_t)(int)__fadd_rn(v, 0.5f);
}

// ------------------------------------------------------------------------------------------ decode
__device__ __forceinline__ double u01(uint64_t seed, uint64_t idx) {  // splitmix64 -> [0,1)
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (idx + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

// inverse mel: X2 = max(pinv(A) * S, 0) (what librosa.util.nnls returns on image-domain inputs: its L-BFGS-B stops at
// iteration 0), mag = sqrt(X2), angles = mag * exp(2 pi i u).   grid (ceil(F/64), ceil(T/64), n), 256 threads, 4x4 tile.
__global__ void __launch_bounds__(256) dec_pinv_kernel(const uint8_t* __restrict__ img, const double* __restrict__ pinv,
                                                       double* __restrict__ mag, double2* __restrict__ ang, MelDims d,
                                                       double top_db, uint64_t seed) {
  __shared__ double sp[16][65];  // pinv tile  [k][f]
  __shared__ double ss[16][65];  // power tile [k][t]
  const int n = blockIdx.z, f0 = blockIdx.x * 64, t0 = blockIdx.y * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // tx -> f, ty -> t
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
  for (int k0 = 0; k0 < d.M; k0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      const int kk = i & 15, ff = i >> 4;  // pinv is [F][M]: consecutive threads read consecutive m
      const int f = f0 + ff;
      sp[kk][ff] = (f < d.F && k0 + kk < d.M) ? pinv[(size_t)f * d.M + k0 + kk] : 0.0;   // y_res need not be a multiple of 16
    }
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      const int tt = i & 63, kk = i >> 6;  // image is [M][T]: consecutive threads read consecutive t
      const int t = t0 + tt;
      double v = 0.0;
      if (t < d.T && k0 + kk < d.M) {
        const double bb = (double)img[((size_t)n * d.M + k0 + kk) * d.T + t];
        const double ldb = bb * top_db / 255.0 - top_db;  // mel.py:163
        v = pow(10.0, 0.1 * ldb);                          // librosa.db_to_power
      }
      ss[kk][tt] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      double pf[4], st[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { pf[i] = sp[kk][tx + 16 * i]; st[i] = ss[kk][ty + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(pf[i], st[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int t = t0 + ty + 16 * j;
    if (t >= d.T) continue;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = f0 + tx + 16 * i;
      if (f >= d.F) continue;
      const double m = sqrt(fmax(acc[i][j], 0.0));
      const size_t o = ((size_t)n * d.T + t) * d.F + f;
      mag[o] = m;
      double s, c;
      sincospi(2.0 * u01(seed, o), &s, &c);
      ang[o] = make_double2(m * c, m * s);
    }
  }
}

// grid (T, n): frame t of image n: irfft of angles[:, t], times the synthesis window -> frames[n][t][N] (fp32)
__global__ void __launch_bounds__(256, 4) gl_istft_kernel(const double2* __restrict__ ang, const double2* __restrict__ tw,
                                                       const double* __restrict__ win, float* __restrict__ frames, MelDims d) {
  extern __shared__ __align__(16) uint8_t msm[];
  const int M = d.N >> 1;
  double2* a = reinterpret_cast<double2*>(msm);
  double2* b = a + M;
  const int t = blockIdx.x, n = blockIdx.y;
  const double2* X = ang + ((size_t)n * d.T + t) * d.F;
  for (int k = threadIdx.x; k <= M / 2; k += blockDim.x) {
    double2 xk = X[k], xm = X[M - k];
    if (k == 0) { xk.y = 0.0; xm.y = 0.0; }       // irfft ignores the imaginary parts of the DC and Nyquist bins
    double2 zk, zm;
    irfft_pair(xk, xm, tw, k, zk, zm);
    a[k] = zk;
    if (k != 0 && 2 * k != M) a[M - k] = zm;
  }
  __syncthreads();
  const double2* z = cfft<true>(a, b, tw, M, d.logN - 1);
  const double inv = 1.0 / (double)M;
  float2* out = reinterpret_cast<float2*>(frames + ((size_t)n * d.T + t) * d.N);
  for (int j = threadIdx.x; j < M; j += blockDim.x)
    out[j] = make_float2((float)(z[j].x * inv * win[2 * j]), (float)(z[j].y * inv * win[2 * j + 1]));
}

// overlap-add of the windowed frames at padded position p, normalised by the window sum-square (librosa.istft)
__device__ __forceinline__ float ola_sample(const float* __restrict__ fr, const float* __restrict__ wss, int p, const MelDims& d) {
  int f_hi = p / d.hop;
  if (f_hi > d.T - 1) f_hi = d.T - 1;
  int f_lo = (p - d.N + d.hop) / d.hop;  // ceil((p - N + 1) / hop) for p - N + 1 >= 0
  if (p - d.N + 1 <= 0) f_lo = 0;
  double acc = 0.0;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int i = p - f * d.hop;
    if (i < 0 || i >= d.N) continue;
    acc += (double)fr[(size_t)f * d.N + i];
  }
  const float y = (float)acc, ws = __ldg(wss + p);
  return (ws > 1.17549435e-38f) ? __fdiv_rn(y, ws) : y;
}

// grid (T, n): STFT of the re-synthesised signal for frame t, then the fast Griffin-Lim phase update
//   angles = rebuilt - momentum/(1+momentum) * tprev;  angles /= |angles| + tiny;  angles *= mag;  tprev = rebuilt
__global__ void __launch_bounds__(256, 5) gl_stft_update_kernel(const float* __restrict__ frames, const double2* __restrict__ tw,
                                                             const double* __restrict__ win, const float* __restrict__ wss,
                                                             const double* __restrict__ mag, double2* __restrict__ ang,
                                                             float2* __restrict__ tprev, int have_prev, MelDims d) {
  extern __shared__ __align__(16) uint8_t msm[];
  const int M = d.N >> 1;
  double2* a = reinterpret_cast<double2*>(msm);
  double2* b = a + M;
  const int t = blockIdx.x, n = blockIdx.y;
  const float* fr = frames + (size_t)n * d.T * d.N;
  const int p_lo = d.N / 2, p_hi = d.N / 2 + (d.T - 1) * d.hop;  // trimmed signal occupies padded [p_lo, p_hi)
  for (int j = threadIdx.x; j < M; j += blockDim.x) {
    const int p = t * d.hop + 2 * j;
    const double v0 = (p >= p_lo && p < p_hi) ? (double)ola_sample(fr, wss, p, d) : 0.0;
    const double v1 = (p + 1 >= p_lo && p + 1 < p_hi) ? (double)ola_sample(fr, wss, p + 1, d) : 0.0;
    a[j] = make_double2(v0 * win[2 * j], v1 * win[2 * j + 1]);
  }
  __syncthreads();
  const double2* Z = cfft<false>(a, b, tw, M, d.logN - 1);
  const double mom = 0.99 / 1.99;
  const size_t o0 = ((size_t)n * d.T + t) * d.F;
  auto update = [&](int f, double2 x) {
    const size_t o = o0 + f;
    const float2 rb = make_float2((float)x.x, (float)x.y);  // rebuilt is complex64
    double re = (double)rb.x, im = (double)rb.y;
    if (have_prev) {
      const float2 tp = tprev[o];
      re -= mom * (double)tp.x;
      im -= mom * (double)tp.y;
    }
    // angles / (|angles| + tiny) * mag: one fp64 rsqrt instead of hypot + two divisions (3/4 of this kernel's instructions);
    // |angles|^2 neither overflows nor underflows for complex64 inputs, and 0 / tiny = 0 in the reference too
    const double r2 = re * re + im * im;
    const double sc = r2 > 0.0 ? mag[o] * rsqrt(r2) : 0.0;
    ang[o] = make_double2(re * sc, im * sc);
    tprev[o] = rb;
  };
  for (int k = threadIdx.x; k <= M / 2; k += blockDim.x) {
    double2 xk, xm;
    rfft_pair(Z, tw, M, k, xk, xm);
    update(k, xk);
    if (2 * k != M) update(M - k, xm);
  }
}

__global__ void gl_out_kernel(const float* __restrict__ frames, const float* __restrict__ wss, float* __restrict__ audio, MelDims d) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = blockIdx.y;
  const int len = (d.T - 1) * d.hop;
  if (j >= len) return;
  audio[(size_t)n * len + j] = ola_sample(frames + (size_t)n * d.T * d.N, wss, j + d.N / 2, d);
}

static int mel_dims(const b200ad_mel_config* c, MelDims* d) {
  if (!c) return set_err("mel: null config");
  int logN = 0;
  while ((1 << logN) < c->n_fft) ++logN;
  if ((1 << logN) != c->n_fft || c->n_fft < 64 || c->n_fft > 4096) return set_err("mel: n_fft must be a power of two in [64, 4096]");
  if (c->hop_length <= 0 || c->hop_length > c->n_fft) return set_err("mel: hop_length out of range");
  d->T = c->x_res; d->M = c->y_res; d->N = c->n_fft; d->logN = logN; d->F = c->n_fft / 2 + 1; d->hop = c->hop_length;
  d->L = c->x_res * c->hop_length - 1;
  return 0;
}
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace b200ad
using namespace b200ad;

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (call);                                                         \
    if (e__ != cudaSuccess) return set_err("%s: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

extern "C" size_t b200ad_mel_scratch_bytes(const b200ad_mel_config* c, int n) {
  MelDims d;
  if (mel_dims(c, &d)) return 0;
  const size_t spec = (size_t)n * d.T * d.F;
  size_t b = al256((size_t)d.N * 16) + al256((size_t)d.N * 8) + al256((size_t)(d.N + (d.T - 1) * d.hop) * 4);   // twiddles, window, window sum-square
  const size_t enc = al256((size_t)n * d.M * d.T * 4) + al256((size_t)n * 4);
  const size_t dec = al256(spec * 8) + al256(spec * 16) + al256(spec * 8) + al256((size_t)n * d.T * d.N * 4);
  return b + (enc > dec ? enc : dec);
}

static int fft_smem_attr(const void* fn, size_t smem) {
  CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}

extern "C" int b200ad_mel_encode_ref(const b200ad_mel_config* c, const float* basis_t, const float* audio, uint8_t* images,
                                     int n, const float* ref_values, float* mel_power_out, void* scratch,
                                     size_t scratch_bytes, void* stream) {
  MelDims d;
  if (mel_dims(c, &d)) return -1;
  if (scratch_bytes < b200ad_mel_scratch_bytes(c, n)) return set_err("mel_encode: scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sb = (uint8_t*)scratch;
  double2* tw = (double2*)sb;
  sb += al256((size_t)d.N * 16);
  double* win = (double*)sb;
  sb += al256((size_t)d.N * 8);
  sb += al256((size_t)(d.N + (d.T - 1) * d.hop) * 4);
  float* mel = (float*)sb;
  sb += al256((size_t)n * d.M * d.T * 4);
  unsigned* smax = (unsigned*)sb;
  mel_tables_kernel<<<(d.N + 255) / 256, 256, 0, st>>>(tw, win, nullptr, d.N, d.T, d.hop);
  CK(cudaGetLastError());
  CK(cudaMemsetAsync(smax, 0, (size_t)n * 4, st));
  // two half-size complex buffers + the power spectrum, padded to 16 B (compute-sanitizer memcheck: the unrolled mel sum
  // reads the spectrum in 12 / 16-byte pieces and the last piece ran 8 bytes past an F * 4-byte allocation)
  const size_t smem = (size_t)d.N * 16 + (size_t)((d.F + 3) & ~3) * 4;
  if (fft_smem_attr((const void*)enc_frame_kernel, smem)) return -1;
  enc_frame_kernel<<<dim3(d.T, n), 256, smem, st>>>(audio, basis_t, tw, win, mel, smax, d);
  CK(cudaGetLastError());
  const int per = d.M * d.T;
  if (mel_power_out) CK(cudaMemcpyAsync(mel_power_out, mel, (size_t)n * per * 4, cudaMemcpyDeviceToDevice, st));
  if (images) {
    enc_db_kernel<<<dim3((per + 255) / 256, n), 256, 0, st>>>(mel, smax, ref_values, images, per, (float)c->top_db);
    CK(cudaGetLastError());
  }
  return 0;
}
extern "C" int b200ad_mel_encode(const b200ad_mel_config* c, const float* basis_t, const float* audio, uint8_t* images,
                                 int n, void* scratch, size_t scratch_bytes, void* stream) {
  if (!images) return set_err("mel_encode: images is null");
  return b200ad_mel_encode_ref(c, basis_t, audio, images, n, nullptr, nullptr, scratch, scratch_bytes, stream);
}

extern "C" int b200ad_mel_decode(const b200ad_mel_config* c, const double* pinv, const uint8_t* images, float* audio, int n,
                                 uint64_t phase_seed, void* scratch, size_t scratch_bytes, void* stream) {
  MelDims d;
  if (mel_dims(c, &d)) return -1;
  if (scratch_bytes < b200ad_mel_scratch_bytes(c, n)) return set_err("mel_decode: scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* sb = (uint8_t*)scratch;
  const size_t spec = (size_t)n * d.T * d.F;
  const int lpad = d.N + (d.T - 1) * d.hop;
  double2* tw = (double2*)sb;       sb += al256((size_t)d.N * 16);
  double* win = (double*)sb;        sb += al256((size_t)d.N * 8);
  float* wss = (float*)sb;          sb += al256((size_t)lpad * 4);
  double* mag = (double*)sb;        sb += al256(spec * 8);
  double2* ang = (double2*)sb;      sb += al256(spec * 16);
  float2* tprev = (float2*)sb;      sb += al256(spec * 8);
  float* frames = (float*)sb;
  mel_tables_kernel<<<(lpad + 255) / 256, 256, 0, st>>>(tw, win, wss, d.N, d.T, d.hop);
  CK(cudaGetLastError());
  dec_pinv_kernel<<<dim3((d.F + 63) / 64, (d.T + 63) / 64, n), 256, 0, st>>>(images, pinv, mag, ang, d, (double)c->top_db,
                                                                            phase_seed);
  CK(cudaGetLastError());
  const size_t smem = (size_t)d.N * 16;        // two half-size complex buffers
  if (fft_smem_attr((const void*)gl_istft_kernel, smem)) return -1;
  if (fft_smem_attr((const void*)gl_stft_update_kernel, smem)) return -1;
  for (int it = 0; it < c->n_iter; ++it) {
    gl_istft_kernel<<<dim3(d.T, n), 256, smem, st>>>(ang, tw, win, frames, d);
    CK(cudaGetLastError());
    gl_stft_update_kernel<<<dim3(d.T, n), 256, smem, st>>>(frames, tw, win, wss, mag, ang, tprev, it > 0 ? 1 : 0, d);
    CK(cudaGetLastError());
  }
  gl_istft_kernel<<<dim3(d.T, n), 256, smem, st>>>(ang, tw, win, frames, d);
  CK(cudaGetLastError());
  const int len = (d.T - 1) * d.hop;
  gl_out_kernel<<<dim3((len + 255) / 256, n), 256, 0, st>>>(frames, wss, audio, d);
  CK(cudaGetLastError());
  return 0;
}
