// Harmonic constant-Q front end, FP32 path.
//
// Replaces the first 213 nodes of the deployed graph (SURVEY.md Appendix A.1/A.2), i.e.
//   CQT2010v2.call        reference: basic_pitch/layers/nnaudio.py:623-661
//   get_cqt_complex       reference: basic_pitch/layers/nnaudio.py:216-256
//   downsampling_by_n     reference: basic_pitch/layers/nnaudio.py:259-284
//   NormalizedLog.call    reference: basic_pitch/layers/signal.py:171-185
//   BatchNormalization    reference: basic_pitch/models.py:188-189 (folded scalar affine)
// Kernels:
//   decimate_kernel  x_{o+1}[n] = sum_k LP[k] * x_o[2n + k - 127]           (4 launches + 1 tail launch per chunk)
//   cqt_kernel       frames(172) x taps(256) x 72 projection per octave, magnitude*sqrt(len),
//                    10*log10(p + 1e-10), per-window min/max (atomics)       (1 launch per chunk)
//   lognorm_kernel   (L - min) / (max - min) * bn_scale + bn_bias            (1 launch per chunk)
#include "kernels.cuh"

namespace bp {

// d.{x,y} += o * w.{x,y}: two FMAs whose tap pair is read from constant memory once (Hopper has no packed FP32 FMA)
__device__ __forceinline__ void ffma2(float2& d, float o, float2 w) {
  d.x = fmaf(o, w.x, d.x);
  d.y = fmaf(o, w.y, d.y);
}

// Low-pass taps as pairs: t[k] = (h[k - 12], h[k - 14]), zero outside the 256 taps.  A thread that owns outputs
// 8t .. 8t+7 feeds sample u of its input run into the output pairs (0,1), (2,3), (4,5), (6,7) with t[u + 12],
// t[u + 8], t[u + 4], t[u].
Lowpass2 lowpass_pairs(const float* h_lp) {
  Lowpass2 lp;
  for (int k = 0; k < kLp2; ++k) {
    const int u = k - 12;
    lp.t[k].x = (u >= 0 && u < kTaps) ? h_lp[u] : 0.f;
    lp.t[k].y = (u - 2 >= 0 && u - 2 < kTaps) ? h_lp[u - 2] : 0.f;
  }
  return lp;
}

// ------------------------------------------------------------------------------------------------
// Half-band FIR + decimate by 2:  x_{o+1}[n] = sum_k LP[k] * x_o[2n + k - 127].
// Input runs live in shared memory de-interleaved into 16 phases (sample li at ph[(li & 15) * S + (li >> 4)], S == 2
// mod 32: conflict-free scatter and gather); thread t owns outputs 8t .. 8t+7, so every loaded sample feeds up to 8
// FMAs whose tap pairs are uniform-register operands from the kernel parameters (constant bank 0; fir8 reads them
// through a reference to the __grid_constant__ parameter, so they are never copied).  Each output still accumulates its
// 256 products in tap order.
//   decimate_kernel       stages 0-3: one CTA = 1024 outputs of one window
//   decimate_tail_kernel  stages 4-7 (2740 -> 171 samples): one CTA per window runs the four stages back to back through
//                         shared memory (as four launches they were latency-bound: 25 % of the chain's time for 6 % of
//                         its work)
// ------------------------------------------------------------------------------------------------
template <int S>
__device__ __forceinline__ void fir8(const Lowpass2& lp, const float* __restrict__ ph, int t, float (&out)[8]) {
  float2 a01 = make_float2(0.f, 0.f), a23 = a01, a45 = a01, a67 = a01;
#pragma unroll
  for (int u = 0; u < kLp2; ++u) {
    const float v = ph[(u & 15) * S + t + (u >> 4)];
    if (u < kTaps + 2) ffma2(a01, v, lp.t[u + 12]);
    if (u >= 4 && u < kTaps + 6) ffma2(a23, v, lp.t[u + 8]);
    if (u >= 8 && u < kTaps + 10) ffma2(a45, v, lp.t[u + 4]);
    if (u >= 12) ffma2(a67, v, lp.t[u]);
  }
  out[0] = a01.x, out[1] = a01.y, out[2] = a23.x, out[3] = a23.y;
  out[4] = a45.x, out[5] = a45.y, out[6] = a67.x, out[7] = a67.y;
}

constexpr int kDecTile = 1024;
constexpr int kDecThreads = 128;
constexpr int kDecS = 162;  // positions per phase: (2 * 1024 + 270) / 16 = 145 -> next value == 2 (mod 32)

__global__ void __launch_bounds__(kDecThreads) decimate_kernel(const __grid_constant__ Lowpass2 lp,
                                                               const float* __restrict__ audio,
                                                               const WinDesc* __restrict__ desc,  // stage 0 only
                                                               const float* __restrict__ src,     // chain, stage >= 1
                                                               float* __restrict__ dst, int src_off, int dst_off,
                                                               int len_in, int len_out, int from_audio) {
  __shared__ float ph[16 * kDecS];
  const int b = blockIdx.y;
  const int n0 = blockIdx.x * kDecTile;
  const int gbase = 2 * n0 - 127;  // input index of local index 0
  constexpr int kLocal = 2 * kDecTile + 272;  // local inputs staged (multiple of 16)

  const float* s;
  int lo = 0, hi = len_in;
  if (from_audio) {
    if (desc) {
      const WinDesc d = desc[b];
      s = audio + d.base;
      lo = d.lo;
      hi = d.hi;
    } else {
      s = audio + (long long)b * kWinSamples;
      hi = kWinSamples;
    }
  } else {
    s = src + (size_t)b * kChainStride + src_off;
  }
  for (int li = threadIdx.x; li < kLocal; li += kDecThreads) {
    const int gi = gbase + li;
    ph[(li & 15) * kDecS + (li >> 4)] = (gi >= lo && gi < hi) ? __ldg(s + gi) : 0.f;
  }
  __syncthreads();

  const int t = threadIdx.x;
  const int n = n0 + 8 * t;
  if (n >= len_out) return;
  float o[8];
  fir8<kDecS>(lp, ph, t, o);
  float* d = dst + (size_t)b * kChainStride + dst_off;
  if (n + 7 < len_out) {
    *reinterpret_cast<float4*>(d + n) = make_float4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<float4*>(d + n + 4) = make_float4(o[4], o[5], o[6], o[7]);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (n + i < len_out) d[n + i] = o[i];
  }
}

constexpr int kTailFirst = 4;     // the tail kernel runs stages 4 .. 7
constexpr int kTailThreads = 256;
constexpr int kTailS = 194;       // (2740 + 127 + 270) / 16 = 197 positions would be needed for reads past the last output's run;
                                  // active threads (8t < 1370) read positions <= 171 + 16, 194 == 2 (mod 32)

__global__ void __launch_bounds__(kTailThreads) decimate_tail_kernel(const __grid_constant__ Lowpass2 lp,
                                                                     float* __restrict__ chain) {
  __shared__ float buf[2][16 * kTailS];
  float* c = chain + (size_t)blockIdx.x * kChainStride;
  const int tid = threadIdx.x;
  {
    const float* s = c + chain_off(kTailFirst);
    const int len = octave_len(kTailFirst);
    for (int li = tid; li < 16 * kTailS; li += kTailThreads) {
      const int gi = li - 127;
      buf[0][(li & 15) * kTailS + (li >> 4)] = (gi >= 0 && gi < len) ? s[gi] : 0.f;
    }
  }
  int cur = 0;
#pragma unroll 1
  for (int stage = kTailFirst; stage < 8; ++stage) {
    const int len_out = octave_len_rt(stage + 1);
    float* nxt = buf[cur ^ 1];
    for (int i = tid; i < 16 * kTailS; i += kTailThreads) nxt[i] = 0.f;
    __syncthreads();  // cur is complete, nxt is zero
    const int n = 8 * tid;
    if (n < len_out) {
      float o[8];
      fir8<kTailS>(lp, buf[cur], tid, o);
      float* d = c + chain_off_rt(stage + 1);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (n + i < len_out) {
          d[n + i] = o[i];
          const int li = n + i + 127;  // local index of this sample in the next stage's input run
          nxt[(li & 15) * kTailS + (li >> 4)] = o[i];
        }
    }
    cur ^= 1;
    __syncthreads();
  }
}

void launch_decimate(const Lowpass2& lp, const float* audio, const WinDesc* desc, float* chain, int stage, int n_windows,
                     cudaStream_t st) {
  if (stage > kTailFirst) return;  // done by the tail launch
  if (stage == kTailFirst) {
    decimate_tail_kernel<<<n_windows, kTailThreads, 0, st>>>(lp, chain);
    return;
  }
  // stage s: x_s -> x_{s+1}
  const int len_in = octave_len(stage), len_out = octave_len(stage + 1);
  dim3 grid((len_out + kDecTile - 1) / kDecTile, n_windows);
  decimate_kernel<<<grid, kDecThreads, 0, st>>>(lp, audio, desc, chain, chain, stage ? chain_off(stage) : 0,
                                                 chain_off(stage + 1), len_in, len_out, stage == 0);
}

// ------------------------------------------------------------------------------------------------
// CQT projection of one (window, octave): C[t][n] = sum_k xpad[t*hop + k] * W[k][n], t < 172,
// n < 72 (columns interleave real/imag of the 36 bins), reflect padding of 128 each side.
// 288 threads; thread (ty, tx) accumulates frames {ty, ty+43, ty+86, ty+129} x columns 12tx..12tx+11.
// K is consumed in chunks of 64 staged through shared memory (A gathered through the reflect map).
// Epilogue: magnitude * sqrt(len_k), power, 10*log10(p + 1e-10), block min/max -> atomics.
// ------------------------------------------------------------------------------------------------
constexpr int kCqtThreads = 288;
constexpr int kCqtKc = 64;
constexpr int kCqtApad = kCqtKc + 1;
constexpr int kCqtCols = 72;

__global__ void __launch_bounds__(kCqtThreads) cqt_kernel(const float* __restrict__ audio,
                                                          const WinDesc* __restrict__ desc,
                                                          const float* __restrict__ chain,
                                                          const float* __restrict__ wt,     // [256][72]
                                                          const float* __restrict__ scale,  // [309]
                                                          float* __restrict__ logmag,       // [B][172][309]
                                                          unsigned int* __restrict__ minmax /* [B][2] */) {
  extern __shared__ float smem[];
  float* As = smem;                       // [172][65]
  float* Ws = smem + kFrames * kCqtApad;  // [64][72]
  __shared__ float red_min[kCqtThreads / 32], red_max[kCqtThreads / 32];

  const int b = blockIdx.y;
  const int o = blockIdx.x;  // octave, 0 = top
  const int hop = 256 >> o;
  const int len = octave_len_rt(o);

  long long base = 0;
  int lo = 0, hi = len;
  const float* src;
  if (o == 0) {
    if (desc) {
      WinDesc d = desc[b];
      base = d.base;
      lo = d.lo;
      hi = d.hi;
    } else {
      base = (long long)b * kWinSamples;
    }
    src = audio;
  } else {
    src = chain + (size_t)b * kChainStride + chain_off_rt(o);
  }

  const int tid = threadIdx.x;
  const bool active = tid < 258;
  const int ty = active ? tid / 6 : 0;
  const int tx = active ? tid % 6 : 0;

  float acc[4][12];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 12; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < kTaps; k0 += kCqtKc) {
    __syncthreads();
    for (int e = tid; e < kFrames * kCqtKc; e += kCqtThreads) {
      int t = e >> 6, kk = e & 63;
      int idx = t * hop + k0 + kk - 128;
      if (idx < 0) idx = -idx;
      if (idx >= len) idx = 2 * (len - 1) - idx;
      float v = (idx >= lo && idx < hi) ? __ldg(src + base + idx) : 0.f;
      As[t * kCqtApad + kk] = v;
    }
    for (int e = tid; e < kCqtKc * kCqtCols / 4; e += kCqtThreads)
      reinterpret_cast<float4*>(Ws)[e] = __ldg(reinterpret_cast<const float4*>(wt + k0 * kCqtCols) + e);
    __syncthreads();
    if (active) {
#pragma unroll 4
      for (int kk = 0; kk < kCqtKc; ++kk) {
        float a[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[(ty + 43 * i) * kCqtApad + kk];
        const float4* wp = reinterpret_cast<const float4*>(Ws + kk * kCqtCols + 12 * tx);
        float4 w0 = wp[0], w1 = wp[1], w2 = wp[2];
        float w[12] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 12; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
      }
    }
  }

  float vmin = INFINITY, vmax = -INFINITY;
  if (active) {
#pragma unroll
    for (int jb = 0; jb < 6; ++jb) {
      int g = (8 - o) * kBinsPerOctave + 6 * tx + jb - 15;
      if (g < 0) continue;
      float s = __ldg(scale + g);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float re = __fmul_rn(acc[i][2 * jb], s), im = __fmul_rn(acc[i][2 * jb + 1], s);
        float mag = sqrtf(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)));
        float p = __fadd_rn(__fmul_rn(mag, mag), 1e-10f);
        float L = __fmul_rn(__fmul_rn(logf(p), 0.4342944622039795f), 10.0f);
        logmag[((size_t)b * kFrames + ty + 43 * i) * kCqtBins + g] = L;
        vmin = fminf(vmin, L);
        vmax = fmaxf(vmax, L);
      }
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, off));
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, off));
  }
  if ((tid & 31) == 0) {
    red_min[tid >> 5] = vmin;
    red_max[tid >> 5] = vmax;
  }
  __syncthreads();
  if (tid == 0) {
    for (int i = 1; i < kCqtThreads / 32; ++i) {
      vmin = fminf(vmin, red_min[i]);
      vmax = fmaxf(vmax, red_max[i]);
    }
    atomicMin(minmax + 2 * b, float_to_ordered(vmin));
    atomicMax(minmax + 2 * b + 1, float_to_ordered(vmax));
  }
}

__global__ void minmax_init_kernel(unsigned int* mm, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    mm[2 * i] = 0xffffffffu;
    mm[2 * i + 1] = 0u;
  }
}

// per-device opt-in to > 48 KB of dynamic shared memory (called from bp_model_create under the device guard)
void hcqt_setup() {
  cudaFuncSetAttribute(cqt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                       (int)((kFrames * kCqtApad + kCqtKc * kCqtCols) * sizeof(float)));
}

void launch_cqt(const float* audio, const WinDesc* desc, const float* chain, const float* wt, const float* scale,
                float* logmag, unsigned int* minmax, int n_windows, cudaStream_t st) {
  const int smem = (kFrames * kCqtApad + kCqtKc * kCqtCols) * sizeof(float);
  minmax_init_kernel<<<(n_windows + 255) / 256, 256, 0, st>>>(minmax, n_windows);
  cqt_kernel<<<dim3(kOctaves, n_windows), kCqtThreads, smem, st>>>(audio, desc, chain, wt, scale, logmag, minmax);
}

// ------------------------------------------------------------------------------------------------
// Per-window normalisation + folded BatchNorm, in place.
// ------------------------------------------------------------------------------------------------
__global__ void lognorm_kernel(float* __restrict__ y, const unsigned int* __restrict__ minmax,
                               const float* __restrict__ bn) {
  const int b = blockIdx.y;
  const float bn_scale = __ldg(bn), bn_bias = __ldg(bn + 1);
  const float mn = ordered_to_float(minmax[2 * b]);
  const float mx = __fsub_rn(ordered_to_float(minmax[2 * b + 1]), mn);
  float* p = y + (size_t)b * kFrames * kCqtBins;
  const int n = kFrames * kCqtBins;  // 53148 = 4 * 13287
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n / 4; i += gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(p)[i];
    float* e = reinterpret_cast<float*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float q = (mx == 0.f) ? 0.f : __fdiv_rn(__fsub_rn(e[j], mn), mx);
      e[j] = __fadd_rn(__fmul_rn(q, bn_scale), bn_bias);
    }
    reinterpret_cast<float4*>(p)[i] = v;
  }
}

void launch_lognorm(float* y, const unsigned int* minmax, const float* bn, int n_windows, cudaStream_t st) {
  lognorm_kernel<<<dim3(13, n_windows), 256, 0, st>>>(y, minmax, bn);
}

}  // namespace bp
