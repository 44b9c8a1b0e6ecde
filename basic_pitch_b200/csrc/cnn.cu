// Convolution stack: the FP32 FFMA kernels (path 0: accuracy reference on device; path 2 uses the channels-last
// contour conv2 below).  On the default path the second convolutions are fused into the epilogues of the tensor-core
// kernels (tc_conv.cu).
//
// Replaces nodes 213-247 of the deployed graph (SURVEY.md Appendix A.2/A.3):
//   HarmonicStacking.call   reference: basic_pitch/nn.py:69-88   (never materialised: the 8 "channels"
//                           are shifted, zero-gated views of the normalised CQT, see StackIn)
//   conv stack              reference: basic_pitch/models.py:241-318 (BatchNorm folded, as exported)
//
// conv_kernel: one generic direct-convolution kernel.  A CTA produces a tile of TT frames x FT=FL*P bins for all
// COUT channels of one window; the input patch and the (transposed) weights are staged in shared
// memory.  Thread (cg, tl, fl) owns COB output channels x P bins {fl + FL*p}: lanes walk consecutive
// bins (conflict-free for stride 1 and 3), every loaded input feeds COB FMAs, weights are warp-uniform
// float4 broadcasts.
// conv1_kernel: the C_out = 1 convolutions with a 4 x 4 register tile per thread (planar or channels-last input).
#include "kernels.cuh"

namespace bp {

__constant__ int c_shift[kHarmonics] = {-36, 0, 36, 57, 72, 84, 93, 101};

// Harmonic stack as a view of y[B][172][309]:  H[ci][t][g] = y[t][g + shift_ci] for 0<=g<264 and
// 0 <= g+shift < 309, else 0 (zeros are inserted AFTER BatchNorm, SURVEY.md Appendix A.2).
struct StackIn {
  static constexpr bool kChannelsLast = false;
  const float* y;
  __device__ __forceinline__ float load(int b, int ci, int t, int g) const {
    if ((unsigned)t >= (unsigned)kFrames || (unsigned)g >= (unsigned)kContourBins) return 0.f;
    int gi = g + c_shift[ci];
    if ((unsigned)gi >= (unsigned)kCqtBins) return 0.f;
    return __ldg(y + ((size_t)b * kFrames + t) * kCqtBins + gi);
  }
};
template <int C, int W>
struct PlanarIn {
  static constexpr bool kChannelsLast = false;
  const float* p;  // [B][C][172][W]
  __device__ __forceinline__ float load(int b, int ci, int t, int g) const {
    if ((unsigned)t >= (unsigned)kFrames || (unsigned)g >= (unsigned)W) return 0.f;
    return __ldg(p + (((size_t)b * C + ci) * kFrames + t) * W + g);
  }
};
// channels-last activations [B][172][W][C] (what the tensor-core contour kernel writes)
template <int C, int W>
struct NhwcIn {
  static constexpr bool kChannelsLast = true;
  const float* p;
  __device__ __forceinline__ float load(int b, int ci, int t, int g) const {
    if ((unsigned)t >= (unsigned)kFrames || (unsigned)g >= (unsigned)W) return 0.f;
    return __ldg(p + (((size_t)b * kFrames + t) * W + g) * C + ci);
  }
  __device__ __forceinline__ float4 load4(int b, int c4, int t, int g) const {
    if ((unsigned)t >= (unsigned)kFrames || (unsigned)g >= (unsigned)W) return make_float4(0.f, 0.f, 0.f, 0.f);
    return __ldg(reinterpret_cast<const float4*>(p + (((size_t)b * kFrames + t) * W + g) * C + c4));
  }
};
// channel 0 = note posteriorgram [B][172][88], channels 1..32 = onset conv1 output [B][32][172][88]
struct ConcatIn {
  static constexpr bool kChannelsLast = false;
  const float* note;
  const float* o1;
  __device__ __forceinline__ float load(int b, int ci, int t, int g) const {
    if ((unsigned)t >= (unsigned)kFrames || (unsigned)g >= (unsigned)kPitches) return 0.f;
    if (ci == 0) return __ldg(note + ((size_t)b * kFrames + t) * kPitches + g);
    return __ldg(o1 + (((size_t)b * 32 + (ci - 1)) * kFrames + t) * kPitches + g);
  }
};

enum { ACT_RELU = 0, ACT_SIGMOID = 1 };

template <int CIN_, int CIC_, int COUT_, int COB_, int KH_, int KW_, int SF_, int PT_, int PL_, int WOUT_, int TT_,
          int FL_, int P_, int ACT_>
struct ConvCfg {
  static constexpr int CIN = CIN_, CIC = CIC_, COUT = COUT_, COB = COB_, KH = KH_, KW = KW_, SF = SF_, PT = PT_,
                       PL = PL_, WOUT = WOUT_, TT = TT_, FL = FL_, P = P_, ACT = ACT_;
  static constexpr int FT = FL * P;
  static constexpr int CG = COUT / COB;
  static constexpr int THREADS = FL * TT * CG;
  static constexpr int NEED = (FT - 1) * SF + KW;
  // row stride == FL*SF (mod 32) so that a warp spanning two frame rows stays conflict-free
  static constexpr int RS = NEED + ((((FL * SF - NEED) % 32) + 32) % 32);
  static constexpr int ROWS = TT + KH - 1;
  static constexpr int IN_ELEMS = CIC * ROWS * RS;
  static constexpr int W_ELEMS = CIC * KH * KW * COUT;
  static constexpr int SMEM_BYTES = (IN_ELEMS + W_ELEMS) * 4;
  static constexpr int FTILES = (WOUT + FT - 1) / FT;
  static constexpr int TTILES = (kFrames + TT - 1) / TT;
  static_assert(COUT % COB == 0 && CIN % CIC == 0, "channel blocking");
  static_assert(COB == 1 || COB % 4 == 0, "COB must be 1 or a multiple of 4");
};

template <class Cfg, class In>
__global__ void __launch_bounds__(Cfg::THREADS, 1) conv_kernel(In in, const float* __restrict__ wT,
                                                            const float* __restrict__ bias,
                                                            float* __restrict__ out) {
  extern __shared__ float smem[];
  float* in_s = smem;
  float* w_s = smem + Cfg::IN_ELEMS;

  const int b = blockIdx.y;
  const int ftile = blockIdx.x % Cfg::FTILES;
  const int ttile = blockIdx.x / Cfg::FTILES;
  const int f0 = ftile * Cfg::FT;
  const int t0 = ttile * Cfg::TT;

  const int tid = threadIdx.x;
  const int fl = tid % Cfg::FL;
  const int tl = (tid / Cfg::FL) % Cfg::TT;
  const int cg = tid / (Cfg::FL * Cfg::TT);

  float acc[Cfg::P][Cfg::COB];
#pragma unroll
  for (int p = 0; p < Cfg::P; ++p)
#pragma unroll
    for (int j = 0; j < Cfg::COB; ++j) acc[p][j] = 0.f;

  for (int c0 = 0; c0 < Cfg::CIN; c0 += Cfg::CIC) {
    if (c0) __syncthreads();
    // stage the input patch: rows t0-PT .. t0-PT+ROWS-1, columns f0*SF-PL .. +NEED-1
    for (int e = tid; e < Cfg::CIC * Cfg::ROWS * Cfg::NEED; e += Cfg::THREADS) {
      int x = e % Cfg::NEED;
      int r = (e / Cfg::NEED) % Cfg::ROWS;
      int c = e / (Cfg::NEED * Cfg::ROWS);
      in_s[(c * Cfg::ROWS + r) * Cfg::RS + x] = in.load(b, c0 + c, t0 - Cfg::PT + r, f0 * Cfg::SF - Cfg::PL + x);
    }
    for (int e = tid; e < Cfg::W_ELEMS; e += Cfg::THREADS) w_s[e] = __ldg(wT + c0 * Cfg::KH * Cfg::KW * Cfg::COUT + e);
    __syncthreads();

#pragma unroll 1
    for (int c = 0; c < Cfg::CIC; ++c) {
#pragma unroll 1
      for (int dt = 0; dt < Cfg::KH; ++dt) {
        const float* row = in_s + (c * Cfg::ROWS + tl + dt) * Cfg::RS + fl * Cfg::SF;
        const float* wrow = w_s + ((c * Cfg::KH + dt) * Cfg::KW) * Cfg::COUT + cg * Cfg::COB;
#pragma unroll
        for (int df = 0; df < Cfg::KW; ++df) {
          float w[Cfg::COB];
          if constexpr (Cfg::COB == 1) {
            w[0] = wrow[df * Cfg::COUT];
          } else {
#pragma unroll
            for (int q = 0; q < Cfg::COB / 4; ++q) {
              float4 v = *reinterpret_cast<const float4*>(wrow + df * Cfg::COUT + 4 * q);
              w[4 * q] = v.x;
              w[4 * q + 1] = v.y;
              w[4 * q + 2] = v.z;
              w[4 * q + 3] = v.w;
            }
          }
#pragma unroll
          for (int p = 0; p < Cfg::P; ++p) {
            float v = row[p * Cfg::FL * Cfg::SF + df];
#pragma unroll
            for (int j = 0; j < Cfg::COB; ++j) acc[p][j] = fmaf(v, w[j], acc[p][j]);
          }
        }
      }
    }
  }

  const int t = t0 + tl;
  if (t < kFrames) {
#pragma unroll
    for (int j = 0; j < Cfg::COB; ++j) {
      const int co = cg * Cfg::COB + j;
      const float bv = __ldg(bias + co);
#pragma unroll
      for (int p = 0; p < Cfg::P; ++p) {
        const int f = f0 + fl + Cfg::FL * p;
        if (f < Cfg::WOUT) {
          float v = acc[p][j] + bv;
          if (Cfg::ACT == ACT_RELU)
            v = fmaxf(v, 0.f);
          else
            v = 1.f / (1.f + expf(-v));
          out[(((size_t)b * Cfg::COUT + co) * kFrames + t) * Cfg::WOUT + f] = v;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Single-output-channel convolutions (contour2 8->1 5x5, note2 32->1 7x3, onset2 33->1 3x3) + sigmoid.
// With one output channel there is no channel blocking to amortise input loads, so each thread owns a
// 4 frames x 4 bins register tile and keeps the (4+KH-1) x (4+KW-1) input patch of the current channel in
// registers: every shared-memory load feeds up to KH*KW*16/patch FMAs.  The patch columns of a thread are
// contiguous, so rows are stored de-interleaved into 4 phases (x -> [x & 3][x >> 2]) to keep lanes on
// consecutive words.  Weights are warp-uniform broadcast loads from shared memory.
// ------------------------------------------------------------------------------------------------
template <int CIN_, int CIC_, int KH_, int KW_, int PT_, int PL_, int WOUT_, int TR_>
struct Conv1Cfg {
  static constexpr int CIN = CIN_, CIC = CIC_, KH = KH_, KW = KW_, PT = PT_, PL = PL_, WOUT = WOUT_, TR = TR_;
  static constexpr int Q = 4, P = 4, FL = 22, FT = FL * P;       // 88 bins per tile
  static constexpr int TT = TR * Q;                             // frames per tile
  static constexpr int THREADS = FL * TR;
  static constexpr int ROWS = TT + KH - 1;
  static constexpr int NEED = FT + KW - 1;
  static constexpr int PH = (NEED + 3) / 4 + 1;                 // words per phase
  static constexpr int RS = 4 * PH;
  static constexpr int IN_ELEMS = CIC * ROWS * RS;
  static constexpr int W_ELEMS = CIN * KH * KW;
  static constexpr int SMEM_BYTES = (IN_ELEMS + W_ELEMS) * 4;
  static constexpr int FTILES = (WOUT + FT - 1) / FT;
  static constexpr int TTILES = (kFrames + TT - 1) / TT;
  static_assert(CIN % CIC == 0, "channel blocking");
};

struct SplitOut {           // optional bf16 hi/lo copy of the output in the tensor-core row layout (tc_conv.cu)
  __nv_bfloat16* planes;    // [2][chunks8][rows_total][8]; nullptr = off
  int rows_total, chunks8, rows_per_window, lead;
};

template <class Cfg, class In>
__global__ void __launch_bounds__(Cfg::THREADS) conv1_kernel(In in, const float* __restrict__ w /* [CIN*KH*KW] */,
                                                             const float* __restrict__ bias,
                                                             float* __restrict__ out /* [B][172][WOUT] */,
                                                             SplitOut so) {
  extern __shared__ float smem[];
  float* in_s = smem;
  float* w_s = smem + Cfg::IN_ELEMS;
  const int b = blockIdx.y;
  const int ftile = blockIdx.x % Cfg::FTILES, ttile = blockIdx.x / Cfg::FTILES;
  const int f0 = ftile * Cfg::FT, t0 = ttile * Cfg::TT;
  const int tid = threadIdx.x;
  const int fp = tid % Cfg::FL, tq = tid / Cfg::FL;

  for (int e = tid; e < Cfg::W_ELEMS; e += Cfg::THREADS) w_s[e] = __ldg(w + e);

  float acc[Cfg::Q][Cfg::P];
#pragma unroll
  for (int q = 0; q < Cfg::Q; ++q)
#pragma unroll
    for (int p = 0; p < Cfg::P; ++p) acc[q][p] = 0.f;

  for (int c0 = 0; c0 < Cfg::CIN; c0 += Cfg::CIC) {
    __syncthreads();
    if constexpr (In::kChannelsLast) {
      // channels-last input: every tile row is one contiguous run of NEED x CIN floats -> float4 loads
      static_assert(Cfg::CIC % 4 == 0, "channels-last staging moves float4 groups of channels");
      constexpr int V = Cfg::CIC / 4;
      for (int e = tid; e < Cfg::ROWS * Cfg::NEED * V; e += Cfg::THREADS) {
        const int c4 = (e % V) * 4;
        const int x = (e / V) % Cfg::NEED;
        const int r = e / (V * Cfg::NEED);
        const float4 v = in.load4(b, c0 + c4, t0 - Cfg::PT + r, f0 - Cfg::PL + x);
        float* d = in_s + (c4 * Cfg::ROWS + r) * Cfg::RS + (x & 3) * Cfg::PH + (x >> 2);
        d[0] = v.x;
        d[Cfg::ROWS * Cfg::RS] = v.y;
        d[2 * Cfg::ROWS * Cfg::RS] = v.z;
        d[3 * Cfg::ROWS * Cfg::RS] = v.w;
      }
    } else {
      for (int e = tid; e < Cfg::CIC * Cfg::ROWS * Cfg::NEED; e += Cfg::THREADS) {
        const int x = e % Cfg::NEED;
        const int r = (e / Cfg::NEED) % Cfg::ROWS;
        const int c = e / (Cfg::NEED * Cfg::ROWS);
        in_s[(c * Cfg::ROWS + r) * Cfg::RS + (x & 3) * Cfg::PH + (x >> 2)] =
            in.load(b, c0 + c, t0 - Cfg::PT + r, f0 - Cfg::PL + x);
      }
    }
    __syncthreads();
#pragma unroll 1
    for (int c = 0; c < Cfg::CIC; ++c) {
      float patch[Cfg::Q + Cfg::KH - 1][Cfg::P + Cfg::KW - 1];
      const float* base = in_s + (c * Cfg::ROWS + tq * Cfg::Q) * Cfg::RS + fp;
#pragma unroll
      for (int r = 0; r < Cfg::Q + Cfg::KH - 1; ++r)
#pragma unroll
        for (int j = 0; j < Cfg::P + Cfg::KW - 1; ++j) patch[r][j] = base[r * Cfg::RS + (j & 3) * Cfg::PH + (j >> 2)];
      const float* wc = w_s + (c0 + c) * Cfg::KH * Cfg::KW;
#pragma unroll
      for (int dt = 0; dt < Cfg::KH; ++dt)
#pragma unroll
        for (int df = 0; df < Cfg::KW; ++df) {
          const float wv = wc[dt * Cfg::KW + df];
#pragma unroll
          for (int q = 0; q < Cfg::Q; ++q)
#pragma unroll
            for (int p = 0; p < Cfg::P; ++p) acc[q][p] = fmaf(wv, patch[q + dt][p + df], acc[q][p]);
        }
    }
  }
  const float bv = __ldg(bias);
#pragma unroll
  for (int q = 0; q < Cfg::Q; ++q) {
    const int t = t0 + tq * Cfg::Q + q;
    const int f = f0 + fp * Cfg::P;
    if (t < kFrames && f < Cfg::WOUT) {
      float4 o;
      o.x = 1.f / (1.f + expf(-(acc[q][0] + bv)));
      o.y = 1.f / (1.f + expf(-(acc[q][1] + bv)));
      o.z = 1.f / (1.f + expf(-(acc[q][2] + bv)));
      o.w = 1.f / (1.f + expf(-(acc[q][3] + bv)));
      *reinterpret_cast<float4*>(out + ((size_t)b * kFrames + t) * Cfg::WOUT + f) = o;
      if (so.planes) {  // hi/lo bf16 split for the tensor-core consumer: 4 bins = half of an 8-bin chunk
        const float ov[4] = {o.x, o.y, o.z, o.w};
        __align__(8) __nv_bfloat16 hi[4], lo[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          hi[j] = __float2bfloat16_rn(ov[j]);
          lo[j] = __float2bfloat16_rn(ov[j] - __bfloat162float(hi[j]));
        }
        const size_t d = (size_t)so.lead + (size_t)b * so.rows_per_window + t;
        const size_t off = ((size_t)(f >> 3) * so.rows_total + d) * 8 + (f & 7);
        const size_t plane = (size_t)so.chunks8 * so.rows_total * 8;
        *reinterpret_cast<uint2*>(so.planes + off) = *reinterpret_cast<const uint2*>(hi);
        *reinterpret_cast<uint2*>(so.planes + plane + off) = *reinterpret_cast<const uint2*>(lo);
      }
    }
  }
}

//                           CIN CIC KH KW PT PL WOUT TR
using Contour2Cfg1 = Conv1Cfg<8, 4, 5, 5, 2, 2, 264, 11>;
using Contour2CfgN = Conv1Cfg<8, 4, 5, 5, 2, 2, 264, 11>;  // channels-last input, two passes of 4 channels
using Note2Cfg1 = Conv1Cfg<32, 4, 7, 3, 3, 1, 88, 11>;
using Onset2Cfg1 = Conv1Cfg<33, 3, 3, 3, 1, 1, 88, 11>;

//                         CIN CIC COUT COB KH  KW SF PT PL  WOUT TT  FL P  ACT
using Contour1Cfg = ConvCfg<8, 8, 8, 8, 3, 39, 1, 1, 19, 264, 12, 22, 4, ACT_RELU>;
using Note1Cfg = ConvCfg<1, 1, 32, 8, 7, 7, 3, 3, 2, 88, 4, 22, 4, ACT_RELU>;
using Onset1Cfg = ConvCfg<8, 8, 32, 8, 5, 5, 3, 2, 1, 88, 4, 22, 4, ACT_RELU>;

template <class Cfg, class In>
static void set_attr() {
  cudaFuncSetAttribute(conv_kernel<Cfg, In>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
}

template <class Cfg, class In>
static void set_attr1() {
  cudaFuncSetAttribute(conv1_kernel<Cfg, In>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES);
}
template <class Cfg, class In>
static void launch1(In in, const float* w, const float* bias, float* out, int n_windows, cudaStream_t st,
                    SplitOut so = SplitOut{nullptr, 0, 0, 0, 0}) {
  dim3 grid(Cfg::FTILES * Cfg::TTILES, n_windows);
  conv1_kernel<Cfg, In><<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(in, w, bias, out, so);
}

void cnn_setup() {
  set_attr1<Contour2Cfg1, PlanarIn<8, 264>>();
  set_attr1<Contour2CfgN, NhwcIn<8, 264>>();
  set_attr1<Note2Cfg1, PlanarIn<32, 88>>();
  set_attr1<Onset2Cfg1, ConcatIn>();
  set_attr<Contour1Cfg, StackIn>();
  set_attr<Note1Cfg, PlanarIn<1, 264>>();
  set_attr<Onset1Cfg, StackIn>();
}

template <class Cfg, class In>
static void launch(In in, const float* wT, const float* bias, float* out, int n_windows, cudaStream_t st) {
  dim3 grid(Cfg::FTILES * Cfg::TTILES, n_windows);
  conv_kernel<Cfg, In><<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(in, wT, bias, out);
}

void launch_contour1(const float* y, const CnnWeights& w, float* c1, int n, cudaStream_t st) {
  launch<Contour1Cfg>(StackIn{y}, w.contour1_wT, w.contour1_b, c1, n, st);
}
void launch_contour2(const float* c1, const CnnWeights& w, float* contour, int n, cudaStream_t st) {
  launch1<Contour2Cfg1>(PlanarIn<8, 264>{c1}, w.contour2_wT, w.contour2_b, contour, n, st);
}
void launch_contour2_tc(const float* c1, const CnnWeights& w, float* contour, __nv_bfloat16* chl, int rows_total, int n,
                        cudaStream_t st) {
  constexpr TcConvSpec sp = tc_spec(2);  // the note conv reads the contour posteriorgram
  launch1<Contour2CfgN>(NhwcIn<8, 264>{c1}, w.contour2_wT, w.contour2_b, contour, n, st,
                        SplitOut{chl, rows_total, sp.chunks8, sp.rows_per_window, sp.lead_rows});
}
void launch_note1(const float* contour, const CnnWeights& w, float* n1, int n, cudaStream_t st) {
  launch<Note1Cfg>(PlanarIn<1, 264>{contour}, w.note1_wT, w.note1_b, n1, n, st);
}
void launch_note2(const float* n1, const CnnWeights& w, float* note, int n, cudaStream_t st) {
  launch1<Note2Cfg1>(PlanarIn<32, 88>{n1}, w.note2_wT, w.note2_b, note, n, st);
}
void launch_onset1(const float* y, const CnnWeights& w, float* o1, int n, cudaStream_t st) {
  launch<Onset1Cfg>(StackIn{y}, w.onset1_wT, w.onset1_b, o1, n, st);
}
void launch_onset2(const float* note, const float* o1, const CnnWeights& w, float* onset, int n, cudaStream_t st) {
  launch1<Onset2Cfg1>(ConcatIn{note, o1}, w.onset2_wT, w.onset2_b, onset, n, st);
}

}  // namespace bp
