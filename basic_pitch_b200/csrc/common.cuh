// Shared definitions for the sm_90a kernels of the basic-pitch hot path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bp {

// ---- geometry (reference: basic_pitch/constants.py:25-47; SURVEY.md Appendix A) -------------
constexpr int kWinSamples = 43844;
constexpr int kSampleRate = 22050;  // reference: basic_pitch/constants.py AUDIO_SAMPLE_RATE
constexpr int kFrames = 172;
constexpr int kCqtBins = 309;
constexpr int kContourBins = 264;
constexpr int kPitches = 88;
constexpr int kOctaves = 9;
constexpr int kBinsPerOctave = 36;
constexpr int kTaps = 256;
constexpr int kHarmonics = 8;
constexpr int kHopSamples = 36164;
constexpr int kHopFrames = 142;
constexpr int kOverlapHalf = 15;
constexpr int kLeadZeros = 3840;

// lengths of the decimation chain x_1..x_8 (x_0 = the 43844-sample window)
__host__ __device__ constexpr int octave_len(int o) {
  int l = kWinSamples;
  for (int i = 0; i < o; ++i) l = (l - 2) / 2 + 1;
  return l;
}
// offsets (floats) of x_1..x_8 inside one window's chain buffer, each aligned to 4 floats
__host__ __device__ constexpr int chain_off(int o) {  // o >= 1
  int off = 0;
  for (int i = 1; i < o; ++i) off += (octave_len(i) + 3) & ~3;
  return off;
}
constexpr int kChainStride = (chain_off(8) + octave_len(8) + 3 + 31) & ~31;
// The same two functions for an octave index only known at run time: a switch over constant-folded values (the loops
// above cost hundreds of cycles per call when `o` is not a compile-time constant — found in the CQT producers' trace).
__device__ __forceinline__ int octave_len_rt(int o) {
  switch (o) {
    case 0: return octave_len(0);
    case 1: return octave_len(1);
    case 2: return octave_len(2);
    case 3: return octave_len(3);
    case 4: return octave_len(4);
    case 5: return octave_len(5);
    case 6: return octave_len(6);
    case 7: return octave_len(7);
    default: return octave_len(8);
  }
}
__device__ __forceinline__ int chain_off_rt(int o) {
  switch (o) {
    case 1: return chain_off(1);
    case 2: return chain_off(2);
    case 3: return chain_off(3);
    case 4: return chain_off(4);
    case 5: return chain_off(5);
    case 6: return chain_off(6);
    case 7: return chain_off(7);
    default: return chain_off(8);
  }
}


// Where window w's samples come from: sample j = (lo <= j < hi) ? audio[base + j] : 0.
struct WinDesc {
  long long base;
  int lo;
  int hi;
};

// Order-preserving float <-> uint mapping for atomicMin/atomicMax on floats of either sign.
__device__ __forceinline__ unsigned int float_to_ordered(float f) {
  unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_float(unsigned int k) {
  unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

// Model parameters as laid out in one device block (float offsets).  The same block is what the
// single NCCL broadcast at init moves (bp_model_param_block).
struct ParamLayout {
  static constexpr int cqt_real = 0;                          // [36][256]
  static constexpr int cqt_imag = cqt_real + 36 * 256;        // [36][256]
  static constexpr int lowpass = cqt_imag + 36 * 256;         // [256]
  static constexpr int cqt_scale = lowpass + 256;             // [309] (+3 pad)
  static constexpr int bn = cqt_scale + 312;                  // scale, bias (+2 pad)
  static constexpr int contour1_w = bn + 4;                   // [8][8][3][39]
  static constexpr int contour1_b = contour1_w + 8 * 8 * 3 * 39;
  static constexpr int contour2_w = contour1_b + 8;           // [1][8][5][5]
  static constexpr int contour2_b = contour2_w + 200;         // (+3 pad)
  static constexpr int note1_w = contour2_b + 4;              // [32][1][7][7]
  static constexpr int note1_b = note1_w + 32 * 49;
  static constexpr int note2_w = note1_b + 32;                // [1][32][7][3]
  static constexpr int note2_b = note2_w + 672;
  static constexpr int onset1_w = note2_b + 4;                // [32][8][5][5]
  static constexpr int onset1_b = onset1_w + 32 * 200;
  static constexpr int onset2_w = onset1_b + 32;              // [1][33][3][3] (297, +3 pad)
  static constexpr int onset2_b = onset2_w + 300;
  static constexpr int total = onset2_b + 4;
};

}  // namespace bp
