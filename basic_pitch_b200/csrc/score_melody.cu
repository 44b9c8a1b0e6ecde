// Melody counts on the device: the sums behind mir_eval.melody.evaluate (0.7) for a grid of (setting, file) pairs read
// from a posteriorgram, or for a list of explicit f0 tracks (include/bp_b200.h, bp_score_melody_grid_*,
// bp_score_melody_host).
//
// The reference -> estimate map depends on the time bases only, so the host builds it once per call (MelodyRef): per
// reference frame the rounded time, the estimate frame of the zero-order sample (which is also the lower end of the
// linear bracket) and the frame whose held cents the upper end takes.  A grid chunk is then three launches: the arg-max
// of every (distinct bin range, frame), one warp each; the held cents of every (setting, file), one warp scan along the
// frames; the counts, one thread per (setting, reference frame), reduced with warp-aggregated integer atomics.  Every
// sum is an integer: the result is deterministic.
// Decoded notes read as a melody (bp_score_note_melody_grid_*) replace the first two launches by one: a warp per
// (setting, file) picks each frame's pitch from the grid decode's count roll and the note posteriorgram, bends it with
// pitch_bend_at (the decode's own arg-max), writes the raw cents and carries the held cents along the file as the hold
// kernel does; the counts kernel then reads those raw cents.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

#include "kernels.cuh"

namespace bp {

namespace {

constexpr int kMelodyThreads = 128;

// ---- arg-max --------------------------------------------------------------------------------------------------------
// Warp w = r * n_frames + frame: the largest float32 value of the row within range r's bins [lo, hi), the lowest bin on
// a tie; a NaN cell never wins (ordered comparisons).  An empty range or a row of NaN cells gives bin -1.
__global__ void __launch_bounds__(kMelodyThreads) melody_argmax_kernel(const float* __restrict__ gram, long long width,
                                                                       const MelodyRange* __restrict__ ranges,
                                                                       long long n_frames, long long n_warps,
                                                                       MelodyArg* __restrict__ arg) {
  const long long w = (long long)blockIdx.x * (kMelodyThreads / 32) + (threadIdx.x >> 5);
  if (w >= n_warps) return;
  const int lane = threadIdx.x & 31;
  const long long r = w / n_frames, frame = w % n_frames;
  const MelodyRange rg = ranges[r];
  const float* row = gram + frame * width;
  float best = 0.0f;
  int bin = -1;
  for (int b = rg.lo + lane; b < rg.hi; b += 32) {  // ascending bins per lane: a strict > keeps the lowest of a tie
    const float v = row[b];
    if (bin < 0 ? v == v : v > best) best = v, bin = b;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_down_sync(0xffffffffu, best, o);
    const int ob = __shfl_down_sync(0xffffffffu, bin, o);
    if (ob >= 0 && (bin < 0 || ov > best || (ov == best && ob < bin))) best = ov, bin = ob;
  }
  if (lane == 0) arg[w] = MelodyArg{best, bin};
}

// Where the counts read the raw estimate: explicit tracks, the arg-max of a posteriorgram, or decoded notes.
enum class MelodySrc { kExplicit, kGram, kNotes };

// Raw cents and voicing of estimate frame e (global) under chunk-local setting s: the grid reads the arg-max of the
// setting's range (include/bp_b200.h, bp_score_melody_grid_*), decoded notes the raw cents note_melody_kernel wrote (voiced
// exactly where nonzero: every bin cents value is > 0), explicit tracks their arrays.
template <MelodySrc kSrc>
__device__ __forceinline__ double raw_cent(const MelodyEst& E, long long s, long long e, int& voiced) {
  if constexpr (kSrc == MelodySrc::kNotes) {
    const double c = E.raw[s * E.n_frames + e];
    voiced = c != 0.0;
    return c;
  } else if constexpr (kSrc == MelodySrc::kGram) {
    const MelodySettingDev p = E.set[s];
    const MelodyArg a = E.arg[p.range * E.n_frames + e];
    if (a.bin < 0) return voiced = 0, 0.0;
    voiced = (double)a.v >= p.threshold;
    return voiced || p.guess ? E.bin_cent[a.bin] : 0.0;
  } else {
    voiced = E.voiced[e];
    return E.cent[e];
  }
}

// ---- hold -------------------------------------------------------------------------------------------------------------
// Warp q = s * n_files + file: held[s][frame] = the cents of the last frame <= frame of the file whose cents are
// nonzero, 0 when there is none (mir_eval's frequencies_held: a zero takes the previous held value).
__global__ void __launch_bounds__(kMelodyThreads) melody_hold_kernel(MelodyEst E, const long long* __restrict__ frame_off,
                                                                     int n_files, long long n_warps) {
  const long long q = (long long)blockIdx.x * (kMelodyThreads / 32) + (threadIdx.x >> 5);
  if (q >= n_warps) return;
  const int lane = threadIdx.x & 31;
  const long long s = q / n_files;
  const int file = (int)(q % n_files);
  const long long e0 = frame_off[file], e1 = frame_off[file + 1];
  double* held = E.held + s * E.n_frames;
  double carry = 0.0;
  for (long long t0 = e0; t0 < e1; t0 += 32) {
    const long long e = t0 + lane;
    int v = 0;
    const double c = e < e1 ? raw_cent<MelodySrc::kGram>(E, s, e, v) : 0.0;
    const unsigned nz = __ballot_sync(0xffffffffu, c != 0.0) & (0xffffffffu >> (31 - lane));  // lanes <= this one
    const double from = __shfl_sync(0xffffffffu, c, nz ? 31 - __clz(nz) : 0);
    const double h = nz ? from : carry;
    if (e < e1) held[e] = h;
    carry = __shfl_sync(0xffffffffu, h, 31);
  }
}

// ---- decoded notes --------------------------------------------------------------------------------------------------
// Warp q = s * n_files + file, one frame per lane: the sounding pitches of the frame are those with a nonzero roll
// count; the winner has the largest float32 note posteriorgram value, the lowest pitch on a tie, and a NaN loses to every
// number (a frame whose sounding cells are all NaN takes its lowest sounding pitch).  raw[s][e] = bin_cent[3 (p - 21) +
// bend] of the winner (its bend under the setting's bend flag), 0 when nothing sounds; held[s][e] as melody_hold_kernel.
__global__ void __launch_bounds__(kMelodyThreads) note_melody_kernel(NoteMelodyEst N, MelodyEst E, int n_files,
                                                                     long long n_warps) {
  const long long q = (long long)blockIdx.x * (kMelodyThreads / 32) + (threadIdx.x >> 5);
  if (q >= n_warps) return;
  const int lane = threadIdx.x & 31;
  const long long s = q / n_files;
  const int file = (int)(q % n_files);
  const long long e0 = N.frame_off[file], T = N.frame_off[file + 1] - e0;
  const int* roll = N.roll + s * N.roll_stride + e0 * kPitches;
  const bool bend = N.bend_on[s] != 0;
  double* raw = E.raw + s * E.n_frames + e0;
  double* held = E.held + s * E.n_frames + e0;
  double carry = 0.0;
  for (long long t0 = 0; t0 < T; t0 += 32) {
    const long long t = t0 + lane;
    double c = 0.0;
    if (t < T) {
      const float* nrow = N.note + (e0 + t) * kPitches;
      int best = -1;
      float bv = 0.0f;
#pragma unroll 1
      for (int p = 0; p < kPitches; ++p) {
        if (roll[p * T + t] == 0) continue;
        const float v = nrow[p];
        if (best < 0 || v > bv || (bv != bv && v == v)) best = p, bv = v;
      }
      if (best >= 0)
        c = E.bin_cent[3 * best + (bend ? pitch_bend_at(N.contour + (e0 + t) * kContourBins, best, N.gauss) : 0)];
      raw[t] = c;
    }
    const unsigned nz = __ballot_sync(0xffffffffu, c != 0.0) & (0xffffffffu >> (31 - lane));  // lanes <= this one
    const double from = __shfl_sync(0xffffffffu, c, nz ? 31 - __clz(nz) : 0);
    const double h = nz ? from : carry;
    if (t < T) held[t] = h;
    carry = __shfl_sync(0xffffffffu, h, 31);
  }
}

// ---- counts -----------------------------------------------------------------------------------------------------------
// Thread x = s * K + k: reference frame k under chunk-local setting s.
template <MelodySrc kSrc>
__global__ void __launch_bounds__(kMelodyThreads) melody_score_kernel(const MelodyRef* __restrict__ R, long long K,
                                                                      MelodyEst E, double tol, int n_owner,
                                                                      long long n_threads, long long* __restrict__ counts) {
  const long long x = (long long)blockIdx.x * kMelodyThreads + threadIdx.x;
  const bool live = x < n_threads;
  long long v[kMelodyCounts] = {0, 0, 0, 0, 0, 0, 0};
  long long pair = -1;
  if (live) {
    const long long s = x / K, k = x % K;
    const MelodyRef r = R[k];
    pair = s * n_owner + r.owner;
    const bool rv = r.flags & 1;
    int ev = 0;
    double ec = 0.0;
    if (r.zero >= 0) {
      const double zc = raw_cent<kSrc>(E, s, r.zero, ev);
      if (r.flags & 2) {
        ec = zc;  // identical time bases: the raw estimate
      } else if (zc != 0.0) {
        // np.interp on the held cents (interp1d(kind='linear') of float64 data): the knot's value on a knot, else
        // slope (x - t_lo) + y_lo; the result is kept where the zero-order raw cents are nonzero
        const double* held = E.held + s * E.n_frames;
        const double y_lo = held[r.zero];
        if (r.hi < 0) {
          ec = y_lo;
        } else {
          const double slope = __ddiv_rn(__dsub_rn(held[r.hi], y_lo), __dsub_rn(r.t_hi, r.t_lo));
          ec = __dadd_rn(__dmul_rn(slope, __dsub_rn(r.x, r.t_lo)), y_lo);
        }
      }
    }
    v[0] = 1;
    v[1] = rv;
    v[2] = rv && ev;
    v[3] = !rv && ev;
    if (rv && r.cent != 0.0 && ec != 0.0) {
      const double d = fabs(__dsub_rn(r.cent, ec));
      const double octave = __dmul_rn(1200.0, floor(__dadd_rn(__ddiv_rn(d, 1200.0), 0.5)));
      v[4] = d < tol;
      v[5] = fabs(__dsub_rn(d, octave)) < tol;
      v[6] = v[4] && ev;
    }
  }
  // lane 0 is live whenever any lane is (threads are contiguous); a warp whose live lanes share one pair adds once
  const long long pair0 = __shfl_sync(0xffffffffu, pair, 0);
  if (__all_sync(0xffffffffu, !live || pair == pair0)) {
#pragma unroll
    for (int c = 0; c < kMelodyCounts; ++c)
#pragma unroll
      for (int o = 16; o; o >>= 1) v[c] += __shfl_down_sync(0xffffffffu, v[c], o);
    if ((threadIdx.x & 31) == 0 && live)
#pragma unroll
      for (int c = 0; c < kMelodyCounts; ++c)
        if (v[c]) atomicAdd(reinterpret_cast<unsigned long long*>(counts + kMelodyCounts * pair0 + c), (unsigned long long)v[c]);
  } else if (live) {
#pragma unroll
    for (int c = 0; c < kMelodyCounts; ++c)
      if (v[c]) atomicAdd(reinterpret_cast<unsigned long long*>(counts + kMelodyCounts * pair + c), (unsigned long long)v[c]);
  }
}

unsigned int blocks_for(long long n, int per_block) { return (unsigned int)std::max(1LL, (n + per_block - 1) / per_block); }

}  // namespace

void launch_melody_grid(const float* gram, long long width, const MelodyRange* ranges, int n_ranges,
                        const long long* frame_off, int n_files, const MelodyRef* refs, long long K, const MelodyEst& E,
                        double tol, int n_settings, long long* counts, cudaStream_t st) {
  const long long F = E.n_frames, per = kMelodyThreads / 32;
  const long long n_arg = F * n_ranges, n_hold = (long long)n_settings * n_files, n = (long long)n_settings * K;
  melody_argmax_kernel<<<blocks_for(n_arg, per), kMelodyThreads, 0, st>>>(gram, width, ranges, std::max(F, 1LL), n_arg,
                                                                           E.arg);
  melody_hold_kernel<<<blocks_for(n_hold, per), kMelodyThreads, 0, st>>>(E, frame_off, n_files, n_hold);
  melody_score_kernel<MelodySrc::kGram><<<blocks_for(n, kMelodyThreads), kMelodyThreads, 0, st>>>(refs, std::max(K, 1LL), E, tol,
                                                                                     n_files, n, counts);
}

void launch_melody_explicit(const MelodyRef* refs, long long K, const MelodyEst& E, double tol, int n_items,
                            long long* counts, cudaStream_t st) {
  melody_score_kernel<MelodySrc::kExplicit><<<blocks_for(K, kMelodyThreads), kMelodyThreads, 0, st>>>(refs, std::max(K, 1LL), E, tol,
                                                                                      n_items, K, counts);
}

void launch_note_melody(const NoteMelodyEst& N, int n_files, const MelodyRef* refs, long long K, const MelodyEst& E,
                        double tol, int n_settings, long long* counts, cudaStream_t st) {
  const long long n_warps = (long long)n_settings * n_files, n = (long long)n_settings * K;
  note_melody_kernel<<<blocks_for(n_warps, kMelodyThreads / 32), kMelodyThreads, 0, st>>>(N, E, n_files, n_warps);
  melody_score_kernel<MelodySrc::kNotes><<<blocks_for(n, kMelodyThreads), kMelodyThreads, 0, st>>>(
      refs, std::max(K, 1LL), E, tol, n_files, n, counts);
}

}  // namespace bp
