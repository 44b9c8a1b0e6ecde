// Frame-level multi-pitch counts on the device: the sums behind mir_eval.multipitch.metrics (0.7) for a grid of
// (setting, file) pairs or a list of items (include/bp_b200.h, bp_score_frames_grid_*, bp_score_multipitch_host,
// bp_score_salience_grid_*).
//
// Grid estimates come from the grid decode's note slots.  Once the sequential loops have run, each setting's private
// "remaining energy" copy is dead; it is exactly an int [88][T] per file, so it becomes a note-count roll: zeroed by the
// host, +1 / -1 scattered at every note's start / end, then a prefix sum along frames.
// The match kernel runs one thread per (setting, reference frame).  The reference values of a frame are sorted by midi
// on the host; the estimate frame is a roll column (88 pitches in ascending order with their multiplicities), explicit
// values sorted by midi, or a posteriorgram row read under a salience setting (bp_score_salience_grid_*: the bins that
// pass its threshold, peak and range tests, in ascending bin order, each once).  Every sum is an integer, reduced with
// integer atomics: the result is deterministic.
// Bent grid estimates (bp_score_bent_frames_grid_*) read the same roll: each sounding pitch of the column becomes one
// group at its contour bin, 3 (p - 21) plus the pitch's bend at that frame (pitch_bend_at, the decode's own arg-max: the
// bend depends on (frame, pitch) only, so a pitch's count of notes all share it).  Bends move a pitch by up to 25 bins, so
// keys of pitches up to 16 semitones apart can cross: the thread insertion-sorts its <= 88 (key, count) groups in a local
// array of 88 int64 (704 bytes of stack in that instantiation only; no spills) before the unchanged passes.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

#include "kernels.cuh"

namespace bp {

namespace {

constexpr int kRollThreads = 128;
constexpr int kMatchThreads = 128;

// ---- count roll ---------------------------------------------------------------------------------------------------
// blockIdx.x: pair q = setting * n_files + file.  Notes are [start, end) in file-relative frames, start < end <= T.
__global__ void __launch_bounds__(kRollThreads) roll_scatter_kernel(const long long* __restrict__ frame_off,
                                                                    const long long* __restrict__ slot_off,
                                                                    const int* __restrict__ note_count,
                                                                    const int* __restrict__ start,
                                                                    const int* __restrict__ end,
                                                                    const int* __restrict__ pitch, int n_files,
                                                                    int* __restrict__ roll, long long roll_stride) {
  const long long q = blockIdx.x;
  const int file = (int)(q % n_files);
  const long long s = q / n_files;
  const long long base = frame_off[file];
  const int T = (int)(frame_off[file + 1] - base);
  int* r = roll + s * roll_stride + base * kPitches;
  const long long s0 = slot_off[q];
  const int n = note_count[q];
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int p = pitch[s0 + j] - 21, a = start[s0 + j], b = end[s0 + j];
    if (p < 0 || p >= kPitches || a < 0 || a >= T || b <= a) continue;  // never produced by the decode
    atomicAdd(r + (long long)p * T + a, 1);
    if (b < T) atomicAdd(r + (long long)p * T + b, -1);
  }
}

// One warp per row (setting, file, pitch): inclusive prefix sum along the file's T frames.
__global__ void __launch_bounds__(kRollThreads) roll_scan_kernel(const long long* __restrict__ frame_off, int n_files,
                                                                 long long n_rows, int* __restrict__ roll,
                                                                 long long roll_stride) {
  const long long row = (long long)blockIdx.x * (kRollThreads / 32) + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const int p = (int)(row % kPitches);
  const long long fs = row / kPitches;
  const int file = (int)(fs % n_files);
  const long long s = fs / n_files;
  const long long base = frame_off[file];
  const int T = (int)(frame_off[file + 1] - base);
  int* r = roll + s * roll_stride + base * kPitches + (long long)p * T;
  int carry = 0;
  for (int t0 = 0; t0 < T; t0 += 32) {
    const int t = t0 + lane;
    int v = t < T ? r[t] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += u;
    }
    v += carry;
    if (t < T) r[t] = v;
    carry = __shfl_sync(0xffffffffu, v, 31);
  }
}

// ---- matching -----------------------------------------------------------------------------------------------------
// The estimate frame as groups g = 0 .. n-1 of equal values in ascending midi: the 88 pitches of a roll column with their
// counts (roll), single explicit values, or the bins bin_lo + g of a posteriorgram row, each counted once when it is an
// estimate of the frame under the setting (gram).
template <EstKind kKind>
struct EstFrame {
  const int* col;  // roll: roll column at frame t, pitch g at col[g * T]
  const long long* kv;  // bent: group g is key kv[g] >> 32 (a contour bin) with count kv[g] & 0xffffffff, keys ascending
  long long T;
  const double *midi, *chroma;  // roll: tables indexed by MIDI number; explicit: this frame's values; gram: bin tables
  int n;
  const float* row;  // gram: the posteriorgram row of the frame, `width` bins
  int width, lo;
  double thresh;
  bool peak;
  // include/bp_b200.h, bp_score_salience_grid_*: bin b is an estimate when thresh <= (double) G[b] and, with peak
  // picking, 1 <= b <= width - 2 and G[b] > both neighbours (float32, the whole row): scipy.signal.argrelmax, then the
  // threshold.  Ordered comparisons, so a NaN cell is never an estimate and never below a peak.
  __device__ __forceinline__ int gram_count(int g) const {
    const int b = lo + g;
    const float v = row[b];
    if (!((double)v >= thresh)) return 0;
    if (!peak) return 1;
    return b >= 1 && b <= width - 2 && v > row[b - 1] && v > row[b + 1];
  }
  __device__ __forceinline__ int count(int g) const {
    if constexpr (kKind == EstKind::kRoll) return col[g * T];
    else if constexpr (kKind == EstKind::kBent) return (int)(kv[g] & 0xffffffffLL);
    else if constexpr (kKind == EstKind::kGram) return gram_count(g);
    else return 1;
  }
  __device__ __forceinline__ double m(int g) const {
    if constexpr (kKind == EstKind::kRoll) return midi[g + 21];
    else if constexpr (kKind == EstKind::kBent) return midi[kv[g] >> 32];
    else if constexpr (kKind == EstKind::kGram) return midi[lo + g];
    else return midi[g];
  }
  __device__ __forceinline__ double c(int g) const {
    if constexpr (kKind == EstKind::kRoll) return chroma[g + 21];
    else if constexpr (kKind == EstKind::kBent) return chroma[kv[g] >> 32];
    else if constexpr (kKind == EstKind::kGram) return chroma[lo + g];
    else return chroma[g];
  }
};

// Plain pass (util._fast_hit_windows): e hits r when fl(e - w) <= r <= fl(e + w).  Both ends of the windows are
// non-decreasing in e (rounding is monotone), so taking the estimates in ascending order, each one's copies take the
// smallest free references at or above the lower end while they stay at or below the upper end, is a maximum matching:
// it is the earliest-deadline greedy for points and intervals sorted by both ends.  A reference skipped for lying below
// one window's lower end lies below every later window, and exchanging the mate of any maximum matching for the
// smallest free hit in that order never loses an edge.
template <EstKind kKind>
__device__ __forceinline__ int plain_tp(const EstFrame<kKind>& E, const double* rm, int n_ref, double w) {
  int i = 0, tp = 0;
  for (int g = 0; g < E.n && i < n_ref; ++g) {
    int c = E.count(g);
    if (c == 0) continue;
    const double e = E.m(g), lo = __dsub_rn(e, w), hi = __dadd_rn(e, w);
    while (i < n_ref && rm[i] < lo) ++i;
    while (c > 0 && i < n_ref && rm[i] <= hi) ++tp, ++i, --c;
  }
  return tp;
}

// util._outer_distance_mod_n on chroma values in [0, 12): d = |r - e|, hit when min(d, 12 - d) <= w.
__device__ __forceinline__ bool chroma_hit(double r, double e, double w) {
  const double d = fabs(__dsub_rn(r, e));
  return fmin(d, __dsub_rn(12.0, d)) <= w;
}

// Chroma pass: the hits wrap around 12, so an exact method: a greedy pass, then augmenting paths (Kuhn) from each group
// that still has free copies.  A group's copies have identical neighbours, so one failed search ends that group (Kuhn's
// lemma for its copies).  Each search marks the references it visits; the explicit stack holds (group, reference
// cursor) and grows by one per newly visited reference, so it never exceeds n_ref + 1 frames.
// ws: mate [n_ref] (group of the reference, -1 free), seen [n_ref] (search stamp), stack [2 (n_ref + 1)].
template <EstKind kKind>
__device__ __forceinline__ int chroma_tp(const EstFrame<kKind>& E, const double* rc, int n_ref, int n_est, double w,
                                         int* ws) {
  const int limit = min(n_ref, n_est);
  if (limit == 0) return 0;
  if (w >= 6.0) return limit;  // min(d, fl(12 - d)) <= 6 for every d in [0, 12)
  int* mate = ws;
  int* seen = ws + n_ref;
  int* stk = ws + 2 * n_ref;
  for (int i = 0; i < n_ref; ++i) mate[i] = seen[i] = -1;
  int matched = 0;
  for (int g = 0; g < E.n && matched < limit; ++g) {
    int c = E.count(g);
    if (c == 0) continue;
    const double e = E.c(g);
    for (int i = 0; i < n_ref && c > 0; ++i)
      if (mate[i] < 0 && chroma_hit(rc[i], e, w)) mate[i] = g, --c, ++matched;
  }
  int stamp = 0;
  for (int g0 = 0; g0 < E.n && matched < limit; ++g0) {
    int spare = E.count(g0);
    if (spare == 0) continue;
    for (int i = 0; i < n_ref; ++i) spare -= mate[i] == g0;
    while (spare > 0 && matched < limit) {
      const int id = stamp++;
      int depth = 0;
      stk[0] = g0, stk[1] = -1;
      bool found = false;
      while (depth >= 0) {
        const int g = stk[2 * depth];
        const double e = E.c(g);
        int i = stk[2 * depth + 1] + 1;
        while (i < n_ref && (seen[i] == id || !chroma_hit(rc[i], e, w))) ++i;
        if (i == n_ref) {
          --depth;
          continue;
        }
        stk[2 * depth + 1] = i;
        seen[i] = id;
        if (mate[i] < 0) {  // flip the path: each level's group takes the reference its cursor stands on
          for (int l = 0; l <= depth; ++l) mate[stk[2 * l + 1]] = stk[2 * l];
          found = true;
          break;
        }
        ++depth;
        stk[2 * depth] = mate[i], stk[2 * depth + 1] = -1;
      }
      if (!found) break;
      ++matched, --spare;
    }
  }
  return matched;
}

// Thread x = s * K + k: reference frame k under chunk-local setting s.
template <EstKind kKind>
__global__ void __launch_bounds__(kMatchThreads) frame_match_kernel(FrameRefs R, FrameEst E, double w,
                                                                    int* __restrict__ ws, int n_owner,
                                                                    long long n_threads, long long* __restrict__ counts) {
  const long long x = (long long)blockIdx.x * kMatchThreads + threadIdx.x;
  const bool live = x < n_threads;
  long long v[kFrameCounts] = {0, 0, 0, 0, 0, 0, 0};
  long long pair = -1;
  if (live) {
    const long long K = R.n_frames;
    const long long s = x / K, k = x % K;
    const int owner = R.owner[k], t = R.est_frame[k];
    const long long r0 = R.voff[k];
    const int n_ref = (int)(R.voff[k + 1] - r0);
    pair = s * n_owner + owner;
    EstFrame<kKind> ef{};
    long long kv[kKind == EstKind::kBent ? kPitches : 1];
    int n_est = 0;
    if (t >= 0) {
      if constexpr (kKind == EstKind::kRoll) {
        const long long base = E.frame_off[owner];
        ef.T = E.frame_off[owner + 1] - base;
        ef.col = E.roll + s * E.roll_stride + base * kPitches + t;
        ef.midi = E.tab_midi;
        ef.chroma = E.tab_chroma;
        ef.n = kPitches;
#pragma unroll 1  // unrolled, ptxas spills
        for (int g = 0; g < kPitches; ++g) n_est += ef.count(g);
      } else if constexpr (kKind == EstKind::kBent) {
        const long long base = E.frame_off[owner], T = E.frame_off[owner + 1] - base;
        const int* col = E.roll + s * E.roll_stride + base * kPitches + t;
        const float* crow = E.contour + (base + t) * kContourBins;  // read only with bends
        const bool bend = E.bend_on[s] != 0;
        int n = 0;
#pragma unroll 1
        for (int p = 0; p < kPitches; ++p) {
          const int c = col[p * T];
          if (c == 0) continue;
          const long long key = (long long)(3 * p + (bend ? pitch_bend_at(crow, p, E.gauss) : 0)) << 32 | (unsigned)c;
          int i = n++;
          for (; i > 0 && kv[i - 1] > key; --i) kv[i] = kv[i - 1];
          kv[i] = key;
          n_est += c;
        }
        ef.kv = kv;
        ef.n = n;
        ef.midi = E.tab_midi;
        ef.chroma = E.tab_chroma;
      } else if constexpr (kKind == EstKind::kGram) {
        const SalienceSettingDev p = E.salience[s];
        ef.row = E.gram + (E.frame_off[owner] + t) * E.width;
        ef.width = (int)E.width;
        ef.lo = p.bin_lo;
        ef.n = p.bin_hi - p.bin_lo;
        ef.thresh = p.threshold;
        ef.peak = p.peak_pick != 0;
        ef.midi = E.tab_midi;
        ef.chroma = E.tab_chroma;
#pragma unroll 1
        for (int g = 0; g < ef.n; ++g) n_est += ef.count(g);
      } else {
        const long long e0 = E.voff[t];
        ef.midi = E.midi + e0;
        ef.chroma = E.chroma + e0;
        ef.n = n_est = (int)(E.voff[t + 1] - e0);
      }
    }
    if (n_ref > 0 && n_est > 0) {
      v[2] = plain_tp(ef, R.midi + r0, n_ref, w);
      v[3] = chroma_tp(ef, R.chroma + r0, n_ref, n_est, w, ws + s * frame_ws_stride(R.voff[K], K) + 4 * r0 + 2 * k);
    }
    v[0] = n_ref;
    v[1] = n_est;
    v[4] = min(n_ref, n_est);
    v[5] = max(0, n_ref - n_est);
    v[6] = max(0, n_est - n_ref);
  }
  // lane 0 is live whenever any lane is (threads are contiguous); a warp whose live lanes share one pair adds once
  const long long pair0 = __shfl_sync(0xffffffffu, pair, 0);
  if (__all_sync(0xffffffffu, !live || pair == pair0)) {
#pragma unroll
    for (int c = 0; c < kFrameCounts; ++c)
#pragma unroll
      for (int o = 16; o; o >>= 1) v[c] += __shfl_down_sync(0xffffffffu, v[c], o);
    if ((threadIdx.x & 31) == 0 && live)
#pragma unroll
      for (int c = 0; c < kFrameCounts; ++c)
        if (v[c]) atomicAdd(reinterpret_cast<unsigned long long*>(counts + kFrameCounts * pair0 + c), (unsigned long long)v[c]);
  } else if (live) {
#pragma unroll
    for (int c = 0; c < kFrameCounts; ++c)
      if (v[c]) atomicAdd(reinterpret_cast<unsigned long long*>(counts + kFrameCounts * pair + c), (unsigned long long)v[c]);
  }
}

}  // namespace

void launch_frame_roll(const long long* frame_off, const long long* slot_off, const int* note_count, const int* start,
                       const int* end, const int* pitch, int n_files, int n_settings, int* roll, long long roll_stride,
                       cudaStream_t st) {
  const long long n_pairs = (long long)n_settings * n_files;
  roll_scatter_kernel<<<(unsigned int)n_pairs, kRollThreads, 0, st>>>(frame_off, slot_off, note_count, start, end, pitch,
                                                                       n_files, roll, roll_stride);
  const long long rows = n_pairs * kPitches, per = kRollThreads / 32;
  roll_scan_kernel<<<(unsigned int)((rows + per - 1) / per), kRollThreads, 0, st>>>(frame_off, n_files, rows, roll,
                                                                                     roll_stride);
}

void launch_frame_match(const FrameRefs& R, const FrameEst& E, double window, int* ws, int n_owner, int n_settings,
                        long long* counts, cudaStream_t st) {
  const long long n = (long long)n_settings * R.n_frames;
  const unsigned int blocks = (unsigned int)std::max(1LL, (n + kMatchThreads - 1) / kMatchThreads);
  if (E.roll && E.bend_on)
    frame_match_kernel<EstKind::kBent><<<blocks, kMatchThreads, 0, st>>>(R, E, window, ws, n_owner, n, counts);
  else if (E.roll)
    frame_match_kernel<EstKind::kRoll><<<blocks, kMatchThreads, 0, st>>>(R, E, window, ws, n_owner, n, counts);
  else if (E.salience)
    frame_match_kernel<EstKind::kGram><<<blocks, kMatchThreads, 0, st>>>(R, E, window, ws, n_owner, n, counts);
  else
    frame_match_kernel<EstKind::kExplicit><<<blocks, kMatchThreads, 0, st>>>(R, E, window, ws, n_owner, n, counts);
}

}  // namespace bp
