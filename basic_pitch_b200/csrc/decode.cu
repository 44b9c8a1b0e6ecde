// Note decode: posteriorgrams -> note events, bit-identical to the reference decode on the same input.
//
// Replaces reference: basic_pitch/note_creation.py
//   constrain_frequency          :314-343   (column range applied on every read; inputs untouched)
//   get_infered_onsets           :289-311   (float64, two file-global maxima)
//   output_to_notes_polyphonic   :360-511   (peak pick :398-404, onset loop :409-447, melodia :449-509)
//   get_pitch_bends              :182-219
// Semantics pinned in SURVEY.md Appendix B; oracle: oracle/decode_ref.py.
//
// Kernels
//   decode_prep_kernel   tiles of 32 frames x 88 pitches staged in shared memory: "remaining energy" E (column-major
//                        per file, frames with the pitch range applied, written frame-fastest), per-file
//                        max(onsets) and max(frame_diff)
//   decode_cand_kernel   same tiles + 1 halo frame: float64 inferred onsets (one division per cell), strict time
//                        peaks, threshold -> one candidate bit per cell (warp ballot -> 32-bit words)
//   decode_seq_kernel    one CTA per file: candidates in (time desc, pitch desc) order through the greedy
//                        onset loop (warp-cooperative run-of-`energy_tol` scan + neighbour zeroing), then the
//                        melodia loop with per-column maxima kept in shared memory
//   note_finish_kernel   one warp per note: amplitude (NumPy pairwise float32 mean) and per-frame pitch-bend
//                        arg-max in float64
// The grid decode (bp_decode_grid_*) runs the same three kernels for many parameter sets at once (template kGrid): the
// prep per distinct pitch range, the candidates per distinct (range, infer_onsets, onset_thresh), the loops per
// (file, setting) on the setting's own copy of E; blockIdx.y picks the group or setting.
#include "kernels.cuh"

namespace bp {

__device__ __forceinline__ int find_file(const long long* __restrict__ off, int n_files, long long frame) {
  int lo = 0, hi = n_files;  // invariant: off[lo] <= frame < off[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (off[mid] <= frame)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

__device__ __forceinline__ float constrained(const float* __restrict__ m, long long frame, int f, int lo, int hi) {
  return (f >= lo && f < hi) ? m[frame * kPitches + f] : 0.f;
}

// ------------------------------------------------------------------------------------------------
// Both cell-parallel kernels work on tiles of 32 consecutive frames of the batch (all 88 pitches) staged in shared
// memory: row-major global reads, the transposed (frame-fastest) writes of E and the time neighbours of the peak pick
// come from the tile.  A tile may straddle files; every row carries its own file.
// ------------------------------------------------------------------------------------------------
constexpr int kTileFrames = 32;

struct RowInfo {
  int file;        // -1: row outside the batch
  int t, T;        // frame index inside the file, frames of the file
  long long base;  // first frame of the file
};

__device__ __forceinline__ RowInfo row_info(const long long* __restrict__ frame_off, int n_files, long long g,
                                            long long total) {
  RowInfo r{-1, 0, 0, 0};
  if (g >= 0 && g < total) {
    r.file = find_file(frame_off, n_files, g);
    r.base = frame_off[r.file];
    r.T = (int)(frame_off[r.file + 1] - r.base);
    r.t = (int)(g - r.base);
  }
  return r;
}

// positive part of min(n[t]-n[t-1], n[t]-n[t-2]) in float64 from three rows of the staged tile (t >= 2)
__device__ __forceinline__ double frame_diff3(float a, float m1, float m2) {
  const double d1 = (double)a - (double)m1, d2 = (double)a - (double)m2;
  const double d = d1 < d2 ? d1 : d2;
  return d < 0.0 ? 0.0 : d;
}

// kGrid: blockIdx.y is a prep group of g (range, maxima and the E copies of its settings); otherwise lo / hi and one E
template <bool kGrid>
__global__ void __launch_bounds__(256) decode_prep_kernel(const float* __restrict__ note, const float* __restrict__ onset,
                                                          const long long* __restrict__ frame_off, int n_files,
                                                          float* __restrict__ energy,
                                                          unsigned int* __restrict__ max_onset,     // [n_files] ordered-uint
                                                          unsigned long long* __restrict__ max_fd,  // [n_files] bits of a double >= 0
                                                          int lo, int hi, DecodeGridDev g) {
  if constexpr (kGrid) {
    lo = g.prep[blockIdx.y].lo;
    hi = g.prep[blockIdx.y].hi;
    max_onset += (size_t)blockIdx.y * n_files;
    max_fd += (size_t)blockIdx.y * n_files;
  }
  __shared__ float s_n[kTileFrames + 2][kPitches + 1];  // rows g0-2 .. g0+31, pitch range applied
  __shared__ RowInfo s_row[kTileFrames];
  __shared__ unsigned int s_mo[8];
  __shared__ unsigned long long s_fd[8];
  const long long total = frame_off[n_files];
  const long long g0 = (long long)blockIdx.x * kTileFrames;
  const int nrows = (int)min((long long)kTileFrames, total - g0);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < kTileFrames) s_row[tid] = row_info(frame_off, n_files, g0 + tid, total);
  for (int idx = tid; idx < (kTileFrames + 2) * kPitches; idx += 256) {
    const int rr = idx / kPitches, f = idx - rr * kPitches;
    const long long g = g0 - 2 + rr;
    s_n[rr][f] = (g >= 0 && g < total) ? constrained(note, g, f, lo, hi) : 0.f;
  }
  __syncthreads();
  const bool one_file = s_row[0].file == s_row[nrows - 1].file;
  unsigned int mo = 0u;  // ordered encoding of -inf is > 0, so 0 is a safe identity for max
  unsigned long long fd_bits = 0ull;
  for (int idx = tid; idx < nrows * kPitches; idx += 256) {
    const int r = idx / kPitches, f = idx - r * kPitches;
    const unsigned int mo_c = float_to_ordered(constrained(onset, g0 + r, f, lo, hi));
    const double fd = s_row[r].t >= 2 ? frame_diff3(s_n[r + 2][f], s_n[r + 1][f], s_n[r][f]) : 0.0;
    const unsigned long long fd_c = (unsigned long long)__double_as_longlong(fd);
    if (one_file) {
      mo = max(mo, mo_c);
      fd_bits = max(fd_bits, fd_c);
    } else {
      atomicMax(max_onset + s_row[r].file, mo_c);
      atomicMax(max_fd + s_row[r].file, fd_c);
    }
  }
  if (one_file) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      mo = max(mo, __shfl_xor_sync(0xffffffffu, mo, o));
      fd_bits = max(fd_bits, __shfl_xor_sync(0xffffffffu, fd_bits, o));
    }
    if (lane == 0) {
      s_mo[warp] = mo;
      s_fd[warp] = fd_bits;
    }
    __syncthreads();
    if (tid == 0) {
      for (int i = 1; i < 8; ++i) {
        mo = max(mo, s_mo[i]);
        fd_bits = max(fd_bits, s_fd[i]);
      }
      if (mo) atomicMax(max_onset + s_row[0].file, mo);
      atomicMax(max_fd + s_row[0].file, fd_bits);
    }
  }
  // E is column-major per file ([88][T]): lanes = consecutive frames -> contiguous 128-byte runs
  if (lane < nrows) {
    const RowInfo ri = s_row[lane];
    if constexpr (kGrid) {  // every setting of the group gets its own copy: its loops zero it
      const int j1 = g.prep[blockIdx.y].set_hi;
      for (int j = g.prep[blockIdx.y].set_lo; j < j1; ++j) {
        float* e = energy + g.sets[j] * g.e_stride + ri.base * kPitches + ri.t;
        for (int f = warp; f < kPitches; f += 8) e[(long long)f * ri.T] = s_n[lane + 2][f];
      }
    } else {
      float* e = energy + ri.base * kPitches + ri.t;
      for (int f = warp; f < kPitches; f += 8) e[(long long)f * ri.T] = s_n[lane + 2][f];
    }
  }
}

// kGrid: blockIdx.y is a candidate group of g (its parameters, its prep group's maxima, its own bitmap)
template <bool kGrid>
__global__ void __launch_bounds__(256) decode_cand_kernel(const float* __restrict__ note, const float* __restrict__ onset,
                                                          const long long* __restrict__ frame_off, int n_files,
                                                          const unsigned int* __restrict__ max_onset,
                                                          const unsigned long long* __restrict__ max_fd,
                                                          unsigned int* __restrict__ candbits, int lo, int hi, int infer,
                                                          double onset_thresh, double* __restrict__ onset64_out,
                                                          DecodeGridDev g) {
  if constexpr (kGrid) {
    const DecodeCandGroup cg = g.cand[blockIdx.y];
    lo = cg.lo;
    hi = cg.hi;
    infer = cg.infer;
    onset_thresh = cg.onset_thresh;
    max_onset += (size_t)cg.prep * n_files;
    max_fd += (size_t)cg.prep * n_files;
    candbits += blockIdx.y * g.cand_stride;
  }
  __shared__ float s_n[kTileFrames + 4][kPitches + 1];  // note rows g0-3 .. g0+32 (inferred onsets only)
  __shared__ double s_v[kTileFrames + 2][kPitches];     // float64 onset value of rows g0-1 .. g0+32
  __shared__ RowInfo s_row[kTileFrames + 2];
  __shared__ double s_maxo[kTileFrames + 2], s_maxfd[kTileFrames + 2];
  const long long total = frame_off[n_files];
  const long long g0 = (long long)blockIdx.x * kTileFrames;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < kTileFrames + 2) {
    const RowInfo ri = row_info(frame_off, n_files, g0 - 1 + tid, total);
    s_row[tid] = ri;
    if (ri.file >= 0) {
      s_maxo[tid] = (double)ordered_to_float(max_onset[ri.file]);
      s_maxfd[tid] = __longlong_as_double((long long)max_fd[ri.file]);
    }
  }
  if (infer) {
    for (int idx = tid; idx < (kTileFrames + 4) * kPitches; idx += 256) {
      const int rr = idx / kPitches, f = idx - rr * kPitches;
      const long long g = g0 - 3 + rr;
      s_n[rr][f] = (g >= 0 && g < total) ? constrained(note, g, f, lo, hi) : 0.f;
    }
  }
  __syncthreads();
  // float64 onset value used for peak picking (NaN when max(frame_diff) == 0, like the reference): once per cell
  for (int idx = tid; idx < (kTileFrames + 2) * kPitches; idx += 256) {
    const int rr = idx / kPitches, f = idx - rr * kPitches;
    const RowInfo ri = s_row[rr];
    double v = 0.0;
    if (ri.file >= 0) {
      const double o = (double)constrained(onset, g0 - 1 + rr, f, lo, hi);
      v = o;
      if (infer) {
        const double fd = ri.t >= 2 ? frame_diff3(s_n[rr + 2][f], s_n[rr + 1][f], s_n[rr][f]) : 0.0;
        const double w = __ddiv_rn(__dmul_rn(s_maxo[rr], fd), s_maxfd[rr]);
        v = (w != w) ? w : (o > w ? o : w);
      }
    }
    s_v[rr][f] = v;
  }
  __syncthreads();
  if (onset64_out) {  // bp_infer_onsets_host: the float64 onset matrix itself (reference: get_infered_onsets)
    for (int idx = tid; idx < kTileFrames * kPitches; idx += 256) {
      const int r = idx / kPitches, f = idx - r * kPitches;
      if (g0 + r < total) onset64_out[(g0 + r) * kPitches + f] = s_v[r + 1][f];
    }
  }
  // strict time peaks >= threshold; a warp ballot is one 32-cell word of the candidate bitmap
  const long long cell0 = g0 * kPitches;  // multiple of 32
  const long long total_cells = total * kPitches;
  for (int word = warp; word < kTileFrames * kPitches / 32; word += 8) {
    const int cl = word * 32 + lane;
    const int r = cl / kPitches, f = cl - r * kPitches;
    const RowInfo ri = s_row[r + 1];
    double val = 0.0;
    if (ri.file >= 0 && ri.t >= 1 && ri.t <= ri.T - 2) {
      const double c = s_v[r + 1][f];
      if (c > s_v[r][f] && c > s_v[r + 2][f]) val = c;
    }
    const bool cand = ri.file >= 0 && val >= onset_thresh;
    const unsigned int bits = __ballot_sync(0xffffffffu, cand);
    if (lane == 0 && cell0 + (long long)word * 32 < total_cells) candbits[(cell0 >> 5) + word] = bits;
  }
}

// ------------------------------------------------------------------------------------------------
// Sequential part, one CTA per file.
// ------------------------------------------------------------------------------------------------
constexpr int kSeqThreads = 128;

// block-maxima entries per pitch column for a batch: file i (frames [base, base + T)) owns entries
// [base / 256 + i, .. + ceil(T / 256)), which never overlap the next file's
long long decode_block_slots(long long total_frames, int n_files) { return total_frames / 256 + n_files + 1; }

// Warp-cooperative scan used by both loops: starting at frame i (step +1 or -1) with run counter 0, walk while
// `in range` and run < tol, counting consecutive cells of column `col` that are below the threshold.
// Returns the exit index and the run length in *run.  `limit`: forward -> stop when i >= limit (= T-1);
// backward -> stop when i <= limit (= 0).
__device__ __forceinline__ int scan_run(const float* col, int i, int dir, int limit, int tol, double thresh,
                                        int* run) {
  const int lane = threadIdx.x & 31;
  int k = 0;
  while (true) {
    int idx = i + dir * lane;
    bool valid = dir > 0 ? (idx < limit) : (idx > limit);
    float e = valid ? col[idx] : 0.f;
    unsigned int mv = __ballot_sync(0xffffffffu, valid);
    unsigned int mb = __ballot_sync(0xffffffffu, valid && ((double)e < thresh));
    bool stop = false;
#pragma unroll 1
    for (int j = 0; j < 32; ++j) {
      if (!((mv >> j) & 1u) || k >= tol) {
        stop = true;
        break;
      }
      k = ((mb >> j) & 1u) ? k + 1 : 0;
      i += dir;
    }
    if (stop || k >= tol) break;
  }
  *run = k;
  return i;
}

__device__ __forceinline__ void zero_cols(float* E, int T, int f, int t_lo, int t_hi /* exclusive */) {
  const int lane = threadIdx.x & 31;
  for (int t = t_lo + lane; t < t_hi; t += 32) {
    E[(long long)f * T + t] = 0.f;
    if (f < kPitches - 1) E[(long long)(f + 1) * T + t] = 0.f;
    if (f > 0) E[(long long)(f - 1) * T + t] = 0.f;
  }
}

// The melodia loop needs, after every note, the maximum (value, lowest frame) of the three columns it touched.  A full
// column scan costs T / 32 dependent loads per warp — 500 for a three-minute file, times thousands of iterations — so
// every column keeps the maxima of its 256-frame blocks: a note touches one or two blocks, and the column maximum is a
// reduction over T / 256 block entries.
constexpr int kDecBlk = 256;

// maximum of frames [t_lo, t_hi) of a column: value and the lowest frame that attains it (warp-cooperative)
__device__ void range_max(const float* col, int t_lo, int t_hi, float* out_v, int* out_t) {
  const int lane = threadIdx.x & 31;
  float bv = -INFINITY;
  int bt = 0x7fffffff;
  for (int t = t_lo + lane; t < t_hi; t += 32) {
    float v = col[t];
    if (v > bv) {
      bv = v;
      bt = t;
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    int ot = __shfl_xor_sync(0xffffffffu, bt, o);
    if (ov > bv || (ov == bv && ot < bt)) {
      bv = ov;
      bt = ot;
    }
  }
  *out_v = bv;
  *out_t = bt;
}

// block maxima of blocks [b_lo, b_hi] of one column, then the column maximum from all its block entries
__device__ void refresh_column(const float* col, int T, float* bmax, int* barg, int nblk, int b_lo, int b_hi, float* out_v,
                               int* out_t) {
  const int lane = threadIdx.x & 31;
  for (int b = b_lo; b <= b_hi; ++b) {
    float v;
    int t;
    range_max(col, b * kDecBlk, min(T, (b + 1) * kDecBlk), &v, &t);
    if (lane == 0) {
      bmax[b] = v;
      barg[b] = t;
    }
  }
  __syncwarp();
  float bv = -INFINITY;
  int bt = 0x7fffffff;
  for (int b = lane; b < nblk; b += 32) {  // blocks ascend with the frame index: ties keep the lower block
    const float v = bmax[b];
    if (v > bv) {
      bv = v;
      bt = barg[b];
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    int ot = __shfl_xor_sync(0xffffffffu, bt, o);
    if (ov > bv || (ov == bv && ot < bt)) {
      bv = ov;
      bt = ot;
    }
  }
  *out_v = bv;
  *out_t = bt;
}

// kGrid: blockIdx.y is a setting of g, with its own parameters, E, block maxima and note slots / count
// (setting * n_files + file), reading its candidate group's bitmap
template <bool kGrid>
__global__ void __launch_bounds__(kSeqThreads) decode_seq_kernel(
    const long long* __restrict__ frame_off, float* __restrict__ energy, const unsigned int* __restrict__ candbits,
    const long long* __restrict__ slot_off, int* __restrict__ note_count, int* __restrict__ note_start,
    int* __restrict__ note_end, int* __restrict__ note_pitch, int* __restrict__ overflow, float* __restrict__ blk_max,
    int* __restrict__ blk_arg, DecodeParamsDev p, DecodeGridDev g) {
  const int file = blockIdx.x;
  if constexpr (kGrid) {
    const int s = blockIdx.y;
    p = g.setting[s].p;
    energy += s * g.e_stride;
    candbits += g.setting[s].cand * g.cand_stride;
    blk_max += s * g.blk_stride;
    blk_arg += s * g.blk_stride;
    slot_off += (long long)s * g.n_files;
    note_count += (long long)s * g.n_files;
  }
  const long long base = frame_off[file];
  const int T = (int)(frame_off[file + 1] - base);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const long long slot0 = slot_off[file];
  const int cap = (int)(slot_off[file + 1] - slot0);
  float* E = energy + base * kPitches;

  __shared__ float s_cmax[kPitches];
  __shared__ int s_carg[kPitches];
  __shared__ int s_pick[5];  // tm, f, done, first and last frame the iteration changed
  __shared__ int s_count;

  int count = 0;
  if (T <= 0) {
    if (threadIdx.x == 0) note_count[file] = 0;
    return;
  }

  // ---------------- onset loop (warp 0) ----------------
  if (warp == 0) {
    const long long c_lo = base * kPitches;             // first cell of this file
    const long long c_hi = c_lo + (long long)T * kPitches;  // one past the last
    long long w_hi = (c_hi - 1) >> 5, w_lo = c_lo >> 5;
    for (long long wbase = w_hi; wbase >= w_lo; wbase -= 32) {
      // lanes look at words wbase, wbase-1, ... (descending)
      long long w = wbase - lane;
      unsigned int bits = 0u;
      if (w >= w_lo) {
        bits = candbits[w];
        long long first = w << 5;
        if (first < c_lo) bits &= 0xffffffffu << (int)(c_lo - first);
        if (first + 32 > c_hi) bits &= 0xffffffffu >> (int)(first + 32 - c_hi);
      }
      unsigned int nonzero = __ballot_sync(0xffffffffu, bits != 0u);
      while (nonzero) {
        int src = __ffs(nonzero) - 1;  // lowest lane = highest word
        nonzero &= nonzero - 1;
        unsigned int wb = __shfl_sync(0xffffffffu, bits, src);
        long long wcell = (wbase - src) << 5;
        while (wb) {
          int bit = 31 - __clz(wb);
          wb &= ~(1u << bit);
          long long cell = wcell + bit - c_lo;
          int t0 = (int)(cell / kPitches);
          int f = (int)(cell - (long long)t0 * kPitches);
          if (t0 >= T - 1) continue;
          int k;
          int i = scan_run(E + (long long)f * T, t0 + 1, +1, T - 1, p.energy_tol, p.frame_thresh, &k);
          i -= k;
          if (i - t0 <= p.min_note_len) continue;
          zero_cols(E, T, f, t0, i);
          __syncwarp();
          if (lane == 0) {
            if (count < cap) {
              note_start[slot0 + count] = t0;
              note_end[slot0 + count] = i;
              note_pitch[slot0 + count] = f + 21;
            } else {
              *overflow = 1;
            }
          }
          ++count;
        }
      }
    }
    if (lane == 0) s_count = count;
  }
  __syncthreads();
  count = s_count;

  // ---------------- melodia loop ----------------
  if (p.melodia) {
    // this file's block entries: [88][nblk] behind those of the files before it (see decode_block_slots)
    const int nblk = (T + kDecBlk - 1) / kDecBlk;
    float* bmax = blk_max + (size_t)kPitches * (size_t)(base / kDecBlk + file);
    int* barg = blk_arg + (size_t)kPitches * (size_t)(base / kDecBlk + file);
    for (int f = warp; f < kPitches; f += kSeqThreads / 32) {
      float v;
      int t;
      refresh_column(E + (long long)f * T, T, bmax + (size_t)f * nblk, barg + (size_t)f * nblk, nblk, 0, nblk - 1, &v, &t);
      if (lane == 0) {
        s_cmax[f] = v;
        s_carg[f] = t;
      }
    }
    while (true) {
      __syncthreads();
      if (warp == 0) {
        float bv = -INFINITY;
        int bt = 0x7fffffff, bf = 0x7fffffff;
        for (int f = lane; f < kPitches; f += 32) {
          float v = s_cmax[f];
          int t = s_carg[f];
          if (v > bv || (v == bv && (t < bt || (t == bt && f < bf)))) {
            bv = v;
            bt = t;
            bf = f;
          }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          int ot = __shfl_xor_sync(0xffffffffu, bt, o);
          int of = __shfl_xor_sync(0xffffffffu, bf, o);
          if (ov > bv || (ov == bv && (ot < bt || (ot == bt && of < bf)))) {
            bv = ov;
            bt = ot;
            bf = of;
          }
        }
        bool go = (double)bv > p.frame_thresh;
        if (go) {
          const int tm = bt, f = bf;
          float* col = E + (long long)f * T;
          if (lane == 0) col[tm] = 0.f;
          __syncwarp();
          int k;
          int i = scan_run(col, tm + 1, +1, T - 1, p.energy_tol, p.frame_thresh, &k);
          zero_cols(E, T, f, tm + 1, i);
          const int t_end = i - 1 - k;
          __syncwarp();
          i = scan_run(col, tm - 1, -1, 0, p.energy_tol, p.frame_thresh, &k);
          zero_cols(E, T, f, i + 1, tm);
          const int t_start = i + 1 + k;
          __syncwarp();
          if (t_end - t_start > p.min_note_len) {
            if (lane == 0) {
              if (count < cap) {
                note_start[slot0 + count] = t_start;
                note_end[slot0 + count] = t_end;
                note_pitch[slot0 + count] = f + 21;
              } else {
                *overflow = 1;
              }
            }
            ++count;
          }
          if (lane == 0) {
            s_pick[0] = tm;
            s_pick[1] = f;
            // zeroed on three columns: [backward exit + 1, forward exit), i.e. within energy_tol of the note's ends
            // (64-bit: energy_tol may be up to INT_MAX, and t_end + energy_tol must not wrap below tm)
            const long long tol = p.energy_tol;
            s_pick[3] = (int)max(0LL, min((long long)t_start - tol, (long long)tm));
            s_pick[4] = (int)min((long long)T - 1, max((long long)t_end + tol, (long long)tm));
          }
        }
        if (lane == 0) s_pick[2] = go ? 0 : 1;
      }
      __syncthreads();
      if (s_pick[2]) break;
      // refresh the maxima of the three touched columns
      {
        const int f = s_pick[1] - 1 + warp;
        if (warp < 3 && f >= 0 && f < kPitches) {
          float v;
          int t;
          refresh_column(E + (long long)f * T, T, bmax + (size_t)f * nblk, barg + (size_t)f * nblk, nblk,
                         s_pick[3] / kDecBlk, s_pick[4] / kDecBlk, &v, &t);
          if (lane == 0) {
            s_cmax[f] = v;
            s_carg[f] = t;
          }
        }
      }
    }
  }
  if (threadIdx.x == 0) note_count[file] = count;
}

void launch_decode_notes(const float* note, const float* onset, const DecodeBuffers& b, int n_files,
                         long long total_frames, const DecodeParamsDev& p, cudaStream_t st) {
  const long long cells = total_frames * kPitches;
  cudaMemsetAsync(b.max_onset, 0, sizeof(unsigned int) * n_files, st);
  cudaMemsetAsync(b.max_fd, 0, sizeof(unsigned long long) * n_files, st);
  if (cells > 0) {
    const int threads = 256;
    const unsigned int blocks = (unsigned int)((total_frames + kTileFrames - 1) / kTileFrames);
    decode_prep_kernel<false><<<blocks, threads, 0, st>>>(note, onset, b.frame_off, n_files, b.energy, b.max_onset,
                                                          b.max_fd, p.lo_col, p.hi_col, DecodeGridDev{});
    decode_cand_kernel<false><<<blocks, threads, 0, st>>>(note, onset, b.frame_off, n_files, b.max_onset, b.max_fd,
                                                          b.candbits, p.lo_col, p.hi_col, p.infer_onsets, p.onset_thresh,
                                                          nullptr, DecodeGridDev{});
  }
  decode_seq_kernel<false><<<n_files, kSeqThreads, 0, st>>>(b.frame_off, b.energy, b.candbits, b.slot_off, b.note_count,
                                                            b.note_start, b.note_end, b.note_pitch, b.overflow, b.blk_max,
                                                            b.blk_arg, p, DecodeGridDev{});
}

long long decode_cand_words(long long total_frames) { return total_frames * kPitches / 32 + 2; }

// The launches of launch_decode_notes for a chunk of settings: prep once per prep group, candidates once per candidate
// group, the loops once per (file, setting).  b.max_onset / b.max_fd hold n_prep * n_files entries.
void launch_decode_grid(const float* note, const float* onset, const DecodeBuffers& b, int n_files,
                        long long total_frames, const DecodeGridDev& g, int n_prep, int n_cand, int n_settings,
                        cudaStream_t st) {
  cudaMemsetAsync(b.max_onset, 0, sizeof(unsigned int) * n_files * n_prep, st);
  cudaMemsetAsync(b.max_fd, 0, sizeof(unsigned long long) * n_files * n_prep, st);
  if (total_frames > 0) {
    const unsigned int blocks = (unsigned int)((total_frames + kTileFrames - 1) / kTileFrames);
    decode_prep_kernel<true><<<dim3(blocks, n_prep), 256, 0, st>>>(note, onset, b.frame_off, n_files, b.energy,
                                                                   b.max_onset, b.max_fd, 0, 0, g);
    decode_cand_kernel<true><<<dim3(blocks, n_cand), 256, 0, st>>>(note, onset, b.frame_off, n_files, b.max_onset,
                                                                   b.max_fd, b.candbits, 0, 0, 0, 0.0, nullptr, g);
  }
  decode_seq_kernel<true><<<dim3(n_files, n_settings), kSeqThreads, 0, st>>>(
      b.frame_off, b.energy, b.candbits, b.slot_off, b.note_count, b.note_start, b.note_end, b.note_pitch, b.overflow,
      b.blk_max, b.blk_arg, DecodeParamsDev{}, g);
}

// float64 inferred onsets of a batch of files (reference: note_creation.py:289-311): the two cell-parallel kernels of the
// decode, with the candidate kernel also writing the onset matrix it peak-picks on.
void launch_infer_onsets(const float* note, const float* onset, const DecodeBuffers& b, int n_files, long long total_frames,
                         double* out64, cudaStream_t st) {
  cudaMemsetAsync(b.max_onset, 0, sizeof(unsigned int) * n_files, st);
  cudaMemsetAsync(b.max_fd, 0, sizeof(unsigned long long) * n_files, st);
  if (total_frames <= 0) return;
  const unsigned int blocks = (unsigned int)((total_frames + kTileFrames - 1) / kTileFrames);
  decode_prep_kernel<false><<<blocks, 256, 0, st>>>(note, onset, b.frame_off, n_files, b.energy, b.max_onset, b.max_fd,
                                                    0, kPitches, DecodeGridDev{});
  decode_cand_kernel<false><<<blocks, 256, 0, st>>>(note, onset, b.frame_off, n_files, b.max_onset, b.max_fd, b.candbits,
                                                    0, kPitches, 1, 0.0, out64, DecodeGridDev{});
}

// ------------------------------------------------------------------------------------------------
// Amplitude + pitch bends.
// ------------------------------------------------------------------------------------------------
// float32 pairwise summation exactly as NumPy's add.reduce inner loop does it (blocks of 8 partial sums up to
// 128 elements, recursive halving above), so that amplitude == np.mean(frames[start:end, f]) bit for bit.
__device__ float np_pairwise_sum(const float* a, int n, int stride) {
  if (n < 8) {
    float res = 0.f;
    for (int i = 0; i < n; ++i) res = __fadd_rn(res, a[(long long)i * stride]);
    return res;
  } else if (n <= 128) {
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[(long long)j * stride];
    int i;
    for (i = 8; i < n - (n % 8); i += 8) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[(long long)(i + j) * stride]);
    }
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, a[(long long)i * stride]);
    return res;
  } else {
    int n2 = n / 2;
    n2 -= n2 % 8;
    return __fadd_rn(np_pairwise_sum(a, n2, stride), np_pairwise_sum(a + (long long)n2 * stride, n - n2, stride));
  }
}

__global__ void note_finish_kernel(const float* __restrict__ note, const float* __restrict__ contour,
                                   const long long* __restrict__ note_base, const int* __restrict__ start,
                                   const int* __restrict__ end, const int* __restrict__ pitch, float* __restrict__ amp,
                                   const int* __restrict__ bend_off, int* __restrict__ bends, int n_notes,
                                   int with_bends, const double* __restrict__ gauss) {
  const int warps_per_block = blockDim.x >> 5;
  const int n = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= n_notes) return;
  const long long base = note_base[n];
  const int t0 = start[n], t1 = end[n], col = pitch[n] - 21;
  if (lane == 0) {
    const int len = t1 - t0;
    float s = np_pairwise_sum(note + (base + t0) * kPitches + col, len, kPitches);
    amp[n] = __fdiv_rn(s, (float)len);
  }
  if (!with_bends || bend_off[n + 1] == bend_off[n]) return;  // empty: a grid setting without pitch bends
  // reference: note_creation.py:198-218 ; contour bin of the note = 3*(pitch-21)
  const int c = 3 * col;
  const int lo = max(c - 25, 0);
  const int hi = min(kContourBins, c + 26);
  const int g0 = max(0, 25 - c);       // first Gaussian tap used
  const int shift = 25 - g0;
  const int width = hi - lo;           // <= 51
  int* out = bends + bend_off[n];
  // one frame per lane (a note has 11 .. a few dozen frames): every lane walks its frame's <= 51 bins in ascending order
  // and keeps the first maximum — np.argmax semantics without any cross-lane reduction
  for (int t = t0 + lane; t < t1; t += 32) {
    const float* row = contour + (base + t) * kContourBins + lo;
    double bv = -INFINITY;  // np.argmax semantics for any input (callers may pass contours < 0)
    int bi = 0;
#pragma unroll 4
    for (int j = 0; j < width; ++j) {
      const double v = __dmul_rn((double)__ldg(row + j), gauss[g0 + j]);
      if (v > bv) {
        bv = v;
        bi = j;
      }
    }
    out[t - t0] = bi - shift;
  }
}

void launch_note_finish(const float* note, const float* contour, const long long* note_base, const int* start,
                        const int* end, const int* pitch, float* amp, const int* bend_off, int* bends, int n_notes,
                        int with_bends, const double* gauss, cudaStream_t st) {
  if (n_notes <= 0) return;
  const int threads = 128;
  const int blocks = (n_notes + 3) / 4;
  note_finish_kernel<<<blocks, threads, 0, st>>>(note, contour, note_base, start, end, pitch, amp, bend_off, bends,
                                                 n_notes, with_bends, gauss);
}

}  // namespace bp
