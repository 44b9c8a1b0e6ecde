// Stream group (bp_stream_group_*, include/bp_b200.h): the kernels that let one device pass serve many streams — the
// copies between the per-stream regions of the group's arenas, the kept frames of each window into its stream's rows,
// the quiet scan of every stream in one launch and the start filter of a batch of segments.
#include "kernels.cuh"

namespace bp {

constexpr int kGroupScanThreads = 256;

// Segment k copies rows [src_row, src_row + rows) of array `arr` to rows dst_row .. (width[arr] elements per row).
__device__ __forceinline__ void copy_segment(const GroupCopySeg s, const GroupCopyArrays& a) {
  const void* vs = nullptr;
  void* vd = nullptr;
  int w = 0, b = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k)  // constant indices: the kernel parameters stay in the parameter space
    if (k == s.arr) vs = a.src[k], vd = a.dst[k], w = a.width[k], b = a.bytes[k];
  const long long n = s.rows * w;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (b == 4) {
    const float* src = static_cast<const float*>(vs) + s.src_row * w;
    float* dst = static_cast<float*>(vd) + s.dst_row * w;
    for (long long i = i0; i < n; i += step) dst[i] = src[i];
  } else {
    const unsigned char* src = static_cast<const unsigned char*>(vs) + s.src_row * w;
    unsigned char* dst = static_cast<unsigned char*>(vd) + s.dst_row * w;
    for (long long i = i0; i < n; i += step) dst[i] = src[i];
  }
}

__global__ void group_copy_kernel(const GroupCopySeg* __restrict__ segs, int n_segs, GroupCopyArrays a) {
  for (int k = blockIdx.y; k < n_segs; k += gridDim.y) copy_segment(segs[k], a);
}

void launch_group_copy(const GroupCopySeg* segs, int n_segs, long long max_elems, const GroupCopyArrays& a,
                       cudaStream_t st) {
  if (n_segs <= 0 || max_elems <= 0) return;
  const unsigned int bx = (unsigned int)std::min<long long>((max_elems + 255) / 256, 1024);
  group_copy_kernel<<<dim3(bx, (unsigned int)std::min(n_segs, 65535)), 256, 0, st>>>(segs, n_segs, a);
}

// Window blockIdx.y of a forward chunk: its 142 kept frames, pm / cm frames y * 142 .. of the chunk's unwrapped
// posteriorgrams (frame stride `stride`), to rows dst_row[y] .. of the row-major arenas.  blockIdx.z 0..2: note pitches
// 32 z .., 3..5 onset, 6: contour.
__global__ void group_unwrap_kernel(const float* __restrict__ pm_note, const float* __restrict__ pm_onset,
                                    const float* __restrict__ cm, long long stride, const long long* __restrict__ dst_row,
                                    float* __restrict__ note, float* __restrict__ onset, float* __restrict__ contour) {
  const long long src0 = (long long)blockIdx.y * kHopFrames, d0 = dst_row[blockIdx.y];
  const int i0 = blockIdx.x * 32;
  const int z = blockIdx.z;
  if (z < 6) {
    __shared__ float tile[32][33];
    const float* pm = z < 3 ? pm_note : pm_onset;
    float* rows = z < 3 ? note : onset;
    const int f0 = (z % 3) * 32;
    for (int c = threadIdx.y; c < 32; c += 8) {
      const int i = i0 + threadIdx.x, f = f0 + c;
      tile[c][threadIdx.x] = (i < kHopFrames && f < kPitches) ? pm[(long long)f * stride + src0 + i] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += 8) {
      const int i = i0 + r, f = f0 + threadIdx.x;
      if (i < kHopFrames && f < kPitches) rows[(d0 + i) * kPitches + f] = tile[threadIdx.x][r];
    }
    return;
  }
  // contour: 8-bin chunk c of frame i is 8 consecutive floats on both sides
  constexpr int kChunks = kContourBins / 8;
  for (int e = threadIdx.y * 32 + threadIdx.x; e < 32 * kChunks; e += 256) {
    const int r = e % 32, c = e / 32, i = i0 + r;
    if (i >= kHopFrames) continue;
    const float4* s = reinterpret_cast<const float4*>(cm + ((long long)c * stride + src0 + i) * 8);
    float4* d = reinterpret_cast<float4*>(contour + (d0 + i) * kContourBins + c * 8);
    d[0] = s[0];
    d[1] = s[1];
  }
}

void launch_group_unwrap(const float* pm_note, const float* pm_onset, const float* cm, long long stride,
                         const long long* dst_row, int n_windows, float* note, float* onset, float* contour,
                         bool with_contour, cudaStream_t st) {
  if (n_windows <= 0) return;
  const dim3 grid((kHopFrames + 31) / 32, n_windows, with_contour ? 7 : 6);
  group_unwrap_kernel<<<grid, dim3(32, 8), 0, st>>>(pm_note, pm_onset, cm, stride, dst_row, note, onset, contour);
}

// stream_scan_kernel for every job at once: blockIdx.y is the job, frames are global and row = frame + shift.  The last
// CTA of a job to finish looks for that job's first cut.
__global__ void __launch_bounds__(kGroupScanThreads) group_scan_kernel(const GroupScanJob* __restrict__ jobs,
                                                                       const float* __restrict__ note, int lo, int hi,
                                                                       double frame_thresh, unsigned char* quiet,
                                                                       long long w, long long* __restrict__ out,
                                                                       unsigned int* done) {
  const GroupScanJob J = jobs[blockIdx.y];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int kWarps = kGroupScanThreads / 32;
  for (long long t = J.flag_from + (long long)blockIdx.x * kWarps + warp; t < J.n; t += (long long)gridDim.x * kWarps) {
    bool q = true;
    for (int f = lane; f < kPitches; f += 32) {
      const float v = (f >= lo && f < hi) ? note[(t + J.shift) * kPitches + f] : 0.f;
      q = q && ((double)v < frame_thresh);
    }
    const bool all = __all_sync(0xffffffffu, q);
    if (lane == 0) quiet[t + J.shift] = all ? 1 : 0;
  }
  __threadfence();
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    s_last = atomicAdd(done + blockIdx.y, 1u) == gridDim.x - 1;
    if (s_last) done[blockIdx.y] = 0u;  // ready for the next launch
  }
  __syncthreads();
  if (!s_last) return;

  __shared__ long long s_warp[kWarps];
  __shared__ long long s_hit;
  const volatile unsigned char* vq = quiet;
  long long L = J.last;
  long long* o = out + 2 * blockIdx.y;
  for (long long base = J.from; base < J.n; base += kGroupScanThreads) {
    const long long t = base + threadIdx.x;
    const bool valid = t < J.n;
    const bool q = valid && vq[t + J.shift];
    long long m = (valid && !q) ? t : kStreamNoRun;  // inclusive prefix maximum of the loud frames up to t
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const long long v = __shfl_up_sync(0xffffffffu, m, k);
      if (lane >= k) m = max(m, v);
    }
    if (lane == 31) s_warp[warp] = m;
    if (threadIdx.x == 0) s_hit = LLONG_MAX;
    __syncthreads();
    for (int i = 0; i < warp; ++i) m = max(m, s_warp[i]);
    const long long Lt = max(L, m);
    if (q && t - Lt == w) atomicMin((unsigned long long*)&s_hit, (unsigned long long)t);  // t >= 0
    for (int i = 0; i < kWarps; ++i) L = max(L, s_warp[i]);
    __syncthreads();
    if (s_hit != LLONG_MAX) {
      if (threadIdx.x == 0) {
        o[0] = s_hit;
        o[1] = L;
      }
      return;
    }
    __syncthreads();  // s_warp / s_hit are rewritten by the next chunk
  }
  if (threadIdx.x == 0) {
    o[0] = -1;
    o[1] = L;
  }
}

void launch_group_scan(const GroupScanJob* jobs, int n_jobs, long long max_rows, const float* note, int lo, int hi,
                       double frame_thresh, unsigned char* quiet, long long w, long long* out, unsigned int* done,
                       cudaStream_t st) {
  constexpr int kWarps = kGroupScanThreads / 32;
  const long long want = (max_rows + kWarps - 1) / kWarps;
  const unsigned int blocks = (unsigned int)std::max(1LL, std::min(want, 4096LL));
  group_scan_kernel<<<dim3(blocks, (unsigned int)n_jobs), kGroupScanThreads, 0, st>>>(jobs, note, lo, hi, frame_thresh,
                                                                                      quiet, w, out, done);
}

// stream_compact_kernel for a batch of segments: warp j handles segments j, j + 32, ...; pass 1 counts each segment's
// kept notes, thread 0 turns the counts into offsets note_off[0 .. n], pass 2 writes them in generation order.
__global__ void __launch_bounds__(1024) group_compact_kernel(const GroupKeep* __restrict__ keep, int n_segs,
                                                             const long long* __restrict__ slot_off,
                                                             const int* __restrict__ count, const int* __restrict__ s_start,
                                                             const int* __restrict__ s_end, const int* __restrict__ s_pitch,
                                                             int* __restrict__ start, int* __restrict__ end,
                                                             int* __restrict__ pitch, long long* __restrict__ note_base,
                                                             int* __restrict__ note_off) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  for (int pass = 0; pass < 2; ++pass) {
    for (int j = warp; j < n_segs; j += n_warps) {
      const GroupKeep K = keep[j];
      const long long s0 = slot_off[j];
      const int n = (int)min((long long)count[j], slot_off[j + 1] - s0);  // an overflowed decode is run again
      int k = 0;
      const int d0 = pass ? note_off[j] : 0;
      for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const int t0 = i < n ? s_start[s0 + i] : -1;
        const bool kp = i < n && t0 >= K.keep_lo && t0 < K.keep_hi;
        const unsigned int bits = __ballot_sync(0xffffffffu, kp);
        if (pass && kp) {
          const int d = d0 + k + __popc(bits & ((1u << lane) - 1u));
          start[d] = K.frame0 + t0;
          end[d] = K.frame0 + s_end[s0 + i];
          pitch[d] = s_pitch[s0 + i];
          note_base[d] = K.base;
        }
        k += __popc(bits);
      }
      if (!pass && lane == 0) note_off[j + 1] = k;
    }
    __syncthreads();
    if (!pass && threadIdx.x == 0) {
      note_off[0] = 0;
      for (int j = 0; j < n_segs; ++j) note_off[j + 1] += note_off[j];
    }
    __syncthreads();
  }
}

void launch_group_compact(const GroupKeep* keep, int n_segs, const long long* slot_off, const int* count,
                          const int* s_start, const int* s_end, const int* s_pitch, int* start, int* end, int* pitch,
                          long long* note_base, int* note_off, cudaStream_t st) {
  group_compact_kernel<<<1, 1024, 0, st>>>(keep, n_segs, slot_off, count, s_start, s_end, s_pitch, start, end, pitch,
                                           note_base, note_off);
}

}  // namespace bp
