// Note stream (bp_stream_*, include/bp_b200.h): where to cut the held frames, and which notes of a segment to keep.
// The segments themselves go through the decode kernels of decode.cu as a batch of one file.
#include "kernels.cuh"

namespace bp {

constexpr int kScanThreads = 256;

// One warp per row sets quiet[t] (a ballot over the 88 columns); the last CTA to finish then looks for the first cut.
__global__ void __launch_bounds__(kScanThreads) stream_scan_kernel(const float* __restrict__ note, long long flag_from,
                                                                   long long n, int lo, int hi, double frame_thresh,
                                                                   unsigned char* quiet, long long from, long long last,
                                                                   long long w, long long* __restrict__ out,
                                                                   unsigned int* done) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = flag_from + (long long)blockIdx.x * (kScanThreads / 32) + warp; t < n;
       t += (long long)gridDim.x * (kScanThreads / 32)) {
    bool q = true;
    for (int f = lane; f < kPitches; f += 32) {
      const float v = (f >= lo && f < hi) ? note[t * kPitches + f] : 0.f;
      q = q && ((double)v < frame_thresh);
    }
    const bool all = __all_sync(0xffffffffu, q);
    if (lane == 0) quiet[t] = all ? 1 : 0;
  }
  __threadfence();
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    s_last = atomicAdd(done, 1u) == gridDim.x - 1;
    if (s_last) *done = 0u;  // ready for the next launch
  }
  __syncthreads();
  if (!s_last) return;

  __shared__ long long s_warp[kScanThreads / 32];
  __shared__ long long s_hit;
  const volatile unsigned char* vq = quiet;
  long long L = last;
  for (long long base = from; base < n; base += kScanThreads) {
    const long long t = base + threadIdx.x;
    const bool valid = t < n;
    const bool q = valid && vq[t];
    // inclusive prefix maximum of the loud rows up to t
    long long m = (valid && !q) ? t : kStreamNoRun;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long v = __shfl_up_sync(0xffffffffu, m, o);
      if (lane >= o) m = max(m, v);
    }
    if (lane == 31) s_warp[warp] = m;
    if (threadIdx.x == 0) s_hit = LLONG_MAX;
    __syncthreads();
    for (int i = 0; i < warp; ++i) m = max(m, s_warp[i]);
    const long long Lt = max(L, m);
    if (q && t - Lt == w) atomicMin((unsigned long long*)&s_hit, (unsigned long long)t);  // t >= 0
    for (int i = 0; i < kScanThreads / 32; ++i) L = max(L, s_warp[i]);
    __syncthreads();
    if (s_hit != LLONG_MAX) {
      if (threadIdx.x == 0) {
        out[0] = s_hit;
        out[1] = L;
      }
      return;
    }
    __syncthreads();  // s_warp / s_hit are rewritten by the next chunk
  }
  if (threadIdx.x == 0) {
    out[0] = -1;
    out[1] = L;
  }
}

void launch_stream_scan(const float* note, long long flag_from, long long n, int lo, int hi, double frame_thresh,
                        unsigned char* quiet, long long from, long long last, long long w, long long* out,
                        unsigned int* done, cudaStream_t st) {
  const long long rows = n > flag_from ? n - flag_from : 0;
  const long long want = (rows + kScanThreads / 32 - 1) / (kScanThreads / 32);
  const unsigned int blocks = (unsigned int)std::max(1LL, std::min(want, 4096LL));
  stream_scan_kernel<<<blocks, kScanThreads, 0, st>>>(note, flag_from, n, lo, hi, frame_thresh, quiet, from, last, w, out,
                                                      done);
}

// One warp: a ballot per 32 notes keeps the generation order.
__global__ void stream_compact_kernel(const int* __restrict__ count, const int* __restrict__ s_start,
                                      const int* __restrict__ s_end, const int* __restrict__ s_pitch, int keep_lo,
                                      int keep_hi, int frame0, long long base, int* __restrict__ start,
                                      int* __restrict__ end, int* __restrict__ pitch, long long* __restrict__ note_base,
                                      int* __restrict__ kept) {
  const int lane = threadIdx.x;
  const int n = *count;
  int k = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const int t0 = i < n ? s_start[i] : -1;
    const bool keep = i < n && t0 >= keep_lo && t0 < keep_hi;
    const unsigned int bits = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int j = k + __popc(bits & ((1u << lane) - 1u));
      start[j] = frame0 + t0;
      end[j] = frame0 + s_end[i];
      pitch[j] = s_pitch[i];
      note_base[j] = base;
    }
    k += __popc(bits);
  }
  if (lane == 0) *kept = k;
}

void launch_stream_compact(const int* count, const int* s_start, const int* s_end, const int* s_pitch, int keep_lo,
                           int keep_hi, int frame0, long long base, int* start, int* end, int* pitch, long long* note_base,
                           int* kept, cudaStream_t st) {
  stream_compact_kernel<<<1, 32, 0, st>>>(count, s_start, s_end, s_pitch, keep_lo, keep_hi, frame0, base, start, end,
                                          pitch, note_base, kept);
}

}  // namespace bp
