// Audio ingest on the device: PCM samples of any rate / channel count -> mono float32 at 22 050 Hz.
// Replaces `librosa.load(path, sr=22050, mono=True)` minus the container decode (reference:
// basic_pitch/inference.py:239): sample-format conversion, channel mean and a rational polyphase resampler in one kernel,
// so that a file crosses PCIe once, as the PCM it was stored as (2 bytes per sample for 16-bit audio).
//
// Resampler = the Kaiser-windowed FIR of basic_pitch_b200/audio_io.py (pass band 0.913 x Nyquist of the lower rate, 125 dB
// stop band: the shape of soxr's HQ preset that librosa uses), applied exactly like scipy.signal.resample_poly:
//   y[k] = sum_i x[i] * up * h[k * down + half - i * up],   n_out = ceil(n_in * up / down),  zero outside the signal
// in polyphase form: phase p = (k * down + half) % up, newest input i_max = (k * down + half) / up,
//   y[k] = sum_j hp[p][j] * x[i_max - j],   hp[p][j] = up * h[p + j * up].
// A CTA produces 256 consecutive outputs from an input span staged (converted and down-mixed) in shared memory.
#include <cmath>
#include <map>
#include <mutex>
#include <vector>

#include "kernels.cuh"

namespace bp {

namespace {
constexpr int kOutPerCta = 256;

struct Resampler {
  int up = 1, down = 1, half = 0, taps_per_phase = 0;
  float* d_hp = nullptr;  // [up][taps_per_phase]
};

double bessel_i0(double x) {  // power series, converges quickly for the arguments of a 125 dB Kaiser window (beta ~ 12.8)
  double sum = 1.0, term = 1.0;
  const double q = x * x / 4.0;
  for (int k = 1; k < 200; ++k) {
    term *= q / ((double)k * k);
    sum += term;
    if (term < 1e-18 * sum) break;
  }
  return sum;
}

constexpr double kStopDb = 125.0;

// taps of the low-pass for the reduced ratio up / down: scipy.signal.kaiserord(125, width), made odd
int filter_length(int up, int down) {
  const int m = std::max(up, down);
  const double pass_edge = 0.913 / m, stop_edge = 1.0 / m, width = stop_edge - pass_edge;
  return (int)std::ceil((kStopDb - 7.95) / 2.285 / (M_PI * width) + 1.0) | 1;
}

// scipy.signal.kaiserord(125, width) + firwin(numtaps | 1, cutoff, window=("kaiser", beta)), as audio_io._resample_filter
std::vector<double> design_filter(int up, int down) {
  const int m = std::max(up, down);
  const double pass_edge = 0.913 / m, stop_edge = 1.0 / m;
  const double A = kStopDb, beta = 0.1102 * (A - 8.7);
  const int numtaps = filter_length(up, down);
  const double cutoff = 0.5 * (pass_edge + stop_edge), alpha = 0.5 * (numtaps - 1);
  std::vector<double> h(numtaps);
  double sum = 0.0;
  const double i0b = bessel_i0(beta);
  for (int n = 0; n < numtaps; ++n) {
    const double t = n - alpha, x = cutoff * t;
    const double sinc = (x == 0.0) ? 1.0 : std::sin(M_PI * x) / (M_PI * x);
    const double r = t / alpha;
    const double w = bessel_i0(beta * std::sqrt(std::max(0.0, 1.0 - r * r))) / i0b;
    h[n] = cutoff * sinc * w;
    sum += h[n];
  }
  for (double& v : h) v /= sum;  // unit gain at DC
  return h;
}

std::mutex g_mu;
std::map<long long, Resampler> g_resamplers[64];  // per device, keyed by up << 32 | down

template <typename T>
__device__ __forceinline__ float to_float(T v);
template <>
__device__ __forceinline__ float to_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_float<short>(short v) { return (float)v / 32768.f; }
template <>
__device__ __forceinline__ float to_float<int>(int v) { return (float)v / 2147483648.f; }
template <>
__device__ __forceinline__ float to_float<unsigned char>(unsigned char v) { return ((float)v - 128.f) / 128.f; }
// 24-bit WAV as stored: three bytes, little-endian, two's complement, 1-byte aligned.  v / 2^23 equals
// to_float<int>(v << 8), the value of the left-justified int32 that scipy reads the same sample as.
struct s24 {
  unsigned char b[3];
};
template <>
__device__ __forceinline__ float to_float<s24>(s24 v) {
  const int x = ((int)((unsigned)v.b[0] << 8 | (unsigned)v.b[1] << 16 | (unsigned)v.b[2] << 24)) >> 8;
  return (float)x / 8388608.f;
}
// float64 WAV: rounded to float32 first, as the host's astype(np.float32) does, then format 0's path.
template <>
__device__ __forceinline__ float to_float<double>(double v) { return __double2float_rn(v); }

// numpy's pairwise_sum of n >= 1 converted values: below 8 a sequential sum from +0, up to 128 eight interleaved
// accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) then the tail in order
template <typename T>
__device__ __forceinline__ float pairwise_block(const T* p, int n) {
  if (n < 8) {
    float s = 0.f;
    for (int c = 0; c < n; ++c) s = __fadd_rn(s, to_float<T>(p[c]));
    return s;
  }
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = to_float<T>(p[j]);
  int c = 8;
  for (; c + 8 <= n; c += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], to_float<T>(p[c + j]));
  float s = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                      __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; c < n; ++c) s = __fadd_rn(s, to_float<T>(p[c]));
  return s;
}

// above 128 numpy splits at n2 = n / 2 - (n / 2) % 8 and adds the two halves' sums; walked here in post-order with an
// explicit stack.  A split leaves at most n / 2 + 7, so any int count takes at most 24 (65 535 channels, the most a WAV
// file can have, 9)
template <typename T>
__device__ float pairwise_sum(const T* p, int n) {
  constexpr int kDepth = 32;
  int right_off[kDepth], right_n[kDepth];
  float left[kDepth];
  bool left_done[kDepth];
  int sp = 0, off = 0;
  for (;;) {
    while (n > 128) {  // descend into the left half, remember the right one
      const int n2 = n / 2 - (n / 2) % 8;
      right_off[sp] = off + n2, right_n[sp] = n - n2, left_done[sp] = false;
      ++sp;
      n = n2;
    }
    float v = pairwise_block<T>(p + off, n);
    while (sp > 0 && left_done[sp - 1]) v = __fadd_rn(left[--sp], v);  // both halves done: combine and climb
    if (sp == 0) return v;
    left[sp - 1] = v, left_done[sp - 1] = true;
    off = right_off[sp - 1], n = right_n[sp - 1];
  }
}

// mono sample i of the interleaved PCM: numpy's float32 mean over the channel axis, `x.mean(axis=1, dtype=float32)`:
// +0 plus the pairwise sum (a frame of -0 gives +0), divided by the integer count in float64 and rounded to float32
// (the same as a float32 division while the count is exact in float32, i.e. up to 2^24 channels)
template <typename T>
__device__ __forceinline__ float mono_sample(const T* pcm, long long i, int channels) {
  const T* p = pcm + i * channels;
  if (channels == 1) return to_float<T>(p[0]);
  const float s = channels <= 128 ? pairwise_block<T>(p, channels) : pairwise_sum<T>(p, channels);
  return __double2float_rn(__ddiv_rn((double)__fadd_rn(0.f, s), (double)channels));
}

// Output k of a resampled signal (up, down not both 1) from inputs staged in s_x, s_x[t] = x[i_lo + t]: the one dot
// product of every ingest kernel, so that an output has the same bits whichever kernel computed it and wherever its
// inputs were staged from.
__device__ __forceinline__ float resample_output(const float* s_x, long long i_lo, long long k, int up, int down,
                                                 int half, int taps, const float* __restrict__ hp) {
  const long long t0 = k * down + half;
  const int p = (int)(t0 % up);
  const int newest = (int)(t0 / up - i_lo);  // index of x[i_max] in the staged span
  const float* h = hp + (size_t)p * taps;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;  // four partial sums: shorter dependency chains, smaller rounding error
  int j = 0;
  for (; j + 4 <= taps; j += 4) {
    a0 = fmaf(__ldg(h + j), s_x[newest - j], a0);
    a1 = fmaf(__ldg(h + j + 1), s_x[newest - j - 1], a1);
    a2 = fmaf(__ldg(h + j + 2), s_x[newest - j - 2], a2);
    a3 = fmaf(__ldg(h + j + 3), s_x[newest - j - 3], a3);
  }
  for (; j < taps; ++j) a0 = fmaf(__ldg(h + j), s_x[newest - j], a0);
  return (a0 + a1) + (a2 + a3);
}

// The work of one CTA, shared by both whole-file kernels so that a file has the same bits whichever launched it:
// outputs [cta * 256, cta * 256 + 256) of one file from its inputs staged (converted and down-mixed) in s_x.
template <typename T>
__device__ __forceinline__ void ingest_cta(const T* __restrict__ pcm, long long n_in, int channels, int up, int down,
                                           int half, int taps, const float* __restrict__ hp, float* __restrict__ out,
                                           long long n_out, int span, long long cta, float* s_x) {
  const long long k0 = cta * kOutPerCta;
  // inputs the CTA's outputs touch: i in [i_lo, i_lo + span)
  const long long i_lo = (k0 * down + half) / up - (taps - 1);
  for (int t = threadIdx.x; t < span; t += kOutPerCta) {
    const long long i = i_lo + t;
    s_x[t] = (i >= 0 && i < n_in) ? mono_sample<T>(pcm, i, channels) : 0.f;
  }
  __syncthreads();
  const long long k = k0 + threadIdx.x;
  if (k >= n_out) return;
  if (up == 1 && down == 1) {  // same rate: format conversion + down-mix only
    out[k] = s_x[(int)(k - i_lo)];
    return;
  }
  out[k] = resample_output(s_x, i_lo, k, up, down, half, taps, hp);
}

template <typename T>
__global__ void __launch_bounds__(kOutPerCta) ingest_kernel(const T* __restrict__ pcm, long long n_in, int channels, int up,
                                                            int down, int half, int taps, const float* __restrict__ hp,
                                                            float* __restrict__ out, long long n_out, int span) {
  extern __shared__ float s_x[];
  ingest_cta<T>(pcm, n_in, channels, up, down, half, taps, hp, out, n_out, span, blockIdx.x, s_x);
}

// Many files in one launch: file i owns CTAs [cta_off[i], cta_off[i + 1]) (none when it is empty), each CTA looks its
// file up and runs that file's format (0..5: the four of ingest_kernel plus packed 24-bit and float64, which only
// whole files read from WAV files reach).
__global__ void __launch_bounds__(kOutPerCta) ingest_batch_kernel(const IngestFile* __restrict__ files,
                                                                  const int* __restrict__ cta_off, int n_files) {
  extern __shared__ float s_x[];
  const int b = blockIdx.x;
  int lo = 0, hi = n_files;  // cta_off[lo] <= b < cta_off[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cta_off[mid] <= b)
      lo = mid;
    else
      hi = mid;
  }
  const IngestFile f = files[lo];
  const long long cta = b - cta_off[lo];
#define BP_INGEST_CTA(T)                                                                                                   \
  ingest_cta<T>(static_cast<const T*>(f.pcm), f.n_in, f.channels, f.up, f.down, f.half, f.taps, f.hp, f.out, f.n_out,     \
                f.span, cta, s_x)
  switch (f.format) {
    case 0: BP_INGEST_CTA(float); break;
    case 1: BP_INGEST_CTA(short); break;
    case 2: BP_INGEST_CTA(int); break;
    case 3: BP_INGEST_CTA(unsigned char); break;
    case 4: BP_INGEST_CTA(s24); break;
    default: BP_INGEST_CTA(double); break;
  }
#undef BP_INGEST_CTA
}

// Input i of a live stream in the push `d` describes: zero before the recording, the held history below n_prev, the new
// block (converted and down-mixed as the whole-file kernels do it) below n_in, zero from there (read only at the end).
template <typename T>
__device__ __forceinline__ float stream_input(const StreamIngest& d, long long i) {
  if (i < d.hist_lo) return 0.f;  // i < 0: no output reads an input before the history otherwise
  if (i < d.n_prev) return d.hist[i - d.hist_lo];
  if (i < d.f.n_in) return mono_sample<T>(static_cast<const T*>(d.f.pcm), i - d.n_prev, d.f.channels);
  return 0.f;
}

// CTA `cta` of one stream's push: outputs [k0 + 256 cta, k0 + 256 cta + 256) of the push, or, as the stream's last CTA,
// the history it keeps for the next push, into the other history buffer (the output CTAs still read this one).
template <typename T>
__device__ __forceinline__ void stream_ingest_cta(const StreamIngest& d, long long cta, float* s_x) {
  const IngestFile& f = d.f;
  const long long out_ctas = (f.n_out + kOutPerCta - 1) / kOutPerCta;
  if (cta == out_ctas) {
    for (long long i = d.new_hist_lo + threadIdx.x; i < f.n_in; i += kOutPerCta)
      d.hist_out[i - d.new_hist_lo] = stream_input<T>(d, i);
    return;
  }
  const long long k0 = d.k0 + cta * kOutPerCta;
  const long long i_lo = (k0 * f.down + f.half) / f.up - (f.taps - 1);  // as ingest_cta, from this CTA's first output
  for (int t = threadIdx.x; t < f.span; t += kOutPerCta) s_x[t] = stream_input<T>(d, i_lo + t);
  __syncthreads();
  const long long k = k0 + threadIdx.x;
  if (k >= d.k0 + f.n_out) return;
  f.out[k - d.k0] = (f.up == 1 && f.down == 1) ? s_x[(int)(k - i_lo)] : resample_output(s_x, i_lo, k, f.up, f.down, f.half, f.taps, f.hp);
}

// One push of many live streams: stream i owns CTAs [cta_off[i], cta_off[i + 1]).
__global__ void __launch_bounds__(kOutPerCta) stream_ingest_kernel(const StreamIngest* __restrict__ streams,
                                                                   const int* __restrict__ cta_off, int n_streams) {
  extern __shared__ float s_x[];
  const int b = blockIdx.x;
  int lo = 0, hi = n_streams;  // cta_off[lo] <= b < cta_off[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cta_off[mid] <= b)
      lo = mid;
    else
      hi = mid;
  }
  const StreamIngest& d = streams[lo];
  const long long cta = b - cta_off[lo];
  switch (d.f.format) {
    case 0: stream_ingest_cta<float>(d, cta, s_x); break;
    case 1: stream_ingest_cta<short>(d, cta, s_x); break;
    case 2: stream_ingest_cta<int>(d, cta, s_x); break;
    default: stream_ingest_cta<unsigned char>(d, cta, s_x); break;
  }
}

long long ceil_div_ll(long long a, long long b) { return a >= 0 ? (a + b - 1) / b : -((-a) / b); }

long long gcd_ll(long long a, long long b) {
  while (b) {
    const long long t = a % b;
    a = b;
    b = t;
  }
  return a;
}
}  // namespace

// host-only: the designed low-pass (before the gain `up`), for tests against scipy's firwin
std::vector<double> ingest_filter(int up, int down) { return design_filter(up, down); }

long long ingest_output_length(long long n_frames, int sample_rate) {
  if (n_frames <= 0 || sample_rate <= 0) return 0;
  const long long g = gcd_ll(kSampleRate, sample_rate);
  const long long up = kSampleRate / g, down = sample_rate / g;
  return (n_frames * up + down - 1) / down;
}

// The resampler of one sample rate without its taps: ratio, filter geometry and the inputs a CTA stages.  Host
// arithmetic only.  0, or -2 when the format (0 .. n_formats - 1) / channel count / rate is unsupported.
int ingest_geometry(int format, int channels, int sample_rate, IngestFile& f, int n_formats) {
  if (channels < 1 || sample_rate < 1 || format < 0 || format >= n_formats) return -2;
  const long long g = gcd_ll(kSampleRate, sample_rate);
  f.format = format, f.channels = channels;
  f.up = (int)(kSampleRate / g), f.down = (int)(sample_rate / g);
  f.half = 0, f.taps = 1;
  if (f.up != 1 || f.down != 1) {
    const int L = filter_length(f.up, f.down);
    f.half = (L - 1) / 2;
    f.taps = (L + f.up - 1) / f.up;
  }
  // staged inputs per CTA: the newest input of the last output minus the oldest of the first, plus one
  const long long span = ((long long)(kOutPerCta - 1) * f.down + f.up - 1) / f.up + f.taps + 1;
  if (span * (long long)sizeof(float) > 200 * 1024) return -2;  // rate ratios beyond ~100:1
  f.span = (int)span;
  return 0;
}

// The polyphase taps of f's ratio on `device` (designed and uploaded on first use) into f.hp.  0, -1 CUDA error.
int ingest_taps(int device, IngestFile& f) {
  if (device < 0 || device >= 64) return -2;
  std::lock_guard<std::mutex> lk(g_mu);
  auto& cache = g_resamplers[device];
  const long long key = ((long long)f.up << 32) | (unsigned)f.down;
  auto it = cache.find(key);
  if (it == cache.end()) {
    Resampler rs;
    rs.up = f.up, rs.down = f.down;
    if (f.up != 1 || f.down != 1) {
      const int up = f.up;
      const std::vector<double> h = design_filter(f.up, f.down);
      const int L = (int)h.size();
      rs.half = (L - 1) / 2;
      rs.taps_per_phase = (L + up - 1) / up;
      std::vector<float> hp((size_t)up * rs.taps_per_phase, 0.f);
      for (int p = 0; p < up; ++p)
        for (int j = 0; p + (long long)j * up < L; ++j) hp[(size_t)p * rs.taps_per_phase + j] = (float)(up * h[p + (size_t)j * up]);
      if (cudaMalloc(&rs.d_hp, hp.size() * sizeof(float)) != cudaSuccess) return -1;
      if (cudaMemcpy(rs.d_hp, hp.data(), hp.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return -1;
    } else {
      rs.taps_per_phase = 1;
    }
    it = cache.emplace(key, rs).first;
  }
  f.hp = it->second.d_hp;
  return 0;
}

// 0 on success; -1 CUDA error, -2 unsupported argument
int launch_ingest(int device, const void* d_pcm, int format, long long n_frames, int channels, int sample_rate, float* d_out,
                  cudaStream_t st) {
  if (n_frames <= 0) return 0;
  IngestFile f{};
  int rc = ingest_geometry(format, channels, sample_rate, f);
  if (rc == 0) rc = ingest_taps(device, f);
  if (rc) return rc;
  const long long n_out = ingest_output_length(n_frames, sample_rate);
  const size_t smem = (size_t)f.span * sizeof(float);
  const unsigned grid = (unsigned)((n_out + kOutPerCta - 1) / kOutPerCta);
#define BP_INGEST(T)                                                                                                       \
  do {                                                                                                                     \
    if (smem > 48 * 1024) cudaFuncSetAttribute(ingest_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
    ingest_kernel<T><<<grid, kOutPerCta, smem, st>>>(static_cast<const T*>(d_pcm), n_frames, channels, f.up, f.down,       \
                                                     f.half, f.taps, f.hp, d_out, n_out, f.span);                          \
  } while (0)
  switch (format) {
    case 0: BP_INGEST(float); break;
    case 1: BP_INGEST(short); break;
    case 2: BP_INGEST(int); break;
    default: BP_INGEST(unsigned char); break;
  }
#undef BP_INGEST
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

long long ingest_ctas(long long n_out) { return (n_out + kOutPerCta - 1) / kOutPerCta; }

int launch_ingest_batch(const IngestFile* d_files, const int* d_cta_off, int n_files, int n_ctas, int max_span,
                        cudaStream_t st) {
  if (n_ctas <= 0) return 0;
  const size_t smem = (size_t)max_span * sizeof(float);
  if (smem > 48 * 1024) cudaFuncSetAttribute(ingest_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  ingest_batch_kernel<<<(unsigned)n_ctas, kOutPerCta, smem, st>>>(d_files, d_cta_off, n_files);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// Output k reads inputs i_max(k) - T + 1 .. i_max(k), i_max(k) = floor((k down + half) / up); after n frames the outputs
// k < F(n) = max(0, ceil((n up - half) / down)) read only inputs that have arrived.
PcmStep pcm_stream_step(const IngestFile& f, long long n, long long add, bool ending) {
  const auto final_outputs = [&](long long frames) {
    return std::max(0LL, ceil_div_ll(frames * f.up - f.half, f.down));
  };
  PcmStep s;
  s.out_lo = final_outputs(n);
  s.out_hi = ending ? ceil_div_ll((n + add) * f.up, f.down) : final_outputs(n + add);
  s.hist_hi = n + add;
  s.hist_lo = ending ? s.hist_hi : std::min(s.hist_hi, std::max(0LL, (s.out_hi * f.down + f.half) / f.up - (f.taps - 1)));
  return s;
}

int stream_ingest_ctas(const StreamIngest& d) {
  return (int)ingest_ctas(d.f.n_out) + (d.f.n_in > d.new_hist_lo ? 1 : 0);
}

int launch_stream_ingest(const StreamIngest* d_streams, const int* d_cta_off, int n_streams, int n_ctas, int max_span,
                         cudaStream_t st) {
  if (n_ctas <= 0) return 0;
  const size_t smem = (size_t)max_span * sizeof(float);
  if (smem > 48 * 1024) cudaFuncSetAttribute(stream_ingest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  stream_ingest_kernel<<<(unsigned)n_ctas, kOutPerCta, smem, st>>>(d_streams, d_cta_off, n_streams);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace bp
