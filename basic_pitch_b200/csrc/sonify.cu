// GPU render of the MIDI sonification of a batch of files, straight from the note arrays: for every file what
//   note_events_to_midi(events, multiple_pitch_bends).synthesize(fs)
// computes with this package's additive stand-in synthesiser (basic_pitch_b200/midi.py:71-108), which stands in for the
// reference's sonify_midi (basic_pitch/note_creation.py:119-128, called by inference.py:586-592).
//
// Host (threads over the files): the MIDI object (midi_events.h, the one writers.cu restates), each instrument's
// time-sorted pitch-bend table, the note spans, each note's bend segments with their frequency and phase prefix, and for
// every tile of kTile output samples the notes that overlap it, in accumulation order (CSR).
// Device: sonify_tile_kernel — one thread per sample sums the tile's notes in that order (no atomics on the samples) and
// folds the tile's peak |y| into its file's peak by atomicMax on the 64-bit pattern (|y| >= 0, so the integer order is
// the value order and the result does not depend on the order of the tiles); sonify_normalise_kernel divides by it.
// All positions are file-relative, so a file renders to the same bits wherever it sits in a batch.
//
// Accuracy: everything that decides a sample position (lengths, spans, fades, bend switch samples) is exact.  The phase
// is the one difference from the stand-in: NumPy's sequential cumsum of the per-sample frequency (midi.py:99) against
// the closed form S0_seg + (k - k_seg + 1) * f_seg inside a bend segment, with the segment prefixes S0 carried
// sequentially on the host; together with ulp-level differences of pow and sin the tests bound it per sample
// (DESIGN.md §4.4, tests/test_gpu_sonify.py).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <thread>
#include <vector>

#include "bp_b200.h"
#include "midi_events.h"

namespace bp {
int sonify_fail(int code, const std::string& msg);  // api.cu: sets bp_last_error
}

namespace {

using namespace bp;

constexpr int kTile = 256; // output samples per CTA (one thread each)
constexpr double kTwoPi = 2.0 * 3.141592653589793;  // 2.0 * np.pi, the scalar midi.py:99 multiplies by

struct SonNote {       // one sounding note (b > a), file-relative samples
  long long a, b;      // span [a, b): a = int(fs * start), b = int(fs * end) (midi.py:90)
  long long fade;      // min(int(0.01 * fs), (b - a) // 2) (midi.py:101)
  double inv_fade;     // the linspace step 1 / fade of the ramp (midi.py:103)
  double vscale;       // velocity / 127.0 (midi.py:106)
};
struct SonSeg {  // samples of a note with one frequency: [k, next segment's k)
  long long k;   // first sample
  double f;      // 440 * 2 ** ((semis - 69) / 12) (midi.py:98)
  double s0;     // sum of the note's frequencies over samples a .. k-1
};
struct SonTile {
  long long out;     // offset of the tile's first sample in the batch's output
  long long k0;      // file-relative first sample
  long long e0, e1;  // entries [e0, e1)
  int file, n;       // samples in the tile (<= kTile)
};
struct SonEntry {  // a note overlapping a tile, and its segment that contains the tile's first sample of the note
  int note, seg, seg_end;
};

struct FilePlan {
  long long n_samples = 0;
  std::vector<SonNote> notes;
  std::vector<SonSeg> segs;
  std::vector<SonTile> tiles;
  std::vector<SonEntry> entries;
};

// int(fs * x) of a Python float (midi.py:80, 90): the double product truncated towards zero
inline long long trunc_samples(double fs, double x) { return (long long)(fs * x); }

// The first sample whose time k / fs (IEEE division, midi.py:93) is >= t: from that sample on, a bend event at time t
// is at or before the sample's time, which is what searchsorted(bt, t, side="right") - 1 picks (midi.py:96).
long long first_sample_at(double t, double fs) {
  if (!(t > 0.0)) return 0;
  long long k = (long long)std::ceil(t * fs);
  while (k > 0 && (double)(k - 1) / fs >= t) --k;
  while ((double)k / fs < t) ++k;
  return k;
}

// One file.  sizes_only: just the sample count (midi.py:79-82).
FilePlan plan_file(std::vector<Ev> ev, bool multiple_pitch_bends, int sample_rate, bool sizes_only) {
  FilePlan p;
  if (ev.empty()) return p;  // no instruments: np.array([]) (midi.py:81-82)
  if (!multiple_pitch_bends) drop_overlapping_pitch_bends(ev);
  const Instruments inst = group_instruments(ev, multiple_pitch_bends);
  const double fs = (double)sample_rate;
  // get_end_time (midi.py:67-69): the latest note end or pitch-bend time
  double end_time = ev[0].end;
  for (const Ev& e : ev) {
    end_time = std::max(end_time, e.end);
    for (int b = 0; b < e.n_bends; ++b) end_time = std::max(end_time, bend_time(e, b));
  }
  p.n_samples = trunc_samples(fs, end_time + 1.0);  // int(fs * (end_time + 1)) (midi.py:80)
  if (sizes_only || p.n_samples <= 0) return p;

  const long long fade_max = (long long)(0.01 * fs);
  std::vector<long long> tile_count((p.n_samples + kTile - 1) / kTile, 0);
  struct Span {
    int note;                        // index into p.notes
    int seg0, seg1;                  // its segments
  };
  std::vector<Span> order;  // sounding notes in accumulation order: instrument order, then note order (midi.py:83-106)
  for (size_t ii = 0; ii < inst.key.size(); ++ii) {
    // the instrument's bend events, stably sorted by time (midi.py:86-88), and the first sample each applies to
    struct Bend {
      double t, semis;
    };
    std::vector<Bend> bt;
    for (int i : inst.events[ii])
      for (int b = 0; b < ev[i].n_bends; ++b)
        bt.push_back({bend_time(ev[i], b), (double)bend_tick(ev[i].bends[b]) * (2.0 / 8192.0)});
    std::stable_sort(bt.begin(), bt.end(), [](const Bend& x, const Bend& y) { return x.t < y.t; });
    std::vector<long long> kb(bt.size());
    for (size_t j = 0; j < bt.size(); ++j) kb[j] = first_sample_at(bt[j].t, fs);
    auto freq_of = [&](long long pitch, long long j) {  // j: active bend event, -1 = none (bend 0)
      const double semis = (double)pitch + (j >= 0 ? bt[j].semis : 0.0);
      return 440.0 * std::pow(2.0, (semis - 69.0) / 12.0);
    };
    for (int i : inst.events[ii]) {
      const Ev& e = ev[i];
      const long long a = trunc_samples(fs, e.start), b = trunc_samples(fs, e.end);
      if (b <= a) continue;  // midi.py:91-92
      SonNote n;
      n.a = a, n.b = b;
      n.fade = std::min(fade_max, (b - a) / 2);
      n.inv_fade = n.fade > 0 ? 1.0 / (double)n.fade : 0.0;
      n.vscale = (double)velocity_of(e.amp) / 127.0;  // velocity not clamped, like Note.velocity
      Span s{(int)p.notes.size(), (int)p.segs.size(), 0};
      p.notes.push_back(n);
      // segments: the bend active at sample a, then one per later switch sample inside [a, b); events sharing a
      // switch sample collapse to the last of them (side="right")
      long long j = (long long)(std::upper_bound(kb.begin(), kb.end(), a) - kb.begin()) - 1;
      p.segs.push_back({a, freq_of(e.pitch, j), 0.0});
      for (++j; j < (long long)kb.size() && kb[j] < b; ++j) {
        while (j + 1 < (long long)kb.size() && kb[j + 1] == kb[j]) ++j;
        const SonSeg& prev = p.segs.back();
        const double s0 = std::fma((double)(kb[j] - prev.k), prev.f, prev.s0);
        p.segs.push_back({kb[j], freq_of(e.pitch, j), s0});
      }
      s.seg1 = (int)p.segs.size();
      order.push_back(s);
      for (long long t = a / kTile; t <= (b - 1) / kTile; ++t) ++tile_count[t];
    }
  }
  // tiles and their entries (CSR, accumulation order within a tile)
  p.tiles.resize(tile_count.size());
  long long e = 0;
  for (size_t t = 0; t < tile_count.size(); ++t) {
    SonTile& tl = p.tiles[t];
    tl.k0 = (long long)t * kTile;
    tl.n = (int)std::min<long long>(kTile, p.n_samples - tl.k0);
    tl.e0 = e;
    e += tile_count[t];
    tl.e1 = tl.e0;  // advanced while filling
  }
  p.entries.resize(e);
  for (const Span& s : order) {
    const SonNote& n = p.notes[s.note];
    int seg = s.seg0;
    for (long long t = n.a / kTile; t <= (n.b - 1) / kTile; ++t) {
      const long long k = std::max(n.a, t * kTile);
      while (seg + 1 < s.seg1 && p.segs[seg + 1].k <= k) ++seg;
      p.entries[p.tiles[t].e1++] = {s.note, seg, s.seg1};
    }
  }
  return p;
}

template <class F>
void parallel_files(int n_files, F&& fn) {
  int n_threads = (int)std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
  n_threads = std::max(1, std::min(n_threads, n_files));
  std::vector<std::thread> th;
  auto work = [&](int t) {
    for (int i = t; i < n_files; i += n_threads) fn(i);
  };
  for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
  work(0);
  for (auto& x : th) x.join();
}

__global__ void __launch_bounds__(kTile) sonify_tile_kernel(const SonTile* __restrict__ tiles,
                                                            const SonEntry* __restrict__ entries,
                                                            const SonNote* __restrict__ notes,
                                                            const SonSeg* __restrict__ segs, double fs,
                                                            double* __restrict__ y, unsigned long long* __restrict__ peak) {
  __shared__ double warp_max[kTile / 32];
  const SonTile t = tiles[blockIdx.x];
  const long long k = t.k0 + threadIdx.x;
  double acc = 0.0;  // out[k] of the zeroed buffer, notes added in instrument order then note order (midi.py:80, 106)
  for (long long i = t.e0; i < t.e1; ++i) {
    const SonEntry en = entries[i];
    const SonNote n = notes[en.note];
    if (k < n.a || k >= n.b) continue;
    int s = en.seg;
    while (s + 1 < en.seg_end && segs[s + 1].k <= k) ++s;
    const SonSeg sg = segs[s];
    // phase = 2 pi * cumsum(freq) / fs (midi.py:99), the cumulative sum in closed form within the segment; the sum
    // starts at the note's first sample, so sample a already has phase 2 pi f / fs
    const double cum = fma((double)(k - sg.k + 1), sg.f, sg.s0);
    const double phase = kTwoPi * cum / fs;
    // linspace(0, 1, fade, endpoint=False) forwards at the head, reversed at the tail (midi.py:100-105)
    const long long m = k - n.a, len = n.b - n.a;
    double env = 1.0;
    if (m < n.fade)
      env = (double)m * n.inv_fade;
    else if (m >= len - n.fade)
      env = (double)(len - 1 - m) * n.inv_fade;
    // (sin(phase) * env) * (velocity / 127.0), rounded before it is added (no contraction into an FMA): midi.py:106
    acc = __dadd_rn(acc, __dmul_rn(sin(phase) * env, n.vscale));
  }
  if ((int)threadIdx.x < t.n) y[t.out + threadIdx.x] = acc;
  double v = (int)threadIdx.x < t.n ? fabs(acc) : 0.0;
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kTile / 32; ++w) v = fmax(v, warp_max[w]);
    atomicMax(peak + t.file, (unsigned long long)__double_as_longlong(v));
  }
}

// out / peak when peak > 0 (midi.py:107-108)
__global__ void __launch_bounds__(kTile) sonify_normalise_kernel(const SonTile* __restrict__ tiles,
                                                                 const unsigned long long* __restrict__ peak,
                                                                 double* __restrict__ y) {
  const SonTile t = tiles[blockIdx.x];
  if ((int)threadIdx.x >= t.n) return;
  const double p = __longlong_as_double((long long)peak[t.file]);
  if (p > 0.0) y[t.out + threadIdx.x] /= p;
}

#define SCK(call)                                                                                               \
  do {                                                                                                          \
    cudaError_t e_ = (call);                                                                                    \
    if (e_ != cudaSuccess)                                                                                      \
      return bp::sonify_fail(BP_E_CUDA, std::string("bp_sonify_notes_host: ") + #call + " failed: " + cudaGetErrorString(e_)); \
  } while (0)

// Device buffers of one call, stream-ordered (cudaMallocAsync / cudaFreeAsync): no device-wide synchronisation.
struct StreamBufs {
  cudaStream_t st;
  std::vector<void*> ptrs;
  explicit StreamBufs(cudaStream_t s) : st(s) {}
  ~StreamBufs() {
    for (void* p : ptrs) cudaFreeAsync(p, st);
    cudaStreamSynchronize(st);
  }
  template <class T>
  cudaError_t alloc(T** p, size_t n) {
    void* q = nullptr;
    const cudaError_t e = cudaMallocAsync(&q, std::max<size_t>(n, 1) * sizeof(T), st);
    if (e == cudaSuccess) ptrs.push_back(q);
    *p = static_cast<T*>(q);
    return e;
  }
};

template <class T>
cudaError_t upload(T* d, const std::vector<T>& h, cudaStream_t st) {
  return h.empty() ? cudaSuccess : cudaMemcpyAsync(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st);
}

}  // namespace

namespace bp {

// bp_sonify_notes_host without the model: api.cu passes the model's stream (made current on its device) and launch
// counter.  h_audio == NULL: size query, host only (st and launches unused).
int sonify_notes(cudaStream_t st, long long* launches, int32_t n_files, const int32_t* note_off, const double* start_s,
                 const double* end_s, const int32_t* pitch_midi, const float* amplitude, const int32_t* bend_off,
                 const int32_t* bends, int32_t multiple_pitch_bends, int32_t sample_rate, int64_t* h_sample_off,
                 double* h_audio, int64_t capacity) {
  if (n_files < 0 || !note_off || !h_sample_off) return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: bad argument");
  for (int i = 0; i <= n_files; ++i) h_sample_off[i] = 0;
  if (sample_rate <= 0) return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: sample_rate must be > 0");
  if (note_off[0] < 0) return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: note_off[0] < 0");
  for (int i = 0; i < n_files; ++i)
    if (note_off[i + 1] < note_off[i]) return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: note_off decreases");
  const int32_t n0 = note_off[0], n1 = note_off[n_files];
  if (n1 > n0 && (!start_s || !end_s || !pitch_midi || !amplitude))
    return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: null note array");
  if (bend_off) {
    if (n1 > n0 && bend_off[n0] < 0) return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: bend_off < 0");
    for (int j = n0; j < n1; ++j)
      if (bend_off[j + 1] < bend_off[j]) return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: bend_off decreases");
    if (n1 > n0 && bend_off[n1] > bend_off[n0] && !bends)
      return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: null bends array");
  }
  // times the stand-in can render: finite, >= 0 (np.zeros of a negative length raises) and a sample count below 2^53
  const double t_max = 9007199254740992.0 / (double)sample_rate - 1.0;
  for (int j = n0; j < n1; ++j)
    if (!(start_s[j] >= 0.0 && end_s[j] >= 0.0 && start_s[j] < t_max && end_s[j] < t_max))
      return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: note times must be finite, >= 0 and below 2^53 samples");

  const bool sizes_only = h_audio == nullptr;
  std::vector<FilePlan> plans(n_files);
  parallel_files(n_files, [&](int i) {
    plans[i] = plan_file(file_events(i, note_off, start_s, end_s, pitch_midi, amplitude, bend_off, bends),
                         multiple_pitch_bends != 0, sample_rate, sizes_only);
  });
  for (int i = 0; i < n_files; ++i) h_sample_off[i + 1] = h_sample_off[i] + plans[i].n_samples;
  const long long total = h_sample_off[n_files];
  if (sizes_only) return BP_OK;
  if (total > capacity)
    return sonify_fail(BP_E_CAPACITY, "bp_sonify_notes_host: capacity too small, need " + std::to_string(total) + " samples");
  if (total == 0) return BP_OK;

  // concatenate the plans: indices and offsets become batch-global
  std::vector<long long> note_base(n_files + 1, 0), seg_base(n_files + 1, 0), tile_base(n_files + 1, 0),
      entry_base(n_files + 1, 0);
  for (int i = 0; i < n_files; ++i) {
    note_base[i + 1] = note_base[i] + (long long)plans[i].notes.size();
    seg_base[i + 1] = seg_base[i] + (long long)plans[i].segs.size();
    tile_base[i + 1] = tile_base[i] + (long long)plans[i].tiles.size();
    entry_base[i + 1] = entry_base[i] + (long long)plans[i].entries.size();
  }
  if (note_base[n_files] > 0x7fffffffLL || seg_base[n_files] > 0x7fffffffLL || tile_base[n_files] > 0x7fffffffLL)
    return sonify_fail(BP_E_INVALID, "bp_sonify_notes_host: more than 2^31 notes, bend segments or tiles in one call");
  std::vector<SonNote> notes(note_base[n_files]);
  std::vector<SonSeg> segs(seg_base[n_files]);
  std::vector<SonTile> tiles(tile_base[n_files]);
  std::vector<SonEntry> entries(entry_base[n_files]);
  parallel_files(n_files, [&](int i) {
    FilePlan& p = plans[i];
    std::copy(p.notes.begin(), p.notes.end(), notes.begin() + note_base[i]);
    std::copy(p.segs.begin(), p.segs.end(), segs.begin() + seg_base[i]);
    for (size_t t = 0; t < p.tiles.size(); ++t) {
      SonTile tl = p.tiles[t];
      tl.out = h_sample_off[i] + tl.k0;
      tl.e0 += entry_base[i], tl.e1 += entry_base[i];
      tl.file = i;
      tiles[tile_base[i] + t] = tl;
    }
    for (size_t j = 0; j < p.entries.size(); ++j) {
      SonEntry en = p.entries[j];
      en.note += (int)note_base[i], en.seg += (int)seg_base[i], en.seg_end += (int)seg_base[i];
      entries[entry_base[i] + j] = en;
    }
    p = FilePlan();
  });

  StreamBufs buf(st);
  SonTile* d_tiles;
  SonEntry* d_entries;
  SonNote* d_notes;
  SonSeg* d_segs;
  double* d_y;
  unsigned long long* d_peak;
  SCK(buf.alloc(&d_tiles, tiles.size()));
  SCK(buf.alloc(&d_entries, entries.size()));
  SCK(buf.alloc(&d_notes, notes.size()));
  SCK(buf.alloc(&d_segs, segs.size()));
  SCK(buf.alloc(&d_y, (size_t)total));
  SCK(buf.alloc(&d_peak, (size_t)n_files));
  SCK(upload(d_tiles, tiles, st));
  SCK(upload(d_entries, entries, st));
  SCK(upload(d_notes, notes, st));
  SCK(upload(d_segs, segs, st));
  SCK(cudaMemsetAsync(d_peak, 0, sizeof(unsigned long long) * n_files, st));
  const unsigned n_tiles = (unsigned)tiles.size();
  sonify_tile_kernel<<<n_tiles, kTile, 0, st>>>(d_tiles, d_entries, d_notes, d_segs, (double)sample_rate, d_y, d_peak);
  SCK(cudaGetLastError());
  sonify_normalise_kernel<<<n_tiles, kTile, 0, st>>>(d_tiles, d_peak, d_y);
  SCK(cudaGetLastError());
  *launches += 2;
  SCK(cudaMemcpyAsync(h_audio, d_y, sizeof(double) * (size_t)total, cudaMemcpyDeviceToHost, st));
  SCK(cudaStreamSynchronize(st));
  return BP_OK;
}

}  // namespace bp
