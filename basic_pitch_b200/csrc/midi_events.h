// Host-side restatement of the MIDI object `note_events_to_midi` builds (reference: basic_pitch/note_creation.py:222-271;
// this package: note_creation.note_events_to_midi), shared by the MIDI writer (writers.cu) and the sonifier (sonify.cu)
// so that both start from the same notes, velocities, instruments and pitch-bend events.  Host code only.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace bp {

struct Ev {  // one note event of a file, bends as a range of the batch's flat array
  double start, end;
  long long pitch;
  float amp;
  const int32_t* bends;  // nullptr = dropped / none
  int n_bends;
};

// The events of file i of a batch: notes [note_off[i], note_off[i+1]), bends of note j [bend_off[j], bend_off[j+1])
// (bend_off may be NULL: no bends).
inline std::vector<Ev> file_events(int i, const int32_t* note_off, const double* start_s, const double* end_s,
                                   const int32_t* pitch_midi, const float* amplitude, const int32_t* bend_off,
                                   const int32_t* bends) {
  std::vector<Ev> ev;
  for (int j = note_off[i]; j < note_off[i + 1]; ++j) {
    const int nb = bend_off ? bend_off[j + 1] - bend_off[j] : 0;
    ev.push_back({start_s[j], end_s[j], pitch_midi[j], amplitude[j], nb > 0 ? bends + bend_off[j] : nullptr, nb});
  }
  return ev;
}

// Python's tuple comparison of (start, end, pitch, amplitude, [bends]) as used by sorted() in drop_overlapping_pitch_bends
inline bool ev_less(const Ev& a, const Ev& b) {
  if (a.start != b.start) return a.start < b.start;
  if (a.end != b.end) return a.end < b.end;
  if (a.pitch != b.pitch) return a.pitch < b.pitch;
  if (a.amp != b.amp) return a.amp < b.amp;
  const int n = std::min(a.n_bends, b.n_bends);
  for (int i = 0; i < n; ++i)
    if (a.bends[i] != b.bends[i]) return a.bends[i] < b.bends[i];
  return a.n_bends < b.n_bends;
}

// reference: note_creation.py:274-286
inline void drop_overlapping_pitch_bends(std::vector<Ev>& ev) {
  std::stable_sort(ev.begin(), ev.end(), ev_less);
  for (size_t i = 0; i + 1 < ev.size(); ++i)
    for (size_t j = i + 1; j < ev.size(); ++j) {
      if (ev[j].start >= ev[i].end) break;
      ev[i].bends = nullptr, ev[i].n_bends = 0;
      ev[j].bends = nullptr, ev[j].n_bends = 0;
    }
}

inline int velocity_of(float amp) { return (int)std::nearbyintf(127.0f * amp); }  // int(np.round(127 * np.float32))

// Instruments in order of first use: one per pitch with multiple_pitch_bends, else a single one (the defaultdict of
// note_creation.py:255-261).  events[k] lists the indices of instrument k's notes in event order.
struct Instruments {
  std::vector<long long> key;
  std::vector<std::vector<int>> events;
};
inline Instruments group_instruments(const std::vector<Ev>& ev, bool multiple_pitch_bends) {
  Instruments in;
  for (int i = 0; i < (int)ev.size(); ++i) {
    const long long key = multiple_pitch_bends ? ev[i].pitch : 0;
    size_t k = 0;
    while (k < in.key.size() && in.key[k] != key) ++k;
    if (k == in.key.size()) in.key.push_back(key), in.events.emplace_back();
    in.events[k].push_back(i);
  }
  return in;
}

// Time of pitch-bend event b of a note: np.linspace(start, end, n)[b] = b * step + start, the last one exactly `end`
inline double bend_time(const Ev& e, int b) {
  if (e.n_bends == 1) return e.start;
  if (b == e.n_bends - 1) return e.end;
  const double step = (e.end - e.start) / (double)(e.n_bends - 1);
  return (step != 0.0) ? (double)b * step + e.start : (double)b * (e.end - e.start) / (double)(e.n_bends - 1) + e.start;
}

// MIDI pitch-bend value of a bend in 1/3 semitones: round(b * PITCH_BEND_SCALE / bins per semitone), clipped to
// [-8192, 8191] (note_creation.py:265-268)
inline long long bend_tick(int32_t bend) {
  const long long v = (long long)std::nearbyint((double)bend * 4096.0 / 3.0);
  return std::max(-8192LL, std::min(8191LL, v));
}

}  // namespace bp
