// Batched file writers (host code; no kernels): Standard MIDI Files and note-event CSVs for a whole batch of files straight
// from the arrays the decode returns, a few host threads over the files.  Replaces the per-file Python path
//   note_events_to_midi (reference: basic_pitch/note_creation.py:222-271) -> PrettyMIDI.write (inference.py:574-584)
//   save_note_events (inference.py:409-428)
// of predict_and_save (inference.py:509-604) for batches: no Note / PitchBend / Instrument objects, no csv module.
// Output bytes are those of the Python path of this package (note_creation.note_events_to_midi + midi.PrettyMIDI.write,
// inference.save_note_events); tests/test_host_logic.py compares them.
#include <algorithm>
#include <charconv>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "bp_b200.h"
#include "midi_events.h"

namespace bp {
int writer_fail(int code, const std::string& msg);  // api.cu: sets bp_last_error
}

namespace {

void put_vlq(std::string& out, long long n) {
  unsigned char buf[10];
  int k = 0;
  buf[k++] = (unsigned char)(n & 0x7F);
  n >>= 7;
  while (n) {
    buf[k++] = (unsigned char)((n & 0x7F) | 0x80);
    n >>= 7;
  }
  while (k) out.push_back((char)buf[--k]);
}
void put_be32(std::string& out, uint32_t v) {
  for (int s = 24; s >= 0; s -= 8) out.push_back((char)((v >> s) & 0xFF));
}
void put_be16(std::string& out, uint32_t v) {
  out.push_back((char)((v >> 8) & 0xFF));
  out.push_back((char)(v & 0xFF));
}

struct MidiMsg {
  long long tick;
  int prio;
  unsigned char b[3];
  int len;
};

// midi.PrettyMIDI.write for the object note_events_to_midi builds (resolution 220, one tempo)
std::string midi_bytes(std::vector<bp::Ev> ev, bool multiple_pitch_bends, double tempo) {
  if (!multiple_pitch_bends) bp::drop_overlapping_pitch_bends(ev);
  const double resolution = 220.0;
  auto tick_of = [&](double t) { return (long long)std::nearbyint(t * resolution * tempo / 60.0); };
  const bp::Instruments inst = bp::group_instruments(ev, multiple_pitch_bends);
  std::vector<std::string> tracks;
  {
    std::string meta;
    const uint32_t tempo_us = (uint32_t)std::nearbyint(6e7 / tempo);
    meta += std::string("\x00\xff\x51\x03", 4);
    meta.push_back((char)((tempo_us >> 16) & 0xFF));
    meta.push_back((char)((tempo_us >> 8) & 0xFF));
    meta.push_back((char)(tempo_us & 0xFF));
    meta += std::string("\x00\xff\x58\x04\x04\x02\x18\x08", 8);
    meta += std::string("\x01\xff\x2f\x00", 4);
    tracks.push_back(meta);
  }
  const int program = 4;  // "Electric Piano 1"
  for (size_t idx = 0; idx < inst.key.size(); ++idx) {
    static const int channels[15] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 11, 12, 13, 14, 15};
    const int ch = channels[idx % 15];
    std::vector<MidiMsg> msgs;
    msgs.push_back({0, 0, {(unsigned char)(0xC0 | ch), (unsigned char)(program & 0x7F), 0}, 2});
    for (int i : inst.events[idx]) {
      const bp::Ev& e = ev[i];
      const int vel = std::max(0, std::min(127, bp::velocity_of(e.amp)));
      msgs.push_back({tick_of(e.start), 2, {(unsigned char)(0x90 | ch), (unsigned char)(e.pitch & 0x7F), (unsigned char)vel}, 3});
      msgs.push_back({tick_of(e.end), 1, {(unsigned char)(0x90 | ch), (unsigned char)(e.pitch & 0x7F), 0}, 3});
    }
    for (int i : inst.events[idx]) {
      const bp::Ev& e = ev[i];
      if (e.n_bends <= 0) continue;
      for (int b = 0; b < e.n_bends; ++b) {
        const long long v = bp::bend_tick(e.bends[b]) + 8192;
        msgs.push_back({tick_of(bp::bend_time(e, b)), 0, {(unsigned char)(0xE0 | ch), (unsigned char)(v & 0x7F), (unsigned char)((v >> 7) & 0x7F)}, 3});
      }
    }
    std::stable_sort(msgs.begin(), msgs.end(),
                     [](const MidiMsg& a, const MidiMsg& b) { return a.tick != b.tick ? a.tick < b.tick : a.prio < b.prio; });
    std::string data;
    long long last = 0;
    for (const MidiMsg& m : msgs) {
      put_vlq(data, std::max(0LL, m.tick - last));
      data.append(reinterpret_cast<const char*>(m.b), m.len);
      last = std::max(last, m.tick);
    }
    data += std::string("\x01\xff\x2f\x00", 4);
    tracks.push_back(data);
  }
  std::string out = "MThd";
  put_be32(out, 6);
  put_be16(out, 1);
  put_be16(out, (uint32_t)tracks.size());
  put_be16(out, 220);
  for (const std::string& t : tracks) {
    out += "MTrk";
    put_be32(out, (uint32_t)t.size());
    out += t;
  }
  return out;
}

// str(np.float64): the shortest digits that round-trip, fixed notation for 1e-4 <= |x| < 1e16, always with a fraction
void put_float_repr(std::string& out, double x) {
  char buf[64];
  if (x == 0.0) {
    out += std::signbit(x) ? "-0.0" : "0.0";
    return;
  }
  if (!std::isfinite(x)) {
    out += std::isnan(x) ? "nan" : (x < 0 ? "-inf" : "inf");
    return;
  }
  const double ax = std::fabs(x);
  if (ax >= 1e-4 && ax < 1e16) {
    auto r = std::to_chars(buf, buf + sizeof(buf), x, std::chars_format::fixed);
    std::string s(buf, r.ptr);
    if (s.find('.') == std::string::npos) s += ".0";
    out += s;
  } else {
    auto r = std::to_chars(buf, buf + sizeof(buf), x, std::chars_format::scientific);
    out.append(buf, r.ptr);  // "1e-05": two exponent digits at least, like Python
  }
}

std::string csv_bytes(const std::vector<bp::Ev>& ev) {
  std::string out = "start_time_s,end_time_s,pitch_midi,velocity,pitch_bend\r\n";
  char buf[32];
  for (const bp::Ev& e : ev) {
    put_float_repr(out, e.start);
    out.push_back(',');
    put_float_repr(out, e.end);
    out.push_back(',');
    out.append(buf, std::to_chars(buf, buf + sizeof(buf), e.pitch).ptr);
    out.push_back(',');
    out.append(buf, std::to_chars(buf, buf + sizeof(buf), bp::velocity_of(e.amp)).ptr);
    for (int b = 0; b < e.n_bends; ++b) {
      out.push_back(',');
      out.append(buf, std::to_chars(buf, buf + sizeof(buf), e.bends[b]).ptr);
    }
    out += "\r\n";
  }
  return out;
}

bool write_file(const char* path, const std::string& bytes) {
  FILE* f = std::fopen(path, "wb");
  if (!f) return false;
  const bool ok = std::fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size();
  return std::fclose(f) == 0 && ok;
}

}  // namespace

extern "C" int bp_write_note_files(int32_t n_files, const char* const* midi_paths, const char* const* csv_paths,
                                   const int32_t* note_off, const double* start_s, const double* end_s,
                                   const int32_t* pitch_midi, const float* amplitude, const int32_t* bend_off,
                                   const int32_t* bends, int32_t multiple_pitch_bends, double midi_tempo, int32_t n_threads) {
  if (n_files < 0 || !note_off || (n_files > 0 && (!start_s || !end_s || !pitch_midi || !amplitude)) || !(midi_tempo > 0))
    return bp::writer_fail(BP_E_INVALID, "bp_write_note_files: bad argument");
  if (n_threads <= 0) n_threads = (int)std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
  n_threads = std::max(1, std::min(n_threads, n_files));
  std::vector<int> failed(n_threads, -1);
  auto work = [&](int t) {
    for (int i = t; i < n_files; i += n_threads) {
      const std::vector<bp::Ev> ev = bp::file_events(i, note_off, start_s, end_s, pitch_midi, amplitude, bend_off, bends);
      bool ok = true;
      if (csv_paths && csv_paths[i]) ok = write_file(csv_paths[i], csv_bytes(ev)) && ok;
      if (midi_paths && midi_paths[i]) ok = write_file(midi_paths[i], midi_bytes(ev, multiple_pitch_bends != 0, midi_tempo)) && ok;
      if (!ok && failed[t] < 0) failed[t] = i;
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
  work(0);
  for (auto& x : th) x.join();
  for (int t = 0; t < n_threads; ++t)
    if (failed[t] >= 0) return bp::writer_fail(BP_E_INVALID, "bp_write_note_files: cannot write the outputs of file " + std::to_string(failed[t]));
  return BP_OK;
}
