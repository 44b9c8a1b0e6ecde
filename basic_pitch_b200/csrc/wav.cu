// WAV header probe (host only, no GPU): which files the library can read by byte range, and where their samples are.
// A file is accepted only when its reading is unambiguous and equals scipy.io.wavfile.read's (DESIGN.md §4.4): RIFF /
// WAVE, chunks walked as id, little-endian size, body, pad byte after an odd body, up to the RIFF size as scipy walks
// them; exactly one `fmt ` before exactly one `data`; PCM 8 / 16 / 24 / 32 bits or IEEE float 32 / 64 bits (plain or
// EXTENSIBLE with the PCM / IEEE-float sub-format GUID); block_align = channels x bytes per sample; a rate the ingest
// takes; a data size that is a multiple of block_align and lies inside the file.  Everything else is declined, and its
// caller reads it as before.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cerrno>
#include <climits>
#include <cstring>
#include <string>

#include "bp_b200.h"
#include "kernels.cuh"

namespace bp {
int wav_fail(int code, const std::string& msg);
}

namespace {

struct Fd {
  int fd;
  explicit Fd(const char* path) : fd(open(path, O_RDONLY | O_CLOEXEC)) {}
  ~Fd() {
    if (fd >= 0) close(fd);
  }
};

bool read_at(int fd, int64_t pos, void* dst, size_t n) {
  unsigned char* p = static_cast<unsigned char*>(dst);
  while (n > 0) {
    const ssize_t r = pread(fd, p, n, (off_t)pos);
    if (r < 0 && errno == EINTR) continue;
    if (r <= 0) return false;
    p += r, pos += r, n -= (size_t)r;
  }
  return true;
}

uint16_t u16(const unsigned char* p) { return (uint16_t)(p[0] | p[1] << 8); }
uint32_t u32(const unsigned char* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

// The sub-format GUID of WAVE_FORMAT_EXTENSIBLE: the format tag, then 00000000-0010-0080-00AA00389B71.
const unsigned char kGuidTail[12] = {0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};

// Fills s (path, pcm.* but pcm.pcm, data_offset) and returns true when the file is accepted.
bool probe_one(const char* path, bp_pcm_source_t& s) {
  Fd f(path);
  if (f.fd < 0) return false;
  struct stat st;
  if (fstat(f.fd, &st) != 0 || !S_ISREG(st.st_mode)) return false;
  const int64_t file_size = (int64_t)st.st_size;
  unsigned char h[40];
  if (file_size < 12 || !read_at(f.fd, 0, h, 12)) return false;
  if (std::memcmp(h, "RIFF", 4) != 0 || std::memcmp(h + 8, "WAVE", 4) != 0) return false;
  const int64_t riff_end = (int64_t)u32(h + 4) + 8;  // scipy reads chunks while its position is below this
  int n_fmt = 0, n_data = 0, format = -1;
  uint32_t channels = 0, rate = 0, block_align = 0;
  int64_t data_pos = 0, data_size = 0;
  for (int64_t pos = 12; pos < riff_end;) {
    if (pos + 8 > file_size) {
      if (pos == file_size && n_data == 1) break;  // the file ends where the RIFF size says more follows: scipy stops
      return false;                              // a partial chunk header
    }
    if (!read_at(f.fd, pos, h, 8)) return false;
    const int64_t size = u32(h + 4), body = pos + 8;
    if (std::memcmp(h, "fmt ", 4) == 0) {
      if (++n_fmt > 1 || n_data > 0 || size < 16) return false;
      const size_t want = size >= 40 ? 40 : 16;
      if (body + (int64_t)want > file_size || !read_at(f.fd, body, h, want)) return false;
      uint32_t tag = u16(h);
      channels = u16(h + 2), rate = u32(h + 4), block_align = u16(h + 12);
      const uint32_t bytes_per_second = u32(h + 8), bits = u16(h + 14);
      if (tag == 0xFFFE) {  // EXTENSIBLE: cbSize >= 22 and a known sub-format, read as scipy reads them
        if (size < 40 || u16(h + 16) < 22 || std::memcmp(h + 24 + 4, kGuidTail, 12) != 0) return false;
        tag = u32(h + 24);
      }
      if (channels < 1 || rate < 1 || rate > INT_MAX) return false;
      if (tag == 1) {
        if ((uint64_t)bytes_per_second != (uint64_t)rate * block_align) return false;  // scipy raises on these
        format = bits == 8 ? 3 : bits == 16 ? 1 : bits == 24 ? 4 : bits == 32 ? 2 : -1;
      } else if (tag == 3) {
        format = bits == 32 ? 0 : bits == 64 ? 5 : -1;
      } else {
        return false;
      }
      if (format < 0 || block_align != channels * (bits / 8)) return false;
    } else if (std::memcmp(h, "data", 4) == 0) {
      if (++n_data > 1 || n_fmt == 0) return false;
      data_pos = body, data_size = size;
    }
    pos = body + size + (size & 1);
  }
  if (n_fmt != 1 || n_data != 1) return false;
  if (data_size % block_align != 0 || data_pos + data_size > file_size) return false;
  bp::IngestFile g{};
  if (bp::ingest_geometry(format, (int)channels, (int)rate, g, bp::kBatchIngestFormats) != 0) return false;
  s.path = path;
  s.data_offset = data_pos;
  s.pcm.pcm = nullptr;
  s.pcm.n_frames = data_size / block_align;
  s.pcm.sample_format = format;
  s.pcm.channels = (int32_t)channels;
  s.pcm.sample_rate = (int32_t)rate;
  s.pcm.reserved = 0;
  return true;
}

}  // namespace

int bp_probe_wav_files(const char* const* paths, int32_t n_files, bp_pcm_source_t* out, int32_t* accepted) {
  if (n_files < 0 || (n_files > 0 && (!paths || !out || !accepted)))
    return bp::wav_fail(BP_E_INVALID, "bp_probe_wav_files: bad argument");
  for (int32_t i = 0; i < n_files; ++i)
    if (!paths[i]) return bp::wav_fail(BP_E_INVALID, "bp_probe_wav_files: path " + std::to_string(i) + " is NULL");
  for (int32_t i = 0; i < n_files; ++i) {
    out[i] = bp_pcm_source_t{};
    accepted[i] = probe_one(paths[i], out[i]) ? 1 : 0;
    if (!accepted[i]) out[i] = bp_pcm_source_t{};
  }
  return BP_OK;
}
