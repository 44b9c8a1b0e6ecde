// C ABI of the hot path (include/bp_b200.h): model lifetime, workspace, chunked launch sequences.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <thread>
#include <string>
#include <vector>

#include "bp_b200.h"
#include "kernels.cuh"

using namespace bp;

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

}  // namespace
namespace bp {
int writer_fail(int code, const std::string& msg) { return fail(code, msg); }  // writers.cu reports through bp_last_error
int sonify_fail(int code, const std::string& msg) { return fail(code, msg); }  // sonify.cu likewise
}
namespace {

#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t e_ = (call);                                                                             \
    if (e_ != cudaSuccess)                                                                               \
      return fail(BP_E_CUDA, std::string(#call) + " failed: " + cudaGetErrorString(e_) + " (" __FILE__ ":" + \
                                 std::to_string(__LINE__) + ")");                                        \
  } while (0)

#define CKL()                                                                                            \
  do {                                                                                                   \
    cudaError_t e_ = cudaGetLastError();                                                                 \
    if (e_ != cudaSuccess)                                                                               \
      return fail(BP_E_CUDA, std::string("kernel launch failed: ") + cudaGetErrorString(e_) + " (" __FILE__ ":" + \
                                 std::to_string(__LINE__) + ")");                                        \
  } while (0)

// A device buffer that only ever grows.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// transposed / interleaved weight layouts derived from the parameter block
struct DerivedLayout {
  static constexpr int cqt_wt = 0;                           // [256][72] columns: re0,im0,re1,im1,...
  static constexpr int contour1_wT = cqt_wt + 256 * 72;      // [936][8]
  static constexpr int contour2_wT = contour1_wT + 936 * 8;  // [200][1]
  static constexpr int note1_wT = contour2_wT + 200;         // [49][32]
  static constexpr int note2_wT = note1_wT + 49 * 32;        // [672][1]
  static constexpr int onset1_wT = note2_wT + 672;           // [200][32]
  static constexpr int onset2_wT = onset1_wT + 200 * 32;     // [297][1] (+3)
  static constexpr int total = onset2_wT + 300;
};

__global__ void derive_kernel(const float* __restrict__ P, float* __restrict__ D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 256 * 72) {
    int k = i / 72, n = i % 72;
    int bin = n >> 1;
    D[DerivedLayout::cqt_wt + i] = (n & 1) ? P[ParamLayout::cqt_imag + bin * 256 + k] : P[ParamLayout::cqt_real + bin * 256 + k];
  }
  auto tr = [&](int src, int dst, int cout, int kk) {  // [cout][kk] -> [kk][cout]
    if (i < cout * kk) {
      int k = i / cout, c = i % cout;
      D[dst + i] = P[src + c * kk + k];
    }
  };
  tr(ParamLayout::contour1_w, DerivedLayout::contour1_wT, 8, 936);
  tr(ParamLayout::contour2_w, DerivedLayout::contour2_wT, 1, 200);
  tr(ParamLayout::note1_w, DerivedLayout::note1_wT, 32, 49);
  tr(ParamLayout::note2_w, DerivedLayout::note2_wT, 1, 672);
  tr(ParamLayout::onset1_w, DerivedLayout::onset1_wT, 32, 200);
  tr(ParamLayout::onset2_w, DerivedLayout::onset2_wT, 1, 297);
}

__global__ void desc_upload_kernel(const int4* __restrict__ a_src, int4* __restrict__ a_dst, const int4* __restrict__ b_src,
                                   int4* __restrict__ b_dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    a_dst[i] = a_src[i];
    b_dst[i] = b_src[i];
  }
}

__global__ void compact_notes_kernel(const long long* __restrict__ frame_off, const long long* __restrict__ slot_off,
                                     const int* __restrict__ note_off, const int* __restrict__ s_start,
                                     const int* __restrict__ s_end, const int* __restrict__ s_pitch,
                                     int* __restrict__ start, int* __restrict__ end, int* __restrict__ pitch,
                                     long long* __restrict__ note_base) {
  const int file = blockIdx.x;
  const long long q = (long long)blockIdx.y * gridDim.x + file;  // grid decode: (setting blockIdx.y, file)
  const int n = note_off[q + 1] - note_off[q];
  const long long s0 = slot_off[q];
  const int d0 = note_off[q];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    start[d0 + i] = s_start[s0 + i];
    end[d0 + i] = s_end[s0 + i];
    pitch[d0 + i] = s_pitch[s0 + i];
    note_base[d0 + i] = frame_off[file];
  }
}

}  // namespace

struct bp_model {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;  // host->device audio copies of the host entry points run ahead of the compute stream
  std::vector<cudaEvent_t> copy_ev;
  float* d_params = nullptr;
  float* d_derived = nullptr;
  double* d_gauss = nullptr;
  CnnWeights cw{};
  int chunk = 206;  // windows per launch sequence: the M-tiles of every tensor-core layer fill whole waves (bp_model_create)
  int path = 1;  // 0 = FP32 FFMA everywhere, 1 = tensor cores with fused epilogues, 2 = tensor cores keeping the contour activations
  int n_sms = 132;
  struct TcLayer {
    TcConvPlan plan;
    TcConvDev dev{};
    DevBuf<uint16_t> tiles, b1, b2;  // tiles: contour only; b1: onset / note only
  } tc[3];                           // by layer: 0 contour, 1 onset, 2 note (tc_spec)
  DevBuf<__nv_bfloat16> yhl, chl;
  Lowpass2 lp2{};  // decimation FIR taps, a parameter of every decimation launch
  DevBuf<uint16_t> cqt_wtc;  // three-way bf16 split of the CQT kernel matrix (tensor-core path)
  size_t chl_zeroed = 0;  // elements of chl known to hold zeros in every row/bin the kernels never write
  int64_t launches = 0;
  // forward workspace (chunk windows)
  DevBuf<float> chain, y, c1, n1, o1;
  DevBuf<float> raw_note, raw_onset, raw_contour;  // row-major raw windows [nb][172][*] (FP32 path inside run_inference)
  DevBuf<float> i_note, i_onset, i_contour;        // internal raw: pm [88][chunk*172], cm [33][chunk*172][8] (tensor-core paths)
  DevBuf<float> u_note, u_onset, u_contour;        // internal unwrapped posteriorgrams of a call: pm [88][F], cm [33][F][8]
  bool y_is_log = false;  // tensor-core paths: `y` still holds the raw log-magnitudes (bp_debug_activation normalises)
  // bp_model_set_debug_frontend: the forward copies the raw log-magnitudes aside before they are normalised
  bool debug_frontend = false;
  bool ylog_valid = false;  // ylog holds the raw log-magnitudes of the last forward chunk
  DevBuf<float> ylog;
  DevBuf<unsigned int> minmax;
  DevBuf<float> edge;  // partial sums where two frequency-tile ranges of a fused conv meet (tc_conv.cu)
  DevBuf<WinDesc> wdesc;
  DevBuf<UnwrapDesc> udesc;
  // staging for the host entry points
  DevBuf<float> st_audio, st_note, st_onset, st_contour;
  DevBuf<unsigned char> st_pcm;  // bp_load_pcm_host
  // pinned gather buffers of per-file input (one sub-batch each: float32 audio, or the descriptors and stored PCM of
  // bp_transcribe_pcm_files_host); the device->host stream of the posteriorgrams and its events
  unsigned char* gather[3] = {nullptr, nullptr, nullptr};
  size_t gather_cap = 0;  // bytes per buffer
  // device side of the PCM sub-batches: upload k + 1 fills one buffer while the ingest of k reads the other;
  // ingest_ev[k] (compute stream, after the ingest of sub-batch k) frees its buffer for sub-batch k + 2
  DevBuf<unsigned char> pcm_ring[2];
  std::vector<cudaEvent_t> ingest_ev;
  // bp_load_pcm_files_device: descriptors in pinned staging and on the device; the events say when the staging has been
  // read (host may rewrite it) and when the kernel is done with the device copy (a later call may overwrite it)
  unsigned char* h_ingest = nullptr;
  size_t h_ingest_cap = 0;
  DevBuf<unsigned char> d_ingest;
  cudaEvent_t ingest_copied = nullptr, ingest_done = nullptr;
  bool ingest_pending = false;
  cudaStream_t d2h_stream = nullptr;
  std::vector<cudaEvent_t> conv_ev;
  // decode workspace
  DevBuf<long long> d_frame_off, d_slot_off, d_note_base;
  DevBuf<float> energy, d_amp;
  DevBuf<double> d_onset64;
  DevBuf<unsigned int> candbits, max_onset;
  DevBuf<float> blk_max;
  DevBuf<int> blk_arg;
  DevBuf<unsigned long long> max_fd;
  DevBuf<int> note_count, slot_start, slot_end, slot_pitch, overflow, d_note_off, d_start, d_end, d_pitch, d_bend_off,
      d_bends;
  DevBuf<unsigned char> grid_tab;  // group and setting tables of a grid-decode chunk (DecodeGridDev)
  // scoring (bp_score_*): the call's references, tables and explicit estimates; match workspace; counts of the call
  DevBuf<unsigned char> score_in;
  DevBuf<int> score_ws_ref, score_ws_est;
  DevBuf<long long> score_counts;
  // matchings (bp_match_*): hits per pair, workspace offsets and workspace, estimate offsets of a grid chunk, matchings
  DevBuf<long long> match_edges, match_off, match_est_off;
  DevBuf<int> match_ws, match_out;
  int64_t last_forward_n = 0;
  int last_path = 0;
  // optional per-kernel timing (bench.py roofline): CUDA events around one kernel family
  WinDesc* h_wd = nullptr;        // pinned staging of the window / unwrap descriptors (bp_run_inference_device)
  UnwrapDesc* h_ud = nullptr;
  size_t h_desc_cap = 0;
  cudaEvent_t desc_ev = nullptr;
  bool desc_pending = false;
  int profile_which = -1;  // -1 off; 0 contour1, 1 onset1, 2 cqt, 3 decimate chain, 4 small convs, 5 decode, 6 note finish
  std::vector<cudaEvent_t> prof_ev;
  size_t prof_used = 0;
  int64_t prof_windows = 0;
};

namespace {

thread_local int64_t g_need_notes = 0, g_need_bends = 0;  // bp_last_required

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

int parse_blob(const void* blob, size_t nbytes, std::vector<float>& params) {
  const unsigned char* b = static_cast<const unsigned char*>(blob);
  if (nbytes < 8 || std::memcmp(b, "BPW1", 4) != 0) return fail(BP_E_INVALID, "weight blob: bad magic (expected BPW1)");
  uint32_t count;
  std::memcpy(&count, b + 4, 4);
  size_t pos = 8;
  params.assign(ParamLayout::total, 0.f);
  struct Slot {
    const char* name;
    int off;
    int n;
  };
  const Slot slots[] = {
      {"cqt_real", ParamLayout::cqt_real, 36 * 256},  {"cqt_imag", ParamLayout::cqt_imag, 36 * 256},
      {"lowpass", ParamLayout::lowpass, 256},         {"cqt_scale", ParamLayout::cqt_scale, 309},
      {"bn_scale", ParamLayout::bn, 1},               {"bn_bias", ParamLayout::bn + 1, 1},
      {"contour1_w", ParamLayout::contour1_w, 7488},  {"contour1_b", ParamLayout::contour1_b, 8},
      {"contour2_w", ParamLayout::contour2_w, 200},   {"contour2_b", ParamLayout::contour2_b, 1},
      {"note1_w", ParamLayout::note1_w, 1568},        {"note1_b", ParamLayout::note1_b, 32},
      {"note2_w", ParamLayout::note2_w, 672},         {"note2_b", ParamLayout::note2_b, 1},
      {"onset1_w", ParamLayout::onset1_w, 6400},      {"onset1_b", ParamLayout::onset1_b, 32},
      {"onset2_w", ParamLayout::onset2_w, 297},       {"onset2_b", ParamLayout::onset2_b, 1},
  };
  unsigned found = 0;
  for (uint32_t t = 0; t < count; ++t) {
    if (pos + 4 > nbytes) return fail(BP_E_INVALID, "weight blob: truncated");
    uint32_t nl;
    std::memcpy(&nl, b + pos, 4);
    pos += 4;
    if (nl > 64 || pos + nl > nbytes) return fail(BP_E_INVALID, "weight blob: bad tensor name");
    std::string name(reinterpret_cast<const char*>(b + pos), nl);
    pos += nl + ((4 - nl % 4) % 4);
    if (pos + 4 > nbytes) return fail(BP_E_INVALID, "weight blob: truncated");
    uint32_t nd;
    std::memcpy(&nd, b + pos, 4);
    pos += 4;
    if (nd > 8 || pos + 4 * nd > nbytes) return fail(BP_E_INVALID, "weight blob: bad rank");
    size_t n = 1;
    for (uint32_t d = 0; d < nd; ++d) {
      uint32_t v;
      std::memcpy(&v, b + pos, 4);
      pos += 4;
      n *= v;
    }
    if (pos + 4 * n > nbytes) return fail(BP_E_INVALID, "weight blob: truncated tensor " + name);
    for (size_t s = 0; s < sizeof(slots) / sizeof(slots[0]); ++s) {
      if (name == slots[s].name) {
        if ((int)n != slots[s].n) return fail(BP_E_INVALID, "weight blob: tensor " + name + " has wrong size");
        std::memcpy(params.data() + slots[s].off, b + pos, 4 * n);
        found |= 1u << s;
      }
    }
    pos += 4 * n;
  }
  if (found != (1u << (sizeof(slots) / sizeof(slots[0]))) - 1) return fail(BP_E_INVALID, "weight blob: missing tensors");
  return BP_OK;
}

int derive(bp_model* m, cudaStream_t st) {
  derive_kernel<<<(256 * 72 + 255) / 256, 256, 0, st>>>(m->d_params, m->d_derived);
  CKL();
  m->launches += 1;
  // host-built from the parameter block: the decimation taps, the tensor-core plans (split-bf16 Toeplitz weight tiles +
  // MMA programs) and the epilogue values of the tensor-core convs
  std::vector<float> hp(ParamLayout::total);
  CK(cudaMemcpyAsync(hp.data(), m->d_params, sizeof(float) * ParamLayout::total, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  m->lp2 = lowpass_pairs(hp.data() + ParamLayout::lowpass);
  // where each layer's conv1 / conv2 weights and biases sit in the parameter block
  struct TcParams {
    int w1, b1, w2, b2;
  };
  static constexpr TcParams params[3] = {
      {ParamLayout::contour1_w, ParamLayout::contour1_b, ParamLayout::contour2_w, ParamLayout::contour2_b},
      {ParamLayout::onset1_w, ParamLayout::onset1_b, ParamLayout::onset2_w, ParamLayout::onset2_b},
      {ParamLayout::note1_w, ParamLayout::note1_b, ParamLayout::note2_w, ParamLayout::note2_b}};
  for (int l = 0; l < 3; ++l) {
    bp_model::TcLayer& L = m->tc[l];
    const float* w1 = hp.data() + params[l].w1;
    if (l == 0) {  // the contour conv: Toeplitz weight tiles + the MMA program
      L.plan.build(tc_spec(l), w1);
      const TcConvPlan& pl = L.plan;
      if (tc_upload_program(pl, st) != 0)
        return fail(BP_E_INVALID, "tensor-core program does not fit its constant-memory area");
      CK(L.tiles.reserve(pl.tiles.size()));
      CK(cudaMemcpyAsync(L.tiles.p, pl.tiles.data(), pl.tiles.size() * 2, cudaMemcpyHostToDevice, st));
    } else {  // onset / note: the two B matrices of the gathered conv1
      std::vector<uint16_t> b1;
      tc_build_b1(l, w1, b1);
      CK(L.b1.reserve(b1.size()));
      CK(cudaMemcpyAsync(L.b1.p, b1.data(), b1.size() * 2, cudaMemcpyHostToDevice, st));
    }
    CK(cudaStreamSynchronize(st));
    std::vector<uint16_t> b2;
    tc_build_b2_full(l, hp.data() + params[l].w2, b2);
    CK(L.b2.reserve(b2.size()));
    CK(cudaMemcpyAsync(L.b2.p, b2.data(), b2.size() * 2, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
    L.dev = TcConvDev{l, L.tiles.p, L.b1.p, L.b2.p};
    std::copy_n(hp.data() + params[l].b1, tc_spec(l).COUT, L.dev.bias1);
    L.dev.bias2 = hp[params[l].b2];
    if (l == 1) std::copy_n(hp.data() + params[l].w2, 9, L.dev.note_w);  // channel 0: the note input
  }
  {
    std::vector<uint16_t> wtc;
    build_cqt_tc_weights(hp.data() + ParamLayout::cqt_real, hp.data() + ParamLayout::cqt_imag, wtc);
    CK(m->cqt_wtc.reserve(wtc.size()));
    CK(cudaMemcpyAsync(m->cqt_wtc.p, wtc.data(), wtc.size() * 2, cudaMemcpyHostToDevice, st));
    CK(cudaStreamSynchronize(st));
  }
  return BP_OK;
}

int ensure_forward_ws(bp_model* m, int nb) {
  CK(m->chain.reserve((size_t)nb * kChainStride));
  CK(m->y.reserve((size_t)nb * kFrames * kCqtBins));
  // the default path never materialises the 8- / 32-channel activations
  if (m->path != 1) CK(m->c1.reserve((size_t)nb * 8 * kFrames * kContourBins));
  if (m->path == 0) {
    CK(m->n1.reserve((size_t)nb * 32 * kFrames * kPitches));
    CK(m->o1.reserve((size_t)nb * 32 * kFrames * kPitches));
  }
  CK(m->minmax.reserve((size_t)nb * 2));
  if (m->debug_frontend) CK(m->ylog.reserve((size_t)nb * kFrames * kCqtBins));
  if (m->path >= 1) {
    const size_t fr = (size_t)m->chunk * kFrames;
    CK(m->i_note.reserve(kPitches * fr));
    CK(m->i_onset.reserve(kPitches * fr));
    if (m->path == 1) CK(m->i_contour.reserve((size_t)kContourBins * fr));
  }
  CK(m->edge.reserve(std::max({tc_edge_floats(tc_spec(0), nb), tc_edge_floats(tc_spec(1), nb),
                               tc_edge_floats(tc_spec(2), nb)})));
  // split layouts use the row stride of a full chunk whatever the batch size (see launch_conv_tc)
  constexpr TcConvSpec cs = tc_spec(0);
  CK(m->yhl.reserve((size_t)2 * cs.chunks8 * 8 * tc_rows_total(m->chunk, cs.rows_per_window)));
  {
    constexpr TcConvSpec ns = tc_spec(2);
    const size_t need = (size_t)2 * ns.chunks8 * 8 * tc_rows_total(m->chunk, ns.rows_per_window);
    const __nv_bfloat16* before = m->chl.p;
    CK(m->chl.reserve(need));
    if (m->chl.p != before || m->chl_zeroed < m->chl.cap) {  // separator rows / pad bins are never written: zero once
      CK(cudaMemset(m->chl.p, 0, m->chl.cap * sizeof(__nv_bfloat16)));
      m->chl_zeroed = m->chl.cap;
    }
  }
  return BP_OK;
}

// Row-major posteriorgram staging of the model (st_note / st_onset / st_contour) for `n_frames` frames.
int reserve_rows(bp_model* m, int64_t n_frames) {
  CK(m->st_note.reserve((size_t)n_frames * kPitches + 4));
  CK(m->st_onset.reserve((size_t)n_frames * kPitches + 4));
  CK(m->st_contour.reserve((size_t)n_frames * kContourBins + 4));
  return BP_OK;
}

int ensure_events(std::vector<cudaEvent_t>& ev, size_t n) {
  while (ev.size() < n) {
    cudaEvent_t e;
    CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ev.push_back(e);
  }
  return BP_OK;
}

struct ProfScope {
  bp_model* m;
  cudaStream_t st;
  bool on;
  ProfScope(bp_model* m_, int which, cudaStream_t st_) : m(m_), st(st_), on(m_->profile_which == which) {
    if (on) rec();
  }
  ~ProfScope() {
    if (on) rec();
  }
  void rec() {
    if (m->prof_used == m->prof_ev.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      m->prof_ev.push_back(e);
    }
    cudaEventRecord(m->prof_ev[m->prof_used++], st);
  }
};

// Internal (frame-fastest) posteriorgrams of a call, see TcOut in kernels.cuh.
struct PostI {
  float *note, *onset, *contour;  // pm [88][stride], pm [88][stride], cm [33][stride][8]
  long long stride;
};

// HCQT + CNN for `nb` windows (nb <= chunk).
// Without `ud` (bp_forward_*): raw row-major outputs note / onset / contour [nb][172][*].
// With `ud` (bp_run_inference_*): the centre frames of every window go to their unwrapped position in the internal
// posteriorgrams `u` — straight from the fused epilogues on the tensor-core path, through a layout conversion of the
// row-major raw windows on the FP32 path; note / onset / contour are then optional row-major scratch.
int forward_chunk(bp_model* m, const float* audio, const WinDesc* desc, int nb, float* note, float* onset,
                  float* contour, cudaStream_t st, const UnwrapDesc* ud = nullptr, const PostI* u = nullptr) {
  float* chain = m->chain.p;
  if (m->profile_which >= 0) m->prof_windows += nb;
  {
    ProfScope ps(m, 3, st);
    for (int s = 0; s < 8; ++s) launch_decimate(m->lp2, audio, desc, chain, s, nb, st);
  }
  constexpr TcConvSpec cs = tc_spec(0), ns = tc_spec(2);
  const int ystride = tc_rows_total(m->chunk, cs.rows_per_window), cstride = tc_rows_total(m->chunk, ns.rows_per_window);
  const long long fr = (long long)m->chunk * kFrames;  // frame stride of the internal raw buffers
  const long long nfr = (long long)nb * kFrames;
  {
    ProfScope ps(m, 2, st);
    if (m->path >= 1) {
      launch_cqt_tc(audio, desc, chain, m->cqt_wtc.p, m->d_params + ParamLayout::cqt_scale, m->y.p, m->minmax.p, nb,
                    m->n_sms, st);
      if (m->debug_frontend) CK(cudaMemcpyAsync(m->ylog.p, m->y.p, sizeof(float) * nb * kFrames * kCqtBins, cudaMemcpyDeviceToDevice, st));
      // NormalizedLog + BatchNorm straight into the bf16 hi/lo split the convs read
      launch_lognorm_split(m->y.p, m->minmax.p, m->d_params + ParamLayout::bn, m->yhl.p, cs, nb, ystride, st);
      m->y_is_log = true;
    } else {
      launch_cqt(audio, desc, chain, m->d_derived + DerivedLayout::cqt_wt, m->d_params + ParamLayout::cqt_scale, m->y.p,
                 m->minmax.p, nb, st);
      if (m->debug_frontend) CK(cudaMemcpyAsync(m->ylog.p, m->y.p, sizeof(float) * nb * kFrames * kCqtBins, cudaMemcpyDeviceToDevice, st));
      launch_lognorm(m->y.p, m->minmax.p, m->d_params + ParamLayout::bn, nb, st);
      m->y_is_log = false;
    }
    m->ylog_valid = m->debug_frontend;
  }
  int extra = 0;  // launches beyond the fixed sequence
  if (m->path >= 1) {
    {
      ProfScope ps(m, 0, st);
      TcOut o;
      o.edge = m->edge.p;
      if (m->path == 1) {  // fused contour conv2: finished posteriorgram (internal layouts) + the note conv's operand
        o.raw = ud ? nullptr : m->i_contour.p;
        o.raw_rows = fr;
        o.ud = ud;
        o.unwrapped = ud ? u->contour : nullptr;
        o.frame_stride = ud ? u->stride : 0;
        o.chl = m->chl.p;
        o.chl_rows = cstride;
        o.chl_chunks = ns.chunks8;
        o.chl_rpw = ns.rows_per_window;
        o.chl_lead = ns.lead_rows;
      } else {
        o.act = m->c1.p;  // channels-last activations
      }
      launch_conv_tc(m->yhl.p, m->tc[0].dev, o, nb, ystride, m->n_sms, st, /*fuse_next=*/m->path == 1);
    }
    {
      ProfScope ps(m, 4, st);
      if (m->path == 2) {
        launch_contour2_tc(m->c1.p, m->cw, contour, m->chl.p, cstride, nb, st);
        if (ud) launch_rows_to_cm(contour, 0, u->contour, u->stride, 0, st, ud, nb), ++extra;
      }
      TcOut o;
      o.raw = m->i_note.p;  // the onset conv2 reads the raw note rows of the whole window
      o.raw_rows = fr;
      o.ud = ud;
      o.unwrapped = ud ? u->note : nullptr;
      o.frame_stride = ud ? u->stride : 0;
      o.edge = m->edge.p;
      launch_conv_tc(m->chl.p, m->tc[2].dev, o, nb, cstride, m->n_sms, st);
    }
    {
      ProfScope ps(m, 1, st);
      TcOut o;
      o.raw = ud ? nullptr : m->i_onset.p;
      o.raw_rows = fr;
      o.ud = ud;
      o.unwrapped = ud ? u->onset : nullptr;
      o.frame_stride = ud ? u->stride : 0;
      o.note_raw = m->i_note.p;
      o.edge = m->edge.p;
      launch_conv_tc(m->yhl.p, m->tc[1].dev, o, nb, ystride, m->n_sms, st);
    }
    if (!ud) {  // raw windows for the caller: internal -> row-major
      launch_pm_to_rows(m->i_note.p, fr, 0, nfr, kPitches, note, st);
      launch_pm_to_rows(m->i_onset.p, fr, 0, nfr, kPitches, onset, st);
      if (m->path == 1) launch_cm_to_rows(m->i_contour.p, fr, 0, nfr, contour, st), ++extra;
      extra += 2;
    }
  } else {
    {
      ProfScope ps(m, 0, st);
      launch_contour1(m->y.p, m->cw, m->c1.p, nb, st);
    }
    {
      ProfScope ps(m, 4, st);
      launch_contour2(m->c1.p, m->cw, contour, nb, st);
      launch_note1(contour, m->cw, m->n1.p, nb, st);
      launch_note2(m->n1.p, m->cw, note, nb, st);
    }
    {
      ProfScope ps(m, 1, st);
      launch_onset1(m->y.p, m->cw, m->o1.p, nb, st);
    }
    {
      ProfScope ps(m, 4, st);
      launch_onset2(note, m->o1.p, m->cw, onset, nb, st);
    }
    if (ud) {
      launch_rows_to_pm(note, 0, kPitches, u->note, u->stride, 0, st, ud, nb);
      launch_rows_to_pm(onset, 0, kPitches, u->onset, u->stride, 0, st, ud, nb);
      launch_rows_to_cm(contour, 0, u->contour, u->stride, 0, st, ud, nb);
      extra += 3;
    }
  }
  CKL();
  // decimation (4 + tail), min/max init + CQT, log-normalise (+ split); tensor-core convs: 3 x (conv + edge fix)
  // (path 2: contour conv2 instead of one edge fix); FP32 path: 6 convs
  m->launches += 5 + 2 + 1 + 6 + extra;
  m->last_path = m->path;
  return BP_OK;
}

// `who` names the parameter set in the message ("decode params[7]" for a setting of a grid decode)
int validate_params(const bp_decode_params_t* p, const std::string& who = "decode params") {
  if (!p) return fail(BP_E_INVALID, who + ": null");
  if (!(p->frame_thresh == p->frame_thresh) || !(p->onset_thresh == p->onset_thresh))
    return fail(BP_E_INVALID, who + ": NaN threshold");
  if (p->melodia_trick && p->frame_thresh < 0)
    return fail(BP_E_INVALID, who + ": frame_thresh < 0 with melodia_trick never terminates (the reference loops forever)");
  if (p->energy_tol < 1) return fail(BP_E_INVALID, who + ": energy_tol must be >= 1");
  if (p->min_note_len < 0) return fail(BP_E_INVALID, who + ": min_note_len must be >= 0");
  return BP_OK;
}

DecodeParamsDev params_dev(const bp_decode_params_t& p) {
  DecodeParamsDev dp;
  dp.onset_thresh = p.onset_thresh;
  dp.frame_thresh = p.frame_thresh;
  dp.min_note_len = p.min_note_len;
  dp.energy_tol = p.energy_tol;
  dp.infer_onsets = p.infer_onsets;
  dp.melodia = p.melodia_trick;
  dp.lo_col = std::max(0, std::min<int>(p.min_pitch_idx, kPitches));
  dp.hi_col = std::max(0, std::min<int>(p.max_pitch_idx, kPitches));
  return dp;
}

// Grid decode: settings per chunk are bounded by this much device workspace (grid_setting_bytes per setting).  A chunk
// always holds every file of the batch, so one setting of a very large batch may exceed it on its own.
constexpr long long kDecodeGridChunkBytes = 2LL << 30;
constexpr long long kDecodeGridMaxChunk = 65535;  // gridDim.y of the sequential kernel

// Device workspace of one setting in a grid-decode chunk (include/bp_b200.h, bp_decode_grid_chunk_params): its E, a
// candidate bitmap and a prep group's maxima (every setting may be its own group), its block maxima, its first-attempt
// note slots (start, end, pitch) and note counts.
long long grid_setting_bytes(long long total_frames, int n_files) {
  const long long cells = total_frames * kPitches;
  return 4 * cells + 4 * decode_cand_words(total_frames) + 8LL * kPitches * decode_block_slots(total_frames, n_files) +
         12 * std::min(cells, 8 * total_frames + 64LL * n_files) + 16LL * n_files + 64;
}

// Everything bp_decode_grid_* checks before anything is enqueued: arguments, every setting (by index), frame offsets.
int check_grid_args(const std::string& api, const bp_model* m, const int64_t* h_frame_off, int n_files,
                    const bp_decode_params_t* params, int n_params, bool* any_bends) {
  if (!m || !h_frame_off || n_files < 0 || n_params < 0 || (n_params > 0 && !params))
    return fail(BP_E_INVALID, api + ": bad argument");
  *any_bends = false;
  for (int k = 0; k < n_params; ++k) {
    const int rc = validate_params(params + k, "decode params[" + std::to_string(k) + "]");
    if (rc) return rc;
    *any_bends |= params[k].include_pitch_bends != 0;
  }
  if (n_files == 0 || n_params == 0) return BP_OK;
  if (h_frame_off[0] != 0) return fail(BP_E_INVALID, api + ": frame_off[0] must be 0");
  for (int i = 1; i <= n_files; ++i)
    if (h_frame_off[i] < h_frame_off[i - 1]) return fail(BP_E_INVALID, api + ": frame offsets must be non-decreasing");
  return BP_OK;
}

// The chunk loop of the grid entry points (bp_decode_grid_*, bp_score_grid_*): per chunk of settings the group tables,
// the decode kernels with the rerun of pairs that outgrew their first allowance of note slots, then
// tail(p0, P, counts, soff) with the chunk's notes in the slots: pair q (setting-major, chunk-local) has counts[q] notes
// from m->slot_*[soff[q]], soff also at m->d_slot_off.  A tail returns BP_OK to go on to the next chunk.
template <class Tail>
int decode_grid_chunks(bp_model* m, const std::string& api, const float* d_note, const float* d_onset,
                       const std::vector<long long>& foff, int n_files, const bp_decode_params_t* params, int n_params,
                       cudaStream_t st, Tail&& tail) {
  const long long total_frames = foff[n_files];
  const long long cells = total_frames * kPitches;
  const long long chunk = bp_decode_grid_chunk_params(total_frames, n_files);
  DecodeGridDev gd{};
  gd.n_files = n_files;
  gd.e_stride = cells;
  gd.cand_stride = decode_cand_words(total_frames);
  gd.blk_stride = (long long)kPitches * decode_block_slots(total_frames, n_files);
  CK(m->d_frame_off.reserve(n_files + 1));
  CK(cudaMemcpyAsync(m->d_frame_off.p, foff.data(), sizeof(long long) * (n_files + 1), cudaMemcpyHostToDevice, st));

  for (long long p0 = 0; p0 < n_params; p0 += chunk) {
    const int P = (int)std::min<long long>(chunk, n_params - p0);
    const long long n_pairs = (long long)P * n_files;  // (setting, file), setting-major
    // ---- groups: settings sharing a pitch range share the prep; those also sharing infer_onsets and onset_thresh
    // share the candidates
    std::vector<DecodeSettingDev> sd(P);
    std::vector<DecodePrepGroup> prep;
    std::vector<DecodeCandGroup> cand;
    std::vector<int> prep_of(P);
    for (int s = 0; s < P; ++s) {
      sd[s].p = params_dev(params[p0 + s]);
      const DecodeParamsDev& q = sd[s].p;
      int pg = 0;
      while (pg < (int)prep.size() && (prep[pg].lo != q.lo_col || prep[pg].hi != q.hi_col)) ++pg;
      if (pg == (int)prep.size()) prep.push_back(DecodePrepGroup{q.lo_col, q.hi_col, 0, 0});
      ++prep[pg].set_hi;  // count for now
      prep_of[s] = pg;
      int cg = 0;
      while (cg < (int)cand.size() && (cand[cg].prep != pg || cand[cg].infer != q.infer_onsets ||
                                       !(cand[cg].onset_thresh == q.onset_thresh)))
        ++cg;
      if (cg == (int)cand.size()) cand.push_back(DecodeCandGroup{q.onset_thresh, q.lo_col, q.hi_col, q.infer_onsets, pg});
      sd[s].cand = cg;
    }
    const int n_prep = (int)prep.size(), n_cand = (int)cand.size();
    for (int k = 0, at = 0; k < n_prep; ++k) {
      const int n = prep[k].set_hi;
      prep[k].set_lo = prep[k].set_hi = at;
      at += n;
    }
    std::vector<int> sets(P);
    for (int s = 0; s < P; ++s) sets[prep[prep_of[s]].set_hi++] = s;
    // one upload of the tables, 16-byte aligned sections
    auto sec = [](size_t bytes) { return (bytes + 15) / 16 * 16; };
    const size_t o_cand = sec(sizeof(DecodePrepGroup) * n_prep), o_sets = o_cand + sec(sizeof(DecodeCandGroup) * n_cand),
                 o_set = o_sets + sec(sizeof(int) * P), tab_bytes = o_set + sizeof(DecodeSettingDev) * P;
    std::vector<unsigned char> tab(tab_bytes);
    std::memcpy(tab.data(), prep.data(), sizeof(DecodePrepGroup) * n_prep);
    std::memcpy(tab.data() + o_cand, cand.data(), sizeof(DecodeCandGroup) * n_cand);
    std::memcpy(tab.data() + o_sets, sets.data(), sizeof(int) * P);
    std::memcpy(tab.data() + o_set, sd.data(), sizeof(DecodeSettingDev) * P);
    CK(m->grid_tab.reserve(tab_bytes));
    CK(cudaMemcpyAsync(m->grid_tab.p, tab.data(), tab_bytes, cudaMemcpyHostToDevice, st));
    gd.prep = reinterpret_cast<const DecodePrepGroup*>(m->grid_tab.p);
    gd.cand = reinterpret_cast<const DecodeCandGroup*>(m->grid_tab.p + o_cand);
    gd.sets = reinterpret_cast<const int*>(m->grid_tab.p + o_sets);
    gd.setting = reinterpret_cast<const DecodeSettingDev*>(m->grid_tab.p + o_set);

    CK(m->energy.reserve((size_t)(P * cells) + 1));
    CK(m->candbits.reserve((size_t)(n_cand * gd.cand_stride)));
    CK(m->max_onset.reserve((size_t)n_prep * n_files));
    CK(m->max_fd.reserve((size_t)n_prep * n_files));
    CK(m->blk_max.reserve((size_t)(P * gd.blk_stride)));
    CK(m->blk_arg.reserve((size_t)(P * gd.blk_stride)));
    CK(m->note_count.reserve((size_t)n_pairs));
    CK(m->d_slot_off.reserve((size_t)n_pairs + 1));
    CK(m->overflow.reserve(1));
    // ---- the loops, with today's two-attempt slot sizing per (setting, file): a pair that ran out of its first
    // allowance gets 88 T slots, and the chunk runs again (the loops consume E)
    std::vector<long long> soff(n_pairs + 1);
    std::vector<char> full(n_pairs, 0);
    std::vector<int> counts(n_pairs);
    for (int attempt = 0; attempt < 2; ++attempt) {
      soff[0] = 0;
      for (long long q = 0; q < n_pairs; ++q) {
        const long long T = foff[q % n_files + 1] - foff[q % n_files];
        soff[q + 1] = soff[q] + (full[q] ? T * kPitches : std::min<long long>(T * kPitches, 8 * T + 64));
      }
      CK(m->slot_start.reserve((size_t)soff[n_pairs] + 1));
      CK(m->slot_end.reserve((size_t)soff[n_pairs] + 1));
      CK(m->slot_pitch.reserve((size_t)soff[n_pairs] + 1));
      CK(cudaMemcpyAsync(m->d_slot_off.p, soff.data(), sizeof(long long) * (n_pairs + 1), cudaMemcpyHostToDevice, st));
      DecodeBuffers b;
      b.frame_off = m->d_frame_off.p;
      b.energy = m->energy.p;
      b.candbits = m->candbits.p;
      b.max_onset = m->max_onset.p;
      b.max_fd = m->max_fd.p;
      b.slot_off = m->d_slot_off.p;
      b.note_count = m->note_count.p;
      b.note_start = m->slot_start.p;
      b.note_end = m->slot_end.p;
      b.note_pitch = m->slot_pitch.p;
      b.overflow = m->overflow.p;
      b.blk_max = m->blk_max.p;
      b.blk_arg = m->blk_arg.p;
      {
        ProfScope ps(m, 5, st);
        launch_decode_grid(d_note, d_onset, b, n_files, total_frames, gd, n_prep, n_cand, P, st);
      }
      CKL();
      m->launches += total_frames > 0 ? 3 : 1;
      CK(cudaMemcpyAsync(counts.data(), m->note_count.p, sizeof(int) * n_pairs, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      bool overflow = false;
      for (long long q = 0; q < n_pairs; ++q)
        if (counts[q] > soff[q + 1] - soff[q]) overflow = full[q] = 1;
      if (!overflow) break;
      if (attempt == 1) return fail(BP_E_CUDA, api + ": note slots overflowed at full capacity (internal error)");
    }
    const int rc = tail(p0, P, counts, soff);
    if (rc) return rc;
  }
  return BP_OK;
}

// Running totals of a grid call that returns its notes (bp_decode_grid_*, bp_match_grid_*) over the chunks so far.
struct GridNotes {
  long long n_notes = 0, n_bends = 0;
  bool notes_fit = true, bends_fit = true;
};

// The note half of a grid chunk's tail (bp_decode_grid_*, bp_match_grid_*): the note offsets of the chunk's pairs into
// notes->note_off (past the note capacity only the counting goes on: bp_last_required totals the whole grid), the
// compaction of their notes into m->d_start / d_end / d_pitch (chunk-relative int offsets at m->d_note_off), their
// amplitudes and, when `bends`, the pitch bends of the settings with include_pitch_bends, all copied into `notes`.
int grid_chunk_notes(bp_model* m, const std::string& api, const float* d_note, const float* d_contour,
                     const bp_decode_params_t* params, bool bends, int n_files, long long p0, int P,
                     const std::vector<int>& counts, bp_notes_t* notes, GridNotes& g, cudaStream_t st) {
  const long long n_pairs = (long long)P * n_files;
  // ---- note offsets; past the note capacity only the counting goes on (bp_last_required totals the whole grid)
  const long long note0 = g.n_notes;
  for (long long q = 0; q < n_pairs; ++q) {
    g.n_notes += counts[q];
    if (g.n_notes > notes->note_capacity) g.notes_fit = false;
    if (g.notes_fit) notes->note_off[p0 * n_files + q + 1] = (int32_t)g.n_notes;
  }
  const long long nc = g.n_notes - note0;  // notes of this chunk
  if (!g.notes_fit || nc == 0) return BP_OK;
  if (!notes->start_frame || !notes->end_frame || !notes->pitch_midi || !notes->amplitude)
    return fail(BP_E_INVALID, api + ": notes arrays missing");
  std::vector<int> noff(n_pairs + 1);  // chunk-relative
  for (long long q = 0; q <= n_pairs; ++q) noff[q] = (int)(notes->note_off[p0 * n_files + q] - note0);
  CK(m->d_note_off.reserve((size_t)n_pairs + 1));
  CK(m->d_start.reserve((size_t)nc));
  CK(m->d_end.reserve((size_t)nc));
  CK(m->d_pitch.reserve((size_t)nc));
  CK(m->d_amp.reserve((size_t)nc));
  CK(m->d_note_base.reserve((size_t)nc));
  CK(m->d_bend_off.reserve((size_t)nc + 1));
  CK(cudaMemcpyAsync(m->d_note_off.p, noff.data(), sizeof(int) * (n_pairs + 1), cudaMemcpyHostToDevice, st));
  compact_notes_kernel<<<dim3(n_files, P), 128, 0, st>>>(m->d_frame_off.p, m->d_slot_off.p, m->d_note_off.p,
                                                         m->slot_start.p, m->slot_end.p, m->slot_pitch.p, m->d_start.p,
                                                         m->d_end.p, m->d_pitch.p, m->d_note_base.p);
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(notes->start_frame + note0, m->d_start.p, sizeof(int) * nc, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(notes->end_frame + note0, m->d_end.p, sizeof(int) * nc, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(notes->pitch_midi + note0, m->d_pitch.p, sizeof(int) * nc, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  // ---- bend offsets: each setting's own include_pitch_bends (without: empty ranges, as bp_decode_device leaves them)
  const long long bend0 = g.n_bends;
  for (int s = 0; s < P; ++s) {
    const bool with = bends && params[p0 + s].include_pitch_bends != 0;
    for (long long j = note0 + noff[(long long)s * n_files]; j < note0 + noff[(long long)(s + 1) * n_files]; ++j) {
      if (with) g.n_bends += notes->end_frame[j] - notes->start_frame[j];
      if (g.n_bends > 0x7fffffffLL) return fail(BP_E_CAPACITY, api + ": more than 2^31 pitch-bend values");
      notes->bend_off[j + 1] = (int32_t)g.n_bends;
    }
  }
  if (g.n_bends > notes->bend_capacity) g.bends_fit = false;
  if (!g.bends_fit) return BP_OK;
  const long long bc = g.n_bends - bend0;  // bends of this chunk
  if (bc > 0 && !notes->bends) return fail(BP_E_INVALID, api + ": bends array missing");
  std::vector<int> boff(nc + 1);
  for (long long j = 0; j <= nc; ++j) boff[j] = (int)(notes->bend_off[note0 + j] - bend0);
  CK(m->d_bends.reserve((size_t)bc + 1));
  CK(cudaMemcpyAsync(m->d_bend_off.p, boff.data(), sizeof(int) * (nc + 1), cudaMemcpyHostToDevice, st));
  {
    ProfScope ps(m, 6, st);
    launch_note_finish(d_note, d_contour, m->d_note_base.p, m->d_start.p, m->d_end.p, m->d_pitch.p, m->d_amp.p,
                       m->d_bend_off.p, m->d_bends.p, (int)nc, bc > 0 ? 1 : 0, m->d_gauss, st);
  }
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(notes->amplitude + note0, m->d_amp.p, sizeof(float) * nc, cudaMemcpyDeviceToHost, st));
  if (bc > 0) CK(cudaMemcpyAsync(notes->bends + bend0, m->d_bends.p, sizeof(int) * bc, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

// BP_OK, or BP_E_CAPACITY with bp_last_required, once a grid call that returns its notes has run every chunk.
int grid_notes_result(const std::string& api, const GridNotes& g) {
  if (!g.notes_fit)
    return g_need_notes = g.n_notes, fail(BP_E_CAPACITY, api + ": note_capacity too small, need " + std::to_string(g.n_notes));
  if (!g.bends_fit)
    return g_need_bends = g.n_bends, fail(BP_E_CAPACITY, api + ": bend_capacity too small, need " + std::to_string(g.n_bends));
  return BP_OK;
}

// The posteriorgrams of a grid call (the salience scorers' one in `contour`), in device memory or, when `host`, in host
// memory.
struct Grams {
  const float *note, *onset, *contour;
  bool host;
};

// Uploads a grid call's host posteriorgrams of `total` frames once for the whole grid on m->stream and points `g` at the
// model's staging; device memory is left where it is.  gram_width 0: the note and onset rows, and the contour rows when
// `contour`, into the row staging; otherwise the salience posteriorgram, total x gram_width, into st_contour.
int stage_grams(bp_model* m, int64_t total, Grams& g, bool contour, int gram_width = 0) {
  if (!g.host) return BP_OK;
  cudaStream_t st = m->stream;
  if (gram_width > 0) {
    if (total > 0) {
      CK(m->st_contour.reserve((size_t)total * gram_width));
      CK(cudaMemcpyAsync(m->st_contour.p, g.contour, sizeof(float) * total * gram_width, cudaMemcpyHostToDevice, st));
    }
    g = Grams{nullptr, nullptr, m->st_contour.p, false};
    return BP_OK;
  }
  const int rc = reserve_rows(m, total);
  if (rc) return rc;
  if (total > 0) {
    CK(cudaMemcpyAsync(m->st_note.p, g.note, sizeof(float) * total * kPitches, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m->st_onset.p, g.onset, sizeof(float) * total * kPitches, cudaMemcpyHostToDevice, st));
    if (contour)
      CK(cudaMemcpyAsync(m->st_contour.p, g.contour, sizeof(float) * total * kContourBins, cudaMemcpyHostToDevice, st));
  }
  g = Grams{m->st_note.p, m->st_onset.p, m->st_contour.p, false};
  return BP_OK;
}

// ---- scoring (bp_score_*) ----------------------------------------------------------------------------------------------

int check_score_params(const std::string& api, const bp_score_params_t* sp) {
  if (!sp) return fail(BP_E_INVALID, api + ": null score params");
  const double v[4] = {sp->onset_tolerance, sp->pitch_tolerance, sp->offset_ratio, sp->offset_min_tolerance};
  const char* name[4] = {"onset_tolerance", "pitch_tolerance", "offset_ratio", "offset_min_tolerance"};
  for (int k = 0; k < 4; ++k)
    if (!std::isfinite(v[k]) || v[k] < 0)
      return fail(BP_E_INVALID, api + ": score params: " + name[k] + " must be finite and >= 0");
  return BP_OK;
}

ScoreTol score_tol(const bp_score_params_t& sp) {
  ScoreTol t{};
  t.onset = sp.onset_tolerance;
  t.pitch = sp.pitch_tolerance;
  t.ratio = sp.offset_ratio;
  t.off_min = sp.offset_min_tolerance;
  // around(x, 4) <= tol needs x <= tol + 0.5e-4 (+ rounding); the kernel adds a margin relative to the onset
  t.window = sp.onset_tolerance * (1 + 1e-12) + 1e-4;
  t.k_buckets = (int)std::min(std::floor((sp.pitch_tolerance + 1e-6) / 100.0) + 1.0, 1073741824.0);
  return t;
}

// Validates n sets of notes (`what` "references" / "estimates", set unit "file" / "item"): note_off[0] = 0 and
// non-decreasing, at most 2^31 - 1 notes per set, every note with finite values, onset >= 0 and offset > onset.
// Without `pitched` log2_hz is not read (intervals only).
int check_note_set(const std::string& api, const char* what, const char* unit, const bp_note_set_t* s, int n,
                   bool pitched = true) {
  const std::string who = api + ": " + what;
  if (!s || !s->note_off) return fail(BP_E_INVALID, who + ": null note set");
  if (s->note_off[0] != 0) return fail(BP_E_INVALID, who + ": note_off[0] must be 0");
  for (int i = 0; i < n; ++i)
    if (s->note_off[i + 1] < s->note_off[i] || s->note_off[i + 1] - s->note_off[i] > INT_MAX)
      return fail(BP_E_INVALID, who + " " + unit + " " + std::to_string(i) + ": bad note_off");
  if (s->note_off[n] > 0 && (!s->onset_s || !s->offset_s || (pitched && !s->log2_hz)))
    return fail(BP_E_INVALID, who + ": null array");
  for (int i = 0; i < n; ++i)
    for (long long j = s->note_off[i]; j < s->note_off[i + 1]; ++j) {
      const double on = s->onset_s[j], off = s->offset_s[j], l2 = pitched ? s->log2_hz[j] : 0.0;
      const char* why = !std::isfinite(on) || !std::isfinite(off) ? "non-finite time"
                        : !std::isfinite(l2)                      ? "non-finite log2_hz"
                        : on < 0                                  ? "onset < 0"
                        : off <= on                               ? "offset <= onset"
                                                                  : nullptr;
      if (why)
        return fail(BP_E_INVALID, who + " " + unit + " " + std::to_string(i) + " note " +
                                      std::to_string(j - s->note_off[i]) + ": " + why);
    }
  return BP_OK;
}

// 16-byte aligned sections of one host->device upload
struct Pack {
  std::vector<unsigned char> buf;
  size_t add(const void* p, size_t bytes) {
    const size_t at = (buf.size() + 15) / 16 * 16;
    buf.resize(at + bytes);
    if (bytes) std::memcpy(buf.data() + at, p, bytes);
    return at;
  }
};

// The references of n sets, sorted by (bucket, onset) within each set, into `pk`; offsets of the sections in `o[6]`
// (note_off, onset, offset, log2_hz, bucket, index within its set before sorting); the range of buckets into tol.
// Without log2_hz (s->log2_hz NULL) every reference is in bucket 0 with log2_hz 0.
void pack_refs(const bp_note_set_t* s, int n, Pack& pk, size_t* o, ScoreTol& tol) {
  const long long R = s->note_off[n];
  std::vector<long long> idx(R);
  std::vector<int> bucket(R), bsorted(R);
  std::vector<double> on(R), off(R), l2(R);
  tol.bucket_lo = 0, tol.bucket_hi = -1;
  for (long long j = 0; j < R; ++j) {
    idx[j] = j;
    bucket[j] = s->log2_hz ? score_bucket(s->log2_hz[j]) : 0;
    if (j == 0 || bucket[j] < tol.bucket_lo) tol.bucket_lo = bucket[j];
    if (j == 0 || bucket[j] > tol.bucket_hi) tol.bucket_hi = bucket[j];
  }
  for (int i = 0; i < n; ++i)
    std::sort(idx.begin() + s->note_off[i], idx.begin() + s->note_off[i + 1], [&](long long a, long long b) {
      if (bucket[a] != bucket[b]) return bucket[a] < bucket[b];
      if (s->onset_s[a] != s->onset_s[b]) return s->onset_s[a] < s->onset_s[b];
      return a < b;
    });
  for (long long j = 0; j < R; ++j) {
    on[j] = s->onset_s[idx[j]];
    off[j] = s->offset_s[idx[j]];
    l2[j] = s->log2_hz ? s->log2_hz[idx[j]] : 0.0;
    bsorted[j] = bucket[idx[j]];
  }
  const std::vector<long long> noff(s->note_off, s->note_off + n + 1);
  o[0] = pk.add(noff.data(), sizeof(long long) * (n + 1));
  o[1] = pk.add(on.data(), sizeof(double) * R);
  o[2] = pk.add(off.data(), sizeof(double) * R);
  o[3] = pk.add(l2.data(), sizeof(double) * R);
  o[4] = pk.add(bsorted.data(), sizeof(int) * R);
  std::vector<int> orig(R);
  for (int i = 0; i < n; ++i)
    for (long long j = s->note_off[i]; j < s->note_off[i + 1]; ++j) orig[j] = (int)(idx[j] - s->note_off[i]);
  o[5] = pk.add(orig.data(), sizeof(int) * R);
}

ScoreRefs refs_at(const unsigned char* d, const size_t* o) {
  return ScoreRefs{reinterpret_cast<const long long*>(d + o[0]), reinterpret_cast<const double*>(d + o[1]),
                   reinterpret_cast<const double*>(d + o[2]), reinterpret_cast<const double*>(d + o[3]),
                   reinterpret_cast<const int*>(d + o[4])};
}

// What the note scorers read, uploaded once per call to m->score_in.
struct NoteRefs {
  ScoreRefs sr;
  const int* r_orig;  // each reference's index within its file or item before sorting
  ScoreTol tol;
  ScoreEst e;  // the uploaded part of the estimates: a grid's frame_t and log2_midi, or the explicit notes
  long long n_refs;
};

// The references of n_files files, the seconds of every frame a note of files of frame offsets foff can start or end
// on and, unless est_log2_hz is NULL, the log2(Hz) table of the estimates; without it the references are intervals only
// (their log2_hz is not read).
int upload_note_refs(bp_model* m, const bp_note_set_t* refs, int n_files, const std::vector<long long>& foff,
                     const bp_score_params_t& sp, const double* est_log2_hz, NoteRefs& nr, cudaStream_t st) {
  long long max_t = 0;
  for (int i = 0; i < n_files; ++i) max_t = std::max(max_t, foff[i + 1] - foff[i]);
  nr.tol = score_tol(sp);
  Pack pk;
  size_t o_ref[6];
  bp_note_set_t r = *refs;
  if (!est_log2_hz) r.log2_hz = nullptr;
  pack_refs(&r, n_files, pk, o_ref, nr.tol);
  std::vector<double> frame_t(max_t + 1);
  bp_frame_times(max_t + 1, frame_t.data());
  const size_t o_ft = pk.add(frame_t.data(), sizeof(double) * (max_t + 1));
  const size_t o_l2 = est_log2_hz ? pk.add(est_log2_hz, sizeof(double) * 128) : 0;
  CK(m->score_in.reserve(pk.buf.size()));
  CK(cudaMemcpyAsync(m->score_in.p, pk.buf.data(), pk.buf.size(), cudaMemcpyHostToDevice, st));
  const unsigned char* d = m->score_in.p;
  nr.sr = refs_at(d, o_ref);
  nr.r_orig = reinterpret_cast<const int*>(d + o_ref[5]);
  nr.e = ScoreEst{};
  nr.e.frame_t = reinterpret_cast<const double*>(d + o_ft);
  if (est_log2_hz) nr.e.log2_midi = reinterpret_cast<const double*>(d + o_l2);
  nr.n_refs = refs->note_off[n_files];
  return BP_OK;
}

// The prologue of the explicit-notes scorers (bp_score_notes_host, bp_match_notes_host,
// bp_score_onset_offset_notes_host): arguments and score params, then, unless there are no items, the output and both
// note sets (intervals only unless `pitched`).
int check_notes_call(const std::string& api, const bp_model* m, const bp_note_set_t* est, const bp_note_set_t* refs,
                     int n_items, const bp_score_params_t* sp, const void* out, bool pitched) {
  if (!m || n_items < 0) return fail(BP_E_INVALID, api + ": bad argument");
  int rc = check_score_params(api, sp);
  if (rc || n_items == 0) return rc;
  if (!out) return fail(BP_E_INVALID, api + ": bad argument");
  rc = check_note_set(api, "estimates", "item", est, n_items, pitched);
  return rc ? rc : check_note_set(api, "references", "item", refs, n_items, pitched);
}

// One upload of an explicit-notes call (bp_*_notes_host) to m->score_in: the references of n items, then the estimates
// (note_off, onset, offset and, when `pitched`, log2_hz); without `pitched` both are intervals only.
int upload_notes(bp_model* m, const bp_note_set_t& est, const bp_note_set_t* refs, int n, const bp_score_params_t& sp,
                 bool pitched, NoteRefs& nr, cudaStream_t st) {
  nr.tol = score_tol(sp);
  Pack pk;
  size_t o_ref[6], o_est[4];
  bp_note_set_t r = *refs;
  if (!pitched) r.log2_hz = nullptr;
  pack_refs(&r, n, pk, o_ref, nr.tol);
  const long long n_est = est.note_off[n];
  o_est[0] = pk.add(est.note_off, sizeof(long long) * (n + 1));
  o_est[1] = pk.add(est.onset_s, sizeof(double) * n_est);
  o_est[2] = pk.add(est.offset_s, sizeof(double) * n_est);
  if (pitched) o_est[3] = pk.add(est.log2_hz, sizeof(double) * n_est);
  CK(m->score_in.reserve(pk.buf.size()));
  CK(cudaMemcpyAsync(m->score_in.p, pk.buf.data(), pk.buf.size(), cudaMemcpyHostToDevice, st));
  const unsigned char* d = m->score_in.p;
  nr.sr = refs_at(d, o_ref);
  nr.r_orig = reinterpret_cast<const int*>(d + o_ref[5]);
  nr.e = ScoreEst{};
  nr.e.off = reinterpret_cast<const long long*>(d + o_est[0]);
  nr.e.onset = reinterpret_cast<const double*>(d + o_est[1]);
  nr.e.offset = reinterpret_cast<const double*>(d + o_est[2]);
  if (pitched) nr.e.log2hz = reinterpret_cast<const double*>(d + o_est[3]);
  nr.n_refs = refs->note_off[n];
  return BP_OK;
}

// Matching workspace per launch (include/bp_b200.h, bp_match_grid_*): consecutive pairs share a launch while their
// workspace stays within this; a pair that needs more runs alone.
constexpr long long kMatchWorkBytes = 2LL << 30;

// mir_eval's matchings of n_pairs pairs (pair q = setting * n_files + file; its estimates from E, est_off[q] .. est_off[q
// + 1] on the host, against file q % n_files's references [ref_off[f], ref_off[f + 1]) of sr) into d_match [n_pairs /
// n_files][2][n_refs] (estimate index or -1): one count launch, then one match launch per range of pairs whose workspace
// fits kMatchWorkBytes.
int match_pairs(bp_model* m, const std::string& api, const ScoreRefs& sr, const int* r_orig, const ScoreEst& E,
                const ScoreTol& tol, int n_files, long long n_pairs, const std::vector<long long>& est_off,
                const int64_t* ref_off, long long n_refs, int* d_match, cudaStream_t st) {
  CK(cudaMemsetAsync(d_match, 0xff, sizeof(int) * 2 * (n_pairs / n_files) * n_refs, st));
  CK(m->match_edges.reserve((size_t)n_pairs));
  launch_match_count(sr, E, tol, n_files, n_pairs, m->match_edges.p, st);
  CKL();
  m->launches += 1;
  std::vector<long long> edges(n_pairs), off(n_pairs + 1);
  CK(cudaMemcpyAsync(edges.data(), m->match_edges.p, sizeof(long long) * n_pairs, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  off[0] = 0;
  for (long long q = 0; q < n_pairs; ++q) {
    const long long n_est = est_off[q + 1] - est_off[q], n_ref = ref_off[q % n_files + 1] - ref_off[q % n_files];
    if (edges[q] > INT_MAX)
      return fail(BP_E_INVALID, api + ": pair " + std::to_string(q) + " (file " + std::to_string(q % n_files) +
                                    "): more than 2^31 - 1 hits");
    off[q + 1] = off[q] + (n_est > 0 && n_ref > 0 ? 2 * match_pass_ints(n_est, n_ref, edges[q]) : 0);
  }
  std::vector<long long> cut{0};  // ranges [cut[k], cut[k + 1])
  long long most = 0;
  for (long long q0 = 0; q0 < n_pairs;) {
    long long q1 = q0 + 1;
    while (q1 < n_pairs && 4 * (off[q1 + 1] - off[q0]) <= kMatchWorkBytes) ++q1;
    most = std::max(most, off[q1] - off[q0]);
    cut.push_back(q0 = q1);
  }
  CK(m->match_off.reserve((size_t)n_pairs + 1));
  CK(m->match_ws.reserve((size_t)most + 1));
  CK(cudaMemcpyAsync(m->match_off.p, off.data(), sizeof(long long) * (n_pairs + 1), cudaMemcpyHostToDevice, st));
  const MatchWork w{m->match_ws.p, m->match_off.p, m->match_edges.p, r_orig, d_match, n_refs};
  for (size_t k = 0; k + 1 < cut.size(); ++k) {
    launch_match(sr, E, tol, w, n_files, cut[k], cut[k + 1], st);
    CKL();
    m->launches += 1;
  }
  return BP_OK;
}

}  // namespace

extern "C" {

int bp_version(void) { return 100; }
const char* bp_last_error(void) { return g_err.c_str(); }

void bp_default_decode_params(bp_decode_params_t* p) {
  if (!p) return;
  p->onset_thresh = 0.5;
  p->frame_thresh = 0.3;
  p->min_note_len = 11;
  p->energy_tol = 11;
  p->infer_onsets = 1;
  p->melodia_trick = 1;
  p->include_pitch_bends = 1;
  p->min_pitch_idx = 0;
  p->max_pitch_idx = BP_N_PITCHES;
  p->reserved = 0;
}

int64_t bp_num_windows(int64_t n_samples) {
  if (n_samples < 0) return 0;
  return (n_samples + kLeadZeros + kHopSamples - 1) / kHopSamples;
}
int64_t bp_num_frames(int64_t n_samples) {
  if (n_samples <= 0) return 0;
  return (int64_t)((double)n_samples / (double)kHopSamples * (double)kHopFrames);
}

static int model_init(bp_model* m, const std::vector<float>& params, const cudaDeviceProp& prop);

int bp_model_create(const void* blob, size_t nbytes, int device, bp_model_t** out) {
  if (!blob || !out) return fail(BP_E_INVALID, "bp_model_create: null argument");
  *out = nullptr;
  std::vector<float> params;
  int rc = parse_blob(blob, nbytes, params);
  if (rc) return rc;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(BP_E_CUDA, std::string("no CUDA device available (") + cudaGetErrorString(e) +
                               "); this library has no CPU path");
  if (device < 0 || device >= ndev) return fail(BP_E_INVALID, "bp_model_create: bad device index");
  DeviceGuard g(device);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(BP_E_CUDA, std::string("device ") + prop.name + " is sm_" + std::to_string(prop.major) +
                               std::to_string(prop.minor) + "; this library is built for sm_90a only");
  bp_model* m = new bp_model();
  m->device = device;
  rc = model_init(m, params, prop);
  if (rc) {  // every failure path releases the streams and device buffers created so far
    const std::string msg = g_err;
    bp_model_destroy(m);
    g_err = msg;
    return rc;
  }
  *out = m;
  return BP_OK;
}

static int model_init(bp_model* m, const std::vector<float>& params, const cudaDeviceProp& prop) {
  int rc;
  CK(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  CK(cudaMalloc(&m->d_params, sizeof(float) * ParamLayout::total));
  CK(cudaMalloc(&m->d_derived, sizeof(float) * DerivedLayout::total));
  CK(cudaMalloc(&m->d_gauss, sizeof(double) * 51));
  // stream-ordered with derive_kernel below (m->stream is non-blocking: it does not wait for the legacy stream)
  CK(cudaMemcpyAsync(m->d_params, params.data(), sizeof(float) * ParamLayout::total, cudaMemcpyHostToDevice, m->stream));
  double gauss[51];
  for (int i = 0; i < 51; ++i) {  // scipy.signal.windows.gaussian(51, std=5): exp(-n^2 / (2*std^2))
    double n = (double)i - 25.0;
    gauss[i] = std::exp(-(n * n) / 50.0);
  }
  CK(cudaMemcpyAsync(m->d_gauss, gauss, sizeof(gauss), cudaMemcpyHostToDevice, m->stream));
  CK(cudaStreamSynchronize(m->stream));  // `gauss` is a stack array
  const float* P = m->d_params;
  const float* D = m->d_derived;
  m->cw = CnnWeights{D + DerivedLayout::contour1_wT, P + ParamLayout::contour1_b, D + DerivedLayout::contour2_wT,
                     P + ParamLayout::contour2_b,    D + DerivedLayout::note1_wT, P + ParamLayout::note1_b,
                     D + DerivedLayout::note2_wT,    P + ParamLayout::note2_b,    D + DerivedLayout::onset1_wT,
                     P + ParamLayout::onset1_b,      D + DerivedLayout::onset2_wT, P + ParamLayout::onset2_b};
  hcqt_setup();
  cnn_setup();
  if (tc_setup() != 0) {
    cudaGetLastError();
    return fail(BP_E_CUDA, "tensor-core conv kernels: shared-memory opt-in failed");
  }
  cqt_tc_setup();
  m->n_sms = prop.multiProcessorCount;
  // chunk of windows: as many as make 2 * n_sms spans of 122 rows in the note layer (175 rows per window), i.e. about four
  // M-tiles per SM in every layer (M-tiles advance by 64 - (KH2 - 1) rows: they overlap by the time taps of the fused
  // conv2) -> 184 windows on 132 SMs
  {
    constexpr TcConvSpec ns = tc_spec(2);
    m->chunk = std::max(1, 2 * m->n_sms * (128 - (ns.KH2 - 1)) / ns.rows_per_window);
  }
  rc = derive(m, m->stream);
  if (rc) return rc;
  CK(cudaStreamSynchronize(m->stream));
  return BP_OK;
}

void bp_model_destroy(bp_model_t* m) {
  if (!m) return;
  DeviceGuard g(m->device);
  cudaDeviceSynchronize();
  m->chain.release(); m->y.release(); m->c1.release(); m->n1.release(); m->o1.release();
  m->raw_note.release(); m->raw_onset.release(); m->raw_contour.release(); m->minmax.release(); m->edge.release();
  m->i_note.release(); m->i_onset.release(); m->i_contour.release(); m->u_note.release(); m->u_onset.release();
  m->u_contour.release();
  m->wdesc.release(); m->udesc.release(); m->st_audio.release(); m->st_note.release(); m->st_onset.release();
  m->st_contour.release(); m->st_pcm.release(); m->pcm_ring[0].release(); m->pcm_ring[1].release(); m->d_ingest.release();
  m->d_frame_off.release(); m->d_slot_off.release(); m->d_note_base.release();
  m->energy.release(); m->d_amp.release(); m->candbits.release(); m->blk_max.release(); m->blk_arg.release(); m->max_onset.release(); m->max_fd.release();
  m->note_count.release(); m->slot_start.release(); m->slot_end.release(); m->slot_pitch.release();
  m->overflow.release(); m->d_note_off.release(); m->d_start.release(); m->d_end.release(); m->d_pitch.release();
  m->d_bend_off.release(); m->d_bends.release(); m->d_onset64.release();
  m->match_edges.release(); m->match_off.release(); m->match_est_off.release(); m->match_ws.release();
  m->match_out.release();
  m->yhl.release();
  m->chl.release();
  m->cqt_wtc.release();
  for (bp_model::TcLayer& L : m->tc) L.tiles.release(), L.b1.release(), L.b2.release();
  if (m->d_params) cudaFree(m->d_params);
  if (m->d_derived) cudaFree(m->d_derived);
  if (m->d_gauss) cudaFree(m->d_gauss);
  for (cudaEvent_t e : m->prof_ev) cudaEventDestroy(e);
  if (m->desc_ev) cudaEventDestroy(m->desc_ev);
  if (m->h_wd) cudaFreeHost(m->h_wd);
  if (m->h_ud) cudaFreeHost(m->h_ud);
  for (cudaEvent_t e : m->copy_ev) cudaEventDestroy(e);
  if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
  if (m->d2h_stream) cudaStreamDestroy(m->d2h_stream);
  for (unsigned char* b : m->gather)
    if (b) cudaFreeHost(b);
  for (cudaEvent_t e : m->conv_ev) cudaEventDestroy(e);
  for (cudaEvent_t e : m->ingest_ev) cudaEventDestroy(e);
  if (m->h_ingest) cudaFreeHost(m->h_ingest);
  if (m->ingest_copied) cudaEventDestroy(m->ingest_copied);
  if (m->ingest_done) cudaEventDestroy(m->ingest_done);
  if (m->stream) cudaStreamDestroy(m->stream);
  delete m;
}

int bp_model_device(const bp_model_t* m) { return m ? m->device : -1; }
int64_t bp_model_launch_count(const bp_model_t* m) { return m ? m->launches : 0; }
int64_t bp_model_chunk_windows(const bp_model_t* m) { return m ? m->chunk : 0; }

int bp_model_param_block(bp_model_t* m, void** d_ptr, size_t* nbytes) {
  if (!m || !d_ptr || !nbytes) return fail(BP_E_INVALID, "bp_model_param_block: null argument");
  *d_ptr = m->d_params;
  *nbytes = sizeof(float) * ParamLayout::total;
  return BP_OK;
}

int bp_model_refresh(bp_model_t* m) {
  if (!m) return fail(BP_E_INVALID, "bp_model_refresh: null model");
  DeviceGuard g(m->device);
  CK(cudaDeviceSynchronize());
  int rc = derive(m, m->stream);
  if (rc) return rc;
  CK(cudaStreamSynchronize(m->stream));
  return BP_OK;
}

int bp_model_set_path(bp_model_t* m, int path) {
  if (!m) return fail(BP_E_INVALID, "bp_model_set_path: null model");
  if (path < 0 || path > 2)
    return fail(BP_E_INVALID, "bp_model_set_path: path must be 0 (FP32 FFMA), 1 (tensor cores, fused epilogues) or 2 (tensor cores, "
                              "contour activations kept)");
  m->path = path;
  return BP_OK;
}

int bp_forward_device(bp_model_t* m, const float* d_audio, int64_t n_windows, float* d_note, float* d_onset,
                      float* d_contour, void* stream) {
  if (!m || !d_audio || !d_note || !d_onset || !d_contour) return fail(BP_E_INVALID, "bp_forward_device: null argument");
  if (n_windows < 0) return fail(BP_E_INVALID, "bp_forward_device: negative window count");
  DeviceGuard g(m->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = ensure_forward_ws(m, (int)std::min<int64_t>(n_windows, m->chunk));
  if (rc) return rc;
  for (int64_t c0 = 0; c0 < n_windows; c0 += m->chunk) {
    int nb = (int)std::min<int64_t>(m->chunk, n_windows - c0);
    rc = forward_chunk(m, d_audio + c0 * kWinSamples, nullptr, nb, d_note + c0 * kFrames * kPitches,
                       d_onset + c0 * kFrames * kPitches, d_contour + c0 * kFrames * kContourBins, st);
    if (rc) return rc;
  }
  m->last_forward_n = n_windows;
  return BP_OK;
}

int bp_forward_host(bp_model_t* m, const float* h_audio, int64_t n_windows, float* h_note, float* h_onset,
                    float* h_contour) {
  if (!m || !h_audio || !h_note || !h_onset || !h_contour) return fail(BP_E_INVALID, "bp_forward_host: null argument");
  if (n_windows < 0) return fail(BP_E_INVALID, "bp_forward_host: negative window count");
  DeviceGuard g(m->device);
  CK(m->st_audio.reserve((size_t)n_windows * kWinSamples));
  int rc = reserve_rows(m, n_windows * kFrames);
  if (rc) return rc;
  cudaStream_t st = m->stream;
  CK(cudaMemcpyAsync(m->st_audio.p, h_audio, sizeof(float) * n_windows * kWinSamples, cudaMemcpyHostToDevice, st));
  rc = bp_forward_device(m, m->st_audio.p, n_windows, m->st_note.p, m->st_onset.p, m->st_contour.p, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_note, m->st_note.p, sizeof(float) * n_windows * kFrames * kPitches, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_onset, m->st_onset.p, sizeof(float) * n_windows * kFrames * kPitches, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h_contour, m->st_contour.p, sizeof(float) * n_windows * kFrames * kContourBins,
                     cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

// HCQT + CNN + unwrap for a batch of files into the internal posteriorgrams `u` (frames of file i at
// frame_base + h_frame_off[i] ..); h_frame_off is relative to the batch (h_frame_off[0] = 0).
static int run_inference_internal(bp_model* m, const float* d_audio, const int64_t* h_sample_off, int32_t n_files,
                                  const PostI& u, int64_t frame_base, int64_t* h_frame_off, cudaStream_t st) {
  std::vector<WinDesc> wd;
  std::vector<UnwrapDesc> ud;
  h_frame_off[0] = 0;
  for (int i = 0; i < n_files; ++i) {
    const int64_t n = h_sample_off[i + 1] - h_sample_off[i];
    if (n < 0) return fail(BP_E_INVALID, "run_inference: sample offsets must be non-decreasing");
    const int64_t nw = bp_num_windows(n), nf = bp_num_frames(n);
    for (int64_t w = 0; w < nw; ++w) {
      const int64_t s = w * kHopSamples - kLeadZeros;  // window start relative to the file
      WinDesc d;
      d.base = h_sample_off[i] + s;
      d.lo = (int)std::max<int64_t>(0, -s);
      d.hi = (int)std::max<int64_t>(d.lo, std::min<int64_t>(kWinSamples, n - s));
      wd.push_back(d);
      UnwrapDesc x;
      x.dst_base = frame_base + h_frame_off[i] + w * kHopFrames;
      x.rows = (int)std::max<int64_t>(0, std::min<int64_t>(kHopFrames, nf - w * kHopFrames));
      x.pad = 0;
      ud.push_back(x);
    }
    h_frame_off[i + 1] = h_frame_off[i] + nf;
  }
  const int64_t nwin = (int64_t)wd.size();
  if (nwin == 0) return BP_OK;
  if (!d_audio) return fail(BP_E_INVALID, "run_inference: null audio");
  const int chunk = m->chunk;
  int rc = ensure_forward_ws(m, (int)std::min<int64_t>(nwin, chunk));
  if (rc) return rc;
  const int nbmax = (int)std::min<int64_t>(nwin, chunk);
  if (m->path == 0) {  // row-major raw windows of the FP32 kernels, converted + unwrapped per chunk
    CK(m->raw_note.reserve((size_t)nbmax * kFrames * kPitches));
    CK(m->raw_onset.reserve((size_t)nbmax * kFrames * kPitches));
  }
  if (m->path != 1) CK(m->raw_contour.reserve((size_t)nbmax * kFrames * kContourBins));
  CK(m->wdesc.reserve(nwin));
  CK(m->udesc.reserve(nwin));
  // descriptors go through pinned staging owned by the model, guarded by an event that completes with the copy (not with
  // the kernels queued behind it): no stream synchronisation here, so back-to-back calls (the sub-batches of
  // bp_transcribe_host) keep the GPU queue full
  if (m->desc_pending) {
    CK(cudaEventSynchronize(m->desc_ev));
    m->desc_pending = false;
  }
  if ((size_t)nwin > m->h_desc_cap) {
    if (m->h_wd) cudaFreeHost(m->h_wd);
    if (m->h_ud) cudaFreeHost(m->h_ud);
    m->h_wd = nullptr;
    m->h_ud = nullptr;
    m->h_desc_cap = 0;
    const size_t cap = std::max<size_t>((size_t)nwin, 4096);
    CK(cudaMallocHost(&m->h_wd, sizeof(WinDesc) * cap));
    CK(cudaMallocHost(&m->h_ud, sizeof(UnwrapDesc) * cap));
    m->h_desc_cap = cap;
  }
  if (!m->desc_ev) CK(cudaEventCreateWithFlags(&m->desc_ev, cudaEventDisableTiming));
  std::memcpy(m->h_wd, wd.data(), sizeof(WinDesc) * nwin);
  std::memcpy(m->h_ud, ud.data(), sizeof(UnwrapDesc) * nwin);
  // a kernel reads the pinned (device-mapped) staging directly: a copy-engine transfer would queue behind the audio
  // uploads that bp_transcribe_host has in flight on the copy stream
  static_assert(sizeof(WinDesc) == 16 && sizeof(UnwrapDesc) == 16, "descriptor upload moves 16-byte records");
  desc_upload_kernel<<<(unsigned)((nwin + 255) / 256), 256, 0, st>>>(
      reinterpret_cast<const int4*>(m->h_wd), reinterpret_cast<int4*>(m->wdesc.p), reinterpret_cast<const int4*>(m->h_ud),
      reinterpret_cast<int4*>(m->udesc.p), (int)nwin);
  CKL();
  m->launches += 1;
  CK(cudaEventRecord(m->desc_ev, st));
  m->desc_pending = true;
  for (int64_t c0 = 0; c0 < nwin; c0 += chunk) {
    const int nb = (int)std::min<int64_t>(chunk, nwin - c0);
    rc = forward_chunk(m, d_audio, m->wdesc.p + c0, nb, m->raw_note.p, m->raw_onset.p, m->raw_contour.p, st,
                       m->udesc.p + c0, &u);
    if (rc) return rc;
  }
  m->last_forward_n = std::min<int64_t>(nwin, chunk) == nwin ? nwin : 0;
  return BP_OK;
}

namespace {
// Host threads that copy the files of one sub-batch after the other into pinned staging buffers, running ahead of the
// caller: worker t copies its share of sub-batch k as soon as the caller has released that buffer (`released` counts the
// sub-batches whose buffer may be overwritten) and reports it in done[k].  The threads live for one call.  Files are
// bytes here: file i is src[i][0 .. len[i]) and lands off[i] - off[first file of its sub-batch] bytes behind the
// sub-batch's header (float32 audio: no header, off = 4 x the sample offsets; stored PCM: gaps that start every file on a
// 16-byte boundary).
struct Gatherer {
  const unsigned char* const* src;
  const int64_t* off;        // [n_files + 1] non-decreasing byte offsets, off[i] + len[i] <= off[i + 1]
  const int64_t* len;        // [n_files]
  const int64_t* head;       // [n_sub] bytes the caller keeps at the front of each sub-batch's buffer
  const int* cut;            // [n_sub + 1] file index where each sub-batch starts
  int n_sub, n_threads;
  unsigned char* const* stage;  // 3 staging buffers
  std::atomic<int> released{0};
  std::vector<std::atomic<int>> done;
  std::vector<std::thread> threads;
  std::atomic<bool> abort{false};

  Gatherer(const unsigned char* const* s, const int64_t* o, const int64_t* l, const int64_t* h, const int* c, int ns, int nt,
           unsigned char* const* st)
      : src(s), off(o), len(l), head(h), cut(c), n_sub(ns), n_threads(nt), stage(st), done(ns) {
    for (auto& d : done) d.store(0);
    for (int t = 0; t < n_threads; ++t) threads.emplace_back([this, t] { run(t); });
  }
  ~Gatherer() {
    abort.store(true);
    for (auto& x : threads) x.join();
  }
  void run(int t) {
    for (int k = 0; k < n_sub; ++k) {
      for (int spins = 0; released.load(std::memory_order_acquire) <= k; ++spins) {  // buffer k % 3 still holds k - 3
        if (abort.load()) return;
        if (spins < 64)
          std::this_thread::yield();
        else
          std::this_thread::sleep_for(std::chrono::microseconds(50));  // do not fight the enqueueing thread for cores
      }
      const int f0 = cut[k], f1 = cut[k + 1];
      const int64_t base = off[f0], total = off[f1] - base;
      unsigned char* dst = stage[k % 3] + head[k];
      // thread t copies bytes [lo, hi) of the sub-batch: whole files where possible, split files otherwise
      const int64_t lo = base + total * t / n_threads, hi = base + total * (t + 1) / n_threads;
      if (hi > lo) {
        int i = (int)(std::upper_bound(off + f0, off + f1 + 1, lo) - off) - 1;
        for (; i < f1 && off[i] < hi; ++i) {
          const int64_t a = std::max(lo, off[i]), b = std::min(hi, off[i] + len[i]);
          if (b > a) std::memcpy(dst + (a - base), src[i] + (a - off[i]), (size_t)(b - a));
        }
      }
      done[k].fetch_add(1, std::memory_order_release);
    }
  }
  void release_upto(int k) { released.store(k, std::memory_order_release); }  // sub-batches < k may be gathered
  void wait(int k) {
    while (done[k].load(std::memory_order_acquire) < n_threads) std::this_thread::yield();
  }
};

// A batch of whole files as an entry point received it: packed back to back (`audio`, in device memory if `on_device`,
// else in host memory), one host pointer per file (`files`), or one host pointer per file to its stored PCM (`pcm`),
// which the device ingest turns into the 22 050 Hz signals the other two kinds start from.
struct Batch {
  const char* api;             // the calling entry point, prefix of every message
  const float* audio;          // packed: the caller's array; describe_batch moves it to the first file's samples
  bool on_device;
  const float* const* files;
  const bp_pcm_file_t* pcm = nullptr;
  std::vector<int64_t> rel{};  // [n_files + 1] sample offsets (22 050 Hz) from the first file (describe_batch)
  int64_t total_frames = 0;    // frames of the posteriorgrams (describe_batch)
  std::vector<IngestFile> ingest{};  // pcm: each file's resampler, lengths and format (describe_pcm)
  std::vector<int64_t> pcm_bytes{};  // pcm: each file's stored size
  int n_files() const { return (int)rel.size() - 1; }
  bool per_file() const { return files || pcm; }  // gathered into pinned staging sub-batch by sub-batch
};

constexpr int kPcmSampleBytes[4] = {4, 2, 4, 1};
constexpr int64_t align16(int64_t n) { return (n + 15) & ~(int64_t)15; }
// The front of a PCM sub-batch of nf files, on the host and on the device: IngestFile [nf], then the CTA prefix
// int [nf + 1], padded so that the PCM behind it starts on a 16-byte boundary.
constexpr int64_t ingest_header_bytes(int nf) {
  return align16((int64_t)nf * (int64_t)sizeof(IngestFile) + ((int64_t)nf + 1) * (int64_t)sizeof(int));
}

struct Rows {
  float *note, *onset, *contour;
};
}  // namespace

// Validates the files of `b` (packed: sample_off [n_files + 1]; per file: n_samples [n_files]) and fills in their
// offsets relative to the first file and the frames of the batch.
static int describe_batch(Batch& b, const int64_t* sample_off, const int64_t* n_samples, int32_t n_files) {
  const std::string api = b.api;
  if (sample_off && b.audio) b.audio += sample_off[0];
  b.rel.assign(n_files + 1, 0);
  b.total_frames = 0;
  for (int i = 0; i < n_files; ++i) {
    const int64_t n = sample_off ? sample_off[i + 1] - sample_off[i] : n_samples[i];
    if (n < 0 && sample_off) return fail(BP_E_INVALID, api + ": sample offsets must be non-decreasing");
    if (n < 0) return fail(BP_E_INVALID, api + ": file " + std::to_string(i) + " has a negative length");
    if (n > 0 && !(b.files ? b.files[i] : b.audio))
      return fail(BP_E_INVALID, api + ": null audio for file " + std::to_string(i));
    b.rel[i + 1] = b.rel[i] + n;
    b.total_frames += bp_num_frames(n);
  }
  return BP_OK;
}

// Validates every stored-PCM file of a batch, host arithmetic only: -> each file's resampler geometry, frame counts in
// and out (`ingest`, pointers unset) and stored bytes.  `device_pcm`: the pointers are dereferenced by the kernel as they
// are, so they must be aligned to their sample type.
static int describe_pcm(const std::string& api, const bp_pcm_file_t* files, int32_t n_files, bool device_pcm,
                        std::vector<IngestFile>& ingest, std::vector<int64_t>& bytes) {
  ingest.assign(n_files, IngestFile{});
  bytes.assign(n_files, 0);
  int64_t ctas = 0;
  for (int i = 0; i < n_files; ++i) {
    const bp_pcm_file_t& f = files[i];
    const std::string who = api + ": file " + std::to_string(i);
    if (f.n_frames < 0) return fail(BP_E_INVALID, who + " has a negative length");
    if (f.sample_format < 0 || f.sample_format > 3)
      return fail(BP_E_INVALID, who + ": sample_format must be 0 (float32), 1 (int16), 2 (int32) or 3 (uint8)");
    if (f.channels < 1) return fail(BP_E_INVALID, who + ": channels must be >= 1");
    if (f.sample_rate < 1) return fail(BP_E_INVALID, who + ": sample_rate must be >= 1");
    if (ingest_geometry(f.sample_format, f.channels, f.sample_rate, ingest[i]) != 0)
      return fail(BP_E_INVALID, who + ": the ratio of " + std::to_string(f.sample_rate) +
                                    " Hz to 22 050 Hz is beyond the resampler's shared-memory limit (~100:1)");
    const int64_t frame_bytes = (int64_t)f.channels * kPcmSampleBytes[f.sample_format];
    if (f.n_frames > (INT64_MAX >> 16) / frame_bytes) return fail(BP_E_INVALID, who + " is too long");
    if (f.n_frames > 0 && !f.pcm) return fail(BP_E_INVALID, who + ": null pcm");
    if (device_pcm && reinterpret_cast<uintptr_t>(f.pcm) % kPcmSampleBytes[f.sample_format] != 0)
      return fail(BP_E_INVALID, who + ": pcm is not aligned to its sample type");
    bytes[i] = f.n_frames * frame_bytes;
    ingest[i].n_in = f.n_frames;
    ingest[i].n_out = ingest_output_length(f.n_frames, f.sample_rate);
    ctas += ingest_ctas(ingest[i].n_out);
    if (ctas > INT_MAX) return fail(BP_E_INVALID, who + ": the batch is too long for one ingest");
  }
  return BP_OK;
}

// The device's polyphase taps for every file (designed and uploaded on the first use of a ratio).
static int load_ingest_taps(const std::string& api, int device, std::vector<IngestFile>& ingest) {
  for (IngestFile& f : ingest) {
    const int rc = ingest_taps(device, f);
    if (rc) {
      cudaGetLastError();
      return fail(rc == -1 ? BP_E_CUDA : BP_E_INVALID, api + ": resampler filter of ratio " + std::to_string(f.up) + "/" +
                                                           std::to_string(f.down) + " could not be set up");
    }
  }
  return BP_OK;
}

// Writes the header of a batched ingest (ingest_header_bytes) over files whose pcm / out pointers are set.
// -> CTAs of the launch; *max_span: the shared memory it needs, in staged inputs.
static int write_ingest_header(unsigned char* h, const IngestFile* f, int nf, int* max_span) {
  std::memcpy(h, f, sizeof(IngestFile) * (size_t)nf);
  int* cta_off = reinterpret_cast<int*>(h + sizeof(IngestFile) * (size_t)nf);
  cta_off[0] = 0;
  *max_span = 1;
  for (int i = 0; i < nf; ++i) {
    cta_off[i + 1] = cta_off[i] + (int)ingest_ctas(f[i].n_out);
    if (f[i].n_out > 0) *max_span = std::max(*max_span, f[i].span);
  }
  return cta_off[nf];
}

// The batched ingest over a header in device memory.
static int launch_ingest_header(bp_model* m, const unsigned char* d_header, int nf, int n_ctas, int max_span, cudaStream_t st) {
  if (n_ctas == 0) return BP_OK;
  const int rc = launch_ingest_batch(reinterpret_cast<const IngestFile*>(d_header),
                                     reinterpret_cast<const int*>(d_header + sizeof(IngestFile) * (size_t)nf), nf, n_ctas,
                                     max_span, st);
  if (rc) return fail(BP_E_CUDA, std::string("batched ingest: ") + cudaGetErrorString(cudaGetLastError()));
  m->launches += 1;
  return BP_OK;
}

// Sub-batches of whole files, as the index of each one's first file plus n_files.  Device input is one sub-batch.  On
// host input the first two hold at most one chunk of windows (their uploads are the ones the kernels cannot hide), the
// next two at most two and the rest at most four; two for per-file input (float32 or PCM), whose three pinned staging
// buffers each hold a whole sub-batch, so that the cap bounds their size.
static std::vector<int> cut_sub_batches(const Batch& b, int64_t chunk) {
  const int n_files = b.n_files();
  if (b.on_device) return {0, n_files};
  const int64_t cap = b.per_file() ? 2 : 4;
  std::vector<int> cut{0};
  int64_t w = 0;
  for (int i = 0; i < n_files; ++i) {
    const size_t k = cut.size() - 1;
    const int64_t limit = std::min<int64_t>(k < 2 ? 1 : (k < 4 ? 2 : 4), cap) * chunk;
    const int64_t nw = bp_num_windows(b.rel[i + 1] - b.rel[i]);
    if (w > 0 && w + nw > limit) {
      cut.push_back(i);
      w = 0;
    }
    w += nw;
  }
  cut.push_back(n_files);
  return cut;
}

// The whole-file pipeline of every bp_run_inference_* / bp_transcribe_* entry point: windows -> forward -> unwrap ->
// row-major posteriorgrams in `rows` (device memory; the model's staging when null), sub-batch by sub-batch
// (cut_sub_batches).  Host input is uploaded on the copy stream ahead of the kernels (stored PCM: followed by one batched
// ingest per sub-batch, which writes its 22 050 Hz signals where the upload of float32 input would have put them), and the
// posteriorgrams of each sub-batch go to `host` (any may be null) on the device->host stream while later ones compute.  Then the decode, if
// `params` is given.  Device input only enqueues on `st` (the decode synchronises it); host input returns synchronised.
static int run_batch(bp_model* m, const Batch& b, const Rows* rows, Rows host, const bp_decode_params_t* params,
                     bp_notes_t* notes, int64_t* h_frame_off, cudaStream_t st) {
  const int n_files = b.n_files();
  int rc = rows ? BP_OK : reserve_rows(m, b.total_frames);
  if (rc) return rc;
  const Rows d = rows ? *rows : Rows{m->st_note.p, m->st_onset.p, m->st_contour.p};
  // internal (frame-fastest) posteriorgrams of the whole batch
  const size_t F = (size_t)((b.total_frames + 31) / 32 * 32 + 32);
  CK(m->u_note.reserve(kPitches * F));
  CK(m->u_onset.reserve(kPitches * F));
  CK(m->u_contour.reserve((size_t)kContourBins * F));
  const PostI u{m->u_note.p, m->u_onset.p, m->u_contour.p, (long long)F};
  const std::vector<int> cut = cut_sub_batches(b, m->chunk);
  const int n_sub = (int)cut.size() - 1;
  const bool from_host = !b.on_device, to_host = host.note || host.onset || host.contour;
  if (from_host) {
    CK(m->st_audio.reserve((size_t)std::max<int64_t>(b.rel[n_files], 1)));
    if ((rc = ensure_events(m->copy_ev, n_sub))) return rc;
  }
  if (to_host) {
    if (!m->d2h_stream) CK(cudaStreamCreateWithFlags(&m->d2h_stream, cudaStreamNonBlocking));
    if ((rc = ensure_events(m->conv_ev, n_sub))) return rc;
  }
  int n_threads = 0;
  // per-file input as the gather threads see it: bytes (Gatherer)
  std::vector<const unsigned char*> src;
  std::vector<int64_t> off, len, head;
  if (b.per_file()) {
    src.resize(n_files);
    off.assign(n_files + 1, 0);
    len.resize(n_files);
    head.assign(n_sub, 0);
    for (int i = 0; i < n_files; ++i) {
      src[i] = static_cast<const unsigned char*>(b.pcm ? b.pcm[i].pcm : static_cast<const void*>(b.files[i]));
      len[i] = b.pcm ? b.pcm_bytes[i] : (int64_t)sizeof(float) * (b.rel[i + 1] - b.rel[i]);
      off[i + 1] = off[i] + (b.pcm ? align16(len[i]) : len[i]);
    }
    size_t max_sub = 1;  // sized by what is staged: PCM bytes can be many times the samples they become
    for (int k = 0; k < n_sub; ++k) {
      if (b.pcm) head[k] = ingest_header_bytes(cut[k + 1] - cut[k]);
      max_sub = std::max<size_t>(max_sub, (size_t)(head[k] + off[cut[k + 1]] - off[cut[k]]));
    }
    if (max_sub > m->gather_cap) {
      for (unsigned char*& g : m->gather) {
        if (g) cudaFreeHost(g);
        g = nullptr;
      }
      m->gather_cap = 0;
      const size_t want = max_sub + max_sub / 8;
      for (unsigned char*& g : m->gather) CK(cudaHostAlloc(&g, want, cudaHostAllocDefault));
      m->gather_cap = want;
    }
    if (b.pcm) {
      for (DevBuf<unsigned char>& d : m->pcm_ring) CK(d.reserve(max_sub));
      if ((rc = ensure_events(m->ingest_ev, n_sub))) return rc;
    }
    n_threads = (int)std::max(1u, std::min(16u, std::thread::hardware_concurrency() > 2 ? std::thread::hardware_concurrency() - 1 : 1u));
  }
  const bool timing = from_host && getenv("BP_B200_TIMING") != nullptr;  // host-side breakdown of this call on stderr
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto ms_since = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(now() - t).count(); };
  const auto t_call = now();
  double t_gather = 0, t_wait = 0, t_launch = 0;
  if (from_host) CK(cudaStreamSynchronize(st));  // st_audio / st_note.. may still be in use by earlier work on the compute stream
  std::unique_ptr<Gatherer> gatherer;
  if (b.per_file()) {
    gatherer.reset(new Gatherer(src.data(), off.data(), len.data(), head.data(), cut.data(), n_sub, n_threads, m->gather));
    gatherer->release_upto(std::min(3, n_sub));  // the three buffers are free: the workers start at once
  }
  h_frame_off[0] = 0;
  // Iteration k queues sub-batch k, then copies the posteriorgrams of k - 1 to the host: a copy into pageable memory
  // returns only once it is done, so the kernels of the next sub-batch must already be queued to keep the device busy.
  for (int k = 0; k <= n_sub; ++k) {
    auto t0 = now();
    if (k < n_sub) {
      const int f0 = cut[k], f1 = cut[k + 1];
      const int64_t s0 = b.rel[f0], s1 = b.rel[f1];
      if (from_host) {
        if (gatherer) {
          gatherer->wait(k);  // sub-batch k is in its staging buffer (gathered while earlier sub-batches were enqueued)
          t_gather += ms_since(t0);
          t0 = now();
        }
        if (b.pcm) {  // descriptors + PCM up in one copy, then the ingest writes st_audio[s0, s1)
          const int nf = f1 - f0;
          unsigned char* d_sub = m->pcm_ring[k % 2].p;
          std::vector<IngestFile> desc(b.ingest.begin() + f0, b.ingest.begin() + f1);
          for (int i = 0; i < nf; ++i) {
            desc[i].pcm = d_sub + head[k] + (off[f0 + i] - off[f0]);
            desc[i].out = m->st_audio.p + b.rel[f0 + i];
          }
          int max_span = 1;
          const int n_ctas = write_ingest_header(m->gather[k % 3], desc.data(), nf, &max_span);
          if (k >= 2) CK(cudaStreamWaitEvent(m->copy_stream, m->ingest_ev[k - 2], 0));  // the ingest that last read d_sub
          CK(cudaMemcpyAsync(d_sub, m->gather[k % 3], (size_t)(head[k] + off[f1] - off[f0]), cudaMemcpyHostToDevice, m->copy_stream));
          CK(cudaEventRecord(m->copy_ev[k], m->copy_stream));
          CK(cudaStreamWaitEvent(st, m->copy_ev[k], 0));
          if ((rc = launch_ingest_header(m, d_sub, nf, n_ctas, max_span, st))) return rc;
          CK(cudaEventRecord(m->ingest_ev[k], st));
        } else {
          const void* from = gatherer ? static_cast<const void*>(m->gather[k % 3]) : b.audio + s0;
          if (s1 > s0)
            CK(cudaMemcpyAsync(m->st_audio.p + s0, from, sizeof(float) * (size_t)(s1 - s0), cudaMemcpyHostToDevice, m->copy_stream));
          CK(cudaEventRecord(m->copy_ev[k], m->copy_stream));
          CK(cudaStreamWaitEvent(st, m->copy_ev[k], 0));
        }
      }
      const int64_t base = h_frame_off[f0];  // run_inference_internal writes the offsets relative to it
      rc = run_inference_internal(m, from_host ? m->st_audio.p : b.audio, b.rel.data() + f0, f1 - f0, u, base,
                                  h_frame_off + f0, st);
      if (rc) return rc;
      for (int i = f0; i <= f1; ++i) h_frame_off[i] += base;
      if (gatherer && k >= 1) {  // buffer (k - 1) % 3 = (k + 2) % 3 is free once the upload of sub-batch k - 1 has left the host
        const auto tw = now();
        CK(cudaEventSynchronize(m->copy_ev[k - 1]));
        t_wait += ms_since(tw);
        gatherer->release_upto(std::min(k + 3, n_sub));
      }
      const int64_t nf = h_frame_off[f1] - base;
      if (nf > 0) {  // this sub-batch's posteriorgrams: internal -> row-major
        launch_pm_to_rows(u.note, u.stride, base, nf, kPitches, d.note + base * kPitches, st);
        launch_pm_to_rows(u.onset, u.stride, base, nf, kPitches, d.onset + base * kPitches, st);
        launch_cm_to_rows(u.contour, u.stride, base, nf, d.contour + base * kContourBins, st);
        m->launches += 3;
        CKL();
        if (to_host) CK(cudaEventRecord(m->conv_ev[k], st));
      }
    }
    if (to_host && k >= 1) {
      const int64_t f0 = h_frame_off[cut[k - 1]], nf = h_frame_off[cut[k]] - f0;
      if (nf > 0) {
        CK(cudaStreamWaitEvent(m->d2h_stream, m->conv_ev[k - 1], 0));
        if (host.note)
          CK(cudaMemcpyAsync(host.note + f0 * kPitches, d.note + f0 * kPitches, sizeof(float) * nf * kPitches,
                             cudaMemcpyDeviceToHost, m->d2h_stream));
        if (host.onset)
          CK(cudaMemcpyAsync(host.onset + f0 * kPitches, d.onset + f0 * kPitches, sizeof(float) * nf * kPitches,
                             cudaMemcpyDeviceToHost, m->d2h_stream));
        if (host.contour)
          CK(cudaMemcpyAsync(host.contour + f0 * kContourBins, d.contour + f0 * kContourBins,
                             sizeof(float) * nf * kContourBins, cudaMemcpyDeviceToHost, m->d2h_stream));
      }
    }
    t_launch += ms_since(t0);
  }
  const auto t_dec = now();
  rc = params ? bp_decode_device(m, d.note, d.onset, d.contour, h_frame_off, n_files, params, notes, st) : BP_OK;
  if (!from_host) return rc;
  const double ms_dec = ms_since(t_dec);
  const auto t_d2h = now();
  const cudaError_t e1 = to_host ? cudaStreamSynchronize(m->d2h_stream) : cudaSuccess;
  if (timing)
    fprintf(stderr, "%s: %d files, %d sub-batches, %d gather threads: gather %.1f ms, staging waits %.1f ms, enqueue %.1f ms, "
            "decode (incl. waiting for the forward pass) %.1f ms, tail of the posteriorgram copies %.1f ms, total %.1f ms\n",
            b.api, n_files, n_sub, n_threads, t_gather, t_wait, t_launch, ms_dec, ms_since(t_d2h), ms_since(t_call));
  if (rc) return rc;
  CK(e1);
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int bp_run_inference_device(bp_model_t* m, const float* d_audio, const int64_t* h_sample_off, int32_t n_files,
                            float* d_note, float* d_onset, float* d_contour, int64_t* h_frame_off, void* stream) {
  if (!m || !h_sample_off || !h_frame_off || n_files < 0)
    return fail(BP_E_INVALID, "bp_run_inference_device: bad argument");
  DeviceGuard g(m->device);
  Batch b{"bp_run_inference_device", d_audio, true, nullptr};
  int rc = describe_batch(b, h_sample_off, nullptr, n_files);
  if (rc) return rc;
  if (b.total_frames > 0 && (!d_note || !d_onset || !d_contour))
    return fail(BP_E_INVALID, "bp_run_inference_device: null buffer");
  if (!aligned16(d_contour)) return fail(BP_E_INVALID, "bp_run_inference_device: d_contour must be 16-byte aligned");
  const Rows rows{d_note, d_onset, d_contour};
  return run_batch(m, b, &rows, Rows{}, nullptr, nullptr, h_frame_off, static_cast<cudaStream_t>(stream));
}

int bp_run_inference_host(bp_model_t* m, const float* h_audio, const int64_t* h_sample_off, int32_t n_files,
                          float* h_note, float* h_onset, float* h_contour, int64_t* h_frame_off) {
  if (!m || !h_sample_off || !h_frame_off || n_files < 0) return fail(BP_E_INVALID, "bp_run_inference_host: bad argument");
  DeviceGuard g(m->device);
  Batch b{"bp_run_inference_host", h_audio, false, nullptr};
  int rc = describe_batch(b, h_sample_off, nullptr, n_files);
  if (rc) return rc;
  if (b.total_frames > 0 && (!h_note || !h_onset || !h_contour))
    return fail(BP_E_INVALID, "bp_run_inference_host: null output");
  return run_batch(m, b, nullptr, Rows{h_note, h_onset, h_contour}, nullptr, nullptr, h_frame_off, m->stream);
}

int bp_decode_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                     const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, bp_notes_t* notes,
                     void* stream) {
  if (!m || !h_frame_off || !notes || n_files < 0) return fail(BP_E_INVALID, "bp_decode_device: bad argument");
  int rc = validate_params(params);
  if (rc) return rc;
  if (!notes->note_off || !notes->bend_off) return fail(BP_E_INVALID, "bp_decode_device: notes arrays missing");
  DeviceGuard g(m->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total_frames = h_frame_off[n_files] - h_frame_off[0];
  notes->note_off[0] = 0;
  notes->bend_off[0] = 0;
  if (n_files == 0) return BP_OK;
  if (h_frame_off[0] != 0) return fail(BP_E_INVALID, "bp_decode_device: frame_off[0] must be 0");
  if (total_frames > 0 && (!d_note || !d_onset || (params->include_pitch_bends && !d_contour)))
    return fail(BP_E_INVALID, "bp_decode_device: null posteriorgram");

  const DecodeParamsDev dp = params_dev(*params);

  std::vector<long long> foff(n_files + 1), soff(n_files + 1);
  for (int i = 0; i <= n_files; ++i) {
    foff[i] = h_frame_off[i];
    if (i && foff[i] < foff[i - 1]) return fail(BP_E_INVALID, "bp_decode_device: frame offsets must be non-decreasing");
  }
  std::vector<int> counts(n_files);
  for (int attempt = 0; attempt < 2; ++attempt) {
    soff[0] = 0;
    for (int i = 0; i < n_files; ++i) {
      long long T = foff[i + 1] - foff[i];
      soff[i + 1] = soff[i] + (attempt == 0 ? std::min<long long>(T * kPitches, 8 * T + 64) : T * kPitches);
    }
    const size_t cells = (size_t)total_frames * kPitches;
    CK(m->d_frame_off.reserve(n_files + 1));
    CK(m->d_slot_off.reserve(n_files + 1));
    CK(m->energy.reserve(cells + 1));
    CK(m->candbits.reserve(cells / 32 + 2));
    CK(m->blk_max.reserve((size_t)kPitches * decode_block_slots(total_frames, n_files)));
    CK(m->blk_arg.reserve((size_t)kPitches * decode_block_slots(total_frames, n_files)));
    CK(m->max_onset.reserve(n_files));
    CK(m->max_fd.reserve(n_files));
    CK(m->note_count.reserve(n_files));
    CK(m->overflow.reserve(1));
    CK(m->slot_start.reserve((size_t)soff[n_files] + 1));
    CK(m->slot_end.reserve((size_t)soff[n_files] + 1));
    CK(m->slot_pitch.reserve((size_t)soff[n_files] + 1));
    CK(cudaMemcpyAsync(m->d_frame_off.p, foff.data(), sizeof(long long) * (n_files + 1), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m->d_slot_off.p, soff.data(), sizeof(long long) * (n_files + 1), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(m->overflow.p, 0, sizeof(int), st));
    DecodeBuffers b;
    b.frame_off = m->d_frame_off.p;
    b.energy = m->energy.p;
    b.candbits = m->candbits.p;
    b.max_onset = m->max_onset.p;
    b.max_fd = m->max_fd.p;
    b.slot_off = m->d_slot_off.p;
    b.note_count = m->note_count.p;
    b.note_start = m->slot_start.p;
    b.note_end = m->slot_end.p;
    b.note_pitch = m->slot_pitch.p;
    b.overflow = m->overflow.p;
    b.blk_max = m->blk_max.p;
    b.blk_arg = m->blk_arg.p;
    {
      ProfScope ps(m, 5, st);
      launch_decode_notes(d_note, d_onset, b, n_files, total_frames, dp, st);
    }
    CKL();
    m->launches += total_frames > 0 ? 3 : 1;
    int overflow = 0;
    CK(cudaMemcpyAsync(counts.data(), m->note_count.p, sizeof(int) * n_files, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&overflow, m->overflow.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (!overflow) break;
    if (attempt == 1) return fail(BP_E_CUDA, "bp_decode_device: note slots overflowed at full capacity (internal error)");
  }
  long long n_notes = 0;
  for (int i = 0; i < n_files; ++i) {
    n_notes += counts[i];
    if (n_notes > notes->note_capacity) {
      long long need = 0;
      for (int j = 0; j < n_files; ++j) need += counts[j];
      return g_need_notes = need, fail(BP_E_CAPACITY, "bp_decode_device: note_capacity too small, need " + std::to_string(need));
    }
    notes->note_off[i + 1] = (int32_t)n_notes;
  }
  if (n_notes == 0) return BP_OK;
  if (!notes->start_frame || !notes->end_frame || !notes->pitch_midi || !notes->amplitude)
    return fail(BP_E_INVALID, "bp_decode_device: notes arrays missing");

  CK(m->d_note_off.reserve(n_files + 1));
  CK(m->d_start.reserve(n_notes));
  CK(m->d_end.reserve(n_notes));
  CK(m->d_pitch.reserve(n_notes));
  CK(m->d_amp.reserve(n_notes));
  CK(m->d_note_base.reserve(n_notes));
  CK(m->d_bend_off.reserve(n_notes + 1));
  CK(cudaMemcpyAsync(m->d_note_off.p, notes->note_off, sizeof(int) * (n_files + 1), cudaMemcpyHostToDevice, st));
  compact_notes_kernel<<<n_files, 128, 0, st>>>(m->d_frame_off.p, m->d_slot_off.p, m->d_note_off.p, m->slot_start.p,
                                                m->slot_end.p, m->slot_pitch.p, m->d_start.p, m->d_end.p, m->d_pitch.p,
                                                m->d_note_base.p);
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(notes->start_frame, m->d_start.p, sizeof(int) * n_notes, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(notes->end_frame, m->d_end.p, sizeof(int) * n_notes, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(notes->pitch_midi, m->d_pitch.p, sizeof(int) * n_notes, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  long long n_bends = 0;
  const int with_bends = params->include_pitch_bends ? 1 : 0;
  for (long long j = 0; j < n_notes; ++j) {
    if (with_bends) n_bends += notes->end_frame[j] - notes->start_frame[j];
    if (n_bends > 0x7fffffffLL) return fail(BP_E_CAPACITY, "bp_decode_device: more than 2^31 pitch-bend values");
    notes->bend_off[j + 1] = (int32_t)n_bends;
  }
  if (with_bends && n_bends > notes->bend_capacity)
    return g_need_bends = n_bends, fail(BP_E_CAPACITY, "bp_decode_device: bend_capacity too small, need " + std::to_string(n_bends));
  if (with_bends && n_bends > 0 && !notes->bends) return fail(BP_E_INVALID, "bp_decode_device: bends array missing");
  CK(m->d_bends.reserve((size_t)n_bends + 1));
  CK(cudaMemcpyAsync(m->d_bend_off.p, notes->bend_off, sizeof(int) * (n_notes + 1), cudaMemcpyHostToDevice, st));
  {
    ProfScope ps(m, 6, st);
    launch_note_finish(d_note, d_contour, m->d_note_base.p, m->d_start.p, m->d_end.p, m->d_pitch.p, m->d_amp.p,
                       m->d_bend_off.p, m->d_bends.p, (int)n_notes, with_bends, m->d_gauss, st);
  }
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(notes->amplitude, m->d_amp.p, sizeof(float) * n_notes, cudaMemcpyDeviceToHost, st));
  if (with_bends && n_bends > 0)
    CK(cudaMemcpyAsync(notes->bends, m->d_bends.p, sizeof(int) * n_bends, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_infer_onsets_host(bp_model_t* m, const float* h_onset, const float* h_note, int64_t n_frames, double* h_out) {
  if (!m || n_frames < 0) return fail(BP_E_INVALID, "bp_infer_onsets_host: bad argument");
  if (n_frames == 0) return BP_OK;
  if (!h_onset || !h_note || !h_out) return fail(BP_E_INVALID, "bp_infer_onsets_host: null array");
  DeviceGuard g(m->device);
  cudaStream_t st = m->stream;
  const size_t cells = (size_t)n_frames * kPitches;
  const int rc = reserve_rows(m, n_frames);
  if (rc) return rc;
  CK(m->energy.reserve(cells + 1));
  CK(m->candbits.reserve(cells / 32 + 2));
  CK(m->max_onset.reserve(1));
  CK(m->max_fd.reserve(1));
  CK(m->d_frame_off.reserve(2));
  CK(m->d_onset64.reserve(cells));
  const long long foff[2] = {0, (long long)n_frames};
  CK(cudaMemcpyAsync(m->d_frame_off.p, foff, sizeof(foff), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(m->st_note.p, h_note, sizeof(float) * cells, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(m->st_onset.p, h_onset, sizeof(float) * cells, cudaMemcpyHostToDevice, st));
  DecodeBuffers b{};
  b.frame_off = m->d_frame_off.p;
  b.energy = m->energy.p;
  b.candbits = m->candbits.p;
  b.max_onset = m->max_onset.p;
  b.max_fd = m->max_fd.p;
  launch_infer_onsets(m->st_note.p, m->st_onset.p, b, 1, (long long)n_frames, m->d_onset64.p, st);
  CKL();
  m->launches += 2;
  CK(cudaMemcpyAsync(h_out, m->d_onset64.p, sizeof(double) * cells, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_pitch_bends_host(bp_model_t* m, const float* h_contour, int64_t n_frames, int32_t n_notes, const int32_t* h_start,
                        const int32_t* h_end, const int32_t* h_pitch_midi, int32_t* h_bend_off, int32_t* h_bends,
                        int64_t bend_capacity) {
  if (!m || n_frames < 0 || n_notes < 0 || !h_bend_off) return fail(BP_E_INVALID, "bp_pitch_bends_host: bad argument");
  h_bend_off[0] = 0;
  if (n_notes == 0) return BP_OK;
  if (!h_contour || !h_start || !h_end || !h_pitch_midi) return fail(BP_E_INVALID, "bp_pitch_bends_host: null array");
  long long total = 0;
  for (int j = 0; j < n_notes; ++j) {
    if (h_start[j] < 0 || h_end[j] <= h_start[j] || h_end[j] > n_frames)
      return fail(BP_E_INVALID, "bp_pitch_bends_host: note frames must satisfy 0 <= start < end <= n_frames");
    if (h_pitch_midi[j] < 21 || h_pitch_midi[j] >= 21 + kPitches)
      return fail(BP_E_INVALID, "bp_pitch_bends_host: pitch outside 21..108");
    total += h_end[j] - h_start[j];
    if (total > 0x7fffffffLL) return fail(BP_E_CAPACITY, "bp_pitch_bends_host: more than 2^31 pitch-bend values");
    h_bend_off[j + 1] = (int32_t)total;
  }
  if (total > bend_capacity) return fail(BP_E_CAPACITY, "bp_pitch_bends_host: bend_capacity too small, need " + std::to_string(total));
  if (!h_bends) return fail(BP_E_INVALID, "bp_pitch_bends_host: bends array missing");
  DeviceGuard g(m->device);
  cudaStream_t st = m->stream;
  const int rc = reserve_rows(m, n_frames);  // the kernel also averages the note posteriorgram: zeros in st_note
  if (rc) return rc;
  CK(m->d_start.reserve(n_notes));
  CK(m->d_end.reserve(n_notes));
  CK(m->d_pitch.reserve(n_notes));
  CK(m->d_amp.reserve(n_notes));
  CK(m->d_note_base.reserve(n_notes));
  CK(m->d_bend_off.reserve(n_notes + 1));
  CK(m->d_bends.reserve((size_t)total + 1));
  CK(cudaMemsetAsync(m->st_note.p, 0, sizeof(float) * (size_t)n_frames * kPitches, st));
  CK(cudaMemsetAsync(m->d_note_base.p, 0, sizeof(long long) * n_notes, st));
  CK(cudaMemcpyAsync(m->st_contour.p, h_contour, sizeof(float) * (size_t)n_frames * kContourBins, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(m->d_start.p, h_start, sizeof(int) * n_notes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(m->d_end.p, h_end, sizeof(int) * n_notes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(m->d_pitch.p, h_pitch_midi, sizeof(int) * n_notes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(m->d_bend_off.p, h_bend_off, sizeof(int) * (n_notes + 1), cudaMemcpyHostToDevice, st));
  launch_note_finish(m->st_note.p, m->st_contour.p, m->d_note_base.p, m->d_start.p, m->d_end.p, m->d_pitch.p, m->d_amp.p,
                     m->d_bend_off.p, m->d_bends.p, n_notes, 1, m->d_gauss, st);
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(h_bends, m->d_bends.p, sizeof(int) * (size_t)total, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_sonify_notes_host(bp_model_t* m, int32_t n_files, const int32_t* note_off, const double* start_s,
                         const double* end_s, const int32_t* pitch_midi, const float* amplitude, const int32_t* bend_off,
                         const int32_t* bends, int32_t multiple_pitch_bends, int32_t sample_rate, int64_t* h_sample_off,
                         double* h_audio, int64_t capacity) {
  if (!m) return fail(BP_E_INVALID, "bp_sonify_notes_host: bad argument");
  if (!h_audio)  // size query: host only
    return sonify_notes(nullptr, nullptr, n_files, note_off, start_s, end_s, pitch_midi, amplitude, bend_off, bends,
                        multiple_pitch_bends, sample_rate, h_sample_off, nullptr, capacity);
  DeviceGuard g(m->device);
  long long launches = 0;
  const int rc = sonify_notes(m->stream, &launches, n_files, note_off, start_s, end_s, pitch_midi, amplitude, bend_off,
                              bends, multiple_pitch_bends, sample_rate, h_sample_off, h_audio, capacity);
  m->launches += launches;
  return rc;
}

int bp_decode_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                   const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, bp_notes_t* notes) {
  if (!m || !h_frame_off || n_files < 0) return fail(BP_E_INVALID, "bp_decode_host: bad argument");
  DeviceGuard g(m->device);
  const int64_t total = h_frame_off[n_files];
  cudaStream_t st = m->stream;
  const int rc = reserve_rows(m, total);
  if (rc) return rc;
  if (total > 0) {
    if (!h_note || !h_onset || !h_contour) return fail(BP_E_INVALID, "bp_decode_host: null posteriorgram");
    CK(cudaMemcpyAsync(m->st_note.p, h_note, sizeof(float) * total * kPitches, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m->st_onset.p, h_onset, sizeof(float) * total * kPitches, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m->st_contour.p, h_contour, sizeof(float) * total * kContourBins, cudaMemcpyHostToDevice, st));
  }
  return bp_decode_device(m, m->st_note.p, m->st_onset.p, m->st_contour.p, h_frame_off, n_files, params, notes, st);
}

int64_t bp_decode_grid_chunk_params(int64_t total_frames, int32_t n_files) {
  const long long per = grid_setting_bytes(std::max<int64_t>(total_frames, 0), std::max<int32_t>(n_files, 0));
  return std::max(1LL, std::min(kDecodeGridMaxChunk, kDecodeGridChunkBytes / per));
}

static int decode_grid(const std::string& api, bp_model_t* m, Grams g, const int64_t* h_frame_off, int32_t n_files,
                       const bp_decode_params_t* params, int32_t n_params, bp_notes_t* notes, cudaStream_t st) {
  bool any_bends = false;
  int rc = check_grid_args(api, m, h_frame_off, n_files, params, n_params, &any_bends);
  if (rc) return rc;
  if (!notes || !notes->note_off || !notes->bend_off) return fail(BP_E_INVALID, api + ": notes arrays missing");
  g_need_notes = g_need_bends = 0;
  notes->note_off[0] = 0;
  notes->bend_off[0] = 0;
  if (n_files == 0 || n_params == 0) return BP_OK;
  const std::vector<long long> foff(h_frame_off, h_frame_off + n_files + 1);
  const long long total_frames = foff[n_files];
  if (total_frames > 0 && (!g.note || !g.onset || (any_bends && !g.contour)))
    return fail(BP_E_INVALID, api + ": null posteriorgram");
  DeviceGuard dg(m->device);
  rc = stage_grams(m, total_frames, g, any_bends);  // uploaded once for the whole grid
  if (rc) return rc;
  GridNotes gn;  // over the grid so far
  rc = decode_grid_chunks(m, api, g.note, g.onset, foff, n_files, params, n_params, st, [&](long long p0, int P,
                          const std::vector<int>& counts, const std::vector<long long>&) -> int {
    return grid_chunk_notes(m, api, g.note, g.contour, params, true, n_files, p0, P, counts, notes, gn, st);
  });
  if (rc) return rc;
  return grid_notes_result(api, gn);
}

int bp_decode_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                          const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                          bp_notes_t* notes, void* stream) {
  return decode_grid("bp_decode_grid_device", m, Grams{d_note, d_onset, d_contour, false}, h_frame_off, n_files, params,
                     n_params, notes, static_cast<cudaStream_t>(stream));
}

int bp_decode_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                        const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                        bp_notes_t* notes) {
  return decode_grid("bp_decode_grid_host", m, Grams{h_note, h_onset, h_contour, true}, h_frame_off, n_files, params,
                     n_params, notes, m ? m->stream : nullptr);
}

void bp_default_score_params(bp_score_params_t* p) {
  if (!p) return;
  p->onset_tolerance = 0.05;
  p->pitch_tolerance = 50.0;
  p->offset_ratio = 0.2;
  p->offset_min_tolerance = 0.05;
}

int bp_frame_times(int64_t n, double* out) {
  if (n < 0 || (n > 0 && !out)) return fail(BP_E_INVALID, "bp_frame_times: bad argument");
  // model_frames_to_time: (FFT_HOP / SR) * (ANNOT_N_FRAMES - AUDIO_N_SAMPLES / FFT_HOP) + MAGIC_ALIGNMENT_OFFSET, then
  // frame * FFT_HOP / SR - offset * floor(frame / ANNOT_N_FRAMES); every product rounded on its own (volatile: never
  // contracted into a multiply-add)
  volatile double hop_s = 256.0 / 22050.0, frac = 172.0 - 43844.0 / 256.0;
  volatile double prod = hop_s * frac;
  const double window_offset = prod + 0.0018;
  for (int64_t i = 0; i < n; ++i) {
    volatile double shift = window_offset * std::floor((double)i / 172.0);
    out[i] = (double)(i * 256) / 22050.0 - shift;
  }
  return BP_OK;
}

}  // extern "C"

namespace {

// Everything bp_score_grid_*, bp_match_grid_* and bp_score_onset_offset_grid_* check before anything is enqueued, in
// addition to check_grid_args.  Without `pitched` (onset-only and offset-only scores) the pitch_tolerance is validated as
// elsewhere but unused, and neither the estimate table nor the references' log2_hz is read.
int check_score_grid(const std::string& api, int n_files, int n_params, const bp_note_set_t* refs,
                     const bp_score_params_t* sp, const double* est_log2_hz, const void* out, bool pitched) {
  int rc = check_score_params(api, sp);
  if (rc || n_files == 0 || n_params == 0) return rc;
  if (!out || (pitched && !est_log2_hz)) return fail(BP_E_INVALID, api + ": bad argument");
  for (int k = 0; pitched && k < 128; ++k)
    if (!std::isfinite(est_log2_hz[k]))
      return fail(BP_E_INVALID, api + ": estimate table entry " + std::to_string(k) + ": non-finite log2_hz");
  return check_note_set(api, "references", "file", refs, n_files, pitched);
}

}  // namespace

extern "C" {

// bp_score_grid_*, and without `pitched` bp_score_onset_offset_grid_* (the references intervals only, no estimate table).
static int score_grid(const std::string& api, bp_model_t* m, Grams g, const int64_t* h_frame_off, int32_t n_files,
                      const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                      const bp_score_params_t* sp, const double* est_log2_hz, int64_t* h_counts, bool pitched,
                      cudaStream_t st) {
  bool any_bends = false;
  int rc = check_grid_args(api, m, h_frame_off, n_files, params, n_params, &any_bends);
  if (!rc) rc = check_score_grid(api, n_files, n_params, refs, sp, est_log2_hz, h_counts, pitched);
  if (rc) return rc;
  if (n_files == 0 || n_params == 0) return BP_OK;
  const std::vector<long long> foff(h_frame_off, h_frame_off + n_files + 1);
  const long long total_frames = foff[n_files];
  if (total_frames > 0 && (!g.note || !g.onset)) return fail(BP_E_INVALID, api + ": null posteriorgram");
  DeviceGuard dg(m->device);
  NoteRefs nr;
  rc = stage_grams(m, total_frames, g, false);
  if (!rc) rc = upload_note_refs(m, refs, n_files, foff, *sp, pitched ? est_log2_hz : nullptr, nr, st);
  if (rc) return rc;
  CK(m->score_counts.reserve((size_t)n_params * n_files * 4));
  rc = decode_grid_chunks(m, api, g.note, g.onset, foff, n_files, params, n_params, st, [&](long long p0, int P,
                          const std::vector<int>&, const std::vector<long long>& soff) -> int {
    const long long n_pairs = (long long)P * n_files;
    CK(m->score_ws_ref.reserve((size_t)((pitched ? 2 : 6) * P * nr.n_refs) + 1));
    CK(m->score_ws_est.reserve((size_t)(4 * soff[n_pairs] + (pitched ? 0 : 2 * n_pairs)) + 1));
    ScoreEst e = nr.e;
    e.off = m->d_slot_off.p;
    e.count = m->note_count.p;
    e.start = m->slot_start.p;
    e.end = m->slot_end.p;
    if (pitched) e.pitch = m->slot_pitch.p;
    (pitched ? launch_score_match : launch_onset_offset)(nr.sr, e, nr.tol,
                                                         ScoreWork{m->score_ws_ref.p, m->score_ws_est.p, nr.n_refs},
                                                         n_files, n_pairs, m->score_counts.p + 4 * p0 * n_files, st);
    CKL();
    m->launches += 1;
    return BP_OK;
  });
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_counts, m->score_counts.p, sizeof(long long) * 4 * n_params * n_files, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_score_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const int64_t* h_frame_off,
                         int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                         const bp_score_params_t* sp, const double* est_log2_hz, int64_t* h_counts, void* stream) {
  return score_grid("bp_score_grid_device", m, Grams{d_note, d_onset, nullptr, false}, h_frame_off, n_files, params,
                    n_params, refs, sp, est_log2_hz, h_counts, true, static_cast<cudaStream_t>(stream));
}

int bp_score_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const int64_t* h_frame_off,
                       int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                       const bp_score_params_t* sp, const double* est_log2_hz, int64_t* h_counts) {
  return score_grid("bp_score_grid_host", m, Grams{h_note, h_onset, nullptr, true}, h_frame_off, n_files, params,
                    n_params, refs, sp, est_log2_hz, h_counts, true, m ? m->stream : nullptr);
}

// bp_score_notes_host, and without `pitched` bp_score_onset_offset_notes_host (intervals only).
static int score_notes(const std::string& api, bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs,
                       int32_t n_items, const bp_score_params_t* sp, int64_t* h_counts, bool pitched) {
  int rc = check_notes_call(api, m, est, refs, n_items, sp, h_counts, pitched);
  if (rc || n_items == 0) return rc;
  const long long n_est = est->note_off[n_items], n_refs = refs->note_off[n_items];
  bp_note_set_t e = *est;
  std::vector<double> on, off;
  if (!pitched) {  // the count does not depend on the order of the estimates: each item's onsets and offsets go up sorted, apart
    on.assign(est->onset_s, est->onset_s + n_est);
    off.assign(est->offset_s, est->offset_s + n_est);
    for (int i = 0; i < n_items; ++i) {
      std::sort(on.begin() + est->note_off[i], on.begin() + est->note_off[i + 1]);
      std::sort(off.begin() + est->note_off[i], off.begin() + est->note_off[i + 1]);
    }
    e = bp_note_set_t{est->note_off, on.data(), off.data(), nullptr};
  }
  DeviceGuard g(m->device);
  cudaStream_t st = m->stream;
  NoteRefs nr;
  rc = upload_notes(m, e, refs, n_items, *sp, pitched, nr, st);
  if (rc) return rc;
  CK(m->score_ws_ref.reserve((size_t)((pitched ? 2 : 6) * n_refs) + 1));
  CK(m->score_ws_est.reserve((size_t)(4 * n_est + (pitched ? 0 : 2 * n_items)) + 1));
  CK(m->score_counts.reserve((size_t)n_items * 4));
  (pitched ? launch_score_match : launch_onset_offset)(nr.sr, nr.e, nr.tol,
                                                       ScoreWork{m->score_ws_ref.p, m->score_ws_est.p, n_refs}, n_items,
                                                       n_items, m->score_counts.p, st);
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(h_counts, m->score_counts.p, sizeof(long long) * 4 * n_items, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_score_notes_host(bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs, int32_t n_items,
                        const bp_score_params_t* sp, int64_t* h_counts) {
  return score_notes("bp_score_notes_host", m, est, refs, n_items, sp, h_counts, true);
}

static int match_grid(const std::string& api, bp_model_t* m, Grams g, const int64_t* h_frame_off, int32_t n_files,
                      const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                      const bp_score_params_t* sp, const double* est_log2_hz, bp_notes_t* notes, int32_t* h_match,
                      cudaStream_t st) {
  bool any_bends = false;
  int rc = check_grid_args(api, m, h_frame_off, n_files, params, n_params, &any_bends);
  if (!rc) rc = check_score_grid(api, n_files, n_params, refs, sp, est_log2_hz, h_match, true);
  if (rc) return rc;
  if (!notes || !notes->note_off || !notes->bend_off) return fail(BP_E_INVALID, api + ": notes arrays missing");
  g_need_notes = g_need_bends = 0;
  notes->note_off[0] = 0;
  notes->bend_off[0] = 0;
  if (n_files == 0 || n_params == 0) return BP_OK;
  const std::vector<long long> foff(h_frame_off, h_frame_off + n_files + 1);
  const long long total_frames = foff[n_files];
  if (total_frames > 0 && (!g.note || !g.onset)) return fail(BP_E_INVALID, api + ": null posteriorgram");
  DeviceGuard dg(m->device);
  NoteRefs nr;
  rc = stage_grams(m, total_frames, g, false);
  if (!rc) rc = upload_note_refs(m, refs, n_files, foff, *sp, est_log2_hz, nr, st);
  if (rc) return rc;
  const long long n_refs = nr.n_refs;
  GridNotes gn;  // over the grid so far
  rc = decode_grid_chunks(m, api, g.note, g.onset, foff, n_files, params, n_params, st, [&](long long p0, int P,
                          const std::vector<int>& counts, const std::vector<long long>&) -> int {
    const long long note0 = gn.n_notes, n_pairs = (long long)P * n_files;
    int rc = grid_chunk_notes(m, api, g.note, nullptr, params, false, n_files, p0, P, counts, notes, gn, st);
    if (rc || !gn.notes_fit || n_refs == 0) return rc;
    int32_t* out = h_match + 2 * p0 * n_refs;
    if (gn.n_notes == note0) {  // no estimated note in this chunk
      std::fill(out, out + 2 * P * n_refs, -1);
      return BP_OK;
    }
    // the compacted notes: pair q's are [est_off[q], est_off[q + 1]) of m->d_start / d_end / d_pitch
    std::vector<long long> est_off(n_pairs + 1);
    for (long long q = 0; q <= n_pairs; ++q) est_off[q] = notes->note_off[p0 * n_files + q] - note0;
    CK(m->match_est_off.reserve((size_t)n_pairs + 1));
    CK(cudaMemcpyAsync(m->match_est_off.p, est_off.data(), sizeof(long long) * (n_pairs + 1), cudaMemcpyHostToDevice,
                       st));
    CK(m->match_out.reserve((size_t)(2 * P * n_refs)));
    ScoreEst e = nr.e;
    e.off = m->match_est_off.p;
    e.start = m->d_start.p;
    e.end = m->d_end.p;
    e.pitch = m->d_pitch.p;
    rc = match_pairs(m, api, nr.sr, nr.r_orig, e, nr.tol, n_files, n_pairs, est_off, refs->note_off, n_refs,
                     m->match_out.p, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out, m->match_out.p, sizeof(int) * 2 * P * n_refs, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return BP_OK;
  });
  if (rc) return rc;
  return grid_notes_result(api, gn);
}

int bp_match_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const int64_t* h_frame_off,
                         int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                         const bp_score_params_t* sp, const double* est_log2_hz, bp_notes_t* notes, int32_t* h_match,
                         void* stream) {
  return match_grid("bp_match_grid_device", m, Grams{d_note, d_onset, nullptr, false}, h_frame_off, n_files, params,
                    n_params, refs, sp, est_log2_hz, notes, h_match, static_cast<cudaStream_t>(stream));
}

int bp_match_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const int64_t* h_frame_off,
                       int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                       const bp_score_params_t* sp, const double* est_log2_hz, bp_notes_t* notes, int32_t* h_match) {
  return match_grid("bp_match_grid_host", m, Grams{h_note, h_onset, nullptr, true}, h_frame_off, n_files, params,
                    n_params, refs, sp, est_log2_hz, notes, h_match, m ? m->stream : nullptr);
}

int bp_match_notes_host(bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs, int32_t n_items,
                        const bp_score_params_t* sp, int32_t* h_match) {
  const std::string api = "bp_match_notes_host";
  int rc = check_notes_call(api, m, est, refs, n_items, sp, h_match, true);
  if (rc || n_items == 0) return rc;
  const long long n_refs = refs->note_off[n_items];
  if (n_refs == 0) return BP_OK;
  DeviceGuard g(m->device);
  cudaStream_t st = m->stream;
  NoteRefs nr;
  rc = upload_notes(m, *est, refs, n_items, *sp, true, nr, st);
  if (rc) return rc;
  CK(m->match_out.reserve((size_t)(2 * n_refs)));
  const std::vector<long long> est_off(est->note_off, est->note_off + n_items + 1);
  rc = match_pairs(m, api, nr.sr, nr.r_orig, nr.e, nr.tol, n_items, n_items, est_off, refs->note_off, n_refs,
                   m->match_out.p, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_match, m->match_out.p, sizeof(int) * 2 * n_refs, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

// ---- onset-only and offset-only scores (bp_score_onset_offset_*) -------------------------------------------------------

int bp_score_onset_offset_grid_device(bp_model_t* m, const float* d_note, const float* d_onset,
                                      const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                      int32_t n_params, const bp_note_set_t* refs, const bp_score_params_t* sp,
                                      const double* est_log2_hz, int64_t* h_counts, void* stream) {
  return score_grid("bp_score_onset_offset_grid_device", m, Grams{d_note, d_onset, nullptr, false}, h_frame_off, n_files,
                    params, n_params, refs, sp, est_log2_hz, h_counts, false, static_cast<cudaStream_t>(stream));
}

int bp_score_onset_offset_grid_host(bp_model_t* m, const float* h_note, const float* h_onset,
                                    const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                    int32_t n_params, const bp_note_set_t* refs, const bp_score_params_t* sp,
                                    const double* est_log2_hz, int64_t* h_counts) {
  return score_grid("bp_score_onset_offset_grid_host", m, Grams{h_note, h_onset, nullptr, true}, h_frame_off, n_files,
                    params, n_params, refs, sp, est_log2_hz, h_counts, false, m ? m->stream : nullptr);
}

int bp_score_onset_offset_notes_host(bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs,
                                     int32_t n_items, const bp_score_params_t* sp, int64_t* h_counts) {
  return score_notes("bp_score_onset_offset_notes_host", m, est, refs, n_items, sp, h_counts, false);
}

}  // extern "C"

// ---- frame-level scoring (bp_score_frames_grid_*, bp_score_multipitch_host, bp_multipitch_map,
// bp_score_salience_grid_*) ----------------------------------------------------------------------------------------------
namespace {

// Validates n multi-pitch series (`what` "references" / "estimates", set unit "file" / "item"): offsets start at 0 and
// never decrease, at most 2^31 - 1 frames per set and values per frame, times finite, >= 0 and non-decreasing within a
// set, midi finite, chroma in [0, 12).
int check_mp_set(const std::string& api, const char* what, const char* unit, const bp_multipitch_set_t* s, int n) {
  const std::string who = api + ": " + what;
  if (!s || !s->frame_off) return fail(BP_E_INVALID, who + ": null multipitch set");
  if (s->frame_off[0] != 0) return fail(BP_E_INVALID, who + ": frame_off[0] must be 0");
  for (int i = 0; i < n; ++i)
    if (s->frame_off[i + 1] < s->frame_off[i] || s->frame_off[i + 1] - s->frame_off[i] > INT_MAX)
      return fail(BP_E_INVALID, who + " " + unit + " " + std::to_string(i) + ": bad frame_off");
  const long long F = s->frame_off[n];
  if (F == 0) return BP_OK;
  if (!s->time_s || !s->value_off) return fail(BP_E_INVALID, who + ": null array");
  if (s->value_off[0] != 0) return fail(BP_E_INVALID, who + ": value_off[0] must be 0");
  for (long long j = 0; j < F; ++j)
    if (s->value_off[j + 1] < s->value_off[j] || s->value_off[j + 1] - s->value_off[j] > INT_MAX) {
      const long long i = std::upper_bound(s->frame_off, s->frame_off + n + 1, j) - s->frame_off - 1;
      return fail(BP_E_INVALID, who + " " + unit + " " + std::to_string(i) + " frame " +
                                    std::to_string(j - s->frame_off[i]) + ": bad value_off");
    }
  if (s->value_off[F] > 0 && (!s->midi || !s->chroma)) return fail(BP_E_INVALID, who + ": null array");
  for (int i = 0; i < n; ++i)
    for (long long j = s->frame_off[i]; j < s->frame_off[i + 1]; ++j) {
      const std::string at = who + " " + unit + " " + std::to_string(i) + " frame " + std::to_string(j - s->frame_off[i]);
      const double t = s->time_s[j];
      const char* why = !std::isfinite(t)                             ? "non-finite time"
                        : t < 0                                       ? "time < 0"
                        : j > s->frame_off[i] && t < s->time_s[j - 1] ? "time decreases"
                                                                      : nullptr;
      if (why) return fail(BP_E_INVALID, at + ": " + why);
      for (long long v = s->value_off[j]; v < s->value_off[j + 1]; ++v) {
        const double c = s->chroma[v];
        why = !std::isfinite(s->midi[v]) ? "non-finite midi" : !(c >= 0 && c < 12) ? "chroma outside [0, 12)" : nullptr;
        if (why) return fail(BP_E_INVALID, at + " value " + std::to_string(v - s->value_off[j]) + ": " + why);
      }
    }
  return BP_OK;
}

int check_window(const std::string& api, double window) {
  if (!std::isfinite(window) || window < 0) return fail(BP_E_INVALID, api + ": window must be finite and >= 0");
  return BP_OK;
}

// Rule 1 of the metric (include/bp_b200.h): the estimate frame each reference time reads, -1 for none.
template <class Out>
void multipitch_map(const double* et, long long ne, const double* rt, long long nr, Out* out) {
  if (ne == 0) {
    for (long long k = 0; k < nr; ++k) out[k] = -1;
    return;
  }
  bool same = ne == nr;  // np.allclose(est_t, ref_t): |a - b| <= 1e-8 + 1e-5 |b|, each operation rounded on its own
  for (long long k = 0; same && k < nr; ++k) {
    volatile double tol = 1e-5 * std::fabs(rt[k]);
    same = std::fabs(et[k] - rt[k]) <= 1e-8 + tol;
  }
  if (same) {
    for (long long k = 0; k < nr; ++k) out[k] = (Out)k;
    return;
  }
  // interp1d(kind='nearest'): x_bds = x / 2, x_bds[1:] + x_bds[:-1], searchsorted(side='left'), clip; outside
  // [x[0], x[-1]] the fill value
  std::vector<double> bds(ne - 1);
  for (long long i = 0; i + 1 < ne; ++i) bds[i] = et[i + 1] / 2.0 + et[i] / 2.0;
  for (long long k = 0; k < nr; ++k) {
    const double t = rt[k];
    const long long i = std::lower_bound(bds.begin(), bds.end(), t) - bds.begin();
    out[k] = t < et[0] || t > et[ne - 1] ? (Out)-1 : (Out)std::min(i, ne - 1);
  }
}

// The values of frames [0, F) of s, each frame's sorted by midi (stable): appended to pk; offsets into o[3]
// (value_off, midi, chroma).
void pack_mp_values(const bp_multipitch_set_t* s, long long F, Pack& pk, size_t* o) {
  const long long V = F > 0 ? s->value_off[F] : 0;
  std::vector<long long> idx(V), voff(F + 1, 0);
  std::vector<double> mi(V), ch(V);
  for (long long v = 0; v < V; ++v) idx[v] = v;
  for (long long j = 0; j < F; ++j) {
    voff[j + 1] = s->value_off[j + 1];
    std::stable_sort(idx.begin() + s->value_off[j], idx.begin() + s->value_off[j + 1],
                     [&](long long a, long long b) { return s->midi[a] < s->midi[b]; });
  }
  for (long long v = 0; v < V; ++v) mi[v] = s->midi[idx[v]], ch[v] = s->chroma[idx[v]];
  o[0] = pk.add(voff.data(), sizeof(long long) * (F + 1));
  o[1] = pk.add(mi.data(), sizeof(double) * V);
  o[2] = pk.add(ch.data(), sizeof(double) * V);
}

// A value table of n MIDI numbers or posteriorgram bins (`what` "estimate table" / "bin table"): midi finite and
// non-decreasing, chroma in [0, 12).
int check_value_table(const std::string& api, const char* what, const double* midi, const double* chroma, int n) {
  for (int k = 0; k < n; ++k) {
    const std::string at = api + ": " + what + " entry " + std::to_string(k);
    if (!std::isfinite(midi[k])) return fail(BP_E_INVALID, at + ": non-finite midi");
    if (k > 0 && midi[k] < midi[k - 1]) return fail(BP_E_INVALID, at + ": midi decreases");
    if (!(chroma[k] >= 0 && chroma[k] < 12)) return fail(BP_E_INVALID, at + ": chroma outside [0, 12)");
  }
  return BP_OK;
}

// Everything bp_score_frames_grid_* check before anything is enqueued, in addition to check_grid_args.
int check_frames_grid(const std::string& api, int n_files, int n_params, const bp_multipitch_set_t* refs, double window,
                      const double* est_midi, const double* est_chroma, const int64_t* h_counts) {
  int rc = check_window(api, window);
  if (rc || n_files == 0 || n_params == 0) return rc;
  if (!h_counts || !est_midi || !est_chroma) return fail(BP_E_INVALID, api + ": bad argument");
  rc = check_value_table(api, "estimate table", est_midi, est_chroma, 128);
  return rc ? rc : check_mp_set(api, "references", "file", refs, n_files);
}

FrameRefs frame_refs_at(const unsigned char* d, size_t o_owner, size_t o_est, const size_t* o_val, long long K) {
  return FrameRefs{reinterpret_cast<const int*>(d + o_owner), reinterpret_cast<const int*>(d + o_est),
                   reinterpret_cast<const long long*>(d + o_val[0]), reinterpret_cast<const double*>(d + o_val[1]),
                   reinterpret_cast<const double*>(d + o_val[2]), K};
}

// The references of a frame-level grid call into `pk`: per reference frame its file and the frame of that file it reads
// at the model's frame times (files of frame offsets foff), then the sorted values; offsets of the sections in o[5]
// (owner, estimate frame, pack_mp_values' three).
void pack_ref_frames(const bp_multipitch_set_t* refs, const std::vector<long long>& foff, int n_files, Pack& pk,
                     size_t* o) {
  const long long K = refs->frame_off[n_files];
  std::vector<int> owner(K), est(K);
  std::vector<double> et;
  for (int f = 0; f < n_files; ++f) {
    const long long T = foff[f + 1] - foff[f], k0 = refs->frame_off[f];
    et.resize(T);
    bp_frame_times(T, et.data());
    multipitch_map(et.data(), T, refs->time_s + k0, refs->frame_off[f + 1] - k0, est.data() + k0);
    std::fill(owner.begin() + k0, owner.begin() + refs->frame_off[f + 1], f);
  }
  o[0] = pk.add(owner.data(), sizeof(int) * K);
  o[1] = pk.add(est.data(), sizeof(int) * K);
  pack_mp_values(refs, K, pk, o + 2);
}

// Salience scoring (bp_score_salience_grid_*): posteriorgram widths up to this many bins; settings per chunk bounded by
// this much chroma-matching workspace (bp_score_salience_chunk_params).
constexpr int kMaxSalienceWidth = 1024;
constexpr long long kSalienceChunkBytes = 2LL << 30;

// Everything bp_score_salience_grid_* check before anything is enqueued (include/bp_b200.h).
int check_salience_grid(const std::string& api, const bp_model* m, int width, const int64_t* h_frame_off, int n_files,
                        const bp_salience_params_t* params, int n_params, const bp_multipitch_set_t* refs, double window,
                        const double* bin_midi, const double* bin_chroma, const int64_t* h_counts) {
  if (!m || n_files < 0 || n_params < 0 || (n_params > 0 && !params)) return fail(BP_E_INVALID, api + ": bad argument");
  if (width < 1 || width > kMaxSalienceWidth)
    return fail(BP_E_INVALID, api + ": width must be in [1, " + std::to_string(kMaxSalienceWidth) + "]");
  for (int k = 0; k < n_params; ++k) {
    const bp_salience_params_t& p = params[k];
    const char* why = !(std::isfinite(p.threshold) && p.threshold > 0)        ? "threshold must be finite and > 0"
                      : p.peak_pick != 0 && p.peak_pick != 1                  ? "peak_pick must be 0 or 1"
                      : !(0 <= p.bin_lo && p.bin_lo <= p.bin_hi && p.bin_hi <= width) ? "need 0 <= bin_lo <= bin_hi <= width"
                                                                              : nullptr;
    if (why) return fail(BP_E_INVALID, api + ": salience params[" + std::to_string(k) + "]: " + why);
  }
  int rc = check_window(api, window);
  if (rc || n_files == 0 || n_params == 0) return rc;
  if (!h_frame_off || !h_counts || !bin_midi || !bin_chroma) return fail(BP_E_INVALID, api + ": bad argument");
  rc = check_value_table(api, "bin table", bin_midi, bin_chroma, width);
  if (rc) return rc;
  if (h_frame_off[0] != 0) return fail(BP_E_INVALID, api + ": frame_off[0] must be 0");
  for (int i = 0; i < n_files; ++i)
    if (h_frame_off[i + 1] < h_frame_off[i] || h_frame_off[i + 1] - h_frame_off[i] > INT_MAX)
      return fail(BP_E_INVALID, api + ": file " + std::to_string(i) + ": bad frame_off");
  return check_mp_set(api, "references", "file", refs, n_files);
}

}  // namespace

extern "C" {

int bp_multipitch_map(const double* est_t, int64_t n_est, const double* ref_t, int64_t n_ref, int64_t* out) {
  if (n_est < 0 || n_ref < 0 || (n_est > 0 && !est_t) || (n_ref > 0 && (!ref_t || !out)))
    return fail(BP_E_INVALID, "bp_multipitch_map: bad argument");
  for (int64_t i = 0; i < n_est; ++i)
    if (!std::isfinite(est_t[i]) || (i > 0 && est_t[i] < est_t[i - 1]))
      return fail(BP_E_INVALID, "bp_multipitch_map: estimate frame " + std::to_string(i) + ": non-finite or decreasing time");
  for (int64_t k = 0; k < n_ref; ++k)
    if (!std::isfinite(ref_t[k]))
      return fail(BP_E_INVALID, "bp_multipitch_map: reference frame " + std::to_string(k) + ": non-finite time");
  multipitch_map(est_t, n_est, ref_t, n_ref, out);
  return BP_OK;
}

static int score_frames_grid(const std::string& api, bp_model_t* m, Grams g, const int64_t* h_frame_off, int32_t n_files,
                             const bp_decode_params_t* params, int32_t n_params, const bp_multipitch_set_t* refs,
                             double window, const double* est_midi, const double* est_chroma, int64_t* h_counts,
                             cudaStream_t st) {
  bool any_bends = false;
  int rc = check_grid_args(api, m, h_frame_off, n_files, params, n_params, &any_bends);
  if (!rc) rc = check_frames_grid(api, n_files, n_params, refs, window, est_midi, est_chroma, h_counts);
  if (rc) return rc;
  if (n_files == 0 || n_params == 0) return BP_OK;
  const std::vector<long long> foff(h_frame_off, h_frame_off + n_files + 1);
  const long long total_frames = foff[n_files], cells = total_frames * kPitches;
  if (total_frames > 0 && (!g.note || !g.onset)) return fail(BP_E_INVALID, api + ": null posteriorgram");
  DeviceGuard dg(m->device);
  rc = stage_grams(m, total_frames, g, false);
  if (rc) return rc;
  // one upload per call: the reference frames and the tables
  const long long K = refs->frame_off[n_files], V = K > 0 ? refs->value_off[K] : 0;
  Pack pk;
  size_t o_ref[5];
  pack_ref_frames(refs, foff, n_files, pk, o_ref);
  const size_t o_tm = pk.add(est_midi, sizeof(double) * 128), o_tc = pk.add(est_chroma, sizeof(double) * 128);
  CK(m->score_in.reserve(pk.buf.size()));
  CK(cudaMemcpyAsync(m->score_in.p, pk.buf.data(), pk.buf.size(), cudaMemcpyHostToDevice, st));
  const long long n_counts = (long long)n_params * n_files * kFrameCounts;
  CK(m->score_counts.reserve((size_t)n_counts));
  CK(cudaMemsetAsync(m->score_counts.p, 0, sizeof(long long) * n_counts, st));
  const FrameRefs R = frame_refs_at(m->score_in.p, o_ref[0], o_ref[1], o_ref + 2, K);
  rc = decode_grid_chunks(m, api, g.note, g.onset, foff, n_files, params, n_params, st, [&](long long p0, int P,
                          const std::vector<int>&, const std::vector<long long>&) -> int {
    // each setting's E is dead once the loops have run: it becomes that setting's count roll
    int* roll = reinterpret_cast<int*>(m->energy.p);
    if (cells > 0) CK(cudaMemsetAsync(roll, 0, sizeof(int) * P * cells, st));
    launch_frame_roll(m->d_frame_off.p, m->d_slot_off.p, m->note_count.p, m->slot_start.p, m->slot_end.p,
                      m->slot_pitch.p, n_files, P, roll, cells, st);
    CKL();
    CK(m->score_ws_ref.reserve((size_t)(P * frame_ws_stride(V, K)) + 1));
    FrameEst e{};
    e.roll = roll;
    e.roll_stride = cells;
    e.frame_off = m->d_frame_off.p;
    e.tab_midi = reinterpret_cast<const double*>(m->score_in.p + o_tm);
    e.tab_chroma = reinterpret_cast<const double*>(m->score_in.p + o_tc);
    launch_frame_match(R, e, window, m->score_ws_ref.p, n_files, P, m->score_counts.p + kFrameCounts * p0 * n_files, st);
    CKL();
    m->launches += 3;
    return BP_OK;
  });
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_counts, m->score_counts.p, sizeof(long long) * n_counts, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_score_frames_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const int64_t* h_frame_off,
                                int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                                const bp_multipitch_set_t* refs, double window, const double* est_midi,
                                const double* est_chroma, int64_t* h_counts, void* stream) {
  return score_frames_grid("bp_score_frames_grid_device", m, Grams{d_note, d_onset, nullptr, false}, h_frame_off,
                           n_files, params, n_params, refs, window, est_midi, est_chroma, h_counts,
                           static_cast<cudaStream_t>(stream));
}

int bp_score_frames_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const int64_t* h_frame_off,
                              int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                              const bp_multipitch_set_t* refs, double window, const double* est_midi,
                              const double* est_chroma, int64_t* h_counts) {
  return score_frames_grid("bp_score_frames_grid_host", m, Grams{h_note, h_onset, nullptr, true}, h_frame_off, n_files,
                           params, n_params, refs, window, est_midi, est_chroma, h_counts, m ? m->stream : nullptr);
}

int bp_score_multipitch_host(bp_model_t* m, const bp_multipitch_set_t* est, const bp_multipitch_set_t* refs,
                             int32_t n_items, double window, int64_t* h_counts) {
  const std::string api = "bp_score_multipitch_host";
  if (!m || n_items < 0) return fail(BP_E_INVALID, api + ": bad argument");
  int rc = check_window(api, window);
  if (rc || n_items == 0) return rc;
  if (!h_counts) return fail(BP_E_INVALID, api + ": bad argument");
  rc = check_mp_set(api, "estimates", "item", est, n_items);
  if (!rc) rc = check_mp_set(api, "references", "item", refs, n_items);
  if (rc) return rc;
  const long long K = refs->frame_off[n_items], V = K > 0 ? refs->value_off[K] : 0, FE = est->frame_off[n_items];
  if (FE > INT_MAX) return fail(BP_E_INVALID, api + ": more than 2^31 - 1 estimate frames");
  std::vector<int> owner(K), emap(K);
  for (int i = 0; i < n_items; ++i) {
    const long long k0 = refs->frame_off[i], e0 = est->frame_off[i];
    multipitch_map(est->time_s + e0, est->frame_off[i + 1] - e0, refs->time_s + k0, refs->frame_off[i + 1] - k0,
                   emap.data() + k0);
    for (long long k = k0; k < refs->frame_off[i + 1]; ++k) {
      owner[k] = i;
      if (emap[k] >= 0) emap[k] += (int)e0;  // global estimate frame
    }
  }
  Pack pk;
  const size_t o_owner = pk.add(owner.data(), sizeof(int) * K), o_est = pk.add(emap.data(), sizeof(int) * K);
  size_t o_val[3], o_eval[3];
  pack_mp_values(refs, K, pk, o_val);
  pack_mp_values(est, FE, pk, o_eval);
  DeviceGuard g(m->device);
  cudaStream_t st = m->stream;
  CK(m->score_in.reserve(pk.buf.size()));
  CK(m->score_ws_ref.reserve((size_t)frame_ws_stride(V, K) + 1));
  CK(m->score_counts.reserve((size_t)n_items * kFrameCounts));
  CK(cudaMemcpyAsync(m->score_in.p, pk.buf.data(), pk.buf.size(), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(m->score_counts.p, 0, sizeof(long long) * kFrameCounts * n_items, st));
  const unsigned char* d = m->score_in.p;
  FrameEst e{};
  e.voff = reinterpret_cast<const long long*>(d + o_eval[0]);
  e.midi = reinterpret_cast<const double*>(d + o_eval[1]);
  e.chroma = reinterpret_cast<const double*>(d + o_eval[2]);
  launch_frame_match(frame_refs_at(d, o_owner, o_est, o_val, K), e, window, m->score_ws_ref.p, n_items, 1,
                     m->score_counts.p, st);
  CKL();
  m->launches += 1;
  CK(cudaMemcpyAsync(h_counts, m->score_counts.p, sizeof(long long) * kFrameCounts * n_items, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int64_t bp_score_salience_chunk_params(int64_t n_ref_frames, int64_t n_ref_values) {
  const long long per = frame_ws_stride(std::max<int64_t>(n_ref_values, 0), std::max<int64_t>(n_ref_frames, 0)) *
                        (long long)sizeof(int);  // 16 V + 8 K bytes
  return std::max(1LL, kSalienceChunkBytes / std::max(1LL, per));
}

static int score_salience_grid(const std::string& api, bp_model_t* m, Grams g, int32_t width,
                               const int64_t* h_frame_off, int32_t n_files, const bp_salience_params_t* params,
                               int32_t n_params, const bp_multipitch_set_t* refs, double window, const double* bin_midi,
                               const double* bin_chroma, int64_t* h_counts, cudaStream_t st) {
  int rc = check_salience_grid(api, m, width, h_frame_off, n_files, params, n_params, refs, window, bin_midi, bin_chroma,
                               h_counts);
  if (rc) return rc;
  if (n_files == 0 || n_params == 0) return BP_OK;
  const std::vector<long long> foff(h_frame_off, h_frame_off + n_files + 1);
  if (foff[n_files] > 0 && !g.contour) return fail(BP_E_INVALID, api + ": null posteriorgram");
  DeviceGuard dg(m->device);
  rc = stage_grams(m, foff[n_files], g, true, width);
  if (rc) return rc;
  // one upload per call: the reference frames, the bin tables and every setting
  const long long K = refs->frame_off[n_files], V = K > 0 ? refs->value_off[K] : 0;
  std::vector<SalienceSettingDev> sal(n_params);
  for (int k = 0; k < n_params; ++k)
    sal[k] = SalienceSettingDev{params[k].threshold, params[k].peak_pick, params[k].bin_lo, params[k].bin_hi, 0};
  Pack pk;
  size_t o_ref[5];
  pack_ref_frames(refs, foff, n_files, pk, o_ref);
  const size_t o_tm = pk.add(bin_midi, sizeof(double) * width), o_tc = pk.add(bin_chroma, sizeof(double) * width),
               o_set = pk.add(sal.data(), sizeof(SalienceSettingDev) * n_params);
  CK(m->score_in.reserve(pk.buf.size()));
  CK(cudaMemcpyAsync(m->score_in.p, pk.buf.data(), pk.buf.size(), cudaMemcpyHostToDevice, st));
  CK(m->d_frame_off.reserve(n_files + 1));
  CK(cudaMemcpyAsync(m->d_frame_off.p, foff.data(), sizeof(long long) * (n_files + 1), cudaMemcpyHostToDevice, st));
  const long long n_counts = (long long)n_params * n_files * kFrameCounts;
  CK(m->score_counts.reserve((size_t)n_counts));
  CK(cudaMemsetAsync(m->score_counts.p, 0, sizeof(long long) * n_counts, st));
  const long long chunk = bp_score_salience_chunk_params(K, V);
  CK(m->score_ws_ref.reserve((size_t)(std::min<long long>(chunk, n_params) * frame_ws_stride(V, K)) + 1));
  const FrameRefs R = frame_refs_at(m->score_in.p, o_ref[0], o_ref[1], o_ref + 2, K);
  FrameEst e{};
  e.gram = g.contour;
  e.width = width;
  e.frame_off = m->d_frame_off.p;
  e.tab_midi = reinterpret_cast<const double*>(m->score_in.p + o_tm);
  e.tab_chroma = reinterpret_cast<const double*>(m->score_in.p + o_tc);
  for (long long p0 = 0; p0 < n_params; p0 += chunk) {
    const int P = (int)std::min<long long>(chunk, n_params - p0);
    e.salience = reinterpret_cast<const SalienceSettingDev*>(m->score_in.p + o_set) + p0;
    launch_frame_match(R, e, window, m->score_ws_ref.p, n_files, P, m->score_counts.p + kFrameCounts * p0 * n_files, st);
    CKL();
    m->launches += 1;
  }
  CK(cudaMemcpyAsync(h_counts, m->score_counts.p, sizeof(long long) * n_counts, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_score_salience_grid_device(bp_model_t* m, const float* d_gram, int32_t width, const int64_t* h_frame_off,
                                  int32_t n_files, const bp_salience_params_t* params, int32_t n_params,
                                  const bp_multipitch_set_t* refs, double window, const double* bin_midi,
                                  const double* bin_chroma, int64_t* h_counts, void* stream) {
  return score_salience_grid("bp_score_salience_grid_device", m, Grams{nullptr, nullptr, d_gram, false}, width,
                             h_frame_off, n_files, params, n_params, refs, window, bin_midi, bin_chroma, h_counts,
                             static_cast<cudaStream_t>(stream));
}

int bp_score_salience_grid_host(bp_model_t* m, const float* h_gram, int32_t width, const int64_t* h_frame_off,
                                int32_t n_files, const bp_salience_params_t* params, int32_t n_params,
                                const bp_multipitch_set_t* refs, double window, const double* bin_midi,
                                const double* bin_chroma, int64_t* h_counts) {
  return score_salience_grid("bp_score_salience_grid_host", m, Grams{nullptr, nullptr, h_gram, true}, width,
                             h_frame_off, n_files, params, n_params, refs, window, bin_midi, bin_chroma, h_counts,
                             m ? m->stream : nullptr);
}

int bp_transcribe_device(bp_model_t* m, const float* d_audio, const int64_t* h_sample_off, int32_t n_files,
                         const bp_decode_params_t* params, int64_t* h_frame_off, bp_notes_t* notes, void* stream) {
  if (!m || !h_sample_off || !h_frame_off || n_files < 0) return fail(BP_E_INVALID, "bp_transcribe_device: bad argument");
  int rc = validate_params(params);
  if (rc) return rc;
  DeviceGuard g(m->device);
  Batch b{"bp_transcribe_device", d_audio, true, nullptr};
  rc = describe_batch(b, h_sample_off, nullptr, n_files);
  if (rc) return rc;
  return run_batch(m, b, nullptr, Rows{}, params, notes, h_frame_off, static_cast<cudaStream_t>(stream));
}

int bp_transcribe_host(bp_model_t* m, const float* h_audio, const int64_t* h_sample_off, int32_t n_files,
                       const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                       int64_t* h_frame_off, bp_notes_t* notes) {
  if (!m || !h_sample_off || !h_frame_off || n_files < 0) return fail(BP_E_INVALID, "bp_transcribe_host: bad argument");
  int rc = validate_params(params);
  if (rc) return rc;
  DeviceGuard g(m->device);
  Batch b{"bp_transcribe_host", h_audio, false, nullptr};
  rc = describe_batch(b, h_sample_off, nullptr, n_files);
  if (rc) return rc;
  return run_batch(m, b, nullptr, Rows{h_note, h_onset, h_contour}, params, notes, h_frame_off, m->stream);
}

void bp_last_required(int64_t* notes, int64_t* bends) {
  if (notes) *notes = g_need_notes;
  if (bends) *bends = g_need_bends;
}

void* bp_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    fail(BP_E_CUDA, "bp_host_alloc: cudaHostAlloc failed");
    return nullptr;
  }
  return p;
}

void bp_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

int bp_transcribe_files_host(bp_model_t* m, const float* const* audio, const int64_t* n_samples, int32_t n_files,
                             const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                             int64_t* h_frame_off, bp_notes_t* notes) {
  if (!m || !h_frame_off || n_files < 0 || (n_files > 0 && (!audio || !n_samples)))
    return fail(BP_E_INVALID, "bp_transcribe_files_host: bad argument");
  int rc = validate_params(params);
  if (rc) return rc;
  DeviceGuard g(m->device);
  Batch b{"bp_transcribe_files_host", nullptr, false, audio};
  rc = describe_batch(b, nullptr, n_samples, n_files);
  if (rc) return rc;
  return run_batch(m, b, nullptr, Rows{h_note, h_onset, h_contour}, params, notes, h_frame_off, m->stream);
}

int64_t bp_resampled_length(int64_t n_frames, int32_t sample_rate) { return ingest_output_length(n_frames, sample_rate); }

int bp_load_pcm_device(bp_model_t* m, const void* d_pcm, int32_t sample_format, int64_t n_frames, int32_t channels,
                       int32_t sample_rate, float* d_audio, void* stream) {
  if (!m || n_frames < 0) return fail(BP_E_INVALID, "bp_load_pcm_device: bad argument");
  if (n_frames == 0) return BP_OK;
  if (!d_pcm || !d_audio) return fail(BP_E_INVALID, "bp_load_pcm_device: null buffer");
  DeviceGuard g(m->device);
  const int rc = launch_ingest(m->device, d_pcm, sample_format, n_frames, channels, sample_rate, d_audio,
                               static_cast<cudaStream_t>(stream));
  if (rc == -2)
    return fail(BP_E_INVALID, "bp_load_pcm_device: unsupported sample format / channel count / sample rate (format 0..3, "
                              "channels >= 1, rate ratio to 22 050 Hz below ~100)");
  if (rc) return fail(BP_E_CUDA, std::string("bp_load_pcm_device: ") + cudaGetErrorString(cudaGetLastError()));
  m->launches += 1;
  return BP_OK;
}

int bp_load_pcm_host(bp_model_t* m, const void* h_pcm, int32_t sample_format, int64_t n_frames, int32_t channels,
                     int32_t sample_rate, float* h_audio) {
  if (!m || n_frames < 0 || channels < 1 || sample_format < 0 || sample_format > 3)
    return fail(BP_E_INVALID, "bp_load_pcm_host: bad argument");
  if (n_frames == 0) return BP_OK;
  if (!h_pcm || !h_audio) return fail(BP_E_INVALID, "bp_load_pcm_host: null buffer");
  DeviceGuard g(m->device);
  cudaStream_t st = m->stream;
  static const int kBytes[4] = {4, 2, 4, 1};
  const size_t in_bytes = (size_t)n_frames * channels * kBytes[sample_format];
  const int64_t n_out = ingest_output_length(n_frames, sample_rate);
  CK(cudaStreamSynchronize(st));
  CK(m->st_pcm.reserve(in_bytes));
  CK(m->st_audio.reserve((size_t)n_out));
  CK(cudaMemcpyAsync(m->st_pcm.p, h_pcm, in_bytes, cudaMemcpyHostToDevice, st));
  const int rc = bp_load_pcm_device(m, m->st_pcm.p, sample_format, n_frames, channels, sample_rate, m->st_audio.p, st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(h_audio, m->st_audio.p, sizeof(float) * (size_t)n_out, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return BP_OK;
}

int bp_load_pcm_files_device(bp_model_t* m, const bp_pcm_file_t* files, int32_t n_files, float* d_audio,
                             int64_t* h_sample_off, void* stream) {
  if (!m || !h_sample_off || n_files < 0 || (n_files > 0 && !files))
    return fail(BP_E_INVALID, "bp_load_pcm_files_device: bad argument");
  const std::string api = "bp_load_pcm_files_device";
  std::vector<IngestFile> desc;
  std::vector<int64_t> bytes;
  int rc = describe_pcm(api, files, n_files, true, desc, bytes);
  if (rc) return rc;
  int64_t total = 0;
  for (const IngestFile& f : desc) total += f.n_out;
  if (total > 0 && !d_audio) return fail(BP_E_INVALID, api + ": null output");
  h_sample_off[0] = 0;
  for (int i = 0; i < n_files; ++i) h_sample_off[i + 1] = h_sample_off[i] + desc[i].n_out;
  if (total == 0) return BP_OK;
  DeviceGuard g(m->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if ((rc = load_ingest_taps(api, m->device, desc))) return rc;
  for (int i = 0; i < n_files; ++i) {
    desc[i].pcm = files[i].pcm;
    desc[i].out = d_audio + h_sample_off[i];
  }
  const size_t hb = (size_t)ingest_header_bytes(n_files);
  if (m->ingest_pending) {  // the previous call's staging has left the host
    CK(cudaEventSynchronize(m->ingest_copied));
    m->ingest_pending = false;
  }
  if (hb > m->h_ingest_cap) {
    if (m->h_ingest) cudaFreeHost(m->h_ingest);
    m->h_ingest = nullptr;
    m->h_ingest_cap = 0;
    const size_t cap = std::max<size_t>(hb, 1 << 16);
    CK(cudaHostAlloc(&m->h_ingest, cap, cudaHostAllocDefault));
    m->h_ingest_cap = cap;
  }
  CK(m->d_ingest.reserve(hb));
  if (!m->ingest_copied) {
    CK(cudaEventCreateWithFlags(&m->ingest_copied, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&m->ingest_done, cudaEventDisableTiming));
  } else {
    CK(cudaStreamWaitEvent(st, m->ingest_done, 0));  // the previous call's kernel may have run on another stream
  }
  int max_span = 1;
  const int n_ctas = write_ingest_header(m->h_ingest, desc.data(), n_files, &max_span);
  CK(cudaMemcpyAsync(m->d_ingest.p, m->h_ingest, hb, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(m->ingest_copied, st));
  m->ingest_pending = true;
  rc = launch_ingest_header(m, m->d_ingest.p, n_files, n_ctas, max_span, st);
  CK(cudaEventRecord(m->ingest_done, st));
  return rc;
}

int bp_transcribe_pcm_files_host(bp_model_t* m, const bp_pcm_file_t* files, int32_t n_files,
                                 const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                                 int64_t* h_frame_off, int64_t* h_sample_off, bp_notes_t* notes) {
  if (!m || !h_frame_off || n_files < 0 || (n_files > 0 && !files))
    return fail(BP_E_INVALID, "bp_transcribe_pcm_files_host: bad argument");
  int rc = validate_params(params);
  if (rc) return rc;
  Batch b{"bp_transcribe_pcm_files_host", nullptr, false, nullptr};
  b.pcm = files;
  if ((rc = describe_pcm(b.api, files, n_files, false, b.ingest, b.pcm_bytes))) return rc;
  b.rel.assign(n_files + 1, 0);
  for (int i = 0; i < n_files; ++i) {
    b.rel[i + 1] = b.rel[i] + b.ingest[i].n_out;
    b.total_frames += bp_num_frames(b.ingest[i].n_out);
  }
  if (h_sample_off) std::copy(b.rel.begin(), b.rel.end(), h_sample_off);
  DeviceGuard g(m->device);
  if ((rc = load_ingest_taps(b.api, m->device, b.ingest))) return rc;
  return run_batch(m, b, nullptr, Rows{h_note, h_onset, h_contour}, params, notes, h_frame_off, m->stream);
}

int bp_debug_pcm_layout(const bp_pcm_file_t* files, int32_t n_files, int64_t* byte_off, int64_t* sample_off) {
  if (n_files < 0 || (n_files > 0 && !files) || !byte_off || !sample_off)
    return fail(BP_E_INVALID, "bp_debug_pcm_layout: bad argument");
  std::vector<IngestFile> desc;
  std::vector<int64_t> bytes;
  const int rc = describe_pcm("bp_debug_pcm_layout", files, n_files, false, desc, bytes);
  if (rc) return rc;
  byte_off[0] = sample_off[0] = 0;
  for (int i = 0; i < n_files; ++i) {
    byte_off[i + 1] = byte_off[i] + align16(bytes[i]);
    sample_off[i + 1] = sample_off[i] + desc[i].n_out;
  }
  return BP_OK;
}

int64_t bp_debug_resample_filter(int32_t up, int32_t down, double* taps, int64_t capacity) {
  if (up < 1 || down < 1) return fail(BP_E_INVALID, "bp_debug_resample_filter: bad argument"), -1;
  const std::vector<double> h = ingest_filter(up, down);
  if (taps && capacity >= (int64_t)h.size()) std::memcpy(taps, h.data(), h.size() * sizeof(double));
  return (int64_t)h.size();
}

int bp_debug_tc_plan(int which, const float* w, int32_t* sizes, uint16_t* tiles, int32_t* tile_seq, uint32_t* slot_words,
                     int32_t* group_step_off, int32_t* group_ft) {
  if (!w || !sizes || which < 0 || which > 2) return fail(BP_E_INVALID, "bp_debug_tc_plan: bad argument");
  TcConvPlan pl;
  pl.build(tc_spec(which), w);
  sizes[0] = pl.n_tiles;
  sizes[1] = (int32_t)pl.tile_seq.size();
  sizes[2] = pl.n_uses;
  sizes[3] = pl.n_groups;
  if (tiles) std::memcpy(tiles, pl.tiles.data(), pl.tiles.size() * 2);
  if (tile_seq) std::memcpy(tile_seq, pl.tile_seq.data(), pl.tile_seq.size() * 4);
  if (slot_words) {
    std::memcpy(slot_words, pl.slot_words[0].data(), pl.slot_words[0].size() * 4);
    std::memcpy(slot_words + pl.slot_words[0].size(), pl.slot_words[1].data(), pl.slot_words[1].size() * 4);
  }
  if (group_step_off) std::memcpy(group_step_off, pl.group_step_off.data(), pl.group_step_off.size() * 4);
  if (group_ft) std::memcpy(group_ft, pl.group_ft.data(), pl.group_ft.size() * 4);
  return BP_OK;
}

int bp_debug_tc_gather(int which, const float* w, int32_t* sizes, uint16_t* b1, int32_t* starts, int32_t* ranges) {
  if (!w || !sizes || which < 1 || which > 2) return fail(BP_E_INVALID, "bp_debug_tc_gather: bad argument");
  const TcGatherGeom g = tc_gather_geometry(which);
  sizes[0] = g.K;
  sizes[1] = g.n_ci;
  sizes[2] = g.KH;
  sizes[3] = g.wout;
  if (b1) {
    std::vector<uint16_t> m;
    tc_build_b1(which, w, m, true);
    std::memcpy(b1, m.data(), m.size() * 2);
  }
  if (starts) std::copy(g.starts.begin(), g.starts.end(), starts);
  if (ranges) std::copy(g.ranges.begin(), g.ranges.end(), ranges);
  return BP_OK;
}

int bp_debug_tc_gather_packed(int which, const float* w, int32_t* sizes, uint16_t* b1, int32_t* kmap) {
  if (!w || !sizes || which < 1 || which > 2) return fail(BP_E_INVALID, "bp_debug_tc_gather_packed: bad argument");
  const TcGatherGeom g = tc_gather_geometry(which);
  sizes[0] = g.K_packed;
  if (b1) {
    std::vector<uint16_t> m;
    tc_build_b1(which, w, m);
    std::memcpy(b1, m.data(), m.size() * 2);
  }
  if (kmap) std::copy(g.kmap.begin(), g.kmap.end(), kmap);
  return BP_OK;
}

int bp_debug_tc_b2(int which, const float* w2, int32_t* sizes, uint16_t* tiles) {
  if (!w2 || !sizes || which < 0 || which > 2) return fail(BP_E_INVALID, "bp_debug_tc_b2: bad argument");
  std::vector<uint16_t> t;
  tc_build_b2(which, w2, t);
  const TcConvSpec sp = tc_spec(which);
  sizes[0] = sp.n2_tiles;
  sizes[1] = sp.n2;
  sizes[2] = sp.KH2;
  sizes[3] = sp.width;
  sizes[4] = sp.js;
  if (tiles) std::memcpy(tiles, t.data(), t.size() * 2);
  return BP_OK;
}

int bp_debug_tc_clocks(bp_model_t* m, int which, uint64_t* cycles, int reset) {
  if (!m || !cycles || which < 0 || which > 2) return fail(BP_E_INVALID, "bp_debug_tc_clocks: bad argument");
  DeviceGuard g(m->device);
  CK(cudaDeviceSynchronize());
  if (tc_read_clocks(which, reinterpret_cast<unsigned long long*>(cycles), reset != 0) != 0)
    return fail(BP_E_INVALID, "bp_debug_tc_clocks: the library was built without -DBP_TC_CLOCKS");
  return BP_OK;
}

int bp_debug_tc_schedule(int which, int fused, int n_windows, int n_sms, int32_t* sizes, int32_t* items, uint32_t* edges) {
  if (!sizes || which < 0 || which > 2 || n_windows < 1 || n_sms < 1)
    return fail(BP_E_INVALID, "bp_debug_tc_schedule: bad argument");
  const TcConvSpec sp = tc_spec(which);
  int ms = 0;
  const TcSchedule s = tc_schedule(which, fused != 0 || which != 0, n_windows, n_sms, &ms);
  sizes[0] = s.n_items();
  sizes[1] = s.grid;
  sizes[2] = s.n_mtiles;
  sizes[3] = s.n_full;
  sizes[4] = s.n_ranges;
  sizes[5] = ms;
  sizes[6] = s.n_full * ms;
  sizes[7] = sp.G0;
  if (items)
    for (int it = 0; it < s.n_items(); ++it) s.item(it, sp.G0, items[3 * it], items[3 * it + 1], items[3 * it + 2]);
  if (edges) {
    edges[0] = tc_edge_mask(sp, 1u);
    edges[1] = tc_edge_mask(sp, s.tail_starts());
  }
  return BP_OK;
}

int bp_debug_tc_cta_busy(bp_model_t* m, int which, uint64_t* ns, int n, int reset) {
  if (!m || (!ns && n) || which < 0 || which > 2 || n < 0 || n > kTcMaxCtas)
    return fail(BP_E_INVALID, "bp_debug_tc_cta_busy: bad argument");
  DeviceGuard g(m->device);
  CK(cudaDeviceSynchronize());
  if (tc_read_busy(which, reinterpret_cast<unsigned long long*>(ns), n, reset != 0) != 0)
    return fail(BP_E_INVALID, "bp_debug_tc_cta_busy: the library was built without -DBP_TC_CLOCKS");
  return BP_OK;
}

int bp_model_profile(bp_model_t* m, int which) {
  if (!m) return fail(BP_E_INVALID, "bp_model_profile: null model");
  if (which < -1 || which > 6) return fail(BP_E_INVALID, "bp_model_profile: unknown kernel family");
  m->profile_which = which;
  m->prof_used = 0;
  m->prof_windows = 0;
  return BP_OK;
}

int bp_model_profile_read(bp_model_t* m, double* total_ms, int64_t* n_intervals, int64_t* n_windows) {
  if (!m || !total_ms || !n_intervals || !n_windows) return fail(BP_E_INVALID, "bp_model_profile_read: null argument");
  DeviceGuard g(m->device);
  CK(cudaDeviceSynchronize());
  double total = 0.0;
  for (size_t i = 0; i + 1 < m->prof_used; i += 2) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, m->prof_ev[i], m->prof_ev[i + 1]));
    total += ms;
  }
  *total_ms = total;
  *n_intervals = (int64_t)(m->prof_used / 2);
  *n_windows = m->prof_windows;
  return BP_OK;
}

int bp_debug_activation(bp_model_t* m, int which, float* h_out, int64_t n_windows) {
  if (!m || !h_out) return fail(BP_E_INVALID, "bp_debug_activation: null argument");
  if (n_windows <= 0 || n_windows > m->chunk || n_windows > m->last_forward_n)
    return fail(BP_E_INVALID, "bp_debug_activation: only valid for the windows of a single-chunk forward call");
  DeviceGuard g(m->device);
  const float* src = nullptr;
  size_t per = 0;
  switch (which) {
    case 0: src = m->y.p; per = (size_t)kFrames * kCqtBins; break;
    case 1: src = m->c1.p; per = (size_t)8 * kFrames * kContourBins; break;
    case 2: src = m->n1.p; per = (size_t)32 * kFrames * kPitches; break;
    case 3: src = m->o1.p; per = (size_t)32 * kFrames * kPitches; break;
    default: return fail(BP_E_INVALID, "bp_debug_activation: unknown activation id");
  }
  if (m->last_path >= 1 && which >= 2)
    return fail(BP_E_INVALID, "bp_debug_activation: the tensor-core paths never materialise the 32-channel activations "
                              "(use bp_model_set_path(m, 0))");
  if (m->last_path == 1 && which == 1)
    return fail(BP_E_INVALID, "bp_debug_activation: path 1 reduces the contour activations in the epilogue "
                              "(use bp_model_set_path(m, 2) or 0)");
  CK(cudaDeviceSynchronize());
  if (which == 0 && m->y_is_log) {  // the tensor-core paths normalise straight into the split operand: finish `y` now
    launch_lognorm(m->y.p, m->minmax.p, m->d_params + ParamLayout::bn, (int)m->last_forward_n, m->stream);
    CK(cudaStreamSynchronize(m->stream));
    m->y_is_log = false;
  }
  CK(cudaMemcpy(h_out, src, sizeof(float) * per * n_windows, cudaMemcpyDeviceToHost));
  if (which == 1 && m->last_path == 2) {  // the tensor-core path keeps this activation channels-last: return NCHW
    std::vector<float> tmp(h_out, h_out + per * n_windows);
    for (int64_t b = 0; b < n_windows; ++b)
      for (int t = 0; t < kFrames; ++t)
        for (int f = 0; f < kContourBins; ++f)
          for (int c = 0; c < 8; ++c)
            h_out[((b * 8 + c) * kFrames + t) * kContourBins + f] = tmp[((b * kFrames + t) * kContourBins + f) * 8 + c];
  }
  return BP_OK;
}

int bp_model_set_debug_frontend(bp_model_t* m, int on) {
  if (!m) return fail(BP_E_INVALID, "bp_model_set_debug_frontend: null model");
  m->debug_frontend = on != 0;
  return BP_OK;
}

int bp_debug_chain_layout(int32_t* offsets, int32_t* lengths, int32_t* stride) {
  if (!offsets || !lengths || !stride) return fail(BP_E_INVALID, "bp_debug_chain_layout: null argument");
  for (int o = 0; o <= 8; ++o) {
    offsets[o] = o ? chain_off(o) : -1;
    lengths[o] = octave_len(o);
  }
  *stride = kChainStride;
  return BP_OK;
}

int bp_debug_split_layout(const bp_model_t* m, int32_t* out) {
  if (!m || !out) return fail(BP_E_INVALID, "bp_debug_split_layout: null argument");
  constexpr TcConvSpec cs = tc_spec(0);
  out[0] = tc_rows_total(m->chunk, cs.rows_per_window);
  out[1] = m->last_forward_n > 0 ? tc_rows_total((int)m->last_forward_n, cs.rows_per_window) : 0;
  out[2] = cs.lead_rows;
  out[3] = cs.rows_per_window;
  out[4] = cs.chunks8;
  return BP_OK;
}

int bp_debug_frontend(bp_model_t* m, int which, void* h_out, int64_t n_windows) {
  if (!m || !h_out) return fail(BP_E_INVALID, "bp_debug_frontend: null argument");
  if (n_windows <= 0 || n_windows > m->chunk || n_windows > m->last_forward_n)
    return fail(BP_E_INVALID, "bp_debug_frontend: only valid for the windows of a single-chunk forward call");
  if (which < 0 || which > 3) return fail(BP_E_INVALID, "bp_debug_frontend: unknown buffer id");
  DeviceGuard g(m->device);
  CK(cudaDeviceSynchronize());
  switch (which) {
    case 0:
      CK(cudaMemcpy(h_out, m->chain.p, sizeof(float) * kChainStride * n_windows, cudaMemcpyDeviceToHost));
      break;
    case 1: {
      const float* src = m->last_path >= 1 && m->y_is_log ? m->y.p : m->ylog_valid ? m->ylog.p : nullptr;
      if (!src)
        return fail(BP_E_INVALID, "bp_debug_frontend: the raw log-magnitudes of the last forward call are gone (path 0 "
                                  "normalises them in place, and bp_debug_activation(0) does so on the tensor-core paths): "
                                  "call bp_model_set_debug_frontend(m, 1) before the forward call");
      CK(cudaMemcpy(h_out, src, sizeof(float) * kFrames * kCqtBins * n_windows, cudaMemcpyDeviceToHost));
      break;
    }
    case 2: {
      std::vector<unsigned int> mm((size_t)2 * n_windows);
      CK(cudaMemcpy(mm.data(), m->minmax.p, sizeof(unsigned int) * mm.size(), cudaMemcpyDeviceToHost));
      float* out = static_cast<float*>(h_out);
      for (size_t i = 0; i < mm.size(); ++i) {  // ordered_to_float on the host
        const uint32_t u = (mm[i] & 0x80000000u) ? (mm[i] & 0x7fffffffu) : ~mm[i];
        std::memcpy(out + i, &u, 4);
      }
      break;
    }
    case 3: {
      if (m->last_path < 1)
        return fail(BP_E_INVALID, "bp_debug_frontend: the split operand exists only on the tensor-core paths (1 and 2)");
      constexpr TcConvSpec cs = tc_spec(0);
      const size_t n = (size_t)2 * cs.chunks8 * 8 * tc_rows_total(m->chunk, cs.rows_per_window);
      CK(cudaMemcpy(h_out, m->yhl.p, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost));
      break;
    }
  }
  return BP_OK;
}

}  // extern "C"
