// Launch wrappers of the hot-path kernels (host-callable; all asynchronous on `st`).
#pragma once
#include <cuda_bf16.h>

#include <cstring>
#include <vector>

#include "common.cuh"

namespace bp {

// ---- hcqt.cu ------------------------------------------------------------------------------------
void hcqt_setup();  // per device: shared-memory opt-in of the FP32 CQT kernel
// The decimation low-pass taps as the zero-padded pairs the FIR reads (hcqt.cu); every decimation launch takes them as
// a kernel parameter (2.2 KB).
constexpr int kLp2 = kTaps + 14;
struct Lowpass2 {
  float2 t[kLp2];
};
Lowpass2 lowpass_pairs(const float* h_lp /* host: the 256 taps of the parameter block */);
void launch_decimate(const Lowpass2& lp, const float* audio, const WinDesc* desc, float* chain, int stage, int n_windows,
                     cudaStream_t st);
void launch_cqt(const float* audio, const WinDesc* desc, const float* chain, const float* wt, const float* scale,
                float* logmag, unsigned int* minmax, int n_windows, cudaStream_t st);
void launch_lognorm(float* y, const unsigned int* minmax, const float* bn /* device: scale, bias */, int n_windows,
                    cudaStream_t st);

// ---- cnn.cu (FP32 FFMA path) -------------------------------------------------------------------
// Transposed weights wT[(ci*KH+dt)*KW+df][COUT]; activations are planar [B][C][172][W].
struct CnnWeights {
  const float *contour1_wT, *contour1_b;
  const float *contour2_wT, *contour2_b;
  const float *note1_wT, *note1_b;
  const float *note2_wT, *note2_b;
  const float *onset1_wT, *onset1_b;
  const float *onset2_wT, *onset2_b;
};
void cnn_setup();
void launch_contour1(const float* y, const CnnWeights& w, float* c1, int n_windows, cudaStream_t st);
void launch_contour2(const float* c1, const CnnWeights& w, float* contour, int n_windows, cudaStream_t st);
void launch_note1(const float* contour, const CnnWeights& w, float* n1, int n_windows, cudaStream_t st);
void launch_note2(const float* n1, const CnnWeights& w, float* note, int n_windows, cudaStream_t st);
void launch_onset1(const float* y, const CnnWeights& w, float* o1, int n_windows, cudaStream_t st);
void launch_onset2(const float* note, const float* o1, const CnnWeights& w, float* onset, int n_windows,
                   cudaStream_t st);


// ---- tc_conv.cu (tensor-core path of the three wide convolutions, each with its following conv fused) --------
// The geometry of one layer (layer 0 contour, 1 onset, 2 note): every shape of its kernels, shared-memory layout, host
// builders and workspaces is derived from this description.
struct TcConvSpec {
  int KH, KW, SF, PT, PL, COUT, FLT, WOUT;  // taps, frequency stride, pads, channels, bins per 128-column tile, output bins
  int n_ci;                                 // input channels (harmonics of y, or 1 for the contour posteriorgram)
  int shifts[8];                            // frequency shift of every input channel (harmonic stacking)
  int data_bins, chunks8;                   // bins of the input rows and 8-bin chunks of the split layout (even)
  int rows_per_window, lead_rows;           // row layout of the split input: 172 frames + zero rows per window
  int layer;                                // 0 contour, 1 onset, 2 note
  int KH2, HALO, G0;                        // fused next conv: time taps, frequency halo; groups of two frequency tiles
  int PD;                                   // pair distance: the two tiles of a group are PD apart (tc_group_tile)
  // fused next conv as a second contraction (tc_conv.cu): weight tiles, their N, accumulator columns per output offset j,
  // accumulator columns, columns staged in shared memory at a time (a multiple of 8 and of js: whole output offsets)
  int n2_tiles, n2, js, width, pass;
  // gathered conv1 (onset / note, tc_conv.cu): window width in K, and for W = 6 the K slot map
  int W;
  int slot[24];
  __host__ __device__ constexpr int n_ft() const { return (WOUT + FLT - 1) / FLT; }  // frequency tiles
  __host__ __device__ constexpr int tile_bins() const { return 8 * (chunks8 - 1); }  // bins of a data tile (the last chunk is padding)
  __host__ __device__ constexpr int ksteps() const { return (KH * n_ci * W + 15) / 16; }  // gathered conv1: K-steps per bin
  // edge-buffer values per side of a range boundary: the 2 HALO partial sums; the contour also keeps the finished bins
  // that share the two 8-bin output chunks around the boundary
  __host__ __device__ constexpr int edge_per_side() const { return 2 * HALO + (layer == 0 ? 8 - HALO : 0); }
};
// clang-format off
__host__ __device__ constexpr TcConvSpec tc_spec(int layer) {
  //                  KH  KW SF PT PL COUT FLT WOUT n_ci shifts                               bins          ch8 rows/win lead layer KH2 HALO G0  PD  n2_tiles n2 js width pass  W
  return layer == 0 ? TcConvSpec{3, 39, 1, 1, 19, 8, 16, 264, 8, {-36, 0, 36, 57, 72, 84, 93, 101}, kCqtBins,     40, 174, 3, 0, 5, 2, 9,  1,  1, 32, 5, 104, 40, 0, {}}
       : layer == 1 ? TcConvSpec{5, 5, 3, 2, 1, 32, 4, 88, 8, {-36, 0, 36, 57, 72, 84, 93, 101},   kCqtBins,     40, 174, 3, 1, 3, 1, 12, 12, 2, 16, 4, 32, 32,   6,
                                 {9, 10, 21, 22, 14, 4, 2, 1, 16, 3, 6, 13, 5, 17, 18, 20, 19, 23, 7, 0, 8, 15, 12, 11}}
                    : TcConvSpec{7, 7, 3, 3, 2, 32, 4, 88, 1, {0, 0, 0, 0, 0, 0, 0, 0},           kContourBins, 34, 175, 6, 2, 7, 1, 12, 12, 2, 32, 8, 64, 64,   8, {}};
}
// clang-format on
// The pairing of frequency tiles into groups, the one rule the planner, the kernels, edge_fix_kernel and the tests read.
// Group g is position i = g % PD of run g / PD; a run holds 2 PD consecutive tiles, slot 0 the lower PD, slot 1 the upper
// PD, so the tiles of group g are {2 PD run + i, 2 PD run + PD + i} (-1: past the last tile, or no such group).
// Contour PD = 1: neighbouring tiles, which read the same weight tiles at A chunks two apart, so the two slots share
// almost every step of the weight ring.  Onset / note PD = G0: tiles {g, g + G0} (no weight ring to share).
__host__ __device__ constexpr int tc_group_tile(const TcConvSpec& s, int g, int slot) {
  if (g < 0 || g >= s.G0) return -1;
  const int run = g / s.PD, i = g - run * s.PD, ft = 2 * s.PD * run + slot * s.PD + i;
  return ft < s.n_ft() ? ft : -1;
}
// group (slot in bit 0, group << 1) of frequency tile ft: the inverse of tc_group_tile
__host__ __device__ constexpr int tc_tile_group(const TcConvSpec& s, int ft) {
  const int run = ft / (2 * s.PD), r = ft - run * 2 * s.PD, slot = r / s.PD;
  return ((run * s.PD + r - slot * s.PD) << 1) | slot;
}
// A slot walks its tiles of an item's groups [g0, g1) in ascending order and carries the frequency halo of the fused
// conv2 from one tile to the next in registers.  Its tile in group g STARTS a range (no carry from below) where the item
// starts or where its tile in g - 1 is not the one below; it ENDS a range where the item ends or its tile in g + 1 is not
// the one above.  Boundary b (between tiles b - 1 and b) goes through the edge buffer iff tile b starts a range, which is
// the case iff tile b - 1 ends one.
__host__ __device__ constexpr bool tc_starts_range(const TcConvSpec& s, int g, int slot, bool item_start) {
  const int ft = tc_group_tile(s, g, slot);
  return item_start || ft <= 0 || tc_group_tile(s, g - 1, slot) != ft - 1;
}
__host__ __device__ constexpr bool tc_ends_range(const TcConvSpec& s, int g, int slot, bool item_end) {
  return item_end || tc_group_tile(s, g + 1, slot) != tc_group_tile(s, g, slot) + 1;
}
// The items of one conv_tc_kernel launch (tc_schedule, tc_conv.cu).  The persistent CTAs walk items it = blockIdx.x,
// + grid, ...  Items [0, n_full) are the M-tiles 0 .. n_full - 1 whole (all G0 groups); n_full is a multiple of the grid,
// so every CTA runs the same number of whole M-tiles.  The n_tail M-tiles after them are each cut into n_ranges group
// ranges [bounds[q], bounds[q + 1]) of balanced cost; tail item j = it - n_full is range q = j / n_tail of M-tile
// n_full + j % n_tail (range-major, so that the CTAs that take a second tail item take another range).
struct TcSchedule {
  int n_mtiles, n_full, n_tail, n_ranges, grid;
  unsigned char bounds[16];  // n_ranges + 1 group boundaries: 0 = bounds[0] < ... < bounds[n_ranges] = G0
  __host__ __device__ int n_items() const { return n_full + n_tail * n_ranges; }
  __host__ __device__ uint32_t tail_starts() const {  // bit g: a tail item starts at group g
    uint32_t m = 0;
    for (int q = 0; q < n_ranges; ++q) m |= 1u << bounds[q];
    return m;
  }
  __host__ __device__ void item(int it, int G0, int& mt, int& g0, int& g1) const {
    if (it < n_full) {
      mt = it, g0 = 0, g1 = G0;
      return;
    }
    const int j = it - n_full, q = j / n_tail;
    mt = n_full + (j - q * n_tail), g0 = bounds[q], g1 = bounds[q + 1];
  }
};
// The boundaries b = 1 .. n_ft - 1 that go through the edge buffer in an M-tile whose items start at the groups of
// `starts` (bit g): those where tile b starts a range.  Whole M-tiles: starts = 1 (group 0 only).
__host__ __device__ constexpr uint32_t tc_edge_mask(const TcConvSpec& s, uint32_t starts) {
  uint32_t m = 0;
  for (int b = 1; b < s.n_ft(); ++b) {
    const int gs = tc_tile_group(s, b);
    if (tc_starts_range(s, gs >> 1, gs & 1, (starts >> (gs >> 1)) & 1u)) m |= 1u << b;
  }
  return m;
}
// every frequency tile belongs to exactly one (group, slot), and tc_tile_group finds it
__host__ __device__ constexpr bool tc_pairing_ok(const TcConvSpec& s) {
  for (int ft = 0; ft < s.n_ft(); ++ft) {
    int n = 0;
    for (int g = 0; g < s.G0; ++g)
      for (int slot = 0; slot < 2; ++slot) n += tc_group_tile(s, g, slot) == ft;
    const int gs = tc_tile_group(s, ft);
    if (n != 1 || tc_group_tile(s, gs >> 1, gs & 1) != ft) return false;
  }
  return true;
}
// Host side: weight tiles + the per-group MMA programs of the Toeplitz form.  The kernels run it for the contour conv
// only; the onset and note convs gather their A operand instead (tc_build_b1), and their plans only serve the tests.
struct TcConvPlan {
  TcConvSpec spec{};
  std::vector<uint16_t> tiles;          // n_tiles x 4096 bf16 : [plane hi/lo][k-chunk 2][n 128][8]
  std::vector<int> tile_seq;            // per step: tile id
  std::vector<uint32_t> slot_words[2];  // per step and accumulator slot: A offset >> 4 | first << 15, or 0xffffffff
  std::vector<int> group_step_off;      // [n_groups + 1]
  std::vector<int> group_ft;            // [n_groups][2] frequency tiles of the group (-1 = none)
  int n_tiles = 0, n_groups = 0, n_uses = 0;
  void build(const TcConvSpec& spec, const float* w /* [COUT][n_ci][KH][KW] */);
};
struct TcConvDev {
  int layer;  // 0 contour, 1 onset, 2 note (tc_spec)
  const uint16_t* tiles;  // contour: Toeplitz weight tiles (the program is in constant memory)
  const uint16_t* b1;     // onset / note: conv1 B matrices (tc_build_b1)
  const uint16_t* b2;     // conv2 weight matrix of the fused epilogue (tc_build_b2_full)
  // epilogue values, passed with every launch: conv1 bias (COUT used), conv2 bias, and for the onset layer the conv2
  // weights of its note input channel (models.py:305: concat[note, onset1]) [dt][df]
  float bias1[32];
  float bias2;
  float note_w[9];
};
int tc_upload_program(const TcConvPlan& contour_plan, cudaStream_t st);  // 0 on success
// conv1 of the onset (layer 1, w = [32][8][5][5]) / note (layer 2, w = [32][1][7][7]) layer as the kernel gathers it: its
// two B matrices [parity 2][plane hi/lo][K / 8][32][8] bf16, and the geometry of the gather (window start of every output
// bin and channel, [wout][n_ci]; the bins [lo, hi) of every channel that hold input, [n_ci][2]).  window8: B in the
// 8-bin-window form (K rows 8 (dt * n_ci + ci) + j) instead of the K order the kernel uses (kmap).
void tc_build_b1(int layer, const float* w, std::vector<uint16_t>& out, bool window8 = false);
struct TcGatherGeom {
  int K, n_ci, KH, wout;  // K of the 8-bin-window form
  int K_packed;           // K the kernel runs
  std::vector<int> starts, ranges;
  std::vector<int> kmap;  // [K_packed][3]: (dt, ci, window bin j) of every row of the kernel's B, -1 for padding
};
TcGatherGeom tc_gather_geometry(int layer);
// bf16 hi/lo weight tiles of the fused second conv (w2 = that conv's weights), see tc_conv.cu
void tc_build_b2(int layer, const float* w2, std::vector<uint16_t>& out);
// the same tiles placed into the K = 128 x N = width conv2 weight matrix the kernel reads (tc_conv.cu)
void tc_build_b2_full(int layer, const float* w2, std::vector<uint16_t>& out);
int tc_rows_total(int n_windows, int rows_per_window);
int tc_rows_used(int n_rows);  // split rows a launch over n_rows rows of a row space reads (lead + rows + the last M-tile)
size_t tc_edge_floats(const TcConvSpec& spec, int n_windows);  // size of the edge buffer of a fused layer
int tc_setup();  // 0 on success
// cycle sums by role of one layer's conv_tc_kernel launches (tc::TcClk order), optionally reset; -1 unless the library
// was built with -DBP_TC_CLOCKS
int tc_read_clocks(int layer, unsigned long long* out, bool reset);
// busy time of every CTA (index = blockIdx.x, n entries) of one layer's conv_tc_kernel launches in ns of %globaltimer,
// summed over the launches, optionally reset; -1 unless built with -DBP_TC_CLOCKS
constexpr int kTcMaxCtas = 256;
int tc_read_busy(int layer, unsigned long long* out, int n, bool reset);
// Where window w's centre frames go in the unwrapped (per-file) posteriorgrams (reference: inference.py:247-279).
struct UnwrapDesc {
  long long dst_base;  // first output frame this window contributes to
  int rows;            // how many of its 142 centre frames are kept (may be <= 0)
  int pad;
};
// The row space of a tensor-core layer (DESIGN §4.1): window b of a launch holds the input rows [base, base + rows) of
// the layer's split operand (row lead + base + i of the buffer = frame first + i of the window); the layer's conv1 rows
// and output frames have the same indices.  Conv1 row / output frame i of a window is live iff lo1 / lo2 <= i < rows -
// lo1 / lo2; a live row reads only rows of its own window, every other row is computed and dropped.
//   uniform (every forward without unwrap, path 2, the debug hooks): base = b * rows_per_window, first 0, rows 172,
//     lo1 = lo2 = 0: whole windows, the zero rows between them are the "same" padding in time;
//   trimmed (path 1 with unwrap): only the frames the kept centre frames [15, 15 + r) depend on, back to back: window b
//     holds frames [15 - M, 15 + r + M) (M = tc_trim_margin), none if r <= 0.
struct TcRowWin {
  int base, first, rows, pad;
};
struct TcRows {
  const TcRowWin* map = nullptr;  // device, [n_windows]
  int n_rows = 0;                 // rows the M-tiles cover (uniform: n_windows * rows_per_window)
  int lo1 = 0, lo2 = 0;
};
// trimmed row maps: input frames kept on each side of the centre frames by the split layout a layer reads (contour and
// onset share the split of y: 10; note: 7), and output frames each side that later layers read (contour 7, onset 0, note 1)
__host__ __device__ constexpr int tc_trim_margin(int layer) { return layer == 2 ? 7 : 10; }
__host__ __device__ constexpr int tc_trim_out(int layer) { return layer == 0 ? 7 : layer == 1 ? 0 : 1; }
// the map of n windows into out[n] (out may be null); kept[b]: the centre frames window b keeps (UnwrapDesc::rows),
// unused when uniform.  Returns the rows of the row space and sets the live margins.
int tc_row_map(int layer, bool trimmed, const int* kept, int n, TcRowWin* out, int* lo1, int* lo2);
// NormalizedLog + folded BatchNorm of the CQT log-magnitudes straight into the bf16 hi/lo split operand (k-chunk-major
// row layout of tc_spec(0) / tc_spec(1)); `y` itself is left untouched (launch_lognorm makes the fp32 copy).
// rows_stride: row stride of the split layout (>= tc_rows_used(rows.n_rows)), fixed per model.  Every row of
// [0, tc_rows_used(rows.n_rows)) is written: frame first + i of window b at row lead + base + i, zero in every other row.
void launch_lognorm_split(const float* y, const unsigned int* minmax, const float* bn, __nv_bfloat16* dst,
                          const TcConvSpec& spec, const TcRows& rows, int n_windows, int rows_stride, cudaStream_t st);
// Outputs of a fused layer.  Device-internal posteriorgram layouts have the FRAME index fastest, so that the epilogue
// threads (one frame each, 32 consecutive frames per warp) store coalesced, and so that the decode kernels read coalesced:
//   note / onset   pitch-major   pm[pitch][frame]                 frame stride = number of frames the buffer holds
//   contour        chunk-major   cm[8-bin chunk (33)][frame][8]
// `raw` holds all 172 frames of every window of the chunk (frame index b*172 + t, stride `raw_rows`); with `ud` the centre
// frames of every window also / instead go to their unwrapped position (reference: inference.py:247-279) in `unwrapped`,
// whose frame stride is `frame_stride`.
struct TcOut {
  float* raw = nullptr;
  float* unwrapped = nullptr;
  long long frame_stride = 0;
  long long raw_rows = 0;           // frame stride of `raw` and `note_raw`
  const UnwrapDesc* ud = nullptr;
  const float* note_raw = nullptr;  // onset layer: the raw pitch-major note posteriorgram (input channel 0 of its conv2)
  __nv_bfloat16* chl = nullptr;     // contour layer: split operand of the note conv [2][chl_chunks][chl_rows][8]
  const TcRowWin* chl_map = nullptr;  // the note layer's row map: frame t of window b goes to row chl_lead + base + t - first
  int chl_rows = 0, chl_chunks = 0, chl_lead = 0;
  float* edge = nullptr;            // >= tc_edge_floats(spec, n_windows) floats of scratch
  float* act = nullptr;             // unfused contour (path 2): channels-last activations [B][172][WOUT][COUT]
};
// fuse_next (contour layer only; the other two always fuse): also compute the following conv in the epilogue instead
// of storing the channels-last activations.  rows: the layer's row space (TcRowWin); nothing is launched without rows.
void launch_conv_tc(const __nv_bfloat16* data, const TcConvDev& dev, const TcOut& out, int n_windows, const TcRows& rows,
                    int rows_stride, int n_sms, cudaStream_t st, bool fuse_next = false);
// The items launch_conv_tc runs over n_rows rows of a layer's row space on n_sms SMs (fused: the M-tiles of the fused
// epilogue, which overlap by KH2 - 1 rows; the onset and note layers always fuse).  ms: frames an M-tile finishes.
TcSchedule tc_schedule_rows(int layer, bool fused, int n_rows, int n_sms, int* ms = nullptr);
// the same for n_windows whole windows (the uniform row map)
TcSchedule tc_schedule(int layer, bool fused, int n_windows, int n_sms, int* ms = nullptr);
// contour conv2 on the channels-last output of the tensor-core contour conv; also emits the bf16 hi/lo split of the
// contour posteriorgram in the layout of tc_spec(2)
void launch_contour2_tc(const float* c1_nhwc, const CnnWeights& w, float* contour, __nv_bfloat16* chl, int rows_total,
                        int n_windows, cudaStream_t st);

// ---- cqt_tc.cu (tensor-core path of the constant-Q projection, three-way bf16 split) ------------------------
void build_cqt_tc_weights(const float* cqt_real, const float* cqt_imag, std::vector<uint16_t>& out);
void cqt_tc_setup();
void launch_cqt_tc(const float* audio, const WinDesc* desc, const float* chain, const uint16_t* wtc, const float* scale,
                   float* logmag, unsigned int* minmax, int n_windows, int n_sms, cudaStream_t st);

// ---- layout.cu: internal frame-fastest layouts (pm / cm, see TcOut) <-> row-major [frame][bins] of the C ABI ------
// rows -> internal: without `ud` frames [0, n_frames) go to dst_frame0 ..; with `ud` `rows` is a chunk of raw windows
// [n_windows][172][bins] and the kept centre frames of every window go to their unwrapped position
void launch_rows_to_pm(const float* rows, long long n_frames, int width, float* pm, long long stride, long long dst_frame0,
                       cudaStream_t st, const UnwrapDesc* ud = nullptr, int n_windows = 0);
void launch_rows_to_cm(const float* rows, long long n_frames, float* cm, long long stride, long long dst_frame0,
                       cudaStream_t st, const UnwrapDesc* ud = nullptr, int n_windows = 0);
void launch_pm_to_rows(const float* pm, long long stride, long long src_frame0, long long n_frames, int width, float* rows,
                       cudaStream_t st);
void launch_cm_to_rows(const float* cm, long long stride, long long src_frame0, long long n_frames, float* rows,
                       cudaStream_t st);

// ---- ingest.cu: PCM of any rate / channel count -> mono float32 at 22 050 Hz (format: 0 f32, 1 s16, 2 s32, 3 u8) ----
long long ingest_output_length(long long n_frames, int sample_rate);
std::vector<double> ingest_filter(int up, int down);  // host-only: the low-pass design (unit DC gain)
int launch_ingest(int device, const void* d_pcm, int format, long long n_frames, int channels, int sample_rate, float* d_out,
                  cudaStream_t st);  // 0 ok, -1 CUDA error, -2 unsupported argument
// One file of a batched ingest, as the kernel reads it: ingest_geometry fills the format, the ratio, the filter geometry
// and `span` (the inputs a CTA stages), ingest_taps the device's polyphase taps `hp` of that ratio (designed on first
// use, shared by the device's models); the caller sets pcm / n_in / out / n_out.  Both return 0, -1 (CUDA error) or -2
// (unsupported), like launch_ingest.
struct IngestFile {
  const void* pcm;  // interleaved frames, aligned to their sample type
  const float* hp;
  float* out;
  long long n_in, n_out;
  int channels, format, up, down, half, taps, span, pad;
};
// Formats 0 float32, 1 int16, 2 int32, 3 uint8 everywhere; 4 packed 24-bit and 5 float64 only in the batched ingest
// (n_formats = kBatchIngestFormats).
constexpr int kBatchIngestFormats = 6;
int ingest_geometry(int format, int channels, int sample_rate, IngestFile& f, int n_formats = 4);
int ingest_taps(int device, IngestFile& f);
long long ingest_ctas(long long n_out);  // CTAs a file of n_out output samples takes
// d_files [n_files] and d_cta_off [n_files + 1] (exclusive prefix sum of ingest_ctas) in device memory; max_span: the
// largest `span` among the files.  One launch; file i gets the bits of launch_ingest on file i alone.
int launch_ingest_batch(const IngestFile* d_files, const int* d_cta_off, int n_files, int n_ctas, int max_span,
                        cudaStream_t st);
// A live PCM stream (bp_stream_group_open_pcm, include/bp_b200.h): a push of `add` frames to a stream of n frames makes
// outputs [out_lo, out_hi) final (ending: and every output left) and leaves the inputs [hist_lo, hist_hi) held.
struct PcmStep {
  long long out_lo, out_hi, hist_lo, hist_hi;
};
PcmStep pcm_stream_step(const IngestFile& f, long long n, long long add, bool ending);
// One stream's push as the stream ingest kernel reads it.  Input i: 0 below hist_lo (i.e. below 0), hist[i - hist_lo]
// below n_prev, mono frame i - n_prev of the new block f.pcm below f.n_in, 0 from there.  Outputs [k0, k0 + f.n_out) go
// to f.out[0 ..] with the bits of the whole-file ingest; inputs [new_hist_lo, f.n_in) to hist_out (not hist).
struct StreamIngest {
  IngestFile f;
  const float* hist;
  float* hist_out;
  long long k0, n_prev, hist_lo, new_hist_lo;
};
int stream_ingest_ctas(const StreamIngest& d);  // the output CTAs, plus one for the history when it keeps any
// d_streams [n] and d_cta_off [n + 1] (exclusive prefix sum of stream_ingest_ctas) in device memory.  One launch.
int launch_stream_ingest(const StreamIngest* d_streams, const int* d_cta_off, int n_streams, int n_ctas, int max_span,
                         cudaStream_t st);

// ---- decode.cu ----------------------------------------------------------------------------------
struct DecodeParamsDev {
  double onset_thresh, frame_thresh;
  int min_note_len, energy_tol, infer_onsets, melodia, lo_col, hi_col;
};
struct DecodeBuffers {
  const long long* frame_off;     // [n_files+1] device; file i covers frames [frame_off[i], frame_off[i+1])
  float* energy;                  // [total_frames*88] "remaining energy", column-major per file
  unsigned int* candbits;         // [(total_frames*88+31)/32 + 1] onset-candidate bit per cell
  unsigned int* max_onset;        // [n_files]
  unsigned long long* max_fd;     // [n_files]
  const long long* slot_off;      // [n_files+1] device; note slots of file i
  int* note_count;                // [n_files]
  int* note_start;                // [slots]
  int* note_end;
  int* note_pitch;
  int* overflow;                  // [1] set when a file ran out of slots
  float* blk_max;                 // [88 * decode_block_slots(total_frames, n_files)] per-column maxima of 256-frame blocks
  int* blk_arg;                   //   (melodia loop of long files) and their frame indices
};
long long decode_block_slots(long long total_frames, int n_files);
void launch_decode_notes(const float* note, const float* onset, const DecodeBuffers& buf, int n_files,
                         long long total_frames, const DecodeParamsDev& p, cudaStream_t st);
void launch_decode_kernels(const float* note, const float* onset, const DecodeBuffers& buf, int n_files,
                           long long total_frames, const DecodeParamsDev& p, cudaStream_t st);
// Note stream (csrc/stream.cu).  Frames are rows of the stream's held buffer.  The scan sets quiet[t] for rows
// [flag_from, n) (every column of [lo, hi) below frame_thresh), then its last CTA walks rows [from, n): `last` is the row
// before the cut-eligible quiet run in progress (kStreamNoRun: none), and the first row t with quiet[t] and
// t - last == w confirms the cut t - energy_tol + 1.  out[0] = that row or -1, out[1] = `last` after row n - 1.
constexpr long long kStreamNoRun = -(1LL << 60);
constexpr long long kStreamCutBefore = 3;  // LB: quiet frames before a cut (include/bp_b200.h)
constexpr long long kStreamCtxBefore = 3;  // decode context before a segment that starts at a cut
void launch_stream_scan(const float* note, long long flag_from, long long n, int lo, int hi, double frame_thresh,
                        unsigned char* quiet, long long from, long long last, long long w, long long* out,
                        unsigned int* done, cudaStream_t st);
// Keeps, in order, the decoded notes of one segment whose start lies in [keep_lo, keep_hi) (decode-range frames) and
// writes them with frames offset by `frame0`, note_base[j] = base and *kept = their number.
void launch_stream_compact(const int* count, const int* s_start, const int* s_end, const int* s_pitch, int keep_lo,
                           int keep_hi, int frame0, long long base, int* start, int* end, int* pitch, long long* note_base,
                           int* kept, cudaStream_t st);
// Stream group (csrc/stream_group.cu).  A copy of rows between arenas: up to four arrays of 4- or 1-byte elements,
// `width` elements per row; segment k copies rows of array arr.
struct GroupCopyArrays {
  const void* src[4];
  void* dst[4];
  int width[4];
  int bytes[4];
};
struct GroupCopySeg {
  long long src_row, dst_row, rows;
  int arr, pad;
};
// max_elems: the most elements (rows x width) any segment copies
void launch_group_copy(const GroupCopySeg* segs, int n_segs, long long max_elems, const GroupCopyArrays& a,
                       cudaStream_t st);
// The 142 kept frames of every window of a forward chunk (unwrapped into pm / cm at frames w * 142 .., frame stride
// `stride`) to rows dst_row[w] .. of the row-major note / onset (/ contour) arenas.
void launch_group_unwrap(const float* pm_note, const float* pm_onset, const float* cm, long long stride,
                         const long long* dst_row, int n_windows, float* note, float* onset, float* contour,
                         bool with_contour, cudaStream_t st);
// launch_stream_scan for many streams in one launch (blockIdx.y = job); frames are global, row = frame + shift of the
// shared arenas `note` / `quiet`; out[2 j], out[2 j + 1] as out[0], out[1] of launch_stream_scan; done[n_jobs].
struct GroupScanJob {
  long long shift, flag_from, n, from, last;
};
void launch_group_scan(const GroupScanJob* jobs, int n_jobs, long long max_rows, const float* note, int lo, int hi,
                       double frame_thresh, unsigned char* quiet, long long w, long long* out, unsigned int* done,
                       cudaStream_t st);
// launch_stream_compact for a batch of decoded segments (file j of the decode): its notes are written from
// note_off[j] on, note_off[0 .. n_segs] the running sum of the kept counts.
struct GroupKeep {
  int keep_lo, keep_hi, frame0, pad;
  long long base;
};
void launch_group_compact(const GroupKeep* keep, int n_segs, const long long* slot_off, const int* count,
                          const int* s_start, const int* s_end, const int* s_pitch, int* start, int* end, int* pitch,
                          long long* note_base, int* note_off, cudaStream_t st);
// Grid decode: a chunk of parameter sets ("settings") over one batch.  The cell-parallel kernels run once per group of
// settings that share their inputs (blockIdx.y = group); the sequential loops once per (file, setting).
struct DecodePrepGroup {  // a distinct pitch range (lo, hi): constrained frames, per-file max(onsets) / max(frame_diff)
  int lo, hi;
  int set_lo, set_hi;     // its settings are grid_sets[set_lo .. set_hi); the prep writes E of each of them
};
struct DecodeCandGroup {  // a distinct (lo, hi, infer_onsets, onset_thresh): one candidate bitmap
  double onset_thresh;
  int lo, hi, infer, prep;  // prep: its prep group
};
struct DecodeSettingDev {
  DecodeParamsDev p;
  int cand;  // candidate group
};
struct DecodeGridDev {
  const DecodePrepGroup* prep;
  const DecodeCandGroup* cand;
  const int* sets;                  // chunk-local setting indices, grouped by prep group
  const DecodeSettingDev* setting;  // [settings of the chunk]
  int n_files;
  // per-setting / per-group strides of the DecodeBuffers arrays: E, candidate bitmap and block maxima per setting (E,
  // blocks) or candidate group (bitmap); max_onset / max_fd have n_files entries per prep group; slot_off and note_count
  // are indexed setting * n_files + file
  long long e_stride, cand_stride, blk_stride;
};
long long decode_cand_words(long long total_frames);  // 32-bit words of one candidate bitmap
void launch_decode_grid(const float* note, const float* onset, const DecodeBuffers& buf, int n_files,
                        long long total_frames, const DecodeGridDev& g, int n_prep, int n_cand, int n_settings,
                        cudaStream_t st);
void launch_infer_onsets(const float* note, const float* onset, const DecodeBuffers& buf, int n_files, long long total_frames,
                         double* out64 /* [total_frames][88] */, cudaStream_t st);
// amplitude (NumPy pairwise mean) + pitch bends for compacted notes; a note whose bend range is empty gets none (the
// notes of a grid setting without pitch bends)
void launch_note_finish(const float* note, const float* contour, const long long* note_frame_base /*[n_notes]*/,
                        const int* start, const int* end, const int* pitch, float* amp, const int* bend_off,
                        int* bends, int n_notes, int with_bends, const double* gauss /*[51] device*/,
                        cudaStream_t st);
// The pitch bend of note column col (MIDI col + 21) at one frame, `row` that frame's 264 contour bins (reference:
// note_creation.py:198-218, n_bins_tolerance 25): the first arg-max of float64(row[b]) * gauss[b - c + 25] over the
// bins b of [c - 25, c + 25] inside [0, 264), c = 3 col, as an offset from c.  It depends on (frame, pitch) only, so every
// note of that pitch sounding at that frame gets the same bend, and c + bend always lies in [0, 263].  The decode
// (note_finish_kernel) and the bent scorers (score_frames.cu, score_melody.cu) all call this one function.
__device__ __forceinline__ int pitch_bend_at(const float* __restrict__ row, int col, const double* __restrict__ gauss) {
  const int c = 3 * col;
  const int lo = max(c - 25, 0);
  const int hi = min(kContourBins, c + 26);
  const int g0 = max(0, 25 - c);  // first Gaussian tap used
  const int width = hi - lo;      // <= 51
  row += lo;
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
  return bi - (25 - g0);
}

// ---- score.cu: note-level match counts (bp_score_*) ----------------------------------------------------------------
// Nearest semitone (MIDI number) of a pitch given as log2(Hz), clamped to +-1e9 so that bucket differences fit an int.
// The host buckets the references with it and the kernel the estimates; a hit lies within floor(cents / 100) + 1
// buckets whichever side of a .5 either note rounds to.
__host__ __device__ inline int score_bucket(double log2_hz) {
  const double m = rint(12.0 * (log2_hz - 8.78135971352466) + 69.0);  // log2(440)
  return (int)fmin(fmax(m, -1e9), 1e9);
}
struct ScoreRefs {  // file i's references are [off[i], off[i+1]), sorted by (bucket, onset)
  const long long* off;
  const double* onset;
  const double* offset;
  const double* log2hz;
  const int* bucket;
};
struct ScoreEst {  // pair q's estimated notes start at off[q]: count[q] decode slots, or off[q+1] - off[q] explicit notes
  const long long* off;
  const int* count;                                   // NULL: explicit notes
  const double *onset, *offset, *log2hz;              // explicit notes (NULL: decode slots)
  const int *start, *end, *pitch;                     // decode slots: file-relative frames, MIDI number
  const double *frame_t, *log2_midi;                  // seconds per frame (bp_frame_times), log2(Hz) per MIDI number
};
struct ScoreTol {
  double onset, pitch, ratio, off_min;
  double window;          // onset half-width of the candidate search beyond the tolerance (rounding margin)
  int k_buckets;          // floor(pitch / 100) + 1 (with a rounding margin)
  int bucket_lo, bucket_hi;  // range of the references' buckets: the scan never leaves it
};
struct ScoreWork {       // int workspace: 2 per reference and setting, 4 per estimated note
  int* ref;              // setting s, file f: ref + 2 (s * n_ref_total + off[f])
  int* est;              // pair q: est + 4 * ScoreEst.off[q]
  long long n_ref_total;
};
// One launch: counts[4 q ..] = {n_ref, n_est, matched without offsets, matched} of pair q = setting * n_files + file.
void launch_score_match(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, const ScoreWork& W, int n_files,
                        long long n_pairs, long long* counts, cudaStream_t st);

// Onset-only and offset-only match counts (bp_score_onset_offset_*): counts[4 q ..] = {n_ref, n_est, onsets matched,
// offsets matched} of pair q = setting * n_files + file, one thread per (pair, test).  Explicit estimates: E.onset and
// E.offset each sorted ascending within every item (they are no longer notes); decode slots: E.start / E.end / E.frame_t.
// Int workspace of one (pair, test) with N estimate slots and R references: sort keys and next-free array 2 N + 1 at
// W.est + 4 E.off[q] + 2 q, runs and order 3 R at W.ref + 6 (s * n_ref_total + off[f]).
void launch_onset_offset(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, const ScoreWork& W, int n_files,
                         long long n_pairs, long long* counts, cudaStream_t st);

// mir_eval's matching pair for pair (bp_match_*).  Int workspace of one (pair, pass) with N estimated notes, R
// references and M hits without the offset test (the with-offset graph is a subgraph): adjacency offsets and lists,
// the preds lists (node estimate, next), per reference its list head / tail, preds state, the new_layer order and the
// unmatched list, the recursion stack (3 per frame, at most R + 1 frames), per estimate pred, key order and two layers.
__host__ __device__ inline long long match_pass_ints(long long n_est, long long n_ref, long long n_edges) {
  return 3 * n_edges + 5 * n_est + 8 * n_ref + 8;
}
struct MatchWork {
  int* ws;                 // pair q, pass p: ws + (off[q] - off[q0]) + p * match_pass_ints(..) of pair q
  const long long* off;    // [n_pairs + 1] int offsets of every pair's workspace (2 passes), chunk-wide
  const long long* edges;  // [n_pairs] hits without the offset test
  const int* r_orig;       // [n_ref_total] index of sorted reference k within its set
  int* match;              // [n_settings][2][n_ref_total]: estimate index or -1, in the caller's reference order
  long long n_ref_total;
};
// One launch: edges[q] = hits without the offset test of pair q = setting * n_files + file.
void launch_match_count(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, int n_files, long long n_pairs,
                        long long* edges, cudaStream_t st);
// One launch: the matchings of pairs [q0, q1), both passes (one thread per pair and pass); W.match must hold -1.
void launch_match(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, const MatchWork& W, int n_files,
                  long long q0, long long q1, cudaStream_t st);

// ---- score_frames.cu: frame-level multi-pitch counts (bp_score_frames_grid_*, bp_score_multipitch_host,
// bp_score_salience_grid_*) -------------------------------------------------------------------------------------------
constexpr int kFrameCounts = 7;  // n_ref, n_est, tp, tp_chroma, sum min, miss, false alarms
enum class EstKind { kExplicit, kRoll, kGram, kBent };  // where the match kernel's estimate frames come from
struct SalienceSettingDev {  // bp_salience_params_t, validated
  double threshold;
  int peak_pick, bin_lo, bin_hi, reserved;
};
struct FrameRefs {         // the call's K reference frames, back to back over files (grid) or items
  const int* owner;        // [K] file or item of frame k
  const int* est_frame;    // [K] the estimate frame it reads (file-relative for the grid, global otherwise), -1: none
  const long long* voff;   // [K + 1] values of frame k, ascending midi
  const double *midi, *chroma;
  long long n_frames;      // K
};
struct FrameEst {
  // grid: the count roll, int [88][T] per file at roll + s * roll_stride + frame_off[f] * 88, and the value tables of
  // MIDI numbers 0..127 (midi non-decreasing)
  const int* roll;
  long long roll_stride;
  const long long* frame_off;
  const double *tab_midi, *tab_chroma;
  // explicit: estimate frame j's values [voff[j], voff[j+1]), ascending midi
  const long long* voff;
  const double *midi, *chroma;
  // gram: the posteriorgram [frame_off[n_owner]][width], row frame_off[f] + t for frame t of file f, chunk-local
  // setting s at salience[s]; tab_midi / tab_chroma are the width bin tables (midi non-decreasing)
  const float* gram;
  const SalienceSettingDev* salience;
  long long width;
  // bent (bend_on set): the count roll as above, each sounding pitch p at contour bin k = 3 (p - 21) + its pitch bend
  // under chunk-local setting s when bend_on[s] (pitch_bend_at on the contour row [frame_off[n_owner]][264] with the 51
  // Gaussian taps `gauss`), else 3 (p - 21); tab_midi / tab_chroma are then the 264 bin tables (midi non-decreasing)
  const int* bend_on;
  const float* contour;
  const double* gauss;
};
// int workspace of the chroma matching: frame k of chunk-local setting s at ws + s * (4 V + 2 K) + 4 voff[k] + 2 k
// (V values, K frames): per reference value its mate and visit stamp, and a stack of 2 (n + 1) for its frame's n.
__host__ __device__ inline long long frame_ws_stride(long long n_values, long long n_frames) { return 4 * n_values + 2 * n_frames; }
// Count roll of a grid chunk (the decode's dead E, reused): after the memset, +1 / -1 at each note's start / end, then a
// prefix sum along frames: roll[p][t] = notes of pitch p + 21 with start <= t < end.  Two launches.
void launch_frame_roll(const long long* frame_off, const long long* slot_off, const int* note_count, const int* start,
                       const int* end, const int* pitch, int n_files, int n_settings, int* roll, long long roll_stride,
                       cudaStream_t st);
// One launch: counts[7 (s * n_owner + owner) ..] += the seven sums of every frame of setting s (E.roll and E.bend_on
// set: bent roll estimates; E.roll alone: roll estimates; else E.salience set: posteriorgram estimates; else explicit estimates, n_settings 1).  counts must be zeroed by
// the caller.
void launch_frame_match(const FrameRefs& R, const FrameEst& E, double window, int* ws, int n_owner, int n_settings,
                        long long* counts, cudaStream_t st);

// ---- score_melody.cu: melody counts (bp_score_melody_grid_*, bp_score_melody_host) ----------------------------------
constexpr int kMelodyCounts = 7;  // n_frames, ref_voiced, voiced_hit, false_alarm, pitch_correct, chroma_correct, oa
struct MelodyRange {  // a distinct bin range [lo, hi) of a grid chunk
  int lo, hi;
};
struct MelodyArg {  // arg-max of a posteriorgram row within a range: its float32 value and bin (-1: none)
  float v;
  int bin;
};
struct MelodySettingDev {  // bp_melody_params_t, validated; range: its MelodyRange in the chunk
  double threshold;
  int range, guess;
};
struct MelodyRef {      // one reference frame (the t = 0 frame inserted) and where it reads the estimate
  double x, t_lo, t_hi;  // rounded reference time, times of the bracket's ends
  double cent;           // reference cents
  int owner;             // file or item
  int zero;              // global estimate frame of the zero-order sample and bracket's lower end; -1: none (cents 0)
  int hi;                // global estimate frame whose held cents the bracket's upper end takes; -1: x on a knot
  int flags;             // bit 0: reference voiced; bit 1: identical time bases (the raw estimate at `zero`)
};
struct MelodyEst {
  // grid: the arg-max of every (chunk range r, global frame e) at arg[r * n_frames + e], the chunk's settings and the
  // bin cents; explicit: cents and voicing of every global estimate frame
  MelodyArg* arg;
  const MelodySettingDev* set;
  const double* bin_cent;
  const double* cent;
  const int* voiced;
  double* held;  // held cents of chunk-local setting s (explicit: 0) at held[s * n_frames + e]
  long long n_frames;
  double* raw;   // decoded notes: raw cents of chunk-local setting s at raw[s * n_frames + e], voiced where nonzero
};
// Decoded notes of a grid chunk read as a melody (bp_score_note_melody_grid_*): the count roll of launch_frame_roll,
// the note posteriorgram [frame][88] and contour [frame][264] of the call (row-major, global frames), the 51 Gaussian
// taps of the bends and each chunk-local setting's bend flag.  MelodyEst.bin_cent holds the 264 bin cents (all > 0).
struct NoteMelodyEst {
  const int* roll;
  long long roll_stride;
  const long long* frame_off;
  const float *note, *contour;
  const double* gauss;
  const int* bend_on;
};
// Grid chunk: arg-max, hold scan and counts, three launches whatever the number of settings and files.
// counts[7 (s * n_files + file) ..] += the seven sums; zeroed by the caller.
void launch_melody_grid(const float* gram, long long width, const MelodyRange* ranges, int n_ranges,
                        const long long* frame_off, int n_files, const MelodyRef* refs, long long K, const MelodyEst& E,
                        double tol, int n_settings, long long* counts, cudaStream_t st);
// Decoded notes of a grid chunk after launch_frame_roll: the per-(setting, file) pick, bend and hold, then the counts,
// two launches.  counts as launch_melody_grid.
void launch_note_melody(const NoteMelodyEst& N, int n_files, const MelodyRef* refs, long long K, const MelodyEst& E,
                        double tol, int n_settings, long long* counts, cudaStream_t st);
// Explicit tracks (E.held filled by the caller): one launch.
void launch_melody_explicit(const MelodyRef* refs, long long K, const MelodyEst& E, double tol, int n_items,
                            long long* counts, cudaStream_t st);

// ---- sonify.cu: bp_sonify_notes_host on the given stream of the current device (h_audio == NULL: size query, no CUDA
// call); adds its kernel launches to *launches ---------------------------------------------------------------------------
int sonify_notes(cudaStream_t st, long long* launches, int32_t n_files, const int32_t* note_off, const double* start_s,
                 const double* end_s, const int32_t* pitch_midi, const float* amplitude, const int32_t* bend_off,
                 const int32_t* bends, int32_t multiple_pitch_bends, int32_t sample_rate, int64_t* h_sample_off,
                 double* h_audio, int64_t capacity);

}  // namespace bp
