// The three wide convolutions — contour (8 -> 8 channels, 3 x 39 taps, 65 % of the model's FLOPs), onset
// (8 -> 32 channels, 5 x 5 taps, frequency stride 3, 18 %) and note (1 -> 32 channels, 7 x 7, stride 3, 4.5 %) —
// on the Hopper tensor cores: warpgroup MMAs (wgmma, bf16 operands, fp32 accumulators in registers), operands staged in
// shared memory by bulk async copies (UBLKCP) signalled through mbarriers, warp-specialised roles.
//
// Replaces nodes 231/232 (contour conv + ReLU, reference: basic_pitch/models.py:241-250) and 230/243 (onset
// conv + ReLU, reference: basic_pitch/models.py:295-304) of the deployed graph, and the harmonic stacking in
// front of them (reference: basic_pitch/nn.py:69-88), which is folded into the weight operand and never
// materialised; node 238/239 (note conv1 + ReLU, models.py:270-279) reads the contour posteriorgram instead.
// One kernel template, instantiated per layer (0 contour, 1 onset, 2 note) and per epilogue; every shape comes from the
// layer's description tc_spec (kernels.cuh).  The fused epilogue (all three layers) also computes the FOLLOWING
// single-output convolution (onset conv2 models.py:305-313, note conv2 :282-290, contour conv2 :254-262)
// completely, so neither the 8- / 32-channel activations nor any partial sums of them reach HBM:
//   * channels and frequency taps are reduced by a SECOND tensor-core contraction whose A operand is bias + ReLU of the
//     conv1 accumulator, split to bf16 hi/lo straight in the registers (the accumulator fragment of wgmma is the A
//     register fragment of the next K = 16 step), against a conv2 weight matrix in shared memory (tc_build_b2_full),
//   * its sums go through a small shared-memory staging area, where the thread of each tile row adds the time taps of
//     the rows below it; M-tiles overlap by KH2 - 1 rows, so every frame is complete in exactly one tile.  The thread
//     of tile row r finishes the output frame r - H (H = KH2 / 2) and adds its taps in the same order whatever its
//     position in the tile, so a frame's value does not depend on the batch around it,
//   * the frequency halo between neighbouring tiles is a register carry: a slot walks its frequency tiles in ascending
//     order; only where two tile RANGES meet (a slot's next tile is not the one above, or an item's group range
//     ends; tc_starts_range) the two partial sums go to a small edge buffer and edge_fix_kernel finishes those
//     4 (contour) / 2 bins,
//   * bias, sigmoid (+ the note input channel of the onset conv2, + unwrap inference.py:247-279) and the store.
// The unfused contour epilogue stores the activations channels-last (path 2, activation-level tests).
//
// Formulation of the contour conv1 ("Toeplitz along frequency on aligned chunks"; the onset and note conv1 gather instead,
// see below)
//   rows  m = b*174 + t            time frames of all windows of the chunk, two zero rows between windows
//   D[m][(fl,co)] (+)= A[m+dt][8c .. 8c+15] x T(dt,off)[16][(fl,co)]
//     A      the normalised CQT y itself (NOT the 8-channel stack), rows shifted by the time tap dt; K = 16 bins that
//            start on an 8-bin chunk of the k-chunk-major layout
//     T      16 x 128 "weight tile": T[k][(fl,co)] = sum_ci W[co][ci][dt][df_ci] with
//            df_ci = (8c + k) - shift_ci - SF*(ft*FLT + fl) + PL   (terms outside 0 <= df < KW or outside the stacked
//            image 0 <= g < 264 dropped).  The harmonic channels are shifted views of one image, so they are MERGED
//            in the weight operand: the stack conv is a single-channel conv of y whose taps are the union of the
//            shifted per-channel taps (contour: 8 x 39 = 312 taps on 176 distinct offsets -> 12 instead of 32
//            K-steps per time tap and frequency tile).
//            N = FLT output bins x COUT channels = 128 (contour 16 x 8, onset / note 4 x 32); a tile depends on
//            (dt, 8c - SF*FLT*ft), so frequency tiles SF*FLT*d = 8*j bins apart share tiles (de-duplicated by
//            structure: equal sets of summed weights, whatever their values)
//   every (ft, dt, c) with a non-empty tile is one K=16 MMA step of shape 64 x 128 x 16
// Precision: both operands are split x = hi + lo (bf16 each) and three products are accumulated
// (hi*hi + hi*lo + lo*hi) in fp32, which keeps the posteriorgrams within ~1e-5 of the FP32 path
// (SURVEY.md Appendix C.4); a single bf16 product would miss the 1e-3 bar.
//
// Formulation of the onset and note conv1 (layers 1 / 2: 5 or 7 frequency taps at stride 3, where a Toeplitz tile would be
// mostly zeros): an implicit GEMM per output bin f,
//   D_f[m][co] = sum over K = (dt, ci, j < 8) of x[m + dt][s(f, ci) + j] * B_{f & 1}[(dt, ci, j)][co]      (m64 n32)
//   s(f, ci)   the even bin at or below the first tap u0 = SF*f - PL + shift_ci, so the taps sit at j = (u0 & 1) + df
//   B_p        [K = KH * n_ci * 8, padded to 16][32 channels]: the weights at those positions for f & 1 = p (tc_build_b1)
// The A operand is GATHERED from the data tile into wgmma A registers: a register holds the bins s + 2 qd, s + 2 qd + 1
// of one row, one aligned 32-bit shared load, masked to zero where the reference has no input (outside the CQT / the
// contour posteriorgram, outside the stacked image).  The two B matrices stay resident in shared memory.  The four bins of
// a frequency tile go to four m64n32 accumulators that, side by side, are the m64n128 fragment of the Toeplitz form, so
// the epilogue is the same for all layers.
//
// Work decomposition: item = (M-tile of 64 rows, range [g0, g1) of the frequency groups); group g = two frequency
// tiles (tc_group_tile: contour the neighbours {2g, 2g + 1}, onset / note {g, g + G0}), one per accumulator slot; the
// contour's two slots share a weight tile where their content is equal, at every step but a few.  A CTA (1 per
// SM, persistent) walks items i = blockIdx.x, +gridDim.x, ... of the launch's schedule (tc_schedule): whole M-tiles, the
// same number per CTA, then the remaining M-tiles cut into group ranges of balanced cost:
//   warp 8      producer: bulk-copies the (64+KH-1) x 320 bf16 hi/lo data tile (k-chunk-major) once per item and
//               (contour) streams the weight tiles of each group's program (8 KB each) through a ring of stages;
//               (onset / note) copies the conv1 B matrices once per CTA
//   warps 0-3, 4-7  one warpgroup per accumulator slot of the group: contour: program words from constant memory, 3 x
//               wgmma m64n128k16 per step (the stage is released once they completed); onset / note: the gather and
//               3 x wgmma m64n32k16 per K-step and bin.  Then the epilogue of the slot's tile from the accumulator
//               registers: bias, ReLU, split, the conv2 MMAs, time taps, finish (see above)
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <unordered_map>
#include <vector>

#include "kernels.cuh"
#include "tc_ptx.cuh"

namespace bp {

namespace tc {
constexpr int kMTile = 64;
constexpr int kTileBytes = 8192;                                 // weight tile: [plane 2][kchunk 2][128][8] bf16
constexpr int kMaxSteps = 1024;                                  // program steps per layer (constant memory)
constexpr int kMaxGroups = 15;
static_assert(tc_spec(0).G0 <= kMaxGroups, "contour groups in constant memory");
static_assert(tc_pairing_ok(tc_spec(0)) && tc_pairing_ok(tc_spec(1)) && tc_pairing_ok(tc_spec(2)), "group -> tile map");
static_assert(tc_spec(0).n_ft() <= 2 * tc_spec(0).G0 && tc_spec(1).n_ft() <= 2 * tc_spec(1).G0 &&
                  tc_spec(2).n_ft() <= 2 * tc_spec(2).G0,
              "every tile has a place in the reference pairing of the summation order (TcConvPlan::build)");
constexpr int kConsumerWarps = 8;  // two warpgroups, one per accumulator slot
constexpr int kProducerWarp = 8;   // the first warp of the third warpgroup; its other three warps only hand back registers
constexpr int kThreads = 32 * kConsumerWarps + 128;
// Registers per thread: the launch gives every warpgroup 168 (65 536 / 384, rounded down to 8); the producer warpgroup
// drops to 24 so that the MMA warpgroups can take 240 (24 + 2 x 240 = 3 x 168, the CTA's pool).  With 168 the consumers
// spill and ptxas serialises their wgmmas (C7512); the contour epilogue still spills at 232.
constexpr int kProducerRegs = 24;
constexpr int kConsumerRegs = 240;
static_assert(kProducerRegs + 2 * kConsumerRegs <= 3 * 168, "register pool of the CTA");
}  // namespace tc

// ------------------------------------------------------------------------------------------------
// The fused second convolution as a second tensor-core contraction.
// After bias + ReLU the conv1 accumulator row (element k = accumulator column k = fl * COUT + c) is split to bf16
// hi/lo.  A K = 16 step therefore covers
//   contour: 2 bins x 8 channels        (step ks = bins 2 ks, 2 ks + 1)
//   onset / note: half the channels of one bin   (step ks = bin ks / 2, channels 16 (ks % 2) ..)
// and it contributes to the partial sums P[j][dt] of only a few output offsets j (frequency taps) of the tile:
//   contour: j = bl + 4 - df  in [2 ks, 2 ks + 5]      onset / note: j = fl + 2 - df in [fl, fl + 2]
// With the conv2 accumulator laid out j-major (column j * JS + dt, JS >= KH2) those are a contiguous WINDOW of columns,
// the same for every step up to its start column: every step multiplies by the same small weight tile
//   B2[kk][j' * JS + dt] = w2[c(kk)][dt][df(kk, j')]          (N = 32 columns; onset 16)
// placed at the window's start column (contour 10 ks, note 8 fl, onset 4 fl: js x the step's first bin) of a K = 128 x
// N = width matrix (tc_build_b2_full), which the MMAs read from shared memory.  The contour stages its sums in 3 passes of
// 8 output offsets (40 columns), which frees 32 KB of staging for four more weight stages.
//
// The gathered conv1 of the onset (layer 1) and note (layer 2), 32 output channels at frequency stride 3 (see the
// header).  K runs over (time tap dt, channel ci, window bin j < W), padded to whole K = 16 steps (tc_gather_k):
//   onset: 5 dt x 8 harmonics x 6 = 240 (15 steps, 83 % of the rows hold a tap): the window's first tap is at j = 0 or 1
//          and KW = 5, so every tap lies in j < 6; k = 48 dt + 2 P + (j & 1) with the slot P of pair (ci, j / 2)
//   note:  7 dt x 1 x 8 = 56 -> 64 (4 steps): k = 8 (dt * n_ci + ci) + j
// W = 6: K slot pair P of a time tap (k = 48 dt + 2 P + {0, 1}) -> bin pair 3 ci + jp of window ci (TcConvSpec::slot).
// Lane qd of a quad loads slot 4 e + qd of register word e; the order keeps the bank conflicts at their minimum (DESIGN §4.1)
// ------------------------------------------------------------------------------------------------
// row k of B for time tap dt, channel ci, window bin j
__host__ __device__ constexpr int tc_gather_k(TcConvSpec g, int dt, int ci, int j) {
  if (g.W == 8) return 8 * (dt * g.n_ci + ci) + j;
  int P = 0;
  while (g.slot[P] != 3 * ci + j / 2) ++P;
  return g.n_ci * g.W * dt + 2 * P + (j & 1);
}
__host__ __device__ constexpr bool tc_gather_slots_ok(TcConvSpec g) {  // W = 6: the slots are a permutation of the pairs
  if (g.W == 8) return true;
  if (g.W != 6 || g.n_ci != 8) return false;
  for (int p = 0; p < 24; ++p) {
    int n = 0;
    for (int P = 0; P < 24; ++P) n += g.slot[P] == p;
    if (n != 1) return false;
  }
  return true;
}
// W = 6: shift of the channel, and bin pair in its window, that K slot P holds
__host__ __device__ constexpr int tc_gather_slot_shift(TcConvSpec g, int P) { return g.shifts[g.slot[P] / 3]; }
__host__ __device__ constexpr int tc_gather_slot_pair(TcConvSpec g, int P) { return g.slot[P] % 3; }
static_assert(tc_gather_slots_ok(tc_spec(1)) && tc_gather_slots_ok(tc_spec(2)), "K slot map of the gather");
static_assert(tc_spec(1).ksteps() == 15 && tc_spec(2).ksteps() == 4, "K-steps per output bin");
// first bin of the 8-bin window of output bin f, channel ci: the even bin at or below its first tap
__host__ __device__ constexpr int tc_gather_start(TcConvSpec g, int f, int ci) {
  return (g.SF * f - g.PL + g.shifts[ci]) & ~1;
}
// the bins u of channel ci that hold input: inside the row (u < data_bins) and inside the stacked image
// (0 <= u - shift < 264, the zero fill of HarmonicStacking); the gather supplies zero everywhere else
__host__ __device__ constexpr int tc_gather_lo(TcConvSpec g, int ci) { return g.shifts[ci] > 0 ? g.shifts[ci] : 0; }
__host__ __device__ constexpr int tc_gather_hi(TcConvSpec g, int ci) {
  return g.data_bins < kContourBins + g.shifts[ci] ? g.data_bins : kContourBins + g.shifts[ci];
}

namespace tc {
// Shared memory is laid out per layer: the data tile; contour: as many weight-tile stages as fit; onset / note: the two
// conv1 B matrices; for the fused layers the conv2 weight matrix and the staging of the conv2 sums.
struct TcSmem {
  int data_bytes;   // [2 planes][chunks8 - 1][64 + KH - 1 rows][16 B], rounded up to 1 KB
  int b1_bytes;     // onset / note conv1 B matrices [parity 2][plane 2][K / 8][32][8] bf16
  int b2_bytes;     // conv2 weight matrix [2 planes][128][width] bf16
  int p_bytes;      // conv2 sums [2 slots][64 rows][pass + 1] fp32
  int stages;       // contour weight-tile stages
  __host__ __device__ constexpr int total() const {
    return data_bytes + stages * kTileBytes + b1_bytes + b2_bytes + p_bytes + 512;
  }
};
constexpr int kMaxSmem = 232448;  // 227 KB opt-in per CTA
constexpr int kMaxStages = 12;
__host__ __device__ constexpr TcSmem tc_smem(int layer, bool fused) {
  TcSmem s{};
  const TcConvSpec L = tc_spec(layer);
  const bool gather = layer != 0;
  s.data_bytes = (2 * (L.chunks8 - 1) * (kMTile + L.KH - 1) * 16 + 1023) / 1024 * 1024;
  s.b1_bytes = gather ? 2 * 2 * 16 * L.ksteps() * 32 * 2 : 0;
  s.b2_bytes = fused ? 2 * 128 * L.width * 2 : 0;
  s.p_bytes = fused ? 2 * 64 * (L.pass + 1) * 4 : 0;
  const int st = (kMaxSmem - 512 - s.data_bytes - s.b1_bytes - s.b2_bytes - s.p_bytes) / kTileBytes;
  s.stages = gather ? 0 : st < kMaxStages ? st : kMaxStages;
  return s;
}
// weight stages of the contour layer (DESIGN §4.1): activations, fused
static_assert(tc_smem(0, false).stages == 12 && tc_smem(0, true).stages == 9, "weight-ring depth per layer");
static_assert(tc_smem(1, true).total() <= kMaxSmem && tc_smem(2, true).total() <= kMaxSmem, "onset / note shared memory");
// step word of a slot: [0,14) A start-address offset >> 4, [15] first MMA into that accumulator; kNoUse = the
// slot's frequency tile does not use this step's weight tile
constexpr uint32_t kUseFirstAcc = 1u << 15, kNoUse = 0xffffffffu;
}  // namespace tc

// ------------------------------------------------------------------------------------------------
// Host: weight tiles + per-group programs
// ------------------------------------------------------------------------------------------------
static inline uint16_t f2bf(float x) {  // round-to-nearest-even float -> bf16 bits
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7f800000u) == 0x7f800000u) return (uint16_t)(u >> 16);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

void TcConvPlan::build(const TcConvSpec& sp, const float* W /* [COUT][n_ci][KH][KW] */) {
  using namespace tc;
  spec = sp;
  tiles.clear();
  tile_seq.clear();
  slot_words[0].clear();
  slot_words[1].clear();
  group_step_off.clear();
  group_ft.clear();
  const int n_ft = sp.n_ft();
  const int data_rows = kMTile + sp.KH - 1;
  const int lbo16 = data_rows;  // (rows * 16 B) >> 4
  // K = 16 steps start on 8-bin chunk boundaries (the k-chunk-major layout makes any chunk index a legal
  // descriptor start), so frequency tiles d apart share weight tiles when SF*FLT*d is a multiple of 8 bins.  The two
  // tiles of a group are the pair tc_group_tile gives (contour: neighbours, which share almost every step); each slot
  // walks its tiles in ascending order (the fused epilogue carries the frequency halo of the next conv in registers).
  // (Every tile has a partner t +- G0 in the reference pairing of the summation order below: n_ft <= 2 G0.)

  // Weight tiles are de-duplicated by STRUCTURE, not by value: two steps share a tile when every element of the two
  // sums the same weights.  The program (tile ids, their count, which steps of a group's two slots merge) then depends on
  // the layer geometry alone, so it is the same for every model, and the __constant__ bank that holds it can be shared.
  // A key word per element: 0 = no term, else 1 + (dt, d = u - SF * f, mask of the contributing channels), which names
  // the summed weights W[co][ci][dt][d - shift_ci + PL] (co is the element's column) one to one.
  std::unordered_map<uint64_t, std::vector<int>> by_hash;
  int n_keys = 0;
  std::vector<uint16_t> scratch(kTileBytes / 2);
  std::vector<uint32_t> key(16 * 128), keys;  // keys: [tile][16 * 128]
  // The n_ci input channels are shifted views of ONE image (harmonic stacking, nn.py:69-88), so the stack conv is a
  // single-channel conv of y with the merged kernel  Wm[co][dt][u] = sum_ci W[co][ci][dt][u - shift_ci + PL]  wherever
  // the stacked pixel exists (0 <= g = u_abs - shift_ci < 264): the contour taps of the 8 harmonics (8 x 39 = 312)
  // cover only 176 distinct bin offsets, the onset clusters of the upper harmonics overlap too.  A tile therefore
  // holds the SUM over the channels: tile for time tap dt, K rows [clip_lo, 16) of the 16 bins that start at bin
  // 8*c, frequency tile ft (rows below clip_lo belong to the previous step when the last chunk pair is clamped).
  auto find_or_add = [&](int dt, int c, int ft, int clip_lo) -> int {
    bool any = false;
    std::fill(scratch.begin(), scratch.end(), (uint16_t)0);
    std::fill(key.begin(), key.end(), 0u);
    for (int kk = clip_lo; kk < 16; ++kk) {
      const int u = 8 * c + kk;  // bin of y
      if (u >= sp.data_bins) continue;
      for (int n = 0; n < 128; ++n) {
        const int fl = n / sp.COUT, co = n % sp.COUT;
        const int f = ft * sp.FLT + fl;  // (columns f >= WOUT are computed like the others and dropped by the epilogue)
        double acc = 0.0;
        uint32_t mask = 0;
        for (int ci = 0; ci < sp.n_ci; ++ci) {
          const int gg = u - sp.shifts[ci];  // bin of the stacked image
          const int df = gg - sp.SF * f + sp.PL;
          if (df < 0 || df >= sp.KW || gg < 0 || gg >= kContourBins) continue;
          acc += (double)W[((co * sp.n_ci + ci) * sp.KH + dt) * sp.KW + df];
          mask |= 1u << ci;
        }
        if (!mask) continue;
        key[kk * 128 + n] = 1u + (((uint32_t)(dt * 1024 + (u - sp.SF * f + 512)) << 8) | mask);  // |d| < 512, n_ci <= 8
        const float w = (float)acc;
        const uint16_t hi = f2bf(w);
        const uint16_t lo = f2bf(w - bf2f(hi));
        const size_t o = (size_t)(kk >> 3) * 128 * 8 + (size_t)n * 8 + (kk & 7);
        scratch[o] = hi;
        scratch[2048 + o] = lo;
        any = true;
      }
    }
    if (!any) return -1;
    uint64_t h = 1469598103934665603ull;
    for (uint32_t v : key) h = (h ^ v) * 1099511628211ull;
    for (int id : by_hash[h])
      if (std::memcmp(keys.data() + (size_t)id * key.size(), key.data(), key.size() * 4) == 0) return id;
    tiles.insert(tiles.end(), scratch.begin(), scratch.end());
    keys.insert(keys.end(), key.begin(), key.end());
    by_hash[h].push_back(n_keys);
    return n_keys++;
  };

  // The order in which every tile sums its steps is fixed, whatever tile the kernels pair it with: the order of the
  // reference pairing {t, t + G0} (t < G0).  There, per time tap, the uses of the two tiles are sorted by their offset
  // relative to the tile, a weight tile both use is one step, and the steps only the lower tile uses come first, then
  // the shared ones, then those only the upper tile uses.  The order is a function of the geometry alone (not of the
  // batch, the schedule of items or the pairing below), and every tile's fp32 sums stay what they are under that reference pairing.
  struct Use {
    int tile;
    uint32_t w;  // A start offset >> 4: chunk c8, row dt
  };
  struct Step {
    int tile;
    uint32_t w[2];
  };
  std::vector<std::vector<Use>> order(n_ft);
  for (int t = 0; t < sp.G0; ++t) {
    const int fts[2] = {t, t + sp.G0 < n_ft ? t + sp.G0 : -1};
    struct Cand {
      int tile, slot, c8, dt, off;
    };
    std::vector<Cand> uses;
    for (int dt = 0; dt < sp.KH; ++dt) {
      std::vector<Cand> cand;
      for (int slot = 0; slot < 2; ++slot) {
        const int ft = fts[slot];
        if (ft < 0) continue;
        // 8-bin blocks of y this frequency tile reads through any channel
        std::vector<bool> need(sp.chunks8, false);
        for (int ci = 0; ci < sp.n_ci; ++ci)
          for (int fl = 0; fl < sp.FLT; ++fl) {
            const int f = ft * sp.FLT + fl;
            if (f >= sp.WOUT) continue;
            for (int df = 0; df < sp.KW; ++df) {
              const int gg = sp.SF * f - sp.PL + df, u = gg + sp.shifts[ci];
              if (gg < 0 || gg >= kContourBins || u < 0 || u >= sp.data_bins) continue;
              need[u / 8] = true;
            }
          }
        // cover the needed blocks with K = 16 steps (two adjacent blocks), left to right
        for (int c8 = 0; c8 < sp.chunks8;) {
          if (!need[c8]) {
            ++c8;
            continue;
          }
          const int c = std::min(c8, sp.chunks8 - 3);  // both k-chunks of the step must exist in the data tile, which
                                                       // holds chunks 0 .. chunks8 - 2 (the last one is padding only)
          const int off = 8 * c - sp.SF * sp.FLT * ft;
          const int tile = find_or_add(dt, c, ft, 8 * (c8 - c));
          if (tile >= 0) cand.push_back(Cand{tile, slot, c, dt, off});
          c8 += 2;
        }
      }
      std::stable_sort(cand.begin(), cand.end(), [](const Cand& a, const Cand& b) {
        return a.off != b.off ? a.off < b.off : (a.tile != b.tile ? a.tile < b.tile : a.slot < b.slot);
      });
      uses.insert(uses.end(), cand.begin(), cand.end());
    }
    std::vector<Step> steps;
    size_t i = 0;
    while (i < uses.size()) {
      size_t j = i;
      while (j < uses.size() && uses[j].tile == uses[i].tile && (j == i || uses[j].slot != uses[j - 1].slot)) ++j;
      Step stp{uses[i].tile, {kNoUse, kNoUse}};
      for (size_t u = i; u < j; ++u) stp.w[uses[u].slot] = (uint32_t)(uses[u].c8 * lbo16 + uses[u].dt);
      steps.push_back(stp);
      i = j;
    }
    std::stable_sort(steps.begin(), steps.end(), [](const Step& a, const Step& b) {
      auto cls = [](const Step& s) { return s.w[1] == kNoUse ? 0 : (s.w[0] == kNoUse ? 2 : 1); };
      return cls(a) < cls(b);
    });
    for (const Step& stp : steps)
      for (int sl = 0; sl < 2; ++sl)
        if (stp.w[sl] != kNoUse) order[fts[sl]].push_back(Use{stp.tile, stp.w[sl]});
  }

  // Groups: the pairs of tc_group_tile (or singles).  The two tiles' orders are merged into one step sequence; a step is
  // shared wherever the longest common subsequence of their weight tiles allows, every other use is a step of one slot
  // (where either slot's own step could come next, slot 1's does).  Each slot still walks its own tile's order.  (Neighbouring tiles use the same weight tiles at A chunks two apart,
  // so for the contour almost every step is shared.)
  group_step_off.push_back(0);
  n_uses = 0;
  const std::vector<Use> none;
  for (int g = 0; g < sp.G0; ++g) {
    const int fts[2] = {tc_group_tile(sp, g, 0), tc_group_tile(sp, g, 1)};
    group_ft.push_back(fts[0]);
    group_ft.push_back(fts[1]);
    const std::vector<Use>& a = fts[0] >= 0 ? order[fts[0]] : none;
    const std::vector<Use>& b = fts[1] >= 0 ? order[fts[1]] : none;
    const size_t na = a.size(), nb = b.size();
    std::vector<int> lcs((na + 1) * (nb + 1), 0);  // [i][j]: common weight tiles of a[i..] and b[j..]
    auto L = [&](size_t i, size_t j) -> int& { return lcs[i * (nb + 1) + j]; };
    for (size_t i = na; i-- > 0;)
      for (size_t j = nb; j-- > 0;)
        L(i, j) = a[i].tile == b[j].tile ? 1 + L(i + 1, j + 1) : std::max(L(i + 1, j), L(i, j + 1));
    bool seen[2] = {false, false};
    for (size_t i = 0, j = 0; i < na || j < nb;) {
      Step stp{-1, {kNoUse, kNoUse}};
      if (i < na && j < nb && a[i].tile == b[j].tile) {
        stp = Step{a[i].tile, {a[i].w, b[j].w}};
        ++i, ++j;
      } else if (j == nb || (i < na && L(i + 1, j) > L(i, j + 1))) {  // (a tie: slot 1's step first)
        stp = Step{a[i].tile, {a[i].w, kNoUse}};
        ++i;
      } else {
        stp = Step{b[j].tile, {kNoUse, b[j].w}};
        ++j;
      }
      for (int sl = 0; sl < 2; ++sl)
        if (stp.w[sl] != kNoUse) {
          if (!seen[sl]) stp.w[sl] |= kUseFirstAcc;
          seen[sl] = true;
          ++n_uses;
        }
      tile_seq.push_back(stp.tile);
      slot_words[0].push_back(stp.w[0]);
      slot_words[1].push_back(stp.w[1]);
    }
    group_step_off.push_back((int)tile_seq.size());
  }
  n_tiles = n_keys;
  n_groups = (int)group_ft.size() / 2;
}

// The contour layer's MMA program lives in constant memory: the issuing warp indexes it with warp-uniform values, so the
// words, the descriptors derived from them and the loop state stay in uniform registers (no per-use R2UR traffic).
// It depends only on the layer geometry (TcConvSpec), not on the weights (tiles are de-duplicated by structure, see
// TcConvPlan::build), so one upload serves every model of the process; the weight tiles it indexes are per model.
// (The onset and note layers gather their A operand and need no program.)
__constant__ uint32_t c_prog[2][tc::kMaxSteps];  // [slot][step]
__constant__ int c_tile_seq[tc::kMaxSteps];       // [step] -> weight tile id
__constant__ int c_group_step_off[tc::kMaxGroups + 1];  // (the tiles of a group are tc_group_tile's)

// tiles: [tile][plane hi/lo][k-chunk 2][n N2][8] bf16 (canonical K-major no-swizzle: LBO = N2 * 16 B, SBO = 128 B)
// Tile tl, row kk holds element k = 16 tl + kk of the conv1 row: bin b = k / COUT of the step, channel c = k % COUT
// (contour: 2 bins x 8 channels in one tile; onset / note: the 32 channels of one bin in two tiles).
void tc_build_b2(int layer, const float* w2, std::vector<uint16_t>& out) {
  const TcConvSpec sp = tc_spec(layer);
  const int tile_elems = 2 * 16 * sp.n2, KW2 = 2 * sp.HALO + 1;  // time / frequency taps of the conv2: KH2 x KW2
  out.assign((size_t)sp.n2_tiles * tile_elems, 0);
  for (int tl = 0; tl < sp.n2_tiles; ++tl)
    for (int kk = 0; kk < 16; ++kk)
      for (int n = 0; n < sp.n2; ++n) {
        const int jp = n / sp.js, dt = n - jp * sp.js;
        const int b = (16 * tl + kk) / sp.COUT, c = (16 * tl + kk) % sp.COUT, df = b + 2 * sp.HALO - jp;
        if (dt >= sp.KH2 || df < 0 || df >= KW2) continue;
        // conv2 weights [1][channels][KH2][KW2]; the onset conv2 has 33 channels, channel 0 = the note input
        const float w = w2[((c + (layer == 1 ? 1 : 0)) * sp.KH2 + dt) * KW2 + df];
        const uint16_t hi = f2bf(w), lo = f2bf(w - bf2f(hi));
        const size_t o = (size_t)tl * tile_elems + (size_t)(kk >> 3) * sp.n2 * 8 + (size_t)n * 8 + (kk & 7);
        out[o] = hi;
        out[o + 16 * sp.n2] = lo;
      }
}

int tc_upload_program(const TcConvPlan& pl, cudaStream_t st) {
  // the kernel walks the G0 groups of tc_spec(0)
  if (pl.spec.layer != 0 || (int)pl.tile_seq.size() > tc::kMaxSteps - 1 || pl.n_groups != tc_spec(0).G0) return -1;
  for (int sl = 0; sl < 2; ++sl)
    cudaMemcpyToSymbolAsync(c_prog, pl.slot_words[sl].data(), pl.slot_words[sl].size() * 4, (size_t)sl * tc::kMaxSteps * 4,
                            cudaMemcpyHostToDevice, st);
  cudaMemcpyToSymbolAsync(c_tile_seq, pl.tile_seq.data(), pl.tile_seq.size() * 4, 0, cudaMemcpyHostToDevice, st);
  cudaMemcpyToSymbolAsync(c_group_step_off, pl.group_step_off.data(), pl.group_step_off.size() * 4, 0,
                          cudaMemcpyHostToDevice, st);
  return cudaStreamSynchronize(st) == cudaSuccess ? 0 : -1;
}

// The two conv1 B matrices of the onset / note layer, f even and f odd, in the layout the MMAs read:
// [parity 2][plane hi/lo][k-chunk K / 8][n 32][8] bf16 (K-major no-swizzle: LBO = 32 * 16 B, SBO = 128 B).
// B_p[tc_gather_k(dt, ci, j)][co] = W[co][ci][dt][j - o], o = the first tap's offset in its window for f & 1 = p.
// window8: the same weights in the 8-bin-window form k = 8 (dt * n_ci + ci) + j, whatever W (bp_debug_tc_gather).
void tc_build_b1(int layer, const float* W /* [32][n_ci][KH][KW] */, std::vector<uint16_t>& out, bool window8) {
  const TcConvSpec g = tc_spec(layer);
  const int wn = window8 ? 8 : g.W;
  const size_t plane = (size_t)16 * ((g.KH * g.n_ci * wn + 15) / 16) * 32;
  out.assign(4 * plane, 0);
  for (int p = 0; p < 2; ++p)
    for (int dt = 0; dt < g.KH; ++dt)
      for (int ci = 0; ci < g.n_ci; ++ci) {
        const int o = g.SF * p - g.PL + g.shifts[ci] - tc_gather_start(g, p, ci);
        for (int j = 0; j < wn; ++j) {
          const int df = j - o, k = window8 ? 8 * (dt * g.n_ci + ci) + j : tc_gather_k(g, dt, ci, j);
          if (df < 0 || df >= g.KW) continue;
          for (int co = 0; co < 32; ++co) {
            const float w = W[((co * g.n_ci + ci) * g.KH + dt) * g.KW + df];
            const uint16_t hi = f2bf(w), lo = f2bf(w - bf2f(hi));
            const size_t e = ((size_t)(k >> 3) * 32 + co) * 8 + (k & 7);
            out[(2 * p) * plane + e] = hi;
            out[(2 * p + 1) * plane + e] = lo;
          }
        }
      }
}

TcGatherGeom tc_gather_geometry(int layer) {
  const TcConvSpec g = tc_spec(layer);
  TcGatherGeom r;
  r.K = 16 * ((g.KH * g.n_ci * 8 + 15) / 16);  // of the 8-bin-window form
  r.K_packed = 16 * g.ksteps();
  for (int k = 0; k < r.K_packed; ++k) {  // which (dt, ci, j) the kernel puts at row k (-1: K padding)
    int hit[3] = {-1, -1, -1};
    for (int dt = 0; dt < g.KH; ++dt)
      for (int ci = 0; ci < g.n_ci; ++ci)
        for (int j = 0; j < g.W; ++j)
          if (tc_gather_k(g, dt, ci, j) == k) hit[0] = dt, hit[1] = ci, hit[2] = j;
    r.kmap.insert(r.kmap.end(), hit, hit + 3);
  }
  r.n_ci = g.n_ci;
  r.KH = g.KH;
  r.wout = g.WOUT;
  for (int f = 0; f < g.WOUT; ++f)
    for (int ci = 0; ci < g.n_ci; ++ci) r.starts.push_back(tc_gather_start(g, f, ci));
  for (int ci = 0; ci < g.n_ci; ++ci) {
    r.ranges.push_back(tc_gather_lo(g, ci));
    r.ranges.push_back(tc_gather_hi(g, ci));
  }
  return r;
}

// The small tiles expanded into the K = 128 x N = width matrix the conv2 MMAs read:
// [plane hi/lo][k-chunk 16][n width][8] bf16 (K-major no-swizzle: LBO = width * 16 B, SBO = 128 B)
void tc_build_b2_full(int layer, const float* w2, std::vector<uint16_t>& out) {
  const TcConvSpec sp = tc_spec(layer);
  std::vector<uint16_t> small;
  tc_build_b2(layer, w2, small);
  const size_t tile_elems = (size_t)2 * 16 * sp.n2, plane = (size_t)128 * sp.width;
  out.assign(2 * plane, 0);
  for (int ks = 0; ks < 8; ++ks) {
    // step ks starts at bin 16 ks / COUT of the tile; its weight tile repeats every n2_tiles steps
    const int col0 = sp.js * (16 * ks / sp.COUT), tl = ks % sp.n2_tiles;
    for (int pl = 0; pl < 2; ++pl)
      for (int kk = 0; kk < 16; ++kk)
        for (int n = 0; n < sp.n2; ++n)
          out[pl * plane + ((size_t)(2 * ks + (kk >> 3)) * sp.width + col0 + n) * 8 + (kk & 7)] =
              small[(size_t)tl * tile_elems + pl * 16 * sp.n2 + (size_t)(kk >> 3) * sp.n2 * 8 + (size_t)n * 8 + (kk & 7)];
  }
}

// ------------------------------------------------------------------------------------------------
// fp32 rows -> bf16 hi/lo planes in the k-chunk-major row layout the MMA reads:
//   dst[plane][q8 (chunks8)][row d (rows_total)][8],  d = lead + b*rows_per_window + t, every other row zero.
// lognorm_split_kernel: the log-magnitude of the CQT kernel -> NormalizedLog (reference: layers/signal.py:177-183:
//   (L - min) / (max - min), 0 when max == min) + folded BatchNorm (models.py:188-189) as the split operand of the
//   contour / onset convs (309 bins -> 40 chunks).  (The fp32 copy is only produced on request: launch_lognorm.)
// The contour posteriorgram reaches the note conv in the same layout (264 bins -> 34 chunks), written by the contour
// epilogue itself.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_split8(const float (&v)[8], __nv_bfloat16* dst, size_t off, size_t plane) {
  __align__(16) __nv_bfloat16 hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    hi[j] = __float2bfloat16_rn(v[j]);
    lo[j] = __float2bfloat16_rn(v[j] - __bfloat162float(hi[j]));
  }
  *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(dst + plane + off) = *reinterpret_cast<const uint4*>(lo);
}

__global__ void lognorm_split_kernel(const float* __restrict__ y, const unsigned int* __restrict__ minmax,
                                     const float* __restrict__ bn, __nv_bfloat16* __restrict__ dst, int n_windows,
                                     int rows_used, int rows_total /* stride */, int chunks8, int rows_per_window, int lead) {
  // one (row, pair of chunks q8, q8 + chunks8 / 2) per thread: the two 32-byte loads are independent (the kernel is bound by
  // load latency, not bandwidth); rows fastest, so the 16-byte stores of a warp are contiguous
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int half = chunks8 / 2;  // chunks8 is even
  const long long total = (long long)rows_used * half;
  if (idx >= total) return;
  const int d = (int)(idx % rows_used);
  const int qa = (int)(idx / rows_used);
  float v[2][8];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 8; ++j) v[h][j] = 0.f;
  const int m = d - lead;
  if (m >= 0) {
    const int b = m / rows_per_window, t = m - b * rows_per_window;
    if (b < n_windows && t < kFrames) {
      const float bn_scale = __ldg(bn), bn_bias = __ldg(bn + 1);
      const float mn = ordered_to_float(minmax[2 * b]);
      const float mx = __fsub_rn(ordered_to_float(minmax[2 * b + 1]), mn);
      const float* p = y + ((size_t)b * kFrames + t) * kCqtBins;
      float raw[2][8];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int bin = (qa + h * half) * 8 + j;
          raw[h][j] = bin < kCqtBins ? __ldg(p + bin) : 0.f;
        }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if ((qa + h * half) * 8 + j < kCqtBins) {
            const float q = (mx == 0.f) ? 0.f : __fdiv_rn(__fsub_rn(raw[h][j], mn), mx);
            v[h][j] = __fadd_rn(__fmul_rn(q, bn_scale), bn_bias);
          }
    }
  }
  const size_t plane = (size_t)chunks8 * rows_total * 8;
  store_split8(v[0], dst, ((size_t)qa * rows_total + d) * 8, plane);
  store_split8(v[1], dst, ((size_t)(qa + half) * rows_total + d) * 8, plane);
}

// ------------------------------------------------------------------------------------------------
// The tensor-core kernel.  The layer's geometry is compile-time (tc_spec); the arguments are what changes per launch.
// ------------------------------------------------------------------------------------------------
struct TcArgs {
  CUtensorMap data_map;         // 4-D tensor map of `data`: (8 elements, rows_total, chunks8, 2 planes); box = one data tile
  int use_tmap;                 // 0: the encoder was not available, the tile is fetched chunk by chunk with 1-D bulk copies
  const __nv_bfloat16* data;    // [2][chunks8][rows_total][8]
  const uint16_t* tiles;        // contour: [n_tiles][8192 B]
  const uint16_t* b1;           // onset / note: the conv1 B matrices (tc_build_b1)
  const uint16_t* b2;           // conv2 weight matrix (tc_build_b2_full), fused layers
  TcOut o;                      // where the results go (kernels.cuh)
  int edge_rows;                // row stride of o.edge: [edge slot][side 2][KE][edge_rows]
  int rows_total, n_windows;
  TcSchedule sch;               // the launch's items: (M-tile, range of frequency groups), see tc_schedule
  int row0;                     // first data row of M-tile 0
  // = tc_spec(layer).chunks8: a run-time trip count keeps the producer's per-chunk copy loop rolled, which keeps the
  // contour's producer and MMA-issue loop state in uniform registers (a compile-time count unrolls it and they move out)
  int chunks8;
  int ms, h2;                   // M-tile stride (64 - 2*h2) and time halo of the fused conv2
  float bias1[32], bias2, note_w[9];  // the layer's epilogue values (TcConvDev)
};

__device__ __forceinline__ float sigmoidf_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }

// Cycle accounting by role, compiled in with -DBP_TC_CLOCKS only (tools/tc_clocks.py): every thread cuts its time into
// consecutive clock64 spans and adds each span to one bucket; lane 0 of every warp adds its sums to g_tc_clocks[layer]
// when the CTA ends.  Without the flag the calls are empty.
namespace tc {
enum TcClk {
  kClkFull,       // consumers: contour: waiting on full_w (the weight tile of the step); onset / note: the gather
  kClkMma,        // consumers: issuing the step's MMAs and waiting for the previous step's
  kClkEpi,        // consumers: the epilogue of a tile (after the last MMA of the group)
  kClkData,       // consumers: waiting on data_full (the item's data tile)
  kClkConsOther,  // consumers: everything else (program reads, skipped steps, row set-up)
  kClkEmpty,      // producer: waiting on empty_w (a free weight stage; contour only)
  kClkDataEmpty,  // producer: waiting on data_empty (both slots done with the previous item's data tile)
  kClkProdOther,  // producer: everything else (issuing the copies)
  kNumClk
};
}  // namespace tc
// With the flag the CTA's busy time (%globaltimer from its start to the end of its last consumer warp) also goes to
// g_tc_busy[layer][blockIdx.x] (tools/tc_balance.py: how evenly a launch's work is spread over the SMs).
#ifdef BP_TC_CLOCKS
__device__ unsigned long long g_tc_clocks[3][tc::kNumClk];
__device__ unsigned long long g_tc_busy[3][kTcMaxCtas];
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
struct TcClocks {
  // 32-bit sums (a thread's share of one launch stays far below 2^32 cycles) keep the instrumented consumers within
  // their register budget
  uint32_t t, c[tc::kNumClk];
  unsigned long long t0;
  __device__ __forceinline__ TcClocks() {
    t = (uint32_t)clock();
    t0 = globaltimer_ns();
#pragma unroll
    for (int k = 0; k < tc::kNumClk; ++k) c[k] = 0;
  }
  // consumers only (named barrier 3 over their 256 threads): the CTA's work ends with the last consumer warp
  __device__ __forceinline__ void cta_end(int layer) {
    asm volatile("bar.sync 3, 256;" ::: "memory");
    if (threadIdx.x == 0 && blockIdx.x < kTcMaxCtas) atomicAdd(&g_tc_busy[layer][blockIdx.x], globaltimer_ns() - t0);
  }
  __device__ __forceinline__ void lap(int k) {
    const uint32_t n = (uint32_t)clock();
    c[k] += n - t;
    t = n;
  }
  __device__ __forceinline__ void flush(int layer) {
    if ((threadIdx.x & 31) == 0)
#pragma unroll
      for (int k = 0; k < tc::kNumClk; ++k) atomicAdd(&g_tc_clocks[layer][k], (unsigned long long)c[k]);
  }
};
#else
struct TcClocks {
  __device__ __forceinline__ void lap(int) {}
  __device__ __forceinline__ void flush(int) {}
  __device__ __forceinline__ void cta_end(int) {}
};
#endif

int tc_read_busy(int layer, unsigned long long* out, int n, bool reset) {
#ifdef BP_TC_CLOCKS
  if (layer < 0 || layer > 2 || n < 0 || n > kTcMaxCtas) return -1;
  const size_t row = kTcMaxCtas * sizeof(unsigned long long);
  if (n && cudaMemcpyFromSymbol(out, g_tc_busy, n * sizeof(unsigned long long), (size_t)layer * row) != cudaSuccess) return -1;
  if (reset) {
    static const unsigned long long zero[kTcMaxCtas] = {};
    if (cudaMemcpyToSymbol(g_tc_busy, zero, row, (size_t)layer * row) != cudaSuccess) return -1;
  }
  return 0;
#else
  (void)layer, (void)out, (void)n, (void)reset;
  return -1;
#endif
}

int tc_read_clocks(int layer, unsigned long long* out, bool reset) {
#ifdef BP_TC_CLOCKS
  if (layer < 0 || layer > 2) return -1;
  if (cudaMemcpyFromSymbol(out, g_tc_clocks, tc::kNumClk * sizeof(unsigned long long),
                           (size_t)layer * tc::kNumClk * sizeof(unsigned long long)) != cudaSuccess)
    return -1;
  if (reset) {
    static const unsigned long long zero[tc::kNumClk] = {};
    if (cudaMemcpyToSymbol(g_tc_clocks, zero, sizeof(zero), (size_t)layer * sizeof(zero)) != cudaSuccess) return -1;
  }
  return 0;
#else
  (void)layer, (void)out, (void)reset;
  return -1;
#endif
}

__device__ __forceinline__ void slot_barrier(int slot) {  // the four warps (one warpgroup) of one accumulator slot
  asm volatile("bar.sync %0, 128;" ::"r"(1 + slot) : "memory");
}

// The edge buffer has one slot per boundary b between tiles b - 1 and b (slot b - 1), with two sides: side 0 from the
// range that starts at tile b, side 1 from the range that ends at tile b - 1 (tc_starts_range / tc_ends_range).

// What the thread that finishes one frame knows about where its results go.  The threads of a warp hold consecutive
// frames, and every layout below has the frame index fastest.
//   pitch layers (note / onset)  pitch-major planes  [pitch][frame]
//   contour                      chunk-major         [8-bin chunk][frame][8]  (fp32), same shape as the bf16 hi/lo
//                                split layout [plane][chunk][row][8] that the note conv reads
struct RowOut {
  float* raw;    // pitch layers: raw_pm + b*172 + t        ; contour: raw_cm + (b*172 + t)*8            (nullptr: not stored)
  float* unw;    // pitch layers: unw_pm + unwrapped frame  ; contour: unw_cm + unwrapped frame * 8      (nullptr: not stored)
  __nv_bfloat16* chl;  // contour: chl + data row * 8
  float* edge;   // edge buffer column of this frame: edge + R (nullptr: row not complete / not live)
  const float* note_col;  // onset: note_raw_pm + b*172 + t
  int t;         // frame inside the window (of the OUTPUT frame this thread finishes)
  bool ok;       // live output frame whose time taps are complete in this M-tile
};

// Frequency halo + finish for the onset / note layers (FLT = 4, HALO = 1): S[j] is the time-complete sum for bin
// FLT ft - HALO + j.
template <int LAYER>
__device__ __forceinline__ void finish_pitch_tile(const TcArgs& a, const RowOut& ro, float (&S)[6], float (&carry)[2], int ft,
                                                  bool first, bool last) {
  constexpr TcConvSpec L = tc_spec(LAYER);
  static_assert(L.FLT + 2 * L.HALO == 6 && L.HALO == 1, "sums and carry of a pitch tile");
  const bool lower = ft > 0;
  if (first) {
    if (lower && ro.edge) {
      float* e = ro.edge + (size_t)((ft - 1) * 2 + 0) * L.edge_per_side() * a.edge_rows;
      e[0] = S[0];
      e[a.edge_rows] = S[1];
    }
  } else {
    S[0] += carry[0];
    S[1] += carry[1];
  }
  const int jlo = first ? (lower ? 2 * L.HALO : L.HALO) : 0;
  const int jhi = (ft == L.n_ft() - 1) ? L.FLT + L.HALO : L.FLT;  // the last tile also finishes its top bin (no tile above)
  if (ro.ok) {
    float nv[3][6];
    if constexpr (LAYER == 1) {  // note frames t-1 .. t+1, pitches FLT ft - 2 .. FLT ft + 3 (zero outside the image)
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const int f = L.FLT * ft - 2 + c;
        const bool fin = (unsigned)f < (unsigned)kPitches;
        const float* col = ro.note_col + (size_t)f * a.o.raw_rows;
#pragma unroll
        for (int r = 0; r < 3; ++r)
          nv[r][c] = (fin && (unsigned)(ro.t + r - 1) < (unsigned)kFrames) ? __ldg(col + r - 1) : 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < L.FLT + L.HALO; ++j) {
      if (j < jlo || j >= jhi) continue;
      const int f = L.FLT * ft - L.HALO + j;
      float x = S[j] + a.bias2;
      if constexpr (LAYER == 1) {
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int df = 0; df < 3; ++df)
            if (j + df < 6) x = fmaf(nv[r][j + df], a.note_w[r * 3 + df], x);  // pitch f + df - 1 = FLT ft - 2 + (j + df)
      }
      const float v = sigmoidf_fast(x);
      if (ro.raw) ro.raw[(size_t)f * a.o.raw_rows] = v;
      if (ro.unw) ro.unw[(size_t)f * a.o.frame_stride] = v;
    }
  }
  carry[0] = S[L.FLT];
  carry[1] = S[L.FLT + 1];
  if (last && ft < L.n_ft() - 1 && ro.edge) {
    float* e = ro.edge + (size_t)(ft * 2 + 1) * L.edge_per_side() * a.edge_rows;
    e[0] = S[L.FLT];
    e[a.edge_rows] = S[L.FLT + 1];
  }
}

// One finished 8-bin chunk of the contour posteriorgram for one frame: bf16 hi/lo into the operand layout of the note
// conv, fp32 into the chunk-major posteriorgram.
__device__ __forceinline__ void store_contour_chunk(const TcArgs& a, const RowOut& ro, int chunk, const float (&v)[8]) {
  store_split8(v, ro.chl, (size_t)chunk * a.o.chl_rows * 8, (size_t)a.o.chl_chunks * a.o.chl_rows * 8);
  const float4 x0 = make_float4(v[0], v[1], v[2], v[3]), x1 = make_float4(v[4], v[5], v[6], v[7]);
  if (ro.raw) {
    float4* d = reinterpret_cast<float4*>(ro.raw + (size_t)chunk * a.o.raw_rows * 8);
    d[0] = x0;
    d[1] = x1;
  }
  if (ro.unw) {
    float4* d = reinterpret_cast<float4*>(ro.unw + (size_t)chunk * a.o.frame_stride * 8);
    d[0] = x0;
    d[1] = x1;
  }
}

// Contour layer (8 -> 1 channels, 5 x 5 taps, models.py:252-259): S[j] = the time-complete sum for output bin 16 ft - 2 + j
// of the thread's frame.  Frequency halo by register carry, then sigmoid and the stores.
__device__ __forceinline__ void finish_contour_tile(const TcArgs& a, const RowOut& ro, float (&S)[20], int ft, bool first,
                                                    bool last, float (&carry)[4], float (&hold)[6]) {
  // Bins 16 ft - 2 .. 16 ft + 1 also get the top four sums of the tile below.  Finished bins leave in aligned 8-bin chunks:
  // chunk 2 ft - 1 = the six bins held back from the previous tile + j = 0, 1; chunk 2 ft = j = 2 .. 9; j = 10 .. 15 are
  // held for the next tile.  Where a range starts / ends, the four partial sums AND the six finished bins next to them go
  // to the edge buffer (10 values per side); edge_fix_kernel assembles the two chunks around the boundary.
  constexpr TcConvSpec L = tc_spec(0);
  static_assert(L.FLT == 16 && L.HALO == 2 && L.edge_per_side() == 10, "sums, carry and edge values of a contour tile");
  const bool lower = ft > 0;
  if (first) {
    if (lower && ro.edge) {
      float* e = ro.edge + (size_t)((ft - 1) * 2 + 0) * L.edge_per_side() * a.edge_rows;
#pragma unroll
      for (int k = 0; k < 4; ++k) e[(size_t)k * a.edge_rows] = S[k];
#pragma unroll
      for (int k = 0; k < 6; ++k) e[(size_t)(4 + k) * a.edge_rows] = sigmoidf_fast(S[4 + k] + a.bias2);  // bins 16 ft + 2 .. + 7
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) S[k] += carry[k];
  }
  float fin[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) fin[j] = sigmoidf_fast(S[j] + a.bias2);
  if (ro.ok) {
    if (!first) {  // chunk 2 ft - 1: bins 16 ft - 8 .. 16 ft - 1
      const float v[8] = {hold[0], hold[1], hold[2], hold[3], hold[4], hold[5], fin[0], fin[1]};
      store_contour_chunk(a, ro, 2 * ft - 1, v);
    }
    if (!first || !lower) {  // chunk 2 ft: bins 16 ft .. 16 ft + 7 (at a range start above tile 0 the fix-up writes it)
      const float v[8] = {fin[2], fin[3], fin[4], fin[5], fin[6], fin[7], fin[8], fin[9]};
      store_contour_chunk(a, ro, 2 * ft, v);
    }
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) hold[k] = fin[10 + k];
#pragma unroll
  for (int k = 0; k < 4; ++k) carry[k] = S[16 + k];
  if (last && ft < L.n_ft() - 1 && ro.edge) {
    float* e = ro.edge + (size_t)(ft * 2 + 1) * L.edge_per_side() * a.edge_rows;
#pragma unroll
    for (int k = 0; k < 4; ++k) e[(size_t)k * a.edge_rows] = S[16 + k];
#pragma unroll
    for (int k = 0; k < 6; ++k) e[(size_t)(4 + k) * a.edge_rows] = fin[10 + k];  // bins 16 ft + 8 .. + 13
  }
}

// The conv2 MMAs of one tile: A = relu(conv1 + bias) of the warpgroup's 64 rows as bf16 hi / lo register fragments
// (ah / al: per K = 16 step four registers), B = the conv2 weight matrix in shared memory; three split products per step.
template <int NW>
__device__ __forceinline__ void conv2_mma(float (&p)[NW / 2], const uint32_t (&ah)[32], const uint32_t (&al)[32], uint32_t b2) {
  constexpr uint32_t kPlane = 128u * NW * 2u;  // bytes of one bf16 plane of the weight matrix
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    const uint64_t bh = make_desc(b2 + (uint32_t)(2 * ks * NW * 16), NW * 16, 128);
    const uint64_t bl = make_desc(b2 + kPlane + (uint32_t)(2 * ks * NW * 16), NW * 16, 128);
    const uint32_t xh[4] = {ah[4 * ks], ah[4 * ks + 1], ah[4 * ks + 2], ah[4 * ks + 3]};
    const uint32_t xl[4] = {al[4 * ks], al[4 * ks + 1], al[4 * ks + 2], al[4 * ks + 3]};
    if constexpr (NW == 104) {
      wgmma_rs_n104(p, xh, bh, ks ? 1u : 0u);
      wgmma_rs_n104(p, xh, bl, 1u);
      wgmma_rs_n104(p, xl, bh, 1u);
    } else if constexpr (NW == 64) {
      wgmma_rs_n64(p, xh, bh, ks ? 1u : 0u);
      wgmma_rs_n64(p, xh, bl, 1u);
      wgmma_rs_n64(p, xl, bh, 1u);
    } else {
      wgmma_rs_n32(p, xh, bh, ks ? 1u : 0u);
      wgmma_rs_n32(p, xh, bl, 1u);
      wgmma_rs_n32(p, xl, bh, 1u);
    }
  }
}

// conv1 of frequency tile ft of the onset / note layer (layer 1 / 2), gathered (see the header): for each bin f = FLT ft + fl
// the K-steps of the layer, three split products m64n32k16 each, into acc[16 fl ..] (= columns 32 fl .. of the m64n128
// fragment).  The A registers are loaded two steps ahead of the MMAs that read them (three register buffers, gather_steps).
// Every output sums its steps in the same order whatever the item: a value depends only on f and the layer.
template <int LAYER>
struct GatherRegs {
  static constexpr TcConvSpec G = tc_spec(LAYER);
  static_assert(G.W == 8 || (G.W == 6 && G.n_ci * G.W == 48), "W = 6: a time tap is 3 whole K-steps, 6 register words");
  // per register word (W = 8: per channel; W = 6: per slot group e, lane qd loads slot 4 e + qd): byte offset of the
  // thread's bin pair (row fr0) in the data tile in bits [0, 24), and in bits 24 / 25 whether its first / second bf16
  // half holds input (one register per word keeps the consumers within budget)
  static constexpr int NWD = G.W == 8 ? G.n_ci : 6;
  uint32_t om[NWD];
  __device__ __forceinline__ static uint32_t word(int u, int lo, int hi, int fr0) {
    const int uc = min(max(u, 0), G.tile_bins() - 2);  // a pair outside the tile is masked; read one inside it
    return (uint32_t)((uc >> 3) * ((tc::kMTile + G.KH - 1) * 16) + (uc & 7) * 2 + fr0 * 16) |
           (u >= lo && u < hi ? 1u << 24 : 0u) | (u + 1 >= lo && u + 1 < hi ? 1u << 25 : 0u);
  }
  // the windows of output bin f for the thread (lane qd of its quad, rows fr0 / fr0 + 8)
  __device__ __forceinline__ void setup(int f, int fr0, int qd) {
    if constexpr (G.W == 8) {
#pragma unroll
      for (int ci = 0; ci < G.n_ci; ++ci)
        om[ci] = word(tc_gather_start(G, f, ci) + 2 * qd, tc_gather_lo(G, ci), tc_gather_hi(G, ci), fr0);
    } else {
      setup_word<0>(f, fr0, qd);
      setup_word<1>(f, fr0, qd);
      setup_word<2>(f, fr0, qd);
      setup_word<3>(f, fr0, qd);
      setup_word<4>(f, fr0, qd);
      setup_word<5>(f, fr0, qd);
    }
  }
  // W = 6: word e = the lane's slot 4 e + qd, bin pair jp of the window of the channel with shift sh (immediates picked
  // by qd, so that the spec's tables are not indexed at run time)
  template <int E>
  __device__ __forceinline__ void setup_word(int f, int fr0, int qd) {
    constexpr int s0 = tc_gather_slot_shift(G, 4 * E), s1 = tc_gather_slot_shift(G, 4 * E + 1),
                  s2 = tc_gather_slot_shift(G, 4 * E + 2), s3 = tc_gather_slot_shift(G, 4 * E + 3);
    constexpr int j0 = tc_gather_slot_pair(G, 4 * E), j1 = tc_gather_slot_pair(G, 4 * E + 1),
                  j2 = tc_gather_slot_pair(G, 4 * E + 2), j3 = tc_gather_slot_pair(G, 4 * E + 3);
    const int sh = qd == 0 ? s0 : qd == 1 ? s1 : qd == 2 ? s2 : s3;
    const int jp = qd == 0 ? j0 : qd == 1 ? j1 : qd == 2 ? j2 : j3;
    const int u = ((G.SF * f - G.PL + sh) & ~1) + 2 * jp;  // tc_gather_start + 2 jp
    om[E] = word(u, sh > 0 ? sh : 0, G.data_bins < kContourBins + sh ? G.data_bins : kContourBins + sh, fr0);
  }
  __device__ __forceinline__ uint32_t mask(int i) const {  // bits 24 / 25 -> 0x0000ffff / 0xffff0000
    const uint32_t m = om[i] >> 24;
    return ((m | (m << 15)) & 0x10001u) * 0xffffu;
  }
  // the A registers of K-step ks, x[0..3] hi, x[4..7] lo: (half 0, row fr0), (half 0, fr0 + 8), (half 1, fr0),
  // (half 1, fr0 + 8).  W = 8: half h is window 2 ks + h; W = 6: time tap ks / 3, word 2 (ks % 3) + h
  template <int KS>
  __device__ __forceinline__ void load(const unsigned char* s_data, uint32_t (&x)[8]) const {
    constexpr int kPlane = G.tile_bins() / 8 * (tc::kMTile + G.KH - 1) * 16;  // bytes of one plane of the data tile
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      constexpr int NW = G.W == 8 ? G.KH * G.n_ci : 2 * G.ksteps();  // halves holding taps; the rest is K padding
      const int wi = 2 * KS + h;
      const int dt = G.W == 8 ? wi / G.n_ci : KS / 3, i = G.W == 8 ? wi % G.n_ci : 2 * (KS % 3) + h;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (wi < NW) {
          const unsigned char* p = s_data + (om[i] & 0xffffffu) + dt * 16 + rr * 128;
          x[2 * h + rr] = *reinterpret_cast<const uint32_t*>(p) & mask(i);
          x[4 + 2 * h + rr] = *reinterpret_cast<const uint32_t*>(p + kPlane) & mask(i);
        } else {
          x[2 * h + rr] = 0u;
          x[4 + 2 * h + rr] = 0u;
        }
      }
    }
  }
};

// Step I of the tile (bin fl = I / KS, K-step I % KS) reads register buffer I % 3.  Once its MMAs are committed and those
// of step I - 1 have completed, buffer (I - 1) % 3 = (I + 2) % 3 takes step I + 2: the registers of step I + 1 were
// loaded a whole step earlier, so their shared-memory latency is hidden behind the MMAs of two steps, not one.
template <int LAYER, int I>
__device__ __forceinline__ void gather_steps(float (&acc)[64], GatherRegs<LAYER>& gr, uint32_t (&x)[3][8], const unsigned char* s_data,
                                             uint64_t d0, int ft, int fr0, int qd, TcClocks& clk) {
  using namespace tc;
  constexpr int FLT = tc_spec(LAYER).FLT, KS = tc_spec(LAYER).ksteps(), NST = FLT * KS;
  constexpr int fl = I / KS, ks = I % KS;
  constexpr uint32_t kB1Plane = 16 * KS * 32 * 2;  // bytes of one B plane
  float(&d)[16] = *reinterpret_cast<float(*)[16]>(acc + 16 * fl);
  // B_{f & 1}, K-step ks (f & 1 = fl & 1: a tile starts on an even bin)
  const uint64_t bh = d0 + (uint64_t)(((fl & 1) * 2 * kB1Plane + ks * 2 * 32 * 16) >> 4), bl = bh + (kB1Plane >> 4);
  const uint32_t xh[4] = {x[I % 3][0], x[I % 3][1], x[I % 3][2], x[I % 3][3]};
  const uint32_t xl[4] = {x[I % 3][4], x[I % 3][5], x[I % 3][6], x[I % 3][7]};
  wgmma_fence();
  wgmma_rs_n32(d, xh, bh, ks ? 1u : 0u);
  wgmma_rs_n32(d, xh, bl, 1u);
  wgmma_rs_n32(d, xl, bh, 1u);
  wgmma_commit();
  if constexpr (I + 2 < NST) {
    wgmma_wait<1>();  // the previous step's MMAs are done: its A registers may be refilled
    clk.lap(kClkMma);
    // the window offsets follow the bin being LOADED (step I + 2); step I + 1's registers are already in place
    if constexpr ((I + 2) % KS == 0) gr.setup(FLT * ft + (I + 2) / KS, fr0, qd);
    gr.template load<(I + 2) % KS>(s_data, x[(I + 2) % 3]);
    clk.lap(kClkFull);
  }
  if constexpr (I + 1 < NST) gather_steps<LAYER, I + 1>(acc, gr, x, s_data, d0, ft, fr0, qd, clk);
}

template <int LAYER>
__device__ __forceinline__ void gather_conv1(float (&acc)[64], const unsigned char* s_data, uint32_t b1, int ft, int fr0, int qd,
                                             TcClocks& clk) {
  using namespace tc;
  static_assert(tc_spec(LAYER).ksteps() >= 2, "the first two K-steps are loaded up front, of the same bin");
  GatherRegs<LAYER> gr;
  const uint64_t d0 = make_desc(b1, 32 * 16, 128);
  uint32_t x[3][8];
  gr.setup(tc_spec(LAYER).FLT * ft, fr0, qd);
  gr.template load<0>(s_data, x[0]);
  gr.template load<1>(s_data, x[1]);
  clk.lap(kClkFull);
  gather_steps<LAYER, 0>(acc, gr, x, s_data, d0, ft, fr0, qd, clk);
  wgmma_wait<0>();
  reg_fence(acc);
  clk.lap(kClkMma);
}

// LAYER: 0 contour, 1 onset, 2 note; FUSED: the epilogue computes the next conv (always for onset / note; the unfused
// contour stores its channels-last activations)
template <int LAYER, bool FUSED>
__global__ void __launch_bounds__(tc::kThreads, 1) conv_tc_kernel(const __grid_constant__ TcArgs a) {
  using namespace tc;
  constexpr TcConvSpec L = tc_spec(LAYER);
  constexpr bool kFused = FUSED;
  constexpr bool kGather = LAYER != 0;  // onset / note: gathered conv1, no weight ring
  static_assert(kFused || !kGather, "the onset and note epilogues always fuse the next conv");
  constexpr int NW = L.width, PC = L.pass, PS = PC + 1;  // conv2 accumulator columns, staged per pass; staging row pitch
  static_assert(PC % 8 == 0 && PC % L.js == 0, "a staging pass holds whole fragment blocks and whole output offsets");
  constexpr int kDataRows = kMTile + L.KH - 1;
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr TcSmem SM = tc_smem(LAYER, FUSED);
  constexpr int kStages = SM.stages;
  static_assert(SM.total() <= kMaxSmem && kStages <= kMaxStages && (kGather || kStages >= 4), "dynamic shared memory per CTA");
  unsigned char* s_data = smem;                    // [2 planes][chunks][data_rows][16 B]
  unsigned char* s_w = smem + SM.data_bytes;       // contour: [kStages][8192]
  unsigned char* s_b1 = s_w + kStages * kTileBytes;  // onset / note: conv1 B matrices (tc_build_b1)
  unsigned char* s_b2 = s_b1 + SM.b1_bytes;          // conv2 weight matrix [plane 2][k-chunk 16][NW][16 B]
  float* s_p = reinterpret_cast<float*>(s_b2 + SM.b2_bytes);  // conv2 sums [slot 2][64 rows][PS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(s_p) + SM.p_bytes);
  uint64_t* full_w = bars;             // [kStages]
  uint64_t* empty_w = bars + kStages;  // [kStages] one arrival per consumer warp
  uint64_t* data_full = bars + 2 * kStages;
  uint64_t* data_empty = data_full + 1;  // one arrival per consumer warp
  uint64_t* b2_full = data_empty + 1;
  uint64_t* b1_full = b2_full + 1;
  uint32_t* issued = reinterpret_cast<uint32_t*>(b1_full + 1);  // weight fills the producer has issued so far

  // Broadcasting the warp index keeps the role branches and the producer loop state in uniform registers.
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  constexpr uint32_t lbo = kDataRows * 16u;
  constexpr uint32_t plane_bytes = (L.chunks8 - 1) * lbo;  // the tile holds chunks 0 .. chunks8 - 2

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_w + s, 1);
      mbar_init(empty_w + s, kConsumerWarps);
    }
    mbar_init(data_full, 1);
    mbar_init(data_empty, kConsumerWarps);
    mbar_init(b2_full, 1);
    mbar_init(b1_full, 1);
    *issued = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int n_items = a.sch.n_items();
  TcClocks clk;

  if (warp >= kConsumerWarps) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp != kProducerWarp) return;
    // ------------------------------ producer ------------------------------
    // The whole warp walks the loop with warp-uniform state; the arrive / copy instructions are predicated on the elected
    // lane (no elect loop and R2UR around every UBLKCP: the weight ring is paced by this loop's latency per step).
    // For a step that one slot does not use, the producer also arrives on the stage's empty_w for that slot's four warps,
    // so the two slots move through the ring independently (see the consumers).  The onset / note layers have no ring:
    // their producer copies the B matrices once and then only the data tile of every item.
    const uint32_t leader = elect_one() ? 1u : 0u;
    if constexpr (kFused) bulk_g2s_expect_pred(s_b2, a.b2, (uint32_t)SM.b2_bytes, b2_full, leader);
    if constexpr (kGather) bulk_g2s_expect_pred(s_b1, a.b1, (uint32_t)SM.b1_bytes, b1_full, leader);
    uint32_t stage = 0, ph_w = 0, ph_d = 0, n_fill = 0;
    const size_t plane_elems = (size_t)L.chunks8 * a.rows_total * 8;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
      int mt, g0, g1;
      a.sch.item(it, L.G0, mt, g0, g1);
      clk.lap(kClkProdOther);
      mbar_wait_wd(data_empty, ph_d ^ 1, 1);
      clk.lap(kClkDataEmpty);
      const size_t row = (size_t)mt * a.ms + a.row0;
      if (leader) {
        mbar_expect_tx(data_full, 2 * plane_bytes);
        if (a.use_tmap) {  // one tensor-map TMA for the whole (planes x chunks x rows x 8 elements) tile
          tma_load_4d(s_data, &a.data_map, 0, (int)row, 0, 0, data_full);
        } else {
          for (int p = 0; p < 2; ++p)
            for (int c = 0; c < a.chunks8 - 1; ++c)
              bulk_g2s(s_data + p * plane_bytes + c * lbo, a.data + p * plane_elems + ((size_t)c * a.rows_total + row) * 8,
                       lbo, data_full);
        }
      }
      __syncwarp();
      ph_d ^= 1;
      if constexpr (kGather) continue;
      const int s0 = c_group_step_off[g0], s1 = c_group_step_off[g1];
      int tile = c_tile_seq[s0];
      for (int s = s0; s < s1; ++s) {
        const int tile_next = c_tile_seq[s + 1];  // (one past the end is inside the array)
        clk.lap(kClkProdOther);
        mbar_wait_wd(empty_w + stage, ph_w ^ 1, 2);
        clk.lap(kClkEmpty);
        bulk_g2s_expect_pred(s_w + stage * kTileBytes, a.tiles + (size_t)tile * (kTileBytes / 2), kTileBytes, full_w + stage,
                             leader);
        // every step has at least one user, so at most one slot skips it
        const bool skip = c_prog[0][s] == kNoUse || c_prog[1][s] == kNoUse;
        mbar_arrive_cnt_pred(empty_w + stage, kConsumerWarps / 2, skip ? leader : 0u);
        counter_publish(issued, ++n_fill);
        if (++stage == kStages) {
          stage = 0;
          ph_w ^= 1;
        }
        tile = tile_next;
      }
    }
    clk.lap(kClkProdOther);
    clk.flush(LAYER);
  } else {
    setmaxnreg_inc<kConsumerRegs>();
    // ------------------------------ consumers: one warpgroup per accumulator slot ------------------------------
    // conv1: the slot's frequency tile of the 64-row M-tile as m64n128k16 MMAs, accumulators in registers.  Fragment of a
    // thread (warp w of the group, lane = 4 gq + qd): rows 16 w + gq and 16 w + gq + 8, columns 8 i + 2 qd + {0, 1}.
    const int slot = warp >> 2, wq = warp & 3, gq = lane >> 2, qd = lane & 3;
    const int tid = threadIdx.x & 127;
    const int fr0 = 16 * wq + gq;  // first of the thread's two fragment rows (the other is fr0 + 8)
    uint32_t stage = 0, ph_w = 0, ph_d = 0, n_fill = 0;  // n_fill: index of the current step's weight fill in the CTA
    const uint32_t a_hi = smem_u32(s_data), a_lo = a_hi + plane_bytes, w_base = smem_u32(s_w);
    const uint32_t* prog = c_prog[slot];
    float* sp_rows = s_p + slot * 64 * PS;
    if constexpr (kFused) mbar_wait_wd(b2_full, 0, 6);
    if constexpr (kGather) mbar_wait_wd(b1_full, 0, 7);
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
      int mt, g0, g1;
      a.sch.item(it, L.G0, mt, g0, g1);
      // conv1 rows of the thread's fragment (relu(conv1) of a row that is not a live frame is the zero padding in time)
      bool live[2];
      int rb[2], rt[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = mt * a.ms - a.h2 + fr0 + 8 * rr;  // row of the (window, frame) space: m = b * rows_per_window + t
        rb[rr] = m >= 0 ? m / L.rows_per_window : 0;
        rt[rr] = m - rb[rr] * L.rows_per_window;
        live[rr] = m >= 0 && (rb[rr] < a.n_windows) && (rt[rr] < kFrames);
      }
      // Fused layers: threads 0..63 of the group each finish the output frame of one tile row, h2 rows earlier than the
      // conv1 row (all time taps of the fused conv2 then lie at or below the row); rows < 2 h2 are finished by the
      // previous M-tile
      RowOut ro{};
      float carry[4] = {0.f, 0.f, 0.f, 0.f};
      float hold[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if constexpr (kFused) {
        const int row = tid;
        const int q = mt * a.ms - 2 * a.h2 + row;
        const int b = q >= 0 ? q / L.rows_per_window : 0, t = q - b * L.rows_per_window;
        ro.ok = row < 64 && row >= 2 * a.h2 && q >= 0 && b < a.n_windows && t < kFrames;
        ro.t = t;
        if (ro.ok) {
          ro.edge = a.o.edge + q;
          int uf = -1;  // unwrapped frame (reference: inference.py:247-279), if this frame is kept
          if (a.o.ud) {
            const UnwrapDesc u = a.o.ud[b];
            const int tt = t - kOverlapHalf;
            if ((unsigned)tt < (unsigned)max(u.rows, 0)) uf = (int)(u.dst_base + tt);
          }
          if constexpr (LAYER == 0) {
            ro.chl = a.o.chl + ((size_t)a.o.chl_lead + (size_t)b * a.o.chl_rpw + t) * 8;
            if (a.o.raw) ro.raw = a.o.raw + ((size_t)b * kFrames + t) * 8;
            if (uf >= 0) ro.unw = a.o.unwrapped + (size_t)uf * 8;
          } else {
            if (a.o.raw) ro.raw = a.o.raw + (size_t)b * kFrames + t;
            if (uf >= 0) ro.unw = a.o.unwrapped + uf;
            if constexpr (LAYER == 1) ro.note_col = a.o.note_raw + (size_t)b * kFrames + t;
          }
        }
      }
      clk.lap(kClkConsOther);
      mbar_wait_wd(data_full, ph_d, 3);
      clk.lap(kClkData);
      ph_d ^= 1;
      for (int g = g0; g < g1; ++g) {
        float acc[64];
        const int ft = tc_group_tile(L, g, slot);
        if constexpr (kGather) {
          if (ft >= 0) gather_conv1<LAYER>(acc, s_data, smem_u32(s_b1), ft, fr0, qd, clk);
        } else {
          const int s0 = c_group_step_off[g], s1 = c_group_step_off[g + 1];
          int pend = -1;  // stage read by the MMA group still in flight
          uint32_t pend_fill = 0;  // and its fill index
          uint32_t w = prog[s0];
          // A slot skips the steps it does not use (kNoUse) completely: no wait on full_w, no arrival on empty_w (the
          // producer arrives for it).  So it does not see every phase of a stage, and its parity wait for fill f (the
          // stage's phase f / kStages) is only exact if the stage is at most one phase off when it waits:
          //   * not ahead: it first waits until the producer has ISSUED fill f.  That happened after the release of fill
          //     f - kStages, whose user(s) waited for it to land, so the previous phase is complete;
          //   * not behind: fill f + kStages cannot land before this slot's own arrival for fill f gates the refill.
          for (int s = s0; s < s1; ++s, ++n_fill) {
            const uint32_t w_next = prog[s + 1];  // (one word past the end is inside the array)
            if (w != kNoUse) {
              if (pend >= 0 && n_fill - pend_fill >= kStages) {
                // fill f is issued after the release of fill f - kStages, which may be the stage still held
                wgmma_wait<0>();
                if (lane == 0) mbar_arrive(empty_w + pend);
                pend = -1;
              }
              clk.lap(kClkConsOther);
              counter_wait_above(issued, n_fill);
              mbar_wait_wd(full_w + stage, ph_w, 5);
              clk.lap(kClkFull);
              const uint32_t off = (w & 0x3fffu) << 4;  // chunk c8, row dt of the data tile
              const uint32_t bw = w_base + stage * kTileBytes;
              const uint64_t dah = make_desc(a_hi + off, lbo, 128), dal = make_desc(a_lo + off, lbo, 128);
              const uint64_t dbh = make_desc(bw, 2048, 128), dbl = make_desc(bw + 4096, 2048, 128);
              wgmma_fence();
              wgmma_ss_n128(acc, dah, dbh, (w & kUseFirstAcc) ? 0u : 1u);
              wgmma_ss_n128(acc, dah, dbl, 1u);
              wgmma_ss_n128(acc, dal, dbh, 1u);
              wgmma_commit();
              wgmma_wait<1>();  // the previous step's MMAs are done: its weight stage may be refilled
              if (pend >= 0 && lane == 0) mbar_arrive(empty_w + pend);
              pend = (int)stage;
              pend_fill = n_fill;
              clk.lap(kClkMma);
            }
            if (++stage == kStages) {
              stage = 0;
              ph_w ^= 1;
            }
            w = w_next;
          }
          clk.lap(kClkConsOther);
          wgmma_wait<0>();
          reg_fence(acc);
          clk.lap(kClkMma);
          if (pend >= 0 && lane == 0) mbar_arrive(empty_w + pend);
        }
        if (g == g1 - 1 && lane == 0) mbar_arrive(data_empty);  // this warp no longer reads the data tile
        if (ft < 0) continue;
        // first / last tile of this slot's ascending range inside the item
        const bool first = tc_starts_range(L, g, slot, g == g0);
        const bool last = tc_ends_range(L, g, slot, g == g1 - 1);
        const int n_valid = min(L.FLT, L.WOUT - ft * L.FLT) * L.COUT;  // a multiple of 32 (contour: 64 in the last tile)
        // conv1 bias of the thread's accumulator columns: channel of column 8 i + 2 qd + e is (8 i + 2 qd + e) % COUT.
        // Read here, after the conv1 MMAs, so that it holds no registers during the gather.
        float bz[4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int e = 0; e < 2; ++e) bz[i][e] = a.bias1[(8 * i + 2 * qd + e) % L.COUT];
        if constexpr (!kFused) {
          // contour: 16 bins x 8 channels, bias + ReLU, channels-last rows of 128 contiguous floats
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            if (!live[rr]) continue;
            float* dst = a.o.act + ((size_t)rb[rr] * kFrames + rt[rr]) * ((size_t)L.WOUT * L.COUT) + (size_t)ft * 128;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int col = 8 * i + 2 * qd;
              if (col < n_valid)
                *reinterpret_cast<float2*>(dst + col) = make_float2(fmaxf(acc[4 * i + 2 * rr] + bz[i & 3][0], 0.f),
                                                                    fmaxf(acc[4 * i + 2 * rr + 1] + bz[i & 3][1], 0.f));
            }
          }
        } else {
          // relu(conv1 + bias) -> bf16 hi / lo A fragments of the conv2 MMAs.  The conv1 accumulator fragment is the A
          // register layout of a K = 16 step (registers: rows gq / gq + 8 x columns 2 qd / 8 + 2 qd of the step), so
          // columns 16 ks .. 16 ks + 15 form step ks: register 4 ks + 2 (i & 1) + rr holds accumulator block i = 2 ks + (i & 1)
          uint32_t ah[32], al[32];
#pragma unroll
          for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const bool ok = live[rr] && 8 * i < n_valid;
              const float o0 = ok ? fmaxf(acc[4 * i + 2 * rr] + bz[i & 3][0], 0.f) : 0.f;
              const float o1 = ok ? fmaxf(acc[4 * i + 2 * rr + 1] + bz[i & 3][1], 0.f) : 0.f;
              const __nv_bfloat162 hh = __floats2bfloat162_rn(o0, o1);
              const uint32_t hu = *reinterpret_cast<const uint32_t*>(&hh);
              const __nv_bfloat162 ll =
                  __floats2bfloat162_rn(o0 - __uint_as_float(hu << 16), o1 - __uint_as_float(hu & 0xffff0000u));
              const int r = 4 * (i >> 1) + 2 * (i & 1) + rr;
              ah[r] = hu;
              al[r] = *reinterpret_cast<const uint32_t*>(&ll);
            }
          // P[row][j * JS + dt] = sum over channels and frequency taps for output offset j and time tap dt
          float p[NW / 2];
          wgmma_fence();
          conv2_mma<NW>(p, ah, al, smem_u32(s_b2));
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(p);
          // time taps: the frame of tile row r takes P_dt from row r - (KH2 - 1 - dt), taps added from the own row down
          // (the same order for every row: a frame's value does not depend on where the M-tile starts).  The sums go
          // through the staging area PC columns (PC / JS output offsets j) at a time.
          constexpr int KH2 = L.KH2, JS = L.js, JP = PC / JS;
          constexpr int NJ = L.FLT + 2 * L.HALO;  // output bins whose sums the tile holds
          float S[NJ];
#pragma unroll
          for (int q = 0; q * JP < NJ; ++q) {
            slot_barrier(slot);  // the previous pass's (or tile's) sums have been read
#pragma unroll
            for (int i = 0; i < NW / 8; ++i) {
              if (8 * i < q * PC || 8 * i >= (q + 1) * PC) continue;
#pragma unroll
              for (int rr = 0; rr < 2; ++rr) {
                float* d = sp_rows + (fr0 + 8 * rr) * PS + 8 * i - q * PC + 2 * qd;
                d[0] = p[4 * i + 2 * rr];
                d[1] = p[4 * i + 2 * rr + 1];
              }
            }
            slot_barrier(slot);
            if (tid < 64) {
#pragma unroll
              for (int j = q * JP; j < NJ && j < (q + 1) * JP; ++j) {
                float s = 0.f;
#pragma unroll
                for (int ta = 0; ta < KH2; ++ta)
                  if (tid - ta >= 0) s += sp_rows[(tid - ta) * PS + j * JS - q * PC + (KH2 - 1 - ta)];
                S[j] = s;
              }
            }
          }
          if (tid < 64) {
            if constexpr (LAYER == 0) {
              finish_contour_tile(a, ro, S, ft, first, last, carry, hold);
            } else {
              float c2[2] = {carry[0], carry[1]};
              finish_pitch_tile<LAYER>(a, ro, S, c2, ft, first, last);
              carry[0] = c2[0];
              carry[1] = c2[1];
            }
          }
        }
        clk.lap(kClkEpi);
      }
    }
    clk.lap(kClkConsOther);
    clk.flush(LAYER);
    clk.cta_end(LAYER);
  }
}


// ------------------------------------------------------------------------------------------------
// Where two tile ranges meet (boundary ft_b: tile ft_b starts a range in the items of an M-tile, see tc_starts_range)
// the 2 * HALO bins FLT * ft_b - HALO + k got one partial sum from each side: finish them here.  Pitch layers: 2 bins
// per frame.  Contour: 4 bins, and with the six finished bins each side left next to them the two 8-bin chunks around
// the boundary.
// ------------------------------------------------------------------------------------------------
struct EdgeFixArgs {
  TcOut o;
  int edge_rows, n_rows;        // rows of the (window, frame) space covered by the M-tiles
  // bit b: boundary b goes through the edge buffer (tc_edge_mask) in the rows finished by a whole M-tile (rows below
  // tail_row0) and by a tail M-tile (the rows from tail_row0 on)
  uint32_t edges_full, edges_tail;
  int tail_row0;
  int n_windows;
  float bias2, note_w[9];  // the layer's conv2 bias; onset: the conv2 weights of the note input channel
};

static_assert(tc_spec(0).n_ft() <= 32 && tc_spec(1).n_ft() <= 32 && tc_spec(2).n_ft() <= 32, "boundary mask");
static_assert(tc_edge_mask(tc_spec(0), 1u) == 0x1fffeu && tc_edge_mask(tc_spec(1), 1u) == 1u << 12 &&
                  tc_edge_mask(tc_spec(2), 1u) == 1u << 12,
              "whole M-tiles: contour: every tile a range of its own; onset / note: the slot boundary only");

// contour: one thread per frame; pitch layers: per (frame, bin); each fixes the boundaries of the mask
template <int LAYER>
constexpr int kEdgeThreads = LAYER == 0 ? 1 : 2 * tc_spec(LAYER).HALO;

template <int LAYER>
__device__ __forceinline__ void edge_fix_boundary(const EdgeFixArgs& a, int ft_b, int R, int b, int t, int uf, int k) {
  constexpr TcConvSpec L = tc_spec(LAYER);
  const int e = ft_b - 1;  // edge slot of the boundary
  if constexpr (LAYER == 0) {
    const float* lo = a.o.edge + (size_t)(e * 2 + 0) * L.edge_per_side() * a.edge_rows + R;  // from the range that starts at ft_b
    const float* hi = a.o.edge + (size_t)(e * 2 + 1) * L.edge_per_side() * a.edge_rows + R;  // from the range that ends at ft_b - 1
    float fx[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)  // (S + carry) + bias, the order of the in-kernel carry
      fx[q] = sigmoidf_fast((lo[(size_t)q * a.edge_rows] + hi[(size_t)q * a.edge_rows]) + a.bias2);
    float va[8], vb[8];
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      va[q] = hi[(size_t)(4 + q) * a.edge_rows];      // bins 16 ft_b - 8 .. - 3
      vb[2 + q] = lo[(size_t)(4 + q) * a.edge_rows];  // bins 16 ft_b + 2 .. + 7
    }
    va[6] = fx[0], va[7] = fx[1], vb[0] = fx[2], vb[1] = fx[3];
    __nv_bfloat16* chl = a.o.chl + ((size_t)a.o.chl_lead + (size_t)b * a.o.chl_rpw + t) * 8;
    const size_t plane = (size_t)a.o.chl_chunks * a.o.chl_rows * 8;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int chunk = 2 * ft_b - 1 + c;
      const float(&v)[8] = c ? vb : va;
      store_split8(v, chl, (size_t)chunk * a.o.chl_rows * 8, plane);
      const float4 x0 = make_float4(v[0], v[1], v[2], v[3]), x1 = make_float4(v[4], v[5], v[6], v[7]);
      if (a.o.raw) {
        float4* d = reinterpret_cast<float4*>(a.o.raw + ((size_t)chunk * a.o.raw_rows + (size_t)b * kFrames + t) * 8);
        d[0] = x0, d[1] = x1;
      }
      if (uf >= 0) {
        float4* d = reinterpret_cast<float4*>(a.o.unwrapped + ((size_t)chunk * a.o.frame_stride + uf) * 8);
        d[0] = x0, d[1] = x1;
      }
    }
    return;
  }
  const int f = L.FLT * ft_b - L.HALO + k;
  if (f < 0 || f >= L.WOUT) return;
  float x = (a.o.edge[((size_t)(e * 2 + 0) * L.edge_per_side() + k) * a.edge_rows + R] +
             a.o.edge[((size_t)(e * 2 + 1) * L.edge_per_side() + k) * a.edge_rows + R]) + a.bias2;  // (S + carry) + bias
  if (a.o.note_raw) {
#pragma unroll
    for (int dt = 0; dt < 3; ++dt)
#pragma unroll
      for (int df = 0; df < 3; ++df) {
        const int tt = t + dt - 1, ff = f + df - 1;
        if ((unsigned)tt < (unsigned)kFrames && (unsigned)ff < (unsigned)kPitches)
          x = fmaf(__ldg(a.o.note_raw + (size_t)ff * a.o.raw_rows + (size_t)b * kFrames + tt), a.note_w[dt * 3 + df], x);
      }
  }
  const float v = sigmoidf_fast(x);
  if (a.o.raw) a.o.raw[(size_t)f * a.o.raw_rows + (size_t)b * kFrames + t] = v;
  if (uf >= 0) a.o.unwrapped[(size_t)f * a.o.frame_stride + uf] = v;
}

template <int LAYER>
__global__ void edge_fix_kernel(const EdgeFixArgs a) {
  constexpr TcConvSpec L = tc_spec(LAYER);
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)a.n_rows * kEdgeThreads<LAYER>) return;
  const int R = (int)(idx % a.n_rows);  // rows fastest: coalesced reads of the edge buffer, coalesced stores
  const int k = (int)(idx / a.n_rows);
  const int b = R / L.rows_per_window, t = R - b * L.rows_per_window;
  if (b >= a.n_windows || t >= kFrames) return;
  int uf = -1;
  if (a.o.ud) {
    const UnwrapDesc u = a.o.ud[b];
    const int tt = t - kOverlapHalf;
    if ((unsigned)tt < (unsigned)max(u.rows, 0)) uf = (int)(u.dst_base + tt);
  }
  // the mask of the M-tile that finishes row R (tc_schedule: whole M-tiles first, then the tail)
  for (uint32_t m = R < a.tail_row0 ? a.edges_full : a.edges_tail; m; m &= m - 1)
    edge_fix_boundary<LAYER>(a, __ffs(m) - 1, R, b, t, uf, k);
}
// ------------------------------------------------------------------------------------------------
int tc_rows_total(int n_windows, int rows_per_window) {
  // lead rows + the rows of the windows + what the last (overlapping) M-tile and its time taps may touch
  return n_windows * rows_per_window + tc::kMTile + 16;
}

int tc_setup() {
  using namespace tc;
  cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem(0, false).total());
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_tc_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem(1, true).total());
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_tc_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem(2, true).total());
  if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_tc_kernel<0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem(0, true).total());
  return e == cudaSuccess ? 0 : -1;
}

void launch_lognorm_split(const float* y, const unsigned int* minmax, const float* bn, __nv_bfloat16* dst,
                          const TcConvSpec& sp, int n_windows, int rows_stride, cudaStream_t st) {
  const int rows_used = tc_rows_total(n_windows, sp.rows_per_window);  // <= rows_stride
  const long long cells = (long long)rows_used * (sp.chunks8 / 2);  // a thread converts two chunks of a row
  lognorm_split_kernel<<<(unsigned)((cells + 255) / 256), 256, 0, st>>>(y, minmax, bn, dst, n_windows, rows_used, rows_stride,
                                                                       sp.chunks8, sp.rows_per_window, sp.lead_rows);
}

size_t tc_edge_floats(const TcConvSpec& sp, int n_windows) {
  const int ms = tc::kMTile - (sp.KH2 - 1);
  const int n_mtiles = (n_windows * sp.rows_per_window + ms - 1) / ms;
  return (size_t)(sp.n_ft() - 1) * 2 * sp.edge_per_side() * ((size_t)n_mtiles * ms);  // one slot per tile boundary
}

// ------------------------------------------------------------------------------------------------
// The items of a launch.  Cutting every M-tile into k equal runs of groups, the item order (it / k, it % k) pinned every
// CTA to one run when k divides the grid (132 = 2 x 2 x 3 x 11), and the runs are not equal work: the launch waited for
// the CTAs of the heaviest run.  Instead the first n_full = floor(n_mtiles / grid) x grid M-tiles run whole, the same
// number per CTA, and only the n_tail < grid M-tiles after them (all of a small batch) are cut, into the number of
// group ranges, with boundaries of balanced estimated cost, that gives the least estimated time of the busiest CTA.
// Cost of a group, contour: its MMA uses (the slot programs' words) plus kEpiUses per tile for the epilogue; onset /
// note: its tiles (every tile of a pitch layer is the same gather).  Per item the data-tile load adds kItemUsesContour /
// kItemTilesPitch.
// The weights follow the cycle accounting of the contour kernel (DESIGN 4.1): the epilogue takes about as many
// consumer cycles as 14 MMA uses per tile, the data-tile wait about 20 per item; the ring steps are not counted on
// their own, since the consumers set the pace (the producer waits for a free stage most of its time).
// ------------------------------------------------------------------------------------------------
namespace tc {
constexpr double kEpiUses = 14.0, kItemUsesContour = 20.0, kItemTilesPitch = 0.25;
}
// per-group cost and per-item cost of a layer, in the units above
static void tc_group_costs(int layer, std::vector<double>& cost, double& item) {
  using namespace tc;
  const TcConvSpec sp = tc_spec(layer);
  cost.assign(sp.G0, 0.0);
  for (int g = 0; g < sp.G0; ++g)
    for (int sl = 0; sl < 2; ++sl) cost[g] += tc_group_tile(sp, g, sl) >= 0 ? (layer == 0 ? kEpiUses : 1.0) : 0.0;
  item = layer == 0 ? kItemUsesContour : kItemTilesPitch;
  if (layer != 0) return;
  // the contour program depends on the geometry alone (TcConvPlan::build): plan it once, with any weights
  static const std::vector<double> uses = [] {
    const TcConvSpec s = tc_spec(0);
    std::vector<float> w((size_t)s.COUT * s.n_ci * s.KH * s.KW, 0.f);
    TcConvPlan pl;
    pl.build(s, w.data());
    std::vector<double> u(s.G0, 0.0);
    for (int g = 0; g < s.G0; ++g)
      for (int st = pl.group_step_off[g]; st < pl.group_step_off[g + 1]; ++st)
        for (int sl = 0; sl < 2; ++sl) u[g] += pl.slot_words[sl][st] != kNoUse ? 1.0 : 0.0;
    return u;
  }();
  for (int g = 0; g < sp.G0; ++g) cost[g] += uses[g];
}

TcSchedule tc_schedule(int layer, bool fused, int n_windows, int n_sms, int* ms_out) {
  const TcConvSpec sp = tc_spec(layer);
  const int h2 = fused || layer != 0 ? (sp.KH2 - 1) / 2 : 0;
  const int ms = tc::kMTile - 2 * h2;
  if (ms_out) *ms_out = ms;
  std::vector<double> cost;
  double item;
  tc_group_costs(layer, cost, item);
  const int G = sp.G0;
  std::vector<double> pre(G + 1, 0.0);
  for (int g = 0; g < G; ++g) pre[g + 1] = pre[g] + cost[g];
  TcSchedule s{};
  s.n_mtiles = (n_windows * sp.rows_per_window + ms - 1) / ms;
  s.n_full = s.n_mtiles / n_sms * n_sms;
  s.n_tail = s.n_mtiles - s.n_full;
  s.n_ranges = 1;
  s.bounds[0] = 0, s.bounds[1] = (unsigned char)G;
  if (s.n_tail > 0) {
    // best[r][g]: the least largest range cost of the groups [g, G) cut into r ranges, cut[r][g] its first range's end
    std::vector<std::vector<double>> best(G + 1, std::vector<double>(G + 1, 1e300));
    std::vector<std::vector<int>> cut(G + 1, std::vector<int>(G + 1, G));
    for (int g = 0; g < G; ++g) best[1][g] = pre[G] - pre[g];
    for (int r = 2; r <= G; ++r)
      for (int g = 0; g + r <= G; ++g)
        for (int e = g + 1; e + r - 1 <= G; ++e) {
          const double v = std::max(pre[e] - pre[g], best[r - 1][e]);
          if (v < best[r][g]) best[r][g] = v, cut[r][g] = e;
        }
    // every CTA runs n_full / grid whole M-tiles; the tail items j = c, c + grid, ... of CTA c decide the busiest one
    double best_t = 1e300;
    for (int r = 1; r <= G; ++r) {
      unsigned char b[16];
      b[0] = 0;
      for (int q = 0; q < r; ++q) b[q + 1] = (unsigned char)(q + 1 < r ? cut[r - q][b[q]] : G);
      const int n_items = s.n_tail * r, grid = s.n_full ? n_sms : std::min(n_items, n_sms);
      double worst = 0.0;
      for (int c = 0; c < grid && c < n_items; ++c) {
        double t = 0.0;
        for (int j = c; j < n_items; j += grid) t += pre[b[j / s.n_tail + 1]] - pre[b[j / s.n_tail]] + item;
        worst = std::max(worst, t);
      }
      if (worst < best_t * (1.0 - 1e-9)) {  // (a tie: fewer ranges, fewer items and edges)
        best_t = worst;
        s.n_ranges = r;
        std::copy_n(b, r + 1, s.bounds);
      }
    }
  }
  s.grid = std::min(s.n_items(), n_sms);
  return s;
}

// The conv kernel of one layer and, for a fused epilogue, the fix-up of the bins where two tile ranges meet.
template <int LAYER, bool FUSED>
static void launch_layer(const TcArgs& a, const EdgeFixArgs& ef, int grid, cudaStream_t st) {
  conv_tc_kernel<LAYER, FUSED><<<grid, tc::kThreads, tc::tc_smem(LAYER, FUSED).total(), st>>>(a);
  if (FUSED) {
    const long long total = (long long)ef.n_rows * kEdgeThreads<LAYER>;
    edge_fix_kernel<LAYER><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ef);
  }
}

void launch_conv_tc(const __nv_bfloat16* data, const TcConvDev& dev, const TcOut& o, int n_windows, int rows_stride,
                    int n_sms, cudaStream_t st, bool fuse_next) {
  const TcConvSpec sp = tc_spec(dev.layer);
  const bool fused = dev.layer != 0 || fuse_next;
  TcArgs a{};
  a.data = data;
  a.tiles = dev.tiles;
  a.b1 = dev.b1;
  a.b2 = dev.b2;
  a.o = o;
  a.rows_total = rows_stride;  // row stride of the split layout (fixed per model, independent of the batch)
  a.h2 = fused ? (sp.KH2 - 1) / 2 : 0;
  // An item is (M-tile, range of frequency groups): whole M-tiles, the same number per CTA, then the last M-tiles cut
  // into group ranges of balanced cost (tc_schedule)
  a.sch = tc_schedule(dev.layer, fused, n_windows, n_sms, &a.ms);
  a.edge_rows = a.sch.n_mtiles * a.ms;
  a.n_windows = n_windows;
  a.row0 = sp.lead_rows - sp.PT - a.h2;
  a.chunks8 = sp.chunks8;
  std::copy_n(dev.bias1, 32, a.bias1);
  a.bias2 = dev.bias2;
  std::copy_n(dev.note_w, 9, a.note_w);
  const int grid = a.sch.grid;
  {
    // tensor map of the split input: dims (innermost first) 8 elements, rows, 8-bin chunks, hi / lo plane
    using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn encode = [] {
      void* fn = nullptr;
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
          q != cudaDriverEntryPointSuccess)
        fn = nullptr;
      return reinterpret_cast<EncodeFn>(fn);
    }();
    // The data tile can be fetched by ONE tensor-map TMA (cp.async.bulk.tensor.4d -> UTMALDG) or by 1-D bulk copies (one
    // per plane and chunk).  The tensor map's innermost box dimension is only 16 bytes, and one box is walked by one TMA
    // pipeline while the bulk copies proceed in parallel (splitting the box is not possible: a chunk is 66 rows x 16 B =
    // 1 056 B, not a multiple of the 128-byte shared-memory alignment a box needs).  Default = bulk copies;
    // BP_B200_TMAP=1 selects the tensor map (GPU-tested).
    a.use_tmap = 0;
    static const bool want_tmap = getenv("BP_B200_TMAP") != nullptr;
    if (encode && want_tmap) {
      const cuuint64_t dims[4] = {8, (cuuint64_t)rows_stride, (cuuint64_t)sp.chunks8, 2};
      const cuuint64_t strides[3] = {16, (cuuint64_t)rows_stride * 16, (cuuint64_t)sp.chunks8 * rows_stride * 16};
      const cuuint32_t box[4] = {8, (cuuint32_t)(tc::kMTile + sp.KH - 1), (cuuint32_t)(sp.chunks8 - 1), 2};
      const cuuint32_t estr[4] = {1, 1, 1, 1};
      if (encode(&a.data_map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<__nv_bfloat16*>(data), dims, strides, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS)
        a.use_tmap = 1;
    }
  }
  EdgeFixArgs ef{};
  ef.o = o;
  ef.edge_rows = a.edge_rows;
  ef.n_rows = n_windows * sp.rows_per_window;
  ef.edges_full = tc_edge_mask(sp, 1u);  // the conv kernel's own range predicate
  ef.edges_tail = tc_edge_mask(sp, a.sch.tail_starts());
  ef.tail_row0 = a.sch.n_full * a.ms;
  ef.n_windows = n_windows;
  ef.bias2 = dev.bias2;
  std::copy_n(dev.note_w, 9, ef.note_w);
  if (dev.layer == 1)
    launch_layer<1, true>(a, ef, grid, st);
  else if (dev.layer == 2)
    launch_layer<2, true>(a, ef, grid, st);
  else if (fuse_next)
    launch_layer<0, true>(a, ef, grid, st);
  else
    launch_layer<0, false>(a, ef, grid, st);
}

}  // namespace bp