// Constant-Q projection on the tensor cores: per octave the 172 x 256 x 72 contraction
//   C[(b,t)][n] = sum_k xpad_o[b][t*hop_o + k] * W[k][n]          (n interleaves real / imaginary parts of 36 bins)
// as warpgroup MMAs (wgmma, bf16 operands, FP32 accumulators in registers) on a three-way bf16 split of both operands
// (x = hi + mid + lo, each round-to-nearest bf16; the six products hi*hi, hi*mid, mid*hi, hi*lo, lo*hi, mid*mid are
// accumulated in FP32; the dropped terms are below 2^-24 of |a||w|).  A single bf16 / TF32 product is far from the 1e-3
// bar for this stage and even a two-way split leaves ~1e-3 in the weak bins of the log spectrum (SURVEY.md F6 / Appendix
// C.4); the three-way split reproduces FP32-class results.
//
// Replaces (together with the unchanged decimation chain) reference: basic_pitch/layers/nnaudio.py:216-256
// (`get_cqt_complex`, reflect pad + two strided conv1d per octave), :642-661 (concat, sqrt(len) scaling, magnitude) and
// layers/signal.py:174-176 (power -> 10*log10(. + 1e-10)); the per-window min / max feed lognorm_kernel (hcqt.cu).
//
// The A operand is an overlapping strided view of the signal (row t starts at sample t*hop), which no wgmma/TMA
// descriptor can express for hop*4 B < 16 B or non-canonical pitches, so it is staged explicitly ("im2col" into the
// canonical K-major core-matrix layout) by producer warps that also do the reflect padding and the three-way split.
//
// item = (M-tile of 128 frames, octave); per item 4 K-chunks of 64 taps, each chunk = 4 k-steps x 6 products:
//   warps 8-23  producers: gather 128 x 64 samples (128-bit loads where aligned), split, st.shared into
//               [plane][k/8][row][8] ; one lane bulk-copies the matching 30 KB slice of the split kernel matrix W
//               (UBLKCP) ; fence.proxy.async ; mbarrier arrive
//   warps 0-7   two consumer warpgroups, frames 0..63 / 64..127 of the M-tile: 24 wgmma m64n80k16 per chunk (the
//               stage is released when they completed), then the epilogue straight from the accumulator registers:
//               magnitude * sqrt(len), log-power, store, per-window min/max (atomics)
// Shared memory: 2 stages x (48 KB A + 30 KB W), the epilogue's staging tiles and the producers' staging rows.
#include <cuda_bf16.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "kernels.cuh"
#include "tc_ptx.cuh"

namespace bp {

namespace cq {
constexpr int kMTile = 128;
constexpr int kKc = 64;                          // taps per chunk
constexpr int kN = 80;                           // 72 columns padded to a multiple of 16
constexpr int kAPlane = (kKc / 8) * kMTile * 16;  // 16384 B : [8 k-chunks of 8][128 rows][16 B]
constexpr int kWPlane = (kKc / 8) * kN * 16;      // 10240 B : [8][80][16 B]
constexpr int kStageBytes = 3 * kAPlane + 3 * kWPlane;  // 79872
constexpr int kStages = 2;
constexpr int kRowsPerWarp = 8;   // rows of the M-tile a producer warp gathers and converts
constexpr int kProducers = 32 * kMTile / kRowsPerWarp;  // 16 producer warps (more warps in flight hide the gather latency)
constexpr int kEpiWarps = 8;                      // two consumer warpgroups (MMAs + epilogue)
constexpr int kThreads = kProducers + 32 * kEpiWarps;
constexpr int kTilePitch = 37;                    // epilogue staging: [8 warps][16 rows][36 bins + 1]
constexpr int kStgPitch = 68;                     // producer staging: [128 rows][64 taps + 4] fp32
constexpr int kSegOctave = 3;                     // octaves >= this (hop <= 32) stage their signal segment once per item
constexpr int kSegPlane = (kMTile * kStgPitch * 4 / (3 * 2)) & ~7;  // bf16 elements per plane of the segment (5800)
static_assert(kSegPlane >= 126 * 32 + 2 * kTaps + 32, "segment of the hop-32 octave");
constexpr int kEpiBytes = kEpiWarps * 16 * kTilePitch * 4;
constexpr int kSmemBytes = kStages * kStageBytes + 256 + kEpiBytes + kMTile * kStgPitch * 4 + kMTile * 24;
static_assert(kThreads <= 1024 && kRowsPerWarp % 2 == 0 && (kKc * kRowsPerWarp / 32) % 8 == 0, "producer geometry");
static_assert(kSmemBytes <= 232448, "shared memory per CTA");
}  // namespace cq

static inline uint16_t f2bf_rn(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static inline float bf2f_(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// kernel matrix, three-way bf16 split, laid out per chunk: wtc[chunk 4][plane 3][k/8 8][n 80][8] (bf16)
void build_cqt_tc_weights(const float* cqt_real /* [36][256] */, const float* cqt_imag, std::vector<uint16_t>& out) {
  out.assign((size_t)4 * 3 * 8 * cq::kN * 8, 0);
  for (int k = 0; k < kTaps; ++k)
    for (int n = 0; n < 72; ++n) {
      const float w = (n & 1) ? cqt_imag[(n >> 1) * kTaps + k] : cqt_real[(n >> 1) * kTaps + k];
      const uint16_t h = f2bf_rn(w);
      const float r1 = w - bf2f_(h);
      const uint16_t m = f2bf_rn(r1);
      const uint16_t l = f2bf_rn(r1 - bf2f_(m));
      const int c = k / cq::kKc, kk = k % cq::kKc;
      const size_t plane = (size_t)8 * cq::kN * 8;
      const size_t base = (size_t)c * 3 * plane;
      const size_t off = ((size_t)(kk >> 3) * cq::kN + n) * 8 + (kk & 7);
      out[base + off] = h;
      out[base + plane + off] = m;
      out[base + 2 * plane + off] = l;
    }
}

struct RowP {  // where one frame row of the current item reads its signal (producer scratch in shared memory)
  const float* src;
  int i0, lo, hi, live;
};

struct CqtTcArgs {
  const float* audio;
  const WinDesc* desc;   // may be null: window b = audio + b*43844
  const float* chain;    // decimated signals x_1..x_8
  const uint16_t* wtc;   // split kernel matrix (bf16), 4 chunks of 30 KB
  const float* scale;    // [309] sqrt(kernel length)
  float* logmag;         // [B][172][309]
  unsigned int* minmax;  // [B][2] ordered-uint min / max
  int n_windows, n_mtiles;
};
__global__ void __launch_bounds__(cq::kThreads, 1) cqt_tc_kernel(const CqtTcArgs a) {
  using namespace cq;
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* full = bars;              // [kStages]  producer-warp arrivals + the bytes of the W slice
  uint64_t* empty = bars + kStages;   // [kStages]  one arrival per consumer warp

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);  // broadcast: warp-uniform role branches and loop state
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full + s, kProducers / 32);  // one arrival per producer warp (512 single arrivals per chunk serialise)
      mbar_init(empty + s, kEpiWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int n_items = a.n_mtiles * kOctaves;
  const int total_frames = a.n_windows * kFrames;

  if (warp >= kEpiWarps) {
    // ------------------------------ producers ------------------------------
    // Phase A (lanes along the taps): warp pw gathers rows RW pw .. RW pw + RW - 1 of the chunk, two rows (2 x 64 taps) per
    // 128-bit load instruction, into the staging tile S[row][64 taps] -- a load instruction touches 4-6 cache lines
    // instead of 32 (one per row), which is what the LSU pipe was saturated with.  Phase B (lanes along the rows): thread
    // (row, half) reads its 32 taps back, splits them three ways and writes the K-major operand tile.
    constexpr int RW = kRowsPerWarp, NI = RW / 2;  // row pairs per warp
    constexpr int KQ = 32 / RW;                    // phase B: lanes per row
    constexpr int TPL = kKc / KQ;                  // taps per lane in phase B (a multiple of 8)
    const int ptid = threadIdx.x - 32 * kEpiWarps;  // producer thread
    const int pw = ptid >> 5;
    const int r = RW * pw + (lane % RW);  // phase B: the warp converts the rows it gathered, no block-wide barrier
    const int kq = lane / RW;
    float* stg = reinterpret_cast<float*>(smem + kStages * kStageBytes + 256 + kEpiBytes);  // [128][kStgPitch]
    RowP* rowp = reinterpret_cast<RowP*>(smem + kStages * kStageBytes + 256 + kEpiBytes +
                                         kMTile * kStgPitch * 4) + RW * pw;  // this warp's rows
    uint32_t stage = 0, ph = 0;
        for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
      const int mt = it / kOctaves, o = it % kOctaves;
      const int hop = 256 >> o;
      const int len = octave_len_rt(o);
      // The staging area is shared by both paths (rows of a warp / planes of the item's segment): nobody may start
      // writing it for this item while another producer warp still reads it for the previous one.
      asm volatile("bar.sync 1, %0;" ::"n"(kProducers) : "memory");
      if (o >= kSegOctave) {
        // ---- octaves with hop <= 32: the 128 rows of the item overlap (by 7/8 .. 255/256 of their 256 taps), so the signal
        // segment they cover is loaded, reflect-padded and split three ways ONCE per item into bf16 planes in shared memory
        // (it fits where the other path stages its rows), and every chunk's operand tile is then assembled with 16-byte
        // copies: 6 per thread and chunk instead of a gather + split of 16 samples per thread.
        // An M-tile may span two windows: part 0 = rows [0, n0) (frames t0.. of window b0), part 1 = rows [n0, 128)
        // (frames 0.. of window b0 + 1).  Each part's segment starts on a multiple of 8 samples at or below its first tap.
        __nv_bfloat16* seg = reinterpret_cast<__nv_bfloat16*>(stg);
        const int m0 = mt * kMTile;
        const int b0 = m0 / kFrames, t0 = m0 - b0 * kFrames;
        const int n0 = min(kMTile, kFrames - t0);
        const int s0 = t0 * hop - 128, a0 = s0 & ~7, d0 = s0 - a0;  // part 0: first tap, aligned start, offset of the tap
        const int L0 = ((n0 - 1) * hop + kTaps + d0 + 7) & ~7;
        const int L1 = n0 < kMTile ? (((kMTile - n0 - 1) * hop + kTaps + 7) & ~7) : 0;  // part 1 starts at sample -128
        {
          // <= 9 samples per thread (126 * 32 + 2 * 256 + slack <= 9 * 512): all loads are issued before the first use
          constexpr int NS = (126 * 32 + 2 * kTaps + 32 + kProducers - 1) / kProducers;
          float xs[NS];
#pragma unroll
          for (int q = 0; q < NS; ++q) {
            const int idx = ptid + q * kProducers;
            const int part = idx >= L0;
            const int b = b0 + part;
            int i = part ? idx - L0 - 128 : a0 + idx;
            if (i < 0) i = -i;
            if (i >= len) i = 2 * (len - 1) - i;
            xs[q] = (idx < L0 + L1 && b < a.n_windows && i >= 0 && i < len)
                        ? __ldg(a.chain + (size_t)b * kChainStride + chain_off_rt(o) + i)
                        : 0.f;
          }
#pragma unroll
          for (int q = 0; q < NS; ++q) {
            const int idx = ptid + q * kProducers;
            if (idx < L0 + L1) {
              const float x = xs[q];
              const __nv_bfloat16 h = __float2bfloat16_rn(x);
              const float r1 = x - __bfloat162float(h);
              const __nv_bfloat16 md = __float2bfloat16_rn(r1);
              seg[idx] = h;
              seg[kSegPlane + idx] = md;
              seg[2 * kSegPlane + idx] = __float2bfloat16_rn(r1 - __bfloat162float(md));
            }
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kProducers) : "memory");
        for (int c = 0; c < kTaps / kKc; ++c) {
          mbar_wait(empty + stage, ph ^ 1);
          unsigned char* sa = smem + stage * kStageBytes;
          if (ptid == 0) {
            mbar_expect_tx_only(full + stage, 3 * kWPlane);
            bulk_g2s(sa + 3 * kAPlane, a.wtc + (size_t)c * (3 * kWPlane / 2), 3 * kWPlane, full + stage);
          }
#pragma unroll
          for (int q = 0; q < 3 * 8 * kMTile / kProducers; ++q) {
            const int id = ptid + q * kProducers;
            const int row = id & (kMTile - 1), kc = (id >> 7) & 7, pl = id >> 10;
            const int e = (row < n0 ? d0 + row * hop : L0 + (row - n0) * hop) + c * kKc + kc * 8;  // element inside a plane
            const __nv_bfloat16* src = seg + pl * kSegPlane + e;
            uint4 v;
            if ((e & 7) == 0) {
              v = *reinterpret_cast<const uint4*>(src);
            } else if ((e & 1) == 0) {
              const uint32_t* w = reinterpret_cast<const uint32_t*>(src);
              v = make_uint4(w[0], w[1], w[2], w[3]);
            } else {  // odd element offset (hop 1): five words, shifted by half a word
              const uint32_t* w = reinterpret_cast<const uint32_t*>(src - 1);
              v = make_uint4(__funnelshift_r(w[0], w[1], 16), __funnelshift_r(w[1], w[2], 16),
                             __funnelshift_r(w[2], w[3], 16), __funnelshift_r(w[3], w[4], 16));
            }
            *reinterpret_cast<uint4*>(sa + pl * kAPlane + (kc * kMTile + row) * 16) = v;
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(full + stage);
          if (++stage == kStages) {
            stage = 0;
            ph ^= 1;
          }
        }
        continue;
      }
      __syncwarp();
      if (lane < RW) {  // per item: where row RW pw + lane reads its signal
        const int m = mt * kMTile + RW * pw + lane;
        RowP p;
        p.live = m < total_frames;
        const int b = p.live ? m / kFrames : 0;
        const int t = m - b * kFrames;
        p.lo = 0;
        p.hi = len;
        if (o == 0) {
          if (a.desc) {
            const WinDesc d = a.desc[b];
            p.src = a.audio + d.base;
            p.lo = d.lo;
            p.hi = d.hi;
          } else {
            p.src = a.audio + (long long)b * kWinSamples;
          }
        } else {
          p.src = a.chain + (size_t)b * kChainStride + chain_off_rt(o);
        }
        p.i0 = t * hop - 128;  // signal index of tap 0 of this frame
        rowp[lane] = p;
      }
      __syncwarp();
      for (int c = 0; c < kTaps / kKc; ++c) {
        float xs[4 * NI];
        unsigned vmask = 0;  // row pairs that took the vector path (warp-uniform)
#pragma unroll
        for (int i = 0; i < NI; ++i) {
          // rows 2i, 2i + 1 of the warp's rows; vector path: lane -> (row of the pair, 4 taps)
          const RowP p = rowp[2 * i + (lane >> 4)];
          const int ibv = p.i0 + c * kKc;  // signal index of the row's first tap in this chunk
          const bool okv = p.live && ibv >= p.lo && ibv + kKc <= p.hi && ibv >= 0 && ibv + kKc <= len &&
                           ((reinterpret_cast<uintptr_t>(p.src + ibv) & 15) == 0);
          if (__all_sync(0xffffffffu, okv)) {
            vmask |= 1u << i;
            const float4 v = __ldg(reinterpret_cast<const float4*>(p.src + ibv) + (lane & 15));
            xs[4 * i] = v.x, xs[4 * i + 1] = v.y, xs[4 * i + 2] = v.z, xs[4 * i + 3] = v.w;
          } else {
            // general path (unaligned low octaves, rows that touch the signal ends): reflect padding, zeros outside
            // [lo, hi); four loads of (row, 32 consecutive taps)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const RowP pq = rowp[2 * i + (q >> 1)];
              int idx = pq.i0 + c * kKc + (q & 1) * 32 + lane;
              float xv = 0.f;
              if (pq.live) {
                if (idx < 0) idx = -idx;
                if (idx >= len) idx = 2 * (len - 1) - idx;
                if (idx >= pq.lo && idx < pq.hi) xv = __ldg(pq.src + idx);
              }
              xs[4 * i + q] = xv;
            }
          }
        }
        __syncwarp();  // the warp's staging rows are free (phase B of its previous chunk is done)
#pragma unroll
        for (int i = 0; i < NI; ++i) {
          if ((vmask >> i) & 1u) {  // lanes hold (row of the pair, 4 taps)
            *reinterpret_cast<float4*>(stg + (RW * pw + 2 * i + (lane >> 4)) * kStgPitch + 4 * (lane & 15)) =
                make_float4(xs[4 * i], xs[4 * i + 1], xs[4 * i + 2], xs[4 * i + 3]);
          } else {  // lanes hold 4 x (row, tap)
#pragma unroll
            for (int q = 0; q < 4; ++q)
              stg[(RW * pw + 2 * i + (q >> 1)) * kStgPitch + (q & 1) * 32 + lane] = xs[4 * i + q];
          }
        }
        __syncwarp();  // rows complete
        // phase B: this lane's TPL taps of row r
        float xb[TPL];
        {
          const float4* sp = reinterpret_cast<const float4*>(stg + r * kStgPitch + TPL * kq);
#pragma unroll
          for (int i = 0; i < TPL / 4; ++i) {
            const float4 v = sp[i];
            xb[4 * i] = v.x, xb[4 * i + 1] = v.y, xb[4 * i + 2] = v.z, xb[4 * i + 3] = v.w;
          }
        }
        mbar_wait(empty + stage, ph ^ 1);
        unsigned char* sa = smem + stage * kStageBytes;
        if (ptid == 0) {
          mbar_expect_tx_only(full + stage, 3 * kWPlane);  // the bulk copy of the W slice completes on the same barrier
          bulk_g2s(sa + 3 * kAPlane, a.wtc + (size_t)c * (3 * kWPlane / 2), 3 * kWPlane, full + stage);
        }
#pragma unroll
        for (int q = 0; q < TPL / 8; ++q) {
          const int kc = kq * (TPL / 8) + q;
          const float* x = xb + 8 * q;
          __align__(16) __nv_bfloat162 h[4], md[4], l[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            h[j] = __floats2bfloat162_rn(x[2 * j], x[2 * j + 1]);
            const float2 hf = __bfloat1622float2(h[j]);
            const float r0 = x[2 * j] - hf.x, r1 = x[2 * j + 1] - hf.y;
            md[j] = __floats2bfloat162_rn(r0, r1);
            const float2 mf = __bfloat1622float2(md[j]);
            l[j] = __floats2bfloat162_rn(r0 - mf.x, r1 - mf.y);
          }
          const int o16 = (kc * kMTile + r) * 16;
          *reinterpret_cast<uint4*>(sa + o16) = *reinterpret_cast<const uint4*>(h);
          *reinterpret_cast<uint4*>(sa + kAPlane + o16) = *reinterpret_cast<const uint4*>(md);
          *reinterpret_cast<uint4*>(sa + 2 * kAPlane + o16) = *reinterpret_cast<const uint4*>(l);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the MMA
        __syncwarp();
        if (lane == 0) mbar_arrive(full + stage);
        if (++stage == kStages) {
          stage = 0;
          ph ^= 1;
        }
      }
    }
  } else {
    // ------------------------------ consumers: MMAs + epilogue (warps 0..7) ------------------------------
    // Warpgroup h computes frames 64 h .. 64 h + 63 of the M-tile.  Accumulator fragment of m64n80: thread (warp w of the
    // group, lane = 4 g + q) holds rows 16 w + g and 16 w + g + 8, columns 8 i + 2 q + {0, 1} = (re, im) of bin 4 i + q.
    const int h = warp >> 2, w = warp & 3, g = lane >> 2, q = lane & 3;
    const int r0 = 64 * h + 16 * w + g;  // first of the thread's two rows (the other is r0 + 8)
    uint32_t stage = 0, ph = 0;
    float* tile = reinterpret_cast<float*>(smem + kStages * kStageBytes + 256) + warp * (16 * kTilePitch);
    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
      const int mt = it / kOctaves, o = it % kOctaves;
      float d[kN / 2];
#pragma unroll
      for (int i = 0; i < kN / 2; ++i) d[i] = 0.f;
      for (int c = 0; c < kTaps / kKc; ++c) {
        mbar_wait(full + stage, ph);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kKc / 16; ++ks) {
          // one k-step = 16 taps = two 16-byte k-chunks, LBO apart; this warpgroup's 64 rows start 64 h rows in
          const uint32_t ao = sa + (uint32_t)(ks * 2 * (kMTile * 16) + h * 64 * 16);
          const uint32_t bo = sa + 3 * kAPlane + (uint32_t)(ks * 2 * (kN * 16));
          uint64_t A[3], B[3];
#pragma unroll
          for (int p = 0; p < 3; ++p) {
            A[p] = make_desc(ao + p * kAPlane, kMTile * 16, 128);
            B[p] = make_desc(bo + p * kWPlane, kN * 16, 128);
          }
          wgmma_ss_n80(d, A[0], B[0], (c | ks) ? 1u : 0u);  // hi * hi
          wgmma_ss_n80(d, A[0], B[1], 1u);                  // hi * mid
          wgmma_ss_n80(d, A[1], B[0], 1u);                  // mid * hi
          wgmma_ss_n80(d, A[0], B[2], 1u);                  // hi * lo
          wgmma_ss_n80(d, A[2], B[0], 1u);                  // lo * hi
          wgmma_ss_n80(d, A[1], B[1], 1u);                  // mid * mid
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(d);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + stage);  // this warp's share of the stage has been read
        if (++stage == kStages) {
          stage = 0;
          ph ^= 1;
        }
      }
      // epilogue: 10*log10(re^2 + im^2 + 1e-10) per bin (MUFU.LG2; the reference's sqrt-then-square differs by < 1e-6 dB),
      // staged per warp in shared memory so that the stores write runs of consecutive bins
      const int gb0 = (8 - o) * kBinsPerOctave - 15;  // global bin of the octave's bin 0 (negative for the lowest of o = 8)
      float vmin[2] = {INFINITY, INFINITY}, vmax[2] = {-INFINITY, -INFINITY};
      int bw[2];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int m = mt * kMTile + r0 + 8 * rr;
        const bool live = m < total_frames;
        bw[rr] = live ? m / kFrames : -1;
#pragma unroll
        for (int i = 0; i < 9; ++i) {
          const int bin = 4 * i + q, gg = gb0 + bin;
          float L = 0.f;
          if (gg >= 0) {
            const float s = __ldg(a.scale + gg);
            const float re = d[4 * i + 2 * rr] * s, im = d[4 * i + 2 * rr + 1] * s;
            L = __log2f(fmaf(re, re, im * im) + 1e-10f) * 3.0102999566398120f;
            if (live) {
              vmin[rr] = fminf(vmin[rr], L);
              vmax[rr] = fmaxf(vmax[rr], L);
            }
          }
          tile[(g + 8 * rr) * kTilePitch + bin] = L;
        }
      }
      __syncwarp();
      {
        const int m0 = mt * kMTile + 64 * h + 16 * w;  // 16 rows x 36 bins, consecutive lanes -> consecutive bins of a row
        for (int e = lane; e < 16 * kBinsPerOctave; e += 32) {
          const int rr = e / kBinsPerOctave, jj = e - rr * kBinsPerOctave;
          if (m0 + rr < total_frames && gb0 + jj >= 0) a.logmag[(size_t)(m0 + rr) * kCqtBins + gb0 + jj] = tile[rr * kTilePitch + jj];
        }
      }
      __syncwarp();  // the staging tile is reused by the next item
      // per-window min / max: one atomic pair per warp when all its rows sit in one window
      const int b0 = __shfl_sync(0xffffffffu, bw[0], 0);
      const bool uniform = __all_sync(0xffffffffu, bw[0] == b0 && bw[1] == b0);
      if (uniform) {
        if (b0 >= 0) {
          float mn = fminf(vmin[0], vmin[1]), mx = fmaxf(vmax[0], vmax[1]);
#pragma unroll
          for (int off = 16; off; off >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, off));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
          }
          if (lane == 0 && mn <= mx) {
            atomicMin(a.minmax + 2 * b0, float_to_ordered(mn));
            atomicMax(a.minmax + 2 * b0 + 1, float_to_ordered(mx));
          }
        }
      } else {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
          if (bw[rr] >= 0 && vmin[rr] <= vmax[rr]) {
            atomicMin(a.minmax + 2 * bw[rr], float_to_ordered(vmin[rr]));
            atomicMax(a.minmax + 2 * bw[rr] + 1, float_to_ordered(vmax[rr]));
          }
      }
    }
  }
}

__global__ void minmax_init_kernel2(unsigned int* mm, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    mm[2 * i] = 0xffffffffu;
    mm[2 * i + 1] = 0u;
  }
}

void cqt_tc_setup() { cudaFuncSetAttribute(cqt_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cq::kSmemBytes); }

void launch_cqt_tc(const float* audio, const WinDesc* desc, const float* chain, const uint16_t* wtc, const float* scale,
                   float* logmag, unsigned int* minmax, int n_windows, int n_sms, cudaStream_t st) {
  minmax_init_kernel2<<<(n_windows + 255) / 256, 256, 0, st>>>(minmax, n_windows);
  CqtTcArgs a;
  a.audio = audio;
  a.desc = desc;
  a.chain = chain;
  a.wtc = wtc;
  a.scale = scale;
  a.logmag = logmag;
  a.minmax = minmax;
  a.n_windows = n_windows;
  a.n_mtiles = (n_windows * kFrames + cq::kMTile - 1) / cq::kMTile;
  const int n_items = a.n_mtiles * kOctaves;
  const int grid = n_items < n_sms ? n_items : n_sms;
  cqt_tc_kernel<<<grid, cq::kThreads, cq::kSmemBytes, st>>>(a);
}

}  // namespace bp
