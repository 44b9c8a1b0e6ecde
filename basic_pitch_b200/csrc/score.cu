// Note-level transcription scores on the device: the counts behind mir_eval.transcription (0.7) match_notes +
// precision_recall_f1_overlap, with and without offsets, for a grid of (setting, file) pairs or a list of items.
//
// One thread per pair.  A pair's reference notes are sorted by (nearest semitone, onset) on the host; its estimated notes
// come either from the grid decode's note slots (frames and MIDI numbers, turned into seconds and log2(Hz) through two
// tables the host built) or from explicit arrays.  The hit graph is never stored: an estimated note's neighbours are
// found by scanning the semitone buckets within reach of the pitch tolerance and binary-searching the onset window, and
// the exact predicates decide.  The maximum matching is a greedy pass followed by one augmenting-path search (Kuhn) per
// estimated note the greedy pass left free, with an explicit stack in global workspace.
//
// The match kernels (bp_match_*) go further: they store each pair's hit graph and reproduce mir_eval's matching itself,
// pair for pair, for one (pair, pass) per thread.  The onset-only and offset-only counts (bp_score_onset_offset_*) need
// no pitch: their graphs are convex, and one thread per (pair, test) matches them greedily.
#include <cuda_runtime.h>

#include <cmath>

#include "kernels.cuh"

namespace bp {

namespace {

constexpr int kScoreThreads = 128;

// np.around(x, 4): multiply, round half to even, divide
__device__ __forceinline__ double around4(double x) { return __ddiv_rn(rint(__dmul_rn(x, 10000.0)), 10000.0); }

struct EstNote {
  double on, off, l2;
  int bucket;
};

struct PairCtx {
  // references of the pair's file: [0, n_ref) relative to r0
  const double* r_on;
  const double* r_off;
  const double* r_l2;
  const int* r_bucket;
  int n_ref;
  ScoreTol tol;
};

__device__ __forceinline__ EstNote est_note(const ScoreEst& e, long long base, int j) {
  EstNote n;
  if (e.onset) {
    n.on = e.onset[base + j];
    n.off = e.offset[base + j];
    n.l2 = e.log2hz[base + j];
  } else {
    n.on = e.frame_t[e.start[base + j]];
    n.off = e.frame_t[e.end[base + j]];
    n.l2 = e.log2_midi[e.pitch[base + j]];
  }
  n.bucket = score_bucket(n.l2);
  return n;
}

__device__ __forceinline__ bool hit(const PairCtx& c, const EstNote& e, int i, bool with_offset) {
  const double r_on = c.r_on[i];
  if (!(around4(fabs(__dsub_rn(r_on, e.on))) <= c.tol.onset)) return false;
  if (!(fabs(__dmul_rn(1200.0, __dsub_rn(c.r_l2[i], e.l2))) <= c.tol.pitch)) return false;
  if (!with_offset) return true;
  const double r_off = c.r_off[i];
  const double lim = fmax(__dmul_rn(c.tol.ratio, fabs(__dsub_rn(r_off, r_on))), c.tol.off_min);
  return around4(fabs(__dsub_rn(r_off, e.off))) <= lim;
}

// first reference at or after (bucket b, onset lo) in (bucket, onset) order
__device__ __forceinline__ int lower_bound(const PairCtx& c, int b, double lo) {
  int a = 0, n = c.n_ref;
  while (n > 0) {
    const int h = n >> 1, m = a + h;
    const int bm = c.r_bucket[m];
    if (bm < b || (bm == b && c.r_on[m] < lo)) {
      a = m + 1;
      n -= h + 1;
    } else {
      n = h;
    }
  }
  return a;
}

// Advances the cursor (db, pos) of estimated note e to its next hit: buckets e.bucket - K .. e.bucket + K, within each
// the references whose onset lies in [e.on - w, e.on + w] (w = onset tolerance + margin).  pos < 0: start of bucket db.
__device__ __forceinline__ bool next_hit(const PairCtx& c, const EstNote& e, int& db, int& pos, bool with_offset) {
  const double w = c.tol.window + fabs(e.on) * 1e-12;
  const double lo = e.on - w, hi = e.on + w;
  const int db_hi = min(c.tol.k_buckets, c.tol.bucket_hi - e.bucket);
  if (pos < 0) db = max(db, c.tol.bucket_lo - e.bucket);
  while (db <= db_hi) {
    const int b = e.bucket + db;
    pos = pos < 0 ? lower_bound(c, b, lo) : pos + 1;
    if (pos < c.n_ref && c.r_bucket[pos] == b && c.r_on[pos] <= hi) {
      if (hit(c, e, pos, with_offset)) return true;
      continue;
    }
    ++db;
    pos = -1;
  }
  return false;
}

// Size of a maximum matching of the hit graph.  match_ref / visit: [n_ref]; match_est: [n_est]; stack: [3 n_est].
__device__ __forceinline__ int max_matching(const PairCtx& c, const ScoreEst& e, long long ebase, int n_est,
                                            bool with_offset, int* match_ref, int* visit, int* match_est, int* stack) {
  const int K = c.tol.k_buckets;
  for (int i = 0; i < c.n_ref; ++i) match_ref[i] = visit[i] = -1;
  int matched = 0;
  for (int j = 0; j < n_est; ++j) {  // greedy: the first free hit
    match_est[j] = -1;
    const EstNote en = est_note(e, ebase, j);
    int db = -K, pos = -1;
    while (next_hit(c, en, db, pos, with_offset))
      if (match_ref[pos] < 0) {
        match_ref[pos] = j;
        match_est[j] = pos;
        ++matched;
        break;
      }
  }
  if (matched == c.n_ref) return matched;
  // augmenting paths from every estimated note still free; a note without one now never gets one later (Kuhn)
  for (int j = 0; j < n_est; ++j) {
    if (match_est[j] >= 0) continue;
    int depth = 1;
    stack[0] = j, stack[1] = -K, stack[2] = -1;  // frame: estimated note, bucket cursor, reference cursor
    while (depth > 0) {
      int* f = stack + 3 * (depth - 1);
      const EstNote en = est_note(e, ebase, f[0]);
      int db = f[1], r = f[2];
      const bool more = next_hit(c, en, db, r, with_offset);
      f[1] = db, f[2] = r;
      if (!more) {
        --depth;
        continue;
      }
      if (visit[r] == j) continue;
      visit[r] = j;
      if (match_ref[r] < 0) {  // flip the path: each frame's note takes the reference its cursor stands on
        for (int k = 0; k < depth; ++k) {
          const int jj = stack[3 * k], rr = stack[3 * k + 2];
          match_est[jj] = rr;
          match_ref[rr] = jj;
        }
        ++matched;
        break;
      }
      int* g = stack + 3 * depth++;
      g[0] = match_ref[r], g[1] = -K, g[2] = -1;
    }
    if (matched == c.n_ref) break;
  }
  return matched;
}

// Pair q = setting * n_files + file (chunk-local).  counts[q] = {n_ref, n_est, matched without offsets, matched}.
__global__ void __launch_bounds__(kScoreThreads) score_match_kernel(ScoreRefs R, ScoreEst E, ScoreTol tol,
                                                                    ScoreWork W, int n_files, long long n_pairs,
                                                                    long long* __restrict__ counts) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_pairs) return;
  const int file = (int)(q % n_files);
  const long long s = q / n_files;
  const long long r0 = R.off[file];
  PairCtx c;
  c.r_on = R.onset + r0;
  c.r_off = R.offset + r0;
  c.r_l2 = R.log2hz + r0;
  c.r_bucket = R.bucket + r0;
  c.n_ref = (int)(R.off[file + 1] - r0);
  c.tol = tol;
  const long long ebase = E.off[q];
  const int n_est = E.count ? E.count[q] : (int)(E.off[q + 1] - ebase);
  int* rw = W.ref + 2 * (s * W.n_ref_total + r0);
  int* ew = W.est + 4 * ebase;
  long long* out = counts + 4 * q;
  out[0] = c.n_ref;
  out[1] = n_est;
  if (c.n_ref == 0 || n_est == 0) {
    out[2] = out[3] = 0;
    return;
  }
  for (int pass = 0; pass < 2; ++pass)  // hits without, then with the offset test
    out[2 + pass] = max_matching(c, E, ebase, n_est, pass == 1, rw, rw + c.n_ref, ew, ew + n_est);
}

// ---- mir_eval's matching pair for pair (bp_match_*) ------------------------------------------------------------------
// mir_eval.transcription.match_notes builds G = {estimate: [references it hits]} from the row-major np.where of the hit
// matrix and runs util._bipartite_match (Hopcroft-Karp, Eppstein's PADS) on it, walking Python dicts in insertion order.
// The thread below rebuilds G with arrays (lists in ascending reference index, keys ordered by (first reference, j)) and
// runs the same steps in the same order, with an explicit stack for the recursion; include/bp_b200.h states them.

// file's references, which start at r0 = R.off[file]
__device__ __forceinline__ PairCtx pair_ctx(const ScoreRefs& R, const ScoreTol& tol, int file, long long r0) {
  PairCtx c;
  c.r_on = R.onset + r0;
  c.r_off = R.offset + r0;
  c.r_l2 = R.log2hz + r0;
  c.r_bucket = R.bucket + r0;
  c.n_ref = (int)(R.off[file + 1] - r0);
  c.tol = tol;
  return c;
}

__global__ void __launch_bounds__(kScoreThreads) match_count_kernel(ScoreRefs R, ScoreEst E, ScoreTol tol, int n_files,
                                                                    long long n_pairs, long long* __restrict__ edges) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_pairs) return;
  const int file = (int)(q % n_files);
  const long long r0 = R.off[file];
  const PairCtx c = pair_ctx(R, tol, file, r0);
  const long long ebase = E.off[q];
  const int n_est = E.count ? E.count[q] : (int)(E.off[q + 1] - ebase);
  long long m = 0;
  for (int j = 0; c.n_ref > 0 && j < n_est; ++j) {
    const EstNote en = est_note(E, ebase, j);
    int db = -c.tol.k_buckets, pos = -1;
    while (next_hit(c, en, db, pos, false)) ++m;
  }
  edges[q] = m;
}

constexpr int kPredUnmatched = -1;  // pred[u] of an estimate of the first layer (the `unmatched` flag value)
constexpr int kPredAbsent = -2;     // u not in pred

// Thread t of the launch: pair q0 + t / 2, pass t % 2 (0: hits without the offset test, 1: with it).  Every thread
// walks its own graph serially; a minimum of one CTA per SM lets ptxas keep the layout pointers in registers (89, no
// spills) instead of spilling them at the 80 it picks for the default occupancy target.
__global__ void __launch_bounds__(kScoreThreads, 1) match_kernel(ScoreRefs R, ScoreEst E, ScoreTol tol, MatchWork W,
                                                              int n_files, long long q0, long long q1) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long q = q0 + (t >> 1);
  if (q >= q1) return;
  const int pass = (int)(t & 1);
  const int file = (int)(q % n_files);
  const long long r0 = R.off[file];
  const PairCtx c = pair_ctx(R, tol, file, r0);
  const long long ebase = E.off[q];
  const int n_est = E.count ? E.count[q] : (int)(E.off[q + 1] - ebase);
  const int n_ref = c.n_ref;
  if (n_ref == 0 || n_est == 0) return;
  const long long M = W.edges[q];
  int* w = W.ws + (W.off[q] - W.off[q0]) + pass * match_pass_ints(n_est, n_ref, M);
  int* adj_off = w;                 // [N + 1]
  int* adj = adj_off + n_est + 1;   // [M]
  int* node_u = adj + M;            // [M]
  int* node_nx = node_u + M;        // [M]
  int* head = node_nx + M;          // [R + 1], first the counts of the key sort
  int* tail = head + n_ref + 1;     // [R]
  int* pst = tail + n_ref;          // [R] preds state: 2 phase + 1 in this layer's new_layer, 2 phase + 2 in preds
  int* order = pst + n_ref;         // [R] new_layer's insertion order
  int* unm = order + n_ref;         // [R]
  int* stack = unm + n_ref;         // [3 (R + 1)] frames (reference, next node, estimate taken)
  int* pred = stack + 3 * (n_ref + 1);  // [N]
  int* keys = pred + n_est;         // [N]
  int* lay = keys + n_est;          // [N]
  int* nxt = lay + n_est;           // [N]
  int* out = W.match + ((q / n_files) * 2 + pass) * W.n_ref_total + r0;
  const int* orig = W.r_orig + r0;

  // G: estimate j's references in ascending original index (insertion sort; the scan visits them by (bucket, onset))
  int k = 0;
  for (int j = 0; j < n_est; ++j) {
    adj_off[j] = k;
    const EstNote en = est_note(E, ebase, j);
    int db = -c.tol.k_buckets, pos = -1;
    while (next_hit(c, en, db, pos, pass == 1)) {
      const int v = orig[pos];
      int i = k++;
      for (; i > adj_off[j] && adj[i - 1] > v; --i) adj[i] = adj[i - 1];
      adj[i] = v;
    }
  }
  adj_off[n_est] = k;
  // keys: estimates with a hit, by (first reference, j) -- a counting sort on the first reference, stable in j
  for (int v = 0; v <= n_ref; ++v) head[v] = 0;
  for (int j = 0; j < n_est; ++j)
    if (adj_off[j + 1] > adj_off[j]) ++head[adj[adj_off[j]] + 1];
  for (int v = 1; v <= n_ref; ++v) head[v] += head[v - 1];
  int n_keys = 0;
  for (int j = 0; j < n_est; ++j)
    if (adj_off[j + 1] > adj_off[j]) keys[head[adj[adj_off[j]]]++] = j, ++n_keys;
  // greedy: each key takes the first reference of its list not yet matched
  for (int a = 0; a < n_keys; ++a) {
    const int u = keys[a];
    for (int e = adj_off[u]; e < adj_off[u + 1]; ++e)
      if (out[adj[e]] < 0) {
        out[adj[e]] = u;
        break;
      }
  }
  for (int v = 0; v < n_ref; ++v) pst[v] = 0;
  for (int phase = 1;; ++phase) {
    const int in_new = 2 * phase + 1, in_preds = 2 * phase + 2;
    for (int a = 0; a < n_keys; ++a) pred[keys[a]] = kPredUnmatched;
    for (int v = 0; v < n_ref; ++v)
      if (out[v] >= 0) pred[out[v]] = kPredAbsent;
    int n_lay = 0;
    for (int a = 0; a < n_keys; ++a)
      if (pred[keys[a]] == kPredUnmatched) lay[n_lay++] = keys[a];
    int n_unm = 0, n_node = 0;
    // layering: the preds lists of this phase hold at most one node per hit, every estimate being in one layer at most
    while (n_lay > 0 && n_unm == 0) {
      int n_order = 0;
      for (int a = 0; a < n_lay; ++a) {
        const int u = lay[a];
        for (int e = adj_off[u]; e < adj_off[u + 1]; ++e) {
          const int v = adj[e];
          if (pst[v] == in_preds) continue;
          if (pst[v] != in_new) {
            pst[v] = in_new;
            head[v] = n_node;
            order[n_order++] = v;
          } else {
            node_nx[tail[v]] = n_node;
          }
          node_u[n_node] = u;
          node_nx[n_node] = -1;
          tail[v] = n_node++;
        }
      }
      n_lay = 0;
      for (int a = 0; a < n_order; ++a) {
        const int v = order[a];
        pst[v] = in_preds;
        const int u = out[v];
        if (u >= 0) {
          nxt[n_lay++] = u;
          pred[u] = v;
        } else {
          unm[n_unm++] = v;
        }
      }
      int* s = lay;
      lay = nxt;
      nxt = s;
    }
    if (n_unm == 0) break;
    // recurse(v) for every unmatched v of the last layer; a frame resumes its list where it left it
    for (int a = 0; a < n_unm; ++a) {
      const int v0 = unm[a];
      if (pst[v0] != in_preds) continue;
      pst[v0] = 0;  // preds.pop(v)
      stack[0] = v0, stack[1] = head[v0], stack[2] = -1;
      int depth = 1;
      while (depth > 0) {
        int* f = stack + 3 * (depth - 1);
        int node = f[1], child = -1;
        bool found = false;
        while (node >= 0) {
          const int u = node_u[node];
          node = node_nx[node];
          const int pu = pred[u];
          if (pu == kPredAbsent) continue;
          pred[u] = kPredAbsent;
          f[2] = u;
          if (pu == kPredUnmatched) {
            found = true;
            break;
          }
          if (pst[pu] == in_preds) {  // recurse(pu); a reference no longer in preds returns False at once
            child = pu;
            break;
          }
        }
        f[1] = node;
        if (found) {  // every frame's reference takes the estimate it stands on
          for (int d = 0; d < depth; ++d) out[stack[3 * d]] = stack[3 * d + 2];
          break;
        }
        if (child < 0) {
          --depth;
          continue;
        }
        pst[child] = 0;
        int* g = stack + 3 * depth++;
        g[0] = child, g[1] = head[child], g[2] = -1;
      }
    }
  }
}

// ---- onset-only and offset-only counts (bp_score_onset_offset_*) -------------------------------------------------------
// Without the pitch test each test's hit graph is convex: with the estimates in ascending order of the tested time, a
// reference hits one contiguous run of them, because around4(|fl(t_r - t_e)|) falls and then rises as t_e grows.  Taking
// the references by ascending run end, each matched to the smallest free estimate of its run, gives a maximum matching.

// Thread t: pair t / 2, test t % 2 (0: onsets, 1: offsets).  The estimates' tested times come sorted per item (explicit
// notes, sorted on the host) or are sorted here by frame index (decode slots; bp_frame_times is strictly increasing).
__global__ void __launch_bounds__(kScoreThreads) onset_offset_kernel(ScoreRefs R, ScoreEst E, ScoreTol tol, ScoreWork W,
                                                                     int n_files, long long n_pairs,
                                                                     long long* __restrict__ counts) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long q = t >> 1;
  if (q >= n_pairs) return;
  const int test = (int)(t & 1);
  const int file = (int)(q % n_files);
  const long long s = q / n_files;
  const long long r0 = R.off[file];
  const int n_ref = (int)(R.off[file + 1] - r0);
  const long long ebase = E.off[q];
  const int n = E.count ? E.count[q] : (int)(E.off[q + 1] - ebase);
  long long* out = counts + 4 * q;
  if (test == 0) out[0] = n_ref, out[1] = n;
  if (n_ref == 0 || n == 0) {
    out[2 + test] = 0;
    return;
  }
  int* keys = W.est + 4 * ebase + 2 * q + (long long)test * (2LL * n + 1);  // [N] frame of the k-th smallest time
  int* cnt = keys + n;                                                      // [N + 1] counts of the sort, then next free
  int* run = W.ref + 6 * (s * W.n_ref_total + r0) + (long long)test * 3 * n_ref;  // [2 R] lo, end (one past hi)
  int* order = run + 2 * n_ref;                                                   // [R] references by run end
  const double* est_t = test ? E.offset + ebase : E.onset + ebase;                // explicit notes, sorted
  const double* r_t = test ? R.offset + r0 : R.onset + r0;
  if (E.count) {  // heap sort of the slots' frames
    const int* fr = (test ? E.end : E.start) + ebase;
    for (int j = 0; j < n; ++j) keys[j] = fr[j];
    auto sift = [&](int h, int v, int end) {  // v down from h in the max-heap keys[0, end)
      for (int c = 2 * h + 1; c < end; c = 2 * h + 1) {
        if (c + 1 < end && keys[c + 1] > keys[c]) ++c;
        if (keys[c] <= v) break;
        keys[h] = keys[c];
        h = c;
      }
      keys[h] = v;
    };
    for (int i = n / 2 - 1; i >= 0; --i) sift(i, keys[i], n);
    for (int end = n - 1; end > 0; --end) {
      const int v = keys[end];
      keys[end] = keys[0];
      sift(0, v, end);
    }
  }
  auto time = [&](int j) { return E.count ? E.frame_t[keys[j]] : est_t[j]; };
  for (int k = 0; k <= n; ++k) cnt[k] = 0;
  for (int r = 0; r < n_ref; ++r) {
    const double tr = r_t[r];
    const double lim =
        test ? fmax(__dmul_rn(tol.ratio, fabs(__dsub_rn(R.offset[r0 + r], R.onset[r0 + r]))), tol.off_min) : tol.onset;
    // lo: estimates before the reference that miss it; end: first estimate after it that misses it
    int a = 0, len = n;
    while (len > 0) {
      const int h = len >> 1, m = a + h;
      const double te = time(m);
      if (te < tr && !(around4(fabs(__dsub_rn(tr, te))) <= lim)) {
        a = m + 1;
        len -= h + 1;
      } else {
        len = h;
      }
    }
    const int lo = a;
    len = n - lo;
    while (len > 0) {
      const int h = len >> 1, m = a + h;
      const double te = time(m);
      if (!(te > tr && !(around4(fabs(__dsub_rn(tr, te))) <= lim))) {
        a = m + 1;
        len -= h + 1;
      } else {
        len = h;
      }
    }
    run[2 * r] = lo;
    run[2 * r + 1] = a;
    if (lo < a) ++cnt[a];
  }
  for (int k = 0, sum = 0; k <= n; ++k) {  // counting sort by run end (in [1, N] for a non-empty run)
    const int c = cnt[k];
    cnt[k] = sum;
    sum += c;
  }
  int n_order = 0;
  for (int r = 0; r < n_ref; ++r)
    if (run[2 * r] < run[2 * r + 1]) order[cnt[run[2 * r + 1]]++] = r, ++n_order;
  // greedy: each reference takes the smallest free estimate of its run (next free, path halving; cnt[N] = N: none)
  int* nf = cnt;
  for (int k = 0; k <= n; ++k) nf[k] = k;
  int matched = 0;
  for (int k = 0; k < n_order; ++k) {
    const int r = order[k];
    int x = run[2 * r];
    while (nf[x] != x) {
      nf[x] = nf[nf[x]];
      x = nf[x];
    }
    if (x < run[2 * r + 1]) {
      nf[x] = x + 1;
      ++matched;
    }
  }
  out[2 + test] = matched;
}

}  // namespace

void launch_onset_offset(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, const ScoreWork& W, int n_files,
                         long long n_pairs, long long* counts, cudaStream_t st) {
  const unsigned int blocks = (unsigned int)((2 * n_pairs + kScoreThreads - 1) / kScoreThreads);
  onset_offset_kernel<<<blocks, kScoreThreads, 0, st>>>(R, E, tol, W, n_files, n_pairs, counts);
}

void launch_match_count(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, int n_files, long long n_pairs,
                        long long* edges, cudaStream_t st) {
  const unsigned int blocks = (unsigned int)((n_pairs + kScoreThreads - 1) / kScoreThreads);
  match_count_kernel<<<blocks, kScoreThreads, 0, st>>>(R, E, tol, n_files, n_pairs, edges);
}

void launch_match(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, const MatchWork& W, int n_files,
                  long long q0, long long q1, cudaStream_t st) {
  const unsigned int blocks = (unsigned int)((2 * (q1 - q0) + kScoreThreads - 1) / kScoreThreads);
  match_kernel<<<blocks, kScoreThreads, 0, st>>>(R, E, tol, W, n_files, q0, q1);
}

void launch_score_match(const ScoreRefs& R, const ScoreEst& E, const ScoreTol& tol, const ScoreWork& W, int n_files,
                        long long n_pairs, long long* counts, cudaStream_t st) {
  const unsigned int blocks = (unsigned int)((n_pairs + kScoreThreads - 1) / kScoreThreads);
  score_match_kernel<<<blocks, kScoreThreads, 0, st>>>(R, E, tol, W, n_files, n_pairs, counts);
}

}  // namespace bp
