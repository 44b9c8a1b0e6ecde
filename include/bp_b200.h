/*
 * bp_b200.h — C ABI of the Hopper-native basic-pitch hot path (libbp_b200.so, sm_90a).
 *
 * The reference has no FFI: its boundary is a Python API in front of a third-party ML runtime
 * (SURVEY.md §8b).  Each entry point below names the reference interface it stands in for
 * (paths relative to the reference repository root).  All pointers are plain host or device
 * pointers; no torch / numpy types cross this boundary.  Unless stated otherwise arrays are
 * C-contiguous float32.
 *
 * Error convention: every function returning `int` returns BP_OK (0) or a negative BP_E_* code;
 * `bp_last_error()` returns a thread-local, human-readable message for the last failure.
 * There is no CPU fallback: without a CUDA device every call fails with BP_E_CUDA.
 *
 * Threading: one `bp_model_t` is bound to one CUDA device and must not be used from two host
 * threads at the same time (the reference's `Model` is likewise single-threaded,
 * basic_pitch/inference.py:71-182).  Different models (e.g. one per GPU) are independent.
 */
#ifndef BP_B200_H
#define BP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BP_OK 0
#define BP_E_INVALID (-1)  /* bad argument / malformed weight blob                     */
#define BP_E_CUDA (-2)     /* CUDA runtime error (message carries cudaGetErrorString)  */
#define BP_E_CAPACITY (-3) /* caller-provided output capacity too small                */
#define BP_E_NOMEM (-4)
#define BP_E_IO (-5)       /* a file could not be read during the call (message names it: index and path)   */

/* Geometry of the model (reference: basic_pitch/constants.py:25-47, inference.py:185-191,302-305). */
#define BP_SAMPLE_RATE 22050
#define BP_WINDOW_SAMPLES 43844 /* AUDIO_N_SAMPLES                                     */
#define BP_WINDOW_FRAMES 172    /* ANNOT_N_FRAMES                                      */
#define BP_N_PITCHES 88         /* note / onset bins                                   */
#define BP_N_CONTOUR_BINS 264   /* contour bins                                        */
#define BP_OVERLAP_FRAMES 30    /* DEFAULT_OVERLAPPING_FRAMES                          */
#define BP_HOP_SAMPLES 36164    /* AUDIO_N_SAMPLES - 30*256                            */
#define BP_HOP_FRAMES 142       /* frames kept per window after unwrapping             */
#define BP_LEAD_ZEROS 3840      /* zeros prepended to every file (overlap_len / 2)     */

typedef struct bp_model bp_model_t;

/* Parameters of the note decode.
 * reference: basic_pitch/note_creation.py:360-371 (output_to_notes_polyphonic arguments) and
 * :52-63 (model_output_to_notes).  The pitch-column range replaces min_freq/max_freq: the host
 * converts Hz to columns exactly as constrain_frequency does (note_creation.py:333-336). */
typedef struct bp_decode_params {
  double onset_thresh;       /* default 0.5  */
  double frame_thresh;       /* default 0.3 ; must be >= 0 when melodia_trick (reference loops forever otherwise) */
  int32_t min_note_len;      /* frames, default 11 */
  int32_t energy_tol;        /* default 11 */
  int32_t infer_onsets;      /* default 1  */
  int32_t melodia_trick;     /* default 1  */
  int32_t include_pitch_bends; /* default 1 */
  int32_t min_pitch_idx;     /* columns < this are zeroed (default 0)   */
  int32_t max_pitch_idx;     /* columns >= this are zeroed (default 88) */
  int32_t reserved;
} bp_decode_params_t;

/* Note events of a batch of files, structure-of-arrays, caller-allocated (host memory).
 * Notes of file i occupy [note_off[i], note_off[i+1]) in generation order (onset-loop notes latest
 * first, then melodia notes — the order of the reference's list, note_creation.py:410-509).
 * Pitch bends of note j occupy bends[bend_off[j] .. bend_off[j+1]) (1/3-semitone units,
 * note_creation.py:215-217); bend_off has note capacity + 1 entries. */
typedef struct bp_notes {
  int32_t note_capacity;  /* in: capacity of the per-note arrays                     */
  int32_t bend_capacity;  /* in: capacity of `bends`                                 */
  int32_t* note_off;      /* out: [n_files + 1]                                      */
  int32_t* start_frame;   /* out: [note_capacity]                                    */
  int32_t* end_frame;     /* out: [note_capacity]                                    */
  int32_t* pitch_midi;    /* out: [note_capacity]  (column + 21)                     */
  float* amplitude;       /* out: [note_capacity]                                    */
  int32_t* bend_off;      /* out: [note_capacity + 1]                                */
  int32_t* bends;         /* out: [bend_capacity]; may be NULL if !include_pitch_bends */
} bp_notes_t;

/* ---- library ---------------------------------------------------------------------------- */
int bp_version(void);
const char* bp_last_error(void);
void bp_default_decode_params(bp_decode_params_t* p);

/* Number of model windows / output frames for a file of n_samples 22 050 Hz samples.
 * reference: basic_pitch/inference.py:194-219 (window_audio_file), :247-279 (unwrap_output). */
int64_t bp_num_windows(int64_t n_samples);
int64_t bp_num_frames(int64_t n_samples);

/* ---- model lifetime ----------------------------------------------------------------------
 * reference: Model.__init__ (basic_pitch/inference.py:78-154) loading
 * the files under basic_pitch/saved_models/icassp_2022.  `blob` is the BPW1 tensor blob
 * (basic_pitch_b200/weights.py); it is copied, the caller keeps ownership. */
int bp_model_create(const void* blob, size_t nbytes, int device, bp_model_t** out);
void bp_model_destroy(bp_model_t* m);
int bp_model_device(const bp_model_t* m);
/* Device pointer + size of the packed parameter block (for the one NCCL broadcast at init). */
int bp_model_param_block(bp_model_t* m, void** d_ptr, size_t* nbytes);
/* Re-derive internal (split / transposed) weight layouts after the block was overwritten. */
int bp_model_refresh(bp_model_t* m);
/* Kernel launches issued by this model since creation (for bench.py's gpu_launches). */
int64_t bp_model_launch_count(const bp_model_t* m);

/* ---- stage 1+2: audio windows -> posteriorgrams -------------------------------------------
 * reference: Model.predict (basic_pitch/inference.py:156-182), batched: audio [n][43844] ->
 * note [n][172][88], onset [n][172][88], contour [n][172][264].
 * _device: pointers are device memory on the model's device; work is enqueued on `stream`
 * (a cudaStream_t) and NOT synchronised.  _host: host pointers, copies inside, synchronous. */
int bp_forward_device(bp_model_t* m, const float* d_audio, int64_t n_windows, float* d_note, float* d_onset,
                      float* d_contour, void* stream);
int bp_forward_host(bp_model_t* m, const float* h_audio, int64_t n_windows, float* h_note, float* h_onset,
                    float* h_contour);

/* ---- run_inference for whole files ---------------------------------------------------------
 * reference: run_inference (basic_pitch/inference.py:282-330) = get_audio_input windowing
 * (:222-244) + Model.predict per window + unwrap_output (:247-279), for a batch of files.
 * audio: the files' samples back to back; sample_off[n_files+1] gives each file's range.
 * Outputs: unwrapped posteriorgrams of all files back to back; file i has
 * bp_num_frames(len_i) frames starting at frame_off[i] (frame_off[n_files+1] is written by the
 * call; host array in both variants).  Output arrays must hold sum_i bp_num_frames(len_i) frames.
 * _host, like every host entry point for a batch of files, runs it in sub-batches of whole files: the upload of each
 * overlaps the kernels of the one before, and its posteriorgrams come back while later ones compute (page-locked
 * outputs from bp_host_alloc make that copy asynchronous). */
int bp_run_inference_device(bp_model_t* m, const float* d_audio, const int64_t* h_sample_off, int32_t n_files,
                            float* d_note, float* d_onset, float* d_contour, int64_t* h_frame_off, void* stream);
int bp_run_inference_host(bp_model_t* m, const float* h_audio, const int64_t* h_sample_off, int32_t n_files,
                          float* h_note, float* h_onset, float* h_contour, int64_t* h_frame_off);

/* ---- stage 3: posteriorgrams -> note events -------------------------------------------------
 * reference: model_output_to_notes without the MIDI object (basic_pitch/note_creation.py:52-111):
 * output_to_notes_polyphonic (:360-511) + get_pitch_bends (:182-219), for a batch of files whose
 * (unwrapped) posteriorgrams lie back to back, file i covering frames [frame_off[i], frame_off[i+1]).
 * The posteriorgrams are not modified (the reference zeroes out-of-range pitch columns in place,
 * note_creation.py:338-341; the Python wrapper reproduces that on its own arrays).
 * `notes` arrays are host memory in both variants; the call synchronises `stream` before returning. */
int bp_decode_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                     const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, bp_notes_t* notes,
                     void* stream);
int bp_decode_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                   const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, bp_notes_t* notes);

/* ---- stage 3 for a streamed recording -------------------------------------------------------------------------------
 * reference: model_output_to_notes (note_creation.py:52-111) for a recording whose posteriorgrams arrive piecewise (as
 * run_inference_stream yields them), decoded as they arrive in bounded device memory.  DESIGN.md §4.5 gives the argument.
 *   quiet frame  every column of [min_pitch_idx, max_pitch_idx) has a note value strictly below frame_thresh (a value
 *                equal to it is "on", as in the decode's tracking); columns outside the range count as 0, so
 *                frame_thresh <= 0 never gives a quiet frame and never cuts.
 *   cut          at frame c when frames [c - LB, c + LA) are quiet and frame c - LB - 1 is not (or c - LB is the first
 *                frame of the recording or of a forced part): one cut per quiet run of at least LA + LB frames, with
 *                LA = energy_tol and LB = 3.  A cut is known once frame c + LA - 1 has been pushed.
 *   segment      frames [a, b) between two cuts, decoded by the decode kernels as one file over [a - 3, b + A) with
 *                A = max(1, energy_tol - 2) (no context before the start of the recording or of a forced part); only
 *                notes that start in [a, b) are kept.  LA and LB are the smallest lengths for which the notes of every
 *                segment are those of the whole-recording decode that start in it, given that the context is quiet:
 *                a candidate on the last quiet frame before c scans energy_tol frames (LA); the peak pick at c reads
 *                frame c - 1, whose inferred onset reads c - 3 (LB); a track whose last loud frame is c - 4 reads up to
 *                c - 4 + energy_tol, which `i < n_frames - 1` must admit (A); every other read or write of the greedy
 *                loops stays within energy_tol frames of a loud cell, so no track crosses a cut.
 *   maxima       segment k infers its onsets with max(onsets) and max(frame_diff) over stream frames [0, e_k), e_k the
 *                end of its decode range (the running maxima): a segment decoded after both recording-wide maxima have
 *                arrived has exactly the notes of bp_decode_device on the whole recording; earlier ones may differ.
 *   forced cut   max_segment_frames = M > 0: when M frames have arrived since the start a of the open segment and no cut
 *                was known within them, the stream cuts at a + M as at a file boundary (the frames before decode as a
 *                recording that ends there, those after as one that starts there; the maxima carry over).  Results
 *                then differ from the whole-recording decode by construction.  M = 0: never.
 * The device holds the frames from the open segment's decode start on: at most the longest stretch without a cut (or M)
 * plus 3 frames of context and the frames pushed since the last cut, 1 760 bytes per frame.
 * bp_stream_create validates params as bp_decode_device does (BP_E_INVALID), and M < 0.  The stream uses its model's
 * device and stream and must be destroyed before it.
 * bp_stream_push_host: n_frames consecutive frames, row-major [n_frames][88 | 88 | 264] host arrays (h_contour may be
 *   NULL when !include_pitch_bends); synchronous.  Launches: one quiet scan (none when n_frames == 0); then per segment
 *   it closes one more scan unless the cut was confirmed by the last frame pushed, the decode's prep, candidate and loop
 *   kernels (twice when the segment yields more notes than the first allowance of min(88 T, 8 T + 64) slots, T its
 *   decode frames), the compaction if the decode found notes, and the note finish if any of them start in the segment.
 *   BP_E_INVALID after bp_stream_end.
 * bp_stream_end: the recording has ended; decodes the open segment with the end-of-file rules.  BP_E_INVALID if called
 *   twice.
 * bp_stream_take: moves the finished notes out, as bp_decode_device's one file: note_off[0..1], global frame indices,
 *   segments in time order and within a segment the reference's generation order, amplitudes and pitch bends as
 *   there.  BP_E_CAPACITY (bp_last_required) leaves them queued.
 * bp_stream_held_frames: frames held on the device, context included. */
typedef struct bp_stream bp_stream_t;
int bp_stream_create(bp_model_t* m, const bp_decode_params_t* params, int64_t max_segment_frames, bp_stream_t** out);
int bp_stream_push_host(bp_stream_t* s, const float* h_note, const float* h_onset, const float* h_contour,
                        int64_t n_frames);
int bp_stream_end(bp_stream_t* s);
int bp_stream_take(bp_stream_t* s, bp_notes_t* notes);
int64_t bp_stream_held_frames(const bp_stream_t* s);
void bp_stream_destroy(bp_stream_t* s);

/* ---- many streamed recordings at once (stream group) ----------------------------------------------------------------
 * A group holds any number of streams with one set of decode params and M, each decoded by exactly the rules of
 * bp_stream_* above, and serves every stream listed in a call with one device pass: the new samples go up in one copy,
 * the windows they complete run through one forward pass (one launch chain per bp_model_chunk_windows windows), the
 * frames stay on the device, one quiet scan covers every stream and the closed segments are decoded in rounds, one
 * segment per stream per round, as one batch.  A stream's notes are those bp_stream_* gives for the same frames whatever
 * the push schedule (DESIGN.md §4.6), and the frames of an audio stream are those run_inference_stream yields for its
 * blocks.  Streams are named by the ids bp_stream_group_open returns; a call lists each at most once.  BP_E_INVALID for
 * an unknown or ended id, an id listed twice, a negative length, a NULL block of nonzero length, and a stream given
 * audio after posteriorgrams or the reverse.  The group uses its model's device and stream and must be destroyed before
 * it; it keeps no model workspace between calls.
 * bp_stream_group_push_host: the next block of each listed stream, mono float32 at 22 050 Hz (any length, 0 included;
 *   PCM streams below take bp_stream_group_push_pcm_host).
 *   Frames a stream commits: those of its windows except the newest two (whose frames the final trim of unwrap_output
 *   can reach), and at its end bp_num_frames(samples) in all.  h_note / h_onset / h_contour (each may be NULL) receive
 *   the frames each listed stream committed in this call, row-major, stream i's from row h_frame_off[i] on
 *   (h_frame_off[n + 1], may be NULL; bp_stream_group_commit_offsets gives the same offsets before the call).
 * bp_stream_group_end: the listed streams have ended: their last windows run (zero-padded), and their open segments are
 *   decoded with the end-of-file rules; posteriorgram outputs as a push.
 * bp_stream_group_push_frames_host: posteriorgrams instead of audio, as bp_stream_push_host takes them, n_frames[i]
 *   rows for stream i (h_contour may be NULL when !include_pitch_bends).
 * bp_stream_group_commit_offsets: h_frame_off[n + 1] of a push of n_samples[i] samples (ending != 0: of the end).
 * bp_stream_group_take: moves the finished notes of the listed streams out, stream i's at note_off[i] .. note_off[i + 1]
 *   (note_off[n + 1]), each as bp_stream_take; ended streams may be listed.  BP_E_CAPACITY (bp_last_required) leaves
 *   them queued.
 * bp_stream_group_held_frames: as bp_stream_held_frames (0 for an unknown id).
 *
 * PCM streams: live input at its capture rate and format (DESIGN.md §4.6).
 * bp_stream_group_open_pcm: a stream whose blocks are interleaved PCM of `channels` channels at `sample_rate` Hz, format
 *   codes and conversions as bp_load_pcm_* (0 float32, 1 int16, 2 int32, 3 uint8), validated as bp_pcm_file_t is
 *   (BP_E_INVALID for a format outside 0..3, channels or sample_rate below 1, or a ratio beyond ~100:1; the group stays
 *   usable).  With the reduced ratio up / down = (22050 / g) / (sample_rate / g), the filter's half = (L - 1) / 2 and T
 *   taps per phase (bp_load_pcm_*'s resampler), output k reads inputs i_max(k) - T + 1 .. i_max(k), i_max(k) =
 *   floor((k down + half) / up), inputs below 0 and (once the recording has ended) at or past its end being zero:
 *     final outputs  after n frames exactly the outputs k < F(n) = max(0, ceil((n up - half) / down)) are final (every
 *                    input they read has arrived); same rate: F(n) = n;
 *     end            bp_stream_group_end emits the rest, F(n) .. ceil(n up / down), zero-filled as the whole-file ingest;
 *     history        between pushes the device keeps only the down-mixed inputs [i_max(F(n)) - T + 1, n), at most T - 1
 *                    floats;
 *     bit-identity   every output is computed by the whole-file ingest's arithmetic, so for every block schedule the
 *                    stream's 22 050 Hz signal is bp_load_pcm_host(whole recording) bit for bit, its frames are
 *                    run_inference_stream's on that signal and its notes predict_stream_notes'.
 *   A stream opened as mono float32 at 22 050 Hz is a plain stream.
 * bp_stream_group_push_pcm_host: the next block of each listed stream, n_frames[i] PCM frames (0 allowed) of that
 *   stream's format; plain streams may be listed with float32 22 050 Hz blocks (n_frames their samples).  The blocks
 *   are packed behind their descriptors in pinned staging, each on a 16-byte boundary, and go up in one copy as stored;
 *   one stream ingest launch (none when no listed stream has frames) writes every stream's new final samples straight
 *   to its tail, in place of the float push's append copy.  The rest, outputs included, is bp_stream_group_push_host.
 *   bp_stream_group_end flushes ending PCM streams with one ingest launch before their last windows run.  For a PCM
 *   stream n_samples of bp_stream_group_commit_offsets counts PCM frames.  BP_E_INVALID (before anything is enqueued)
 *   for bp_stream_group_push_host on a PCM stream, this call on a posteriorgram stream, a NULL block with frames, a
 *   negative length and a block whose byte count overflows.
 * bp_stream_group_debug_tail: copies the stream's held 22 050 Hz tail, samples [*first_sample, *first_sample + *n) of
 *   its signal, to h_out (BP_E_CAPACITY when capacity < *n, which is still set).
 * bp_debug_pcm_stream_plan: host-only (no GPU).  For a stream of that format pushed frames[0 .. n_pushes) (and ended when
 *   `ending`: one more entry), per push the outputs it makes final [out_lo, out_hi) and the inputs it holds afterwards
 *   [hist_lo, hist_hi), from the function the push itself uses. */
typedef struct bp_stream_group bp_stream_group_t;
int bp_stream_group_create(bp_model_t* m, const bp_decode_params_t* params, int64_t max_segment_frames,
                           bp_stream_group_t** out);
int bp_stream_group_open(bp_stream_group_t* g, int32_t* id);
int bp_stream_group_commit_offsets(const bp_stream_group_t* g, int32_t n, const int32_t* ids, const int64_t* n_samples,
                                   int32_t ending, int64_t* h_frame_off);
int bp_stream_group_push_host(bp_stream_group_t* g, int32_t n, const int32_t* ids, const float* const* audio,
                              const int64_t* n_samples, float* h_note, float* h_onset, float* h_contour,
                              int64_t* h_frame_off);
int bp_stream_group_push_frames_host(bp_stream_group_t* g, int32_t n, const int32_t* ids, const float* const* h_note,
                                     const float* const* h_onset, const float* const* h_contour,
                                     const int64_t* n_frames);
int bp_stream_group_end(bp_stream_group_t* g, int32_t n, const int32_t* ids, float* h_note, float* h_onset,
                        float* h_contour, int64_t* h_frame_off);
int bp_stream_group_take(bp_stream_group_t* g, int32_t n, const int32_t* ids, bp_notes_t* notes);
int64_t bp_stream_group_held_frames(const bp_stream_group_t* g, int32_t id);
void bp_stream_group_destroy(bp_stream_group_t* g);
int bp_stream_group_open_pcm(bp_stream_group_t* g, int32_t sample_format, int32_t channels, int32_t sample_rate,
                             int32_t* id);
int bp_stream_group_push_pcm_host(bp_stream_group_t* g, int32_t n, const int32_t* ids, const void* const* pcm,
                                  const int64_t* n_frames, float* h_note, float* h_onset, float* h_contour,
                                  int64_t* h_frame_off);
int bp_stream_group_debug_tail(const bp_stream_group_t* g, int32_t id, float* h_out, int64_t capacity,
                               int64_t* first_sample, int64_t* n);
int bp_debug_pcm_stream_plan(int32_t sample_format, int32_t channels, int32_t sample_rate, int32_t n_pushes,
                             const int64_t* frames, int32_t ending, int64_t* out_lo, int64_t* out_hi, int64_t* hist_lo,
                             int64_t* hist_hi);

/* ---- stage 3 under a grid of decode parameters ------------------------------------------------
 * reference: note_creation.py:52-111 (model_output_to_notes without the MIDI object), called once per parameter set.
 * One call decodes the batch under each of params[0 .. n_params): every (setting, file) gets exactly the notes
 * bp_decode_device gives for that setting.  Settings that share a pitch range share the per-cell preparation; those
 * also sharing infer_onsets and onset_thresh share the onset candidates; the greedy loops run once per (file, setting),
 * in parallel.
 * Output layout: notes->note_off has n_params * n_files + 1 entries, parameter-major: the notes of setting p, file i
 * occupy [note_off[p*n_files+i], note_off[p*n_files+i+1]) in the reference's generation order; bend_off per note as in
 * bp_decode_device (a setting without include_pitch_bends has empty bend ranges).  Posteriorgrams are not modified.
 * Every setting is validated before anything is enqueued: a bad one returns BP_E_INVALID naming its index
 * ("decode params[7]: ...").  BP_E_CAPACITY: bp_last_required gives the capacities of the whole grid.  n_params == 0 or
 * n_files == 0: BP_OK with note_off[0] = 0.  The settings run in chunks (bp_decode_grid_chunk_params); the kernel
 * launches of a call depend on the number of chunks, not on n_params.  _device: posteriorgrams in device memory, work
 * on `stream`, synchronised before returning; _host: host posteriorgrams, uploaded once for all settings (h_contour may
 * be NULL when no setting has include_pitch_bends). */
int bp_decode_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                          const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                          int32_t n_params, bp_notes_t* notes, void* stream);
int bp_decode_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                        const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                        bp_notes_t* notes);
/* Host-only: settings per chunk of a grid decode over a batch of this shape (>= 1).  A chunk of c settings keeps its
 * device workspace within 2 GiB, c * W <= 2^31 bytes, unless one setting alone needs more (c = 1), where
 *   W = 4 C + 4 (C / 32 + 2) + 8 * 88 * (F / 256 + n_files + 1) + 12 min(C, 8 F + 64 n_files) + 16 n_files + 64
 * bytes, F = total_frames, C = 88 F: per setting its "remaining energy" copy, a candidate bitmap, the block maxima of the
 * melodia loop, the first allowance of note slots and per-file counters.  A (setting, file) that outgrows its first
 * allowance of note slots reruns its chunk with 88 T slots for that pair, beyond this budget. */
int64_t bp_decode_grid_chunk_params(int64_t total_frames, int32_t n_files);

/* ---- note-level scores of decoded notes against reference notes ------------------------------------------------------
 * No reference counterpart: the counts behind mir_eval.transcription 0.7 (match_notes + precision_recall_f1_overlap)
 * with strict=False, with and without offsets.  A reference note i and an estimated note j of the same file match when,
 * in float64 and in this order of operations,
 *   onset:  rint(|on_i - on_j| * 10000) / 10000 <= onset_tolerance            (np.around(., 4), round half to even)
 *   pitch:  |1200 * (log2_hz_i - log2_hz_j)| <= pitch_tolerance               (cents)
 *   offset: rint(|off_i - off_j| * 10000) / 10000 <= max(offset_ratio * |off_i - on_i|, offset_min_tolerance)
 * (the offset test in the "with offsets" pass only).  The matched count of a pass is the size of a maximum matching of
 * that hit graph.  Per (setting, file) or item the result is four counts: {n_ref, n_est, matched without offsets,
 * matched}; precision, recall and F follow from them (basic_pitch_b200/evaluate.py).
 * Notes of set i are [note_off[i], note_off[i+1]); note_off[0] must be 0.  Every note needs finite values, onset >= 0
 * and offset > onset; every tolerance must be finite and >= 0.  Violations return BP_E_INVALID before anything is
 * enqueued, naming the file or item and the note index ("references file 3 note 17: offset <= onset"). */
typedef struct bp_note_set {
  const int64_t* note_off;  /* [n + 1] */
  const double* onset_s;
  const double* offset_s;
  const double* log2_hz;    /* np.log2 of the pitch in Hz */
} bp_note_set_t;

typedef struct bp_score_params {
  double onset_tolerance;      /* seconds, default 0.05 */
  double pitch_tolerance;      /* cents, default 50 */
  double offset_ratio;         /* default 0.2 */
  double offset_min_tolerance; /* seconds, default 0.05 */
} bp_score_params_t;
void bp_default_score_params(bp_score_params_t* p);

/* Host-only: the seconds of frames 0 .. n-1, the bits model_frames_to_time gives (basic_pitch_b200/note_creation.py;
 * reference: note_creation.py:346-357). */
int bp_frame_times(int64_t n, double* out);

/* Grid scoring: bp_decode_grid_* without the contour, and instead of returning the notes, each (setting, file)'s notes
 * are scored on the device against file i's references (refs: one set per file, uploaded once per call).  An estimated
 * note (start_frame, end_frame, pitch_midi) has onset / offset bp_frame_times of its frames and log2_hz
 * est_log2_hz[pitch_midi] (a 128-entry host table, finite).  Amplitudes and pitch bends are not computed
 * (include_pitch_bends is ignored) and no note crosses to the host.  h_counts [n_params][n_files][4] (host).
 * Settings are validated, grouped and chunked as in bp_decode_grid_*.  Kernel launches per chunk: those of the grid
 * decode (3, or 1 when every file is empty; again as many when a pair outgrows its first allowance of note slots and
 * the chunk reruns) + 1 match kernel, whatever the number of settings in the chunk.  Device workspace beyond the
 * decode's: 8 bytes per reference and setting of a chunk, 16 bytes per note slot.
 * _device: posteriorgrams in device memory, work on `stream`, synchronised before returning; _host: host
 * posteriorgrams, uploaded once. */
int bp_score_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const int64_t* h_frame_off,
                         int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                         const bp_score_params_t* score, const double* est_log2_hz, int64_t* h_counts, void* stream);
int bp_score_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const int64_t* h_frame_off,
                       int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                       const bp_score_params_t* score, const double* est_log2_hz, int64_t* h_counts);
/* Item i's estimated notes (est, explicit) scored against item i's references; h_counts [n_items][4].  One kernel
 * launch (none for n_items == 0), synchronous. */
int bp_score_notes_host(bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs, int32_t n_items,
                        const bp_score_params_t* score, int64_t* h_counts);

/* ---- mir_eval's note matching pair for pair ------------------------------------------------------------------------
 * No reference counterpart: which estimated note mir_eval.transcription 0.7 (match_notes, strict=False) matches to each
 * reference note, with and without offsets.  The average overlap ratio and the note scores with velocity
 * (mir_eval.transcription_velocity) depend on these pairs, not only on their number; the host turns them into floats
 * with mir_eval's own NumPy expressions (basic_pitch_b200/evaluate.py, matching_scores).
 * Hits are those of bp_score_* above.  With the references and estimates of one (setting, file) or item:
 *  1. Graph (match_notes): G maps each estimate j with at least one hit to the list of references it hits, in ascending
 *     reference index; its keys are ordered by (smallest reference index hitting j, then j), the order in which j first
 *     appears in the row-major np.where of the hit matrix.  Indices are the caller's order within the set (not the
 *     (bucket, onset) order the library sorts references into), so the matching depends on the order of the estimate
 *     list: grid estimates are in the order bp_decode_grid_* returns them; callers wanting another order pass explicit
 *     notes to bp_match_notes_host.
 *  2. Matching (util._bipartite_match, Hopcroft-Karp), with "for x in d" walking dict d in insertion order:
 *       matching = {}                                        # reference v -> estimate u
 *       for u in G: for v in G[u]: if v not in matching: matching[v] = u; break
 *       loop:
 *         preds = {}; unmatched = []
 *         pred = {u: UNMATCHED for u in G}; del pred[matching[v]] for every v in matching
 *         layer = list(pred)                                 # the free estimates, in key order
 *         while layer and not unmatched:
 *           new_layer = {}                                   # v -> [u, ...], insertion-ordered
 *           for u in layer: for v in G[u]: if v not in preds: new_layer.setdefault(v, []).append(u)
 *           layer = []
 *           for v in new_layer:
 *             preds[v] = new_layer[v]
 *             if v in matching: layer.append(matching[v]); pred[matching[v]] = v
 *             else: unmatched.append(v)
 *         if not unmatched: return matching
 *         recurse(v): if v in preds: L = preds.pop(v)
 *                         for u in L: if u in pred: pu = pred.pop(u)
 *                                         if pu is UNMATCHED or recurse(pu): matching[v] = u; return True
 *                     return False
 *         for v in unmatched: recurse(v)
 *  3. The result is sorted(matching.items()): h_match gives, per reference in the caller's order, the estimate index it
 *     is matched to or -1.  Its number of matches is the matched count of bp_score_*.
 * Pass 0 has no offset test (offset_ratio=None), pass 1 has it.  Each (pair, pass) is one device thread that builds its
 * G (lists by insertion sort, keys by a counting sort on the first reference, stable in j) and runs these steps with
 * arrays and an explicit stack in place of the recursion.
 * Kernel launches: one count launch (hits without the offset test per pair, which size the workspace), then one match
 * launch per range of consecutive pairs whose workspace fits 2 GiB; a pair that needs more runs alone.  Workspace of a
 * pair with N estimates, R references and M hits without the offset test: 8 (3 M + 5 N + 8 R + 8) bytes (both passes).
 * No launch for a chunk without estimated notes or a call without references (every entry -1).
 *
 * Grid: bp_score_grid_*'s inputs; the notes come back in `notes` exactly as bp_decode_grid_* gives them (amplitudes,
 * empty bend ranges: include_pitch_bends is ignored; capacities and BP_E_CAPACITY / bp_last_required as there), and
 * h_match [n_params][2][n_refs_total] (int32, host).  Per chunk: the grid decode's launches, the compaction and
 * amplitude launches of bp_decode_grid_*, then the count and match launches above.  Settings, references and
 * tolerances are validated as in bp_score_grid_* before anything is enqueued. */
int bp_match_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const int64_t* h_frame_off,
                         int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                         const bp_score_params_t* score, const double* est_log2_hz, bp_notes_t* notes, int32_t* h_match,
                         void* stream);
int bp_match_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const int64_t* h_frame_off,
                       int32_t n_files, const bp_decode_params_t* params, int32_t n_params, const bp_note_set_t* refs,
                       const bp_score_params_t* score, const double* est_log2_hz, bp_notes_t* notes, int32_t* h_match);
/* Item i's estimated notes (est, explicit, in the order given) matched against item i's references; h_match
 * [2][n_refs_total].  Validation as bp_score_notes_host; synchronous. */
int bp_match_notes_host(bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs, int32_t n_items,
                        const bp_score_params_t* score, int32_t* h_match);

/* ---- onset-only and offset-only note scores --------------------------------------------------------------------------
 * No reference counterpart: the counts behind mir_eval.transcription 0.7's onset_precision_recall_f1 (match_note_onsets)
 * and offset_precision_recall_f1 (match_note_offsets) with strict=False.  A reference note i and an estimated note j of
 * the same file or item hit, in float64 and with the operations and order of bp_score_* above, when
 *   onset test:  rint(|on_i - on_j| * 10000) / 10000 <= onset_tolerance
 *   offset test: rint(|off_i - off_j| * 10000) / 10000 <= max(offset_ratio * |off_i - on_i|, offset_min_tolerance)
 * Pitch plays no part.  The matched count of a test is the size of a maximum matching of its hit graph.  Per (setting,
 * file) or item the result is four int64 counts: {n_ref, n_est, onsets matched, offsets matched}; precision, recall and
 * F follow from them as for bp_score_* (basic_pitch_b200/evaluate.py, onset_offset_scores).
 * Inputs are those of bp_score_*, except that the pitches are not read: log2_hz of a note set and est_log2_hz may be
 * NULL.  pitch_tolerance is validated as elsewhere and then ignored; intervals are validated as in bp_score_* (finite,
 * onset >= 0, offset > onset, the failing file or item and note named), before anything is enqueued.
 * Method: with a pair's estimates in ascending order of the tested time, every reference hits one contiguous run of
 * them (|fl(t_i - t_j)| does not decrease as t_j moves away from t_i, and the rounding is monotone), so the graph is
 * convex.  One device thread per (pair, test) sorts the tested times (decode slots: a heap sort of the frame indices,
 * bp_frame_times being strictly increasing; explicit estimates: sorted on the host), finds each reference's run by two
 * binary searches with the exact predicate, counting-sorts the references by run end and gives each in turn the smallest
 * free estimate of its run (a next-free array with path halving).  That greedy is exact on a convex graph.  Workspace of
 * a pair with N estimate slots and R references: 8 (2 N + 3 R + 1) bytes (both tests).
 *
 * Grid: bp_score_grid_*'s arguments and h_counts [n_params][n_files][4] (host).  Settings are validated, grouped and
 * chunked, and slot reruns happen, as in bp_decode_grid_*.  Kernel launches per chunk: those of the grid decode + 1,
 * whatever the number of settings.  Device workspace beyond the decode's: 24 bytes per reference and setting of a
 * chunk, 16 bytes per note slot and 8 bytes per (setting, file).  No note crosses to the host.  _device: posteriorgrams
 * in device memory, work on `stream`, synchronised before returning; _host: host posteriorgrams, uploaded once. */
int bp_score_onset_offset_grid_device(bp_model_t* m, const float* d_note, const float* d_onset,
                                      const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                      int32_t n_params, const bp_note_set_t* refs, const bp_score_params_t* score,
                                      const double* est_log2_hz, int64_t* h_counts, void* stream);
int bp_score_onset_offset_grid_host(bp_model_t* m, const float* h_note, const float* h_onset,
                                    const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                    int32_t n_params, const bp_note_set_t* refs, const bp_score_params_t* score,
                                    const double* est_log2_hz, int64_t* h_counts);
/* Item i's estimated notes (explicit, in any order: the counts do not depend on it) against item i's references;
 * h_counts [n_items][4].  One kernel launch (none for n_items == 0), synchronous. */
int bp_score_onset_offset_notes_host(bp_model_t* m, const bp_note_set_t* est, const bp_note_set_t* refs,
                                     int32_t n_items, const bp_score_params_t* score, int64_t* h_counts);

/* ---- frame-level multi-pitch scores of decoded notes against reference frames -------------------------------------
 * No reference counterpart: the sums behind mir_eval.multipitch.metrics 0.7 (window = 0.5 semitones by default).
 * A series is a time array time[0 .. N) (seconds, non-decreasing) and per frame a multiset of values, each carried as
 * two float64 numbers computed by the caller: midi = 69 + 12 log2(hz / 440) and chroma = mod(mod(midi, 12), 12), in
 * [0, 12) (basic_pitch_b200/evaluate.py, multipitch_values).  The library only subtracts, adds, takes absolute values
 * and compares, in float64, round to nearest, never contracted.
 *  1. Time base: reference frame k reads estimate frame k when n_est == n_ref and every
 *     |est_t - ref_t| <= 1e-8 + 1e-5 |ref_t| (np.allclose); otherwise the frame scipy.interpolate.interp1d(est_t,
 *     arange(n_est), kind='nearest', bounds_error=False, fill_value=n_est) gives at ref_t: bounds x_k / 2 + x_k+1 / 2,
 *     the number of bounds below ref_t, clipped to n_est - 1; ref_t < est_t[0] or > est_t[n_est - 1] reads an empty
 *     frame, as does every frame of an empty estimate.  bp_multipitch_map returns this map.
 *  2. Hits within a frame: plain, r and e hit when fl(e - w) <= r <= fl(e + w) (midi values); chroma, d = |r - e| and
 *     min(d, fl(12 - d)) <= w (chroma values).
 *  3. tp_k is the size of a maximum matching of frame k's hit graph; every element of a multiset is a vertex.
 *  4. Per (setting, file) or item, seven int64 sums over the reference frames k, with R_k, E_k the frame's multisets:
 *     {n_ref = sum |R_k|, n_est = sum |E_k|, tp = sum tp_k, tp_chroma = sum tp_chroma_k, n_min = sum min(|R_k|, |E_k|),
 *      miss = sum max(0, |R_k| - |E_k|), fa = sum max(0, |E_k| - |R_k|)}.
 *     Precision tp / n_est, recall tp / n_ref, accuracy tp / (n_est + n_ref - tp), and the error rates
 *     (n_min - tp, miss, fa, n_min + miss + fa - tp) / n_ref follow bit for bit in float64 (0 for a zero denominator;
 *     evaluate.frame_scores); the chroma versions use tp_chroma.
 * Validation, before anything is enqueued, returns BP_E_INVALID naming the file or item and the frame or value
 * ("references file 3 frame 17 value 2: chroma outside [0, 12)"): offsets starting at 0 and never decreasing, at most
 * 2^31 - 1 frames per set and values per frame, times finite, >= 0 and non-decreasing within a set, midi finite, chroma
 * in [0, 12); window finite and >= 0. */
typedef struct bp_multipitch_set {
  const int64_t* frame_off; /* [n + 1]: frames of set i are [frame_off[i], frame_off[i+1]) */
  const double* time_s;     /* [frames] */
  const int64_t* value_off; /* [frames + 1]: values of frame j are [value_off[j], value_off[j+1]); value_off[0] == 0 */
  const double* midi;       /* [values] */
  const double* chroma;     /* [values] */
} bp_multipitch_set_t;

/* Host-only: the reference -> estimate frame map of rule 1 (out[k] = -1: empty frame).  est_t must be finite and
 * non-decreasing, ref_t finite. */
int bp_multipitch_map(const double* est_t, int64_t n_est, const double* ref_t, int64_t n_ref, int64_t* out);

/* Grid frame scoring: bp_score_grid_* with frame-level counts.  The estimate series of (setting, file) has the file's
 * T model frames, times bp_frame_times(T); frame t holds one value per decoded note with start_frame <= t < end_frame,
 * est_midi[pitch_midi] / est_chroma[pitch_midi] (two 128-entry host tables: midi finite and non-decreasing, chroma in
 * [0, 12)).  Pitch bends are not applied (bp_score_bent_frames_grid_* applies them).  That is the piano roll of the
 * note events, sampled at the model frames.
 * refs: one series per file.  h_counts [n_params][n_files][7] (host), in the order of rule 4.
 * Settings are validated, grouped, chunked and rerun as in bp_decode_grid_*.  Kernel launches per chunk: those of the
 * grid decode + 3 (note-count roll scatter, its prefix sum along frames, the match kernel), whatever the number of
 * settings and files; the roll is zeroed with one memset.  Device workspace beyond the decode's: the roll reuses each
 * setting's "remaining energy" copy (int [88][T] per file); the chroma matching takes 16 bytes per reference value and 8
 * per reference frame, per setting of a chunk.
 * _device: posteriorgrams in device memory, work on `stream`, synchronised before returning; _host: host
 * posteriorgrams, uploaded once. */
int bp_score_frames_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const int64_t* h_frame_off,
                                int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                                const bp_multipitch_set_t* refs, double window, const double* est_midi,
                                const double* est_chroma, int64_t* h_counts, void* stream);
int bp_score_frames_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const int64_t* h_frame_off,
                              int32_t n_files, const bp_decode_params_t* params, int32_t n_params,
                              const bp_multipitch_set_t* refs, double window, const double* est_midi,
                              const double* est_chroma, int64_t* h_counts);
/* Grid frame scoring of the bent notes: the series `predict` hands its users, notes with their pitch bends.
 * Bent value: a decoded note of pitch p sounding at model frame t (start_frame <= t < end_frame) has the contour bin
 * k = 3 (p - 21) + b, b its pitch bend at t as bp_decode_grid_* returns it (reference: get_pitch_bends,
 * n_bins_tolerance 25: the arg-max window is clipped to the 264 contour bins, so k lies in [0, 263]); b = 0 under a
 * setting without include_pitch_bends.  The bend is an arg-max over contour row t around bin 3 (p - 21): it depends on
 * (file, p, t) only, so notes of one pitch overlapping at t carry the same bend and the count roll of
 * bp_score_frames_grid_* still describes the estimate.
 * The estimate series of (setting, file) has the file's T model frames at bp_frame_times(T); frame t holds
 * bin_midi[k] / bin_chroma[k] once per sounding note (264-entry host tables: midi finite and non-decreasing, chroma in
 * [0, 12); evaluate.bent_bins passes multipitch_values of evaluate.BENT_HZ, 440 * 2^((21 + k / 3 - 69) / 12), whose
 * entries 3 c are bit for bit midi_to_hz(21 + c)).  Rules 1 to 4 then apply unchanged; evaluate.note_frames_to_multipitch
 * is the host definition.  With every setting's bends off the counts equal bp_score_frames_grid_*'s with the matching
 * 128-entry tables.
 * Arguments as bp_score_frames_grid_* plus the contour posteriorgram, float32 row-major [total_frames][264], which may
 * be NULL only when no setting has include_pitch_bends (as for bp_decode_grid_*; the message names the first setting
 * that has).  Validation as bp_score_frames_grid_*, the tables named "bin table entry k".
 * Kernel launches per chunk: those of the grid decode + 3 (roll scatter, roll prefix sum, match), whatever the number of
 * settings and files; per call one memset of the counts, per chunk one of the roll.  The match thread of a frame puts
 * its sounding pitches' (key, count) groups in ascending key order (bends can move a pitch past others up to 16
 * semitones away) with an insertion sort in a 704-byte local array.  Device workspace as bp_score_frames_grid_*, plus 4
 * bytes per setting; chunks as bp_decode_grid_chunk_params. */
int bp_score_bent_frames_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                                     const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                     int32_t n_params, const bp_multipitch_set_t* refs, double window,
                                     const double* bin_midi, const double* bin_chroma, int64_t* h_counts, void* stream);
int bp_score_bent_frames_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                                   const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                   int32_t n_params, const bp_multipitch_set_t* refs, double window,
                                   const double* bin_midi, const double* bin_chroma, int64_t* h_counts);
/* Item i's estimate series (est, explicit) scored against item i's reference series; h_counts [n_items][7].  One
 * kernel launch and one memset (none for n_items == 0), synchronous.  Workspace: 16 bytes per reference value and 8 per
 * reference frame. */
int bp_score_multipitch_host(bp_model_t* m, const bp_multipitch_set_t* est, const bp_multipitch_set_t* refs,
                             int32_t n_items, double window, int64_t* h_counts);

/* ---- frame-level multi-pitch scores of a posteriorgram read as a multi-f0 estimate ---------------------------------
 * No reference counterpart: the estimate the reference's training targets define (the contour posteriorgram is trained
 * against multi-f0 annotations on FREQ_BINS_CONTOURS), scored by rules 1 to 4 above for a grid of settings.
 * The posteriorgram G has `width` bins per frame, float32 row-major [total_frames][width]; file i is frames
 * [h_frame_off[i], h_frame_off[i+1]), the layout of bp_run_inference_*.  bin_midi[width] / bin_chroma[width] carry the
 * value of each bin (host tables: midi finite and non-decreasing, chroma in [0, 12)); basic_pitch_b200/evaluate.py,
 * salience_bins, passes multipitch_values of constants.FREQ_BINS_CONTOURS or FREQ_BINS_NOTES, the reference's target
 * grids (not midi_to_hz: the bits differ).
 * Under a setting, bin b of frame t is an estimate of that frame when
 *   bin_lo <= b < bin_hi, and
 *   (double) G[t][b] >= threshold, in float64, and
 *   with peak_pick: 1 <= b <= width - 2, G[t][b] > G[t][b-1] and G[t][b] > G[t][b+1], in float32 on the whole row
 *   (not only [bin_lo, bin_hi)).
 * The peak test is scipy.signal.argrelmax(G, axis=1) (order 1, mode 'clip': the edge bins are never peaks), picked
 * before the threshold as DeepSalience's pitch_activations_to_mf0 does.  Every comparison is an IEEE ordered comparison:
 * a NaN cell is never an estimate and never below a peak.  The threshold test is in float64 because NumPy 2 compares a
 * float32 array with a Python float in float32, which answers differently for a threshold between two float32 values;
 * the host definition (evaluate.salience_to_multipitch) casts the posteriorgram to float64 first.
 * The estimate series of (setting, file) has the file's T model frames at bp_frame_times(T); frame t holds its estimate
 * bins in ascending bin order (ascending midi).  Rules 1 to 4 then apply unchanged.
 * h_counts [n_params][n_files][7] (host), in the order of rule 4.
 * Validation, before anything is enqueued, returns BP_E_INVALID naming the index ("salience params[3]: threshold must
 * be finite and > 0", "bin table entry 17: midi decreases"): 1 <= width <= 1024; every threshold finite and > 0;
 * peak_pick 0 or 1; 0 <= bin_lo <= bin_hi <= width; the bin tables as above; h_frame_off starting at 0, never
 * decreasing, at most 2^31 - 1 frames per file; the references and the window as for bp_score_frames_grid_*.
 * n_files == 0 or n_params == 0: BP_OK, nothing enqueued.  The settings run in chunks (bp_score_salience_chunk_params);
 * per call one memset of the counts, per chunk one launch of the match kernel, whatever the number of settings and
 * files: the predicate is evaluated from the posteriorgram row in the kernel, with no per-setting copy.  Device
 * workspace: the chroma matching's 16 bytes per reference value and 8 per reference frame, per setting of a chunk.
 * _device: posteriorgram in device memory, work on `stream`, synchronised before returning; _host: host posteriorgram,
 * uploaded once for all settings. */
typedef struct bp_salience_params {
  double threshold;  /* > 0, compared in float64 */
  int32_t peak_pick; /* 0 or 1 */
  int32_t bin_lo;    /* estimate bins are [bin_lo, bin_hi) */
  int32_t bin_hi;
  int32_t reserved;
} bp_salience_params_t;
int bp_score_salience_grid_device(bp_model_t* m, const float* d_gram, int32_t width, const int64_t* h_frame_off,
                                  int32_t n_files, const bp_salience_params_t* params, int32_t n_params,
                                  const bp_multipitch_set_t* refs, double window, const double* bin_midi,
                                  const double* bin_chroma, int64_t* h_counts, void* stream);
int bp_score_salience_grid_host(bp_model_t* m, const float* h_gram, int32_t width, const int64_t* h_frame_off,
                                int32_t n_files, const bp_salience_params_t* params, int32_t n_params,
                                const bp_multipitch_set_t* refs, double window, const double* bin_midi,
                                const double* bin_chroma, int64_t* h_counts);
/* Host-only: settings per chunk of bp_score_salience_grid_* for references of this size (>= 1): a chunk of c settings
 * keeps the chroma matching's workspace within 2 GiB, c = max(1, 2^31 / max(1, 16 n_ref_values + 8 n_ref_frames)). */
int64_t bp_score_salience_chunk_params(int64_t n_ref_frames, int64_t n_ref_values);

/* ---- melody scores: a posteriorgram or an f0 track read as a single-f0 estimate -----------------------------------
 * No reference counterpart: the counts behind mir_eval.melody.evaluate 0.7 with its defaults (hop=None, kind='linear',
 * base_frequency=10, binary voicing, no est_voicing / ref_reward), cent_tolerance as given (50 by default).
 * A series is a time array time[0 .. N) (seconds) and per frame cents and a voicing, computed by the caller from Hz f
 * (basic_pitch_b200/evaluate.py, melody_values): voiced = f > 0; cents = 1200 log2(|f| / 10) for f != 0, else 0 (a
 * negative f is an unvoiced pitch guess).  The library never takes a log; it subtracts, adds, multiplies, divides and
 * rounds in float64, round to nearest, never contracted.
 *  1. t = 0: a series whose first time is > 0 gets a frame at t = 0 copying its first frame's cents and voicing.  An
 *     inserted reference frame counts in every sum.
 *  2. Identity: when both series (after rule 1) have the same length and every |est_t - ref_t| <= 1e-8 + 1e-5 |ref_t|
 *     (np.allclose), reference frame k reads estimate frame k's raw cents and voicing.
 *  3. Otherwise both time arrays are rounded as np.round(x, 10) (x * 1e10, rint, / 1e10); estimate times must then be
 *     strictly increasing.  When the largest reference time exceeds the last estimate time, a sample at that time
 *     with cents 0 and voicing 0 is appended.  Held cents: a sample whose cents are 0 takes the previous sample's held
 *     cents; sample 0 keeps its own.  At a reference time x, with j the last sample whose time is <= x:
 *       voicing = voicing[j] (interp1d kind='zero');
 *       cents = 0 when cents[j] == 0; else held[j] when t_j == x; else slope (x - t_j) + held[j], slope =
 *       (held[j+1] - held[j]) / (t_{j+1} - t_j) (interp1d kind='linear' on float64 data, which is np.interp).
 *     bp_melody_map returns this map.  An estimate of no frames reads as voicing 0, cents 0 everywhere.
 *  4. Per (setting, file) or item, seven int64 counts over the reference frames (evaluate.MELODY_FIELDS): n_frames;
 *     ref_voiced; voiced_hit (both voiced); false_alarm (reference unvoiced, estimate voiced); pitch_correct (reference
 *     voiced, both cents != 0, d = |ref - est| < tol); chroma_correct (the same with |d - 1200 floor(d / 1200 + 0.5)|
 *     < tol); oa_voiced_correct (pitch_correct and the estimate voiced).
 *     Voicing recall voiced_hit / ref_voiced (1 without voiced reference frames), voicing false alarm false_alarm /
 *     (n_frames - ref_voiced) (0 for a zero denominator), raw pitch and raw chroma accuracy pitch_correct / ref_voiced
 *     and chroma_correct / ref_voiced (0 without voiced reference frames), overall accuracy (oa_voiced_correct +
 *     n_frames - ref_voiced - false_alarm) / n_frames (without voiced reference frames the first term is 0) follow bit
 *     for bit (all five 0 when n_frames == 0; evaluate.melody_scores).
 * Validation, before anything is enqueued, returns BP_E_INVALID naming the file or item and the frame ("references
 * file 3 frame 17: voiced where cents is 0"): offsets starting at 0 and never decreasing, at most 2^31 - 1 frames per
 * set; times finite, >= 0, non-decreasing and small enough to round (x * 1e10 finite), estimate times strictly
 * increasing after rules 1 and 3; cents finite; voiced 0 or 1, and 0 where cents is 0; cent_tolerance finite and > 0. */
typedef struct bp_melody_set {
  const int64_t* frame_off; /* [n + 1]: frames of set i are [frame_off[i], frame_off[i+1]) */
  const double* time_s;     /* [frames] */
  const double* cent;       /* [frames] */
  const int32_t* voiced;    /* [frames], 0 or 1 */
} bp_melody_set_t;

/* Host-only: the map of rules 1 to 3 for one pair of time bases, over the n_ref + (ref_t[0] > 0) reference frames of
 * rule 1.  out_t[3 k ..] = {x, t_j, t_{j+1}} and out_i[3 k ..] = {j, j + 1 (j on a knot), identity}, with j counted in
 * the estimate series after rule 1 and the appended sample (identity: x = t_j = t_{j+1} = ref_t, j = k).  An empty
 * estimate gives j = -1.  est_t and ref_t as in the validation above (est_t strictly increasing after rounding). */
int bp_melody_map(const double* est_t, int64_t n_est, const double* ref_t, int64_t n_ref, double* out_t, int64_t* out_i);

/* Grid melody scoring of a posteriorgram G (`width` bins per frame, float32 row-major [total_frames][width], file i
 * frames [h_frame_off[i], h_frame_off[i+1]): the layout of bp_run_inference_*).  bin_cent[width] holds the cents of
 * each bin (host table, finite and non-decreasing; evaluate.melody_bins passes melody_values of FREQ_BINS_CONTOURS /
 * FREQ_BINS_NOTES).  Under a setting, frame t of file i (time bp_frame_times(T)[t]) has
 *   b* = the bin in [bin_lo, bin_hi) with the largest float32 value, the lowest on a tie; NaN cells never win;
 *   voiced = (double) G[t][b*] >= threshold (float64, as for bp_score_salience_grid_*);
 *   cents = bin_cent[b*] when voiced, or when unvoiced with guess_unvoiced; else 0.  An empty range or a row of NaN
 *   cells in range gives cents 0, unvoiced.
 * (evaluate.salience_to_melody is the host definition.)  refs: one series per file.  h_counts [n_params][n_files][7]
 * (host), in the order of rule 4.  Validation as above, plus: 1 <= width <= 1024; every threshold finite and > 0;
 * 0 <= bin_lo <= bin_hi <= width; guess_unvoiced 0 or 1; the bin table; h_frame_off as for bp_score_salience_grid_*.
 * n_files == 0 or n_params == 0: BP_OK, nothing enqueued.  Per call one memset of the counts; per chunk of settings
 * (bp_score_melody_chunk_params) three launches whatever the number of settings and files: the arg-max of every
 * (distinct bin range, frame), the held cents of every (setting, file), the counts of every (setting, reference frame).
 * Device workspace: 16 bytes per frame and setting of a chunk, and 48 bytes per reference frame.
 * _device: posteriorgram in device memory, work on `stream`, synchronised before returning; _host: host posteriorgram,
 * uploaded once for all settings. */
typedef struct bp_melody_params {
  double threshold;       /* > 0, compared in float64 */
  int32_t bin_lo, bin_hi; /* b* is taken over [bin_lo, bin_hi) */
  int32_t guess_unvoiced; /* 0 or 1 */
  int32_t reserved;
} bp_melody_params_t;
int bp_score_melody_grid_device(bp_model_t* m, const float* d_gram, int32_t width, const int64_t* h_frame_off,
                                int32_t n_files, const bp_melody_params_t* params, int32_t n_params,
                                const bp_melody_set_t* refs, double cent_tolerance, const double* bin_cent,
                                int64_t* h_counts, void* stream);
int bp_score_melody_grid_host(bp_model_t* m, const float* h_gram, int32_t width, const int64_t* h_frame_off,
                              int32_t n_files, const bp_melody_params_t* params, int32_t n_params,
                              const bp_melody_set_t* refs, double cent_tolerance, const double* bin_cent,
                              int64_t* h_counts);
/* Item i's estimate track (explicit) scored against item i's reference track; h_counts [n_items][7].  One kernel
 * launch and one memset (none for n_items == 0), synchronous. */
int bp_score_melody_host(bp_model_t* m, const bp_melody_set_t* est, const bp_melody_set_t* refs, int32_t n_items,
                         double cent_tolerance, int64_t* h_counts);
/* Grid melody scoring of the bent notes: the decoded notes of every (setting, file), with their pitch bends, read as a
 * single-f0 track and scored by rules 1 to 4 above.  Frame t of the estimate (time bp_frame_times(T)[t]) holds the f0 of
 * one sounding pitch: among the pitches p with a note sounding at t, the one with the largest float32 note
 * posteriorgram value N[t][p - 21], the lowest pitch on a tie; a NaN loses to every number, so a frame whose sounding
 * cells are all NaN takes its lowest sounding pitch.  Its cents are bin_cent[k], k the bent value of
 * bp_score_bent_frames_grid_* (the setting's include_pitch_bends applies), voiced.  A frame with no sounding note has
 * cents 0, unvoiced; there is no unvoiced guess.  evaluate.note_frames_to_melody is the host definition; evaluate.bent_bins
 * gives the cents of evaluate.BENT_HZ.
 * Arguments: the grid decode's inputs (posteriorgrams, h_frame_off, settings; the contour as for
 * bp_score_bent_frames_grid_*), refs one reference track per file, cent_tolerance, bin_cent[264] (host table: finite,
 * non-decreasing and > 0).  h_counts [n_params][n_files][7] (host) in the order of rule 4 (evaluate.MELODY_FIELDS).
 * Validation before anything is enqueued: the grid decode's, cent_tolerance, the bin table ("bin table entry 17: cents
 * must be > 0"), at most 2^31 - 1 frames in all, the references as for bp_score_melody_grid_*.  n_files == 0 or
 * n_params == 0: BP_OK, nothing enqueued.
 * Kernel launches per chunk: those of the grid decode + 4 (roll scatter, roll prefix sum, one warp per (setting, file)
 * that picks, bends and holds every frame, the counts of every (setting, reference frame)); per call one memset of the
 * counts, per chunk one of the roll.  No note crosses to the host; the counts are integers reduced with integer atomics.
 * Device workspace beyond the decode's: the roll reuses the decode's "remaining energy" copies; 16 bytes per frame and
 * setting of a chunk (raw and held cents), at most 1/22 of the decode's own workspace (bp_decode_grid_chunk_params bounds
 * the chunk), and 48 bytes per reference frame.
 * _device: posteriorgrams in device memory, work on `stream`, synchronised before returning; _host: host
 * posteriorgrams, uploaded once. */
int bp_score_note_melody_grid_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                                     const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                     int32_t n_params, const bp_melody_set_t* refs, double cent_tolerance,
                                     const double* bin_cent, int64_t* h_counts, void* stream);
int bp_score_note_melody_grid_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                                   const int64_t* h_frame_off, int32_t n_files, const bp_decode_params_t* params,
                                   int32_t n_params, const bp_melody_set_t* refs, double cent_tolerance,
                                   const double* bin_cent, int64_t* h_counts);
/* Host-only: settings per chunk of bp_score_melody_grid_* for posteriorgrams of this many frames (>= 1): the arg-max
 * and held cents of a chunk of c settings stay within 2 GiB, c = max(1, 2^31 / max(1, 16 total_frames)). */
int64_t bp_score_melody_chunk_params(int64_t total_frames);

/* ---- every metric family of a batch under a settings grid, in one device pass --------------------------------------
 * No reference counterpart.  One request asks for any subset of the grid scorers above over the same batch; each
 * family's outputs are bit for bit those of its standalone call on the same posteriorgrams.  A family is requested when
 * its output pointer is non-NULL; its inputs are then those of its standalone entry point:
 *   notes            notes_counts [n_params][n_files][4]          bp_score_grid_*              (note_refs, score, est_log2_hz)
 *   onset_offset     onset_offset_counts [n_params][n_files][4]   bp_score_onset_offset_grid_* (note_refs, score)
 *   pairs            pair_notes + pair_match [n_params][2][R]     bp_match_grid_*              (note_refs, score, est_log2_hz)
 *   frames           frames_counts [n_params][n_files][7]         bp_score_frames_grid_*       (mp_refs, window, est_midi/chroma)
 *   bent_frames      bent_frames_counts [n_params][n_files][7]    bp_score_bent_frames_grid_*  (mp_refs, window, bin_midi/chroma)
 *   note_melody      note_melody_counts [n_params][n_files][7]    bp_score_note_melody_grid_*  (f0_refs, cent_tolerance, bin_cent)
 *   flat_note_melody flat_note_melody_counts, the same with every setting's include_pitch_bends taken as 0
 *   salience         salience_counts [n_salience][n_files][7]     bp_score_salience_grid_*     (own settings and references)
 *   melody           melody_counts [n_melody][n_files][7]         bp_score_melody_grid_*       (own settings and references)
 * The first seven are note-derived: they share params[0 .. n_params).  salience_gram / melody_gram pick the posteriorgram
 * the last two read: 0 the contour (264 bins), 1 the note posteriorgram (88 bins).
 * Order of work: every requested family is validated, with its standalone checks and messages prefixed by its name
 * ("bp_evaluate_host: frames: references file 3 frame 17 value 2: chroma outside [0, 12)"), before anything is
 * enqueued; each family's references are uploaded once.  Then one grid-decode chunk loop (chunk size
 * bp_evaluate_chunk_params) runs the decode once per chunk and, on that chunk's notes, the tail of every requested
 * note-derived family in the order of the table, each with the launches and workspace of its standalone tail.  Then
 * the salience and melody chunk loops run on the posteriorgrams as they are.  All counts come back in one copy, with one
 * synchronisation; the pairs' notes come back per chunk, as in bp_match_grid_* (BP_E_CAPACITY and bp_last_required as
 * there, after every family has run).
 * Kernel launches per decode chunk: those of the grid decode (3, or 1 when every file is empty; doubled when the chunk
 * reruns) + 1 (notes) + 1 (onset_offset) + bp_match_grid_*'s tail (pairs) + 3 (frames) + 3 (bent_frames) + 4
 * (note_melody) + 4 (flat_note_melody), for the requested families; k note-derived families thus save (k - 1) times the
 * decode's launches against k standalone calls.  Per salience chunk (bp_score_salience_chunk_params) 1 launch, per
 * melody chunk (bp_score_melody_chunk_params) 3.
 * n_files == 0 or no family requested: BP_OK, nothing enqueued.
 * _device: posteriorgrams (row-major, the layout of bp_run_inference_*) in device memory, work on `stream`, synchronised
 * before returning; _host: host posteriorgrams, uploaded once (the contour only when a family reads it). */
typedef struct bp_eval_request {
  const bp_decode_params_t* params; /* the grid of every note-derived family */
  int32_t n_params;
  int32_t reserved0;
  const bp_note_set_t* note_refs; /* one set per file */
  const bp_score_params_t* score;
  const double* est_log2_hz; /* [128] */
  int64_t* notes_counts;
  int64_t* onset_offset_counts;
  bp_notes_t* pair_notes; /* pairs: both non-NULL */
  int32_t* pair_match;
  const bp_multipitch_set_t* mp_refs; /* one series per file */
  double window;
  const double* est_midi, *est_chroma; /* [128] */
  int64_t* frames_counts;
  const double* bin_midi, *bin_chroma; /* [264] */
  int64_t* bent_frames_counts;
  const bp_melody_set_t* f0_refs; /* one track per file */
  double cent_tolerance;
  const double* bin_cent; /* [264] */
  int64_t* note_melody_counts;
  int64_t* flat_note_melody_counts;
  const bp_salience_params_t* salience_params;
  int32_t n_salience;
  int32_t salience_gram;
  const bp_multipitch_set_t* salience_refs;
  double salience_window;
  const double* salience_midi, *salience_chroma; /* [width] */
  int64_t* salience_counts;
  const bp_melody_params_t* melody_params;
  int32_t n_melody;
  int32_t melody_gram;
  const bp_melody_set_t* melody_refs;
  double melody_tolerance;
  const double* melody_cent; /* [width] */
  int64_t* melody_counts;
} bp_eval_request_t;
typedef struct bp_pcm_file bp_pcm_file_t; /* stored PCM of one file, defined below */
int bp_evaluate_device(bp_model_t* m, const float* d_note, const float* d_onset, const float* d_contour,
                       const int64_t* h_frame_off, int32_t n_files, const bp_eval_request_t* req, void* stream);
int bp_evaluate_host(bp_model_t* m, const float* h_note, const float* h_onset, const float* h_contour,
                     const int64_t* h_frame_off, int32_t n_files, const bp_eval_request_t* req);
/* The model's output and the evaluation of a batch in one call: the input of bp_run_inference_host (packed float32
 * audio) or of bp_transcribe_pcm_files_host (stored PCM).  The batch runs through the whole-file pipeline without a
 * decode; its posteriorgrams stay in the model's staging, where the request is scored as by bp_evaluate_device.
 * h_frame_off [n_files + 1] is always written; h_note / h_onset / h_contour (row-major, may be NULL) receive the
 * posteriorgrams, h_sample_off (PCM, may be NULL) the resampled lengths as offsets.  The request is validated against
 * the batch's frame offsets before any upload or launch.  Synchronous. */
int bp_evaluate_audio_host(bp_model_t* m, const float* h_audio, const int64_t* h_sample_off, int32_t n_files,
                           const bp_eval_request_t* req, float* h_note, float* h_onset, float* h_contour,
                           int64_t* h_frame_off);
int bp_evaluate_pcm_files_host(bp_model_t* m, const bp_pcm_file_t* files, int32_t n_files, const bp_eval_request_t* req,
                               float* h_note, float* h_onset, float* h_contour, int64_t* h_frame_off,
                               int64_t* h_sample_off);
/* Host-only: settings per decode chunk of bp_evaluate_* over a batch of this shape (>= 1): a chunk of c settings keeps
 * c * (W + X) <= 2^31 bytes unless c = 1, capped at 65535, where W is the grid decode's per-setting workspace
 * (bp_decode_grid_chunk_params) and X sums, over the requested note-derived families, with F = total_frames,
 * S = min(88 F, 8 F + 64 n_files) (a setting's first allowance of note slots), R the reference notes, K the reference
 * frames and V the reference values of mp_refs:
 *   notes 8 R + 16 S;  onset_offset 24 R + 16 S + 8 n_files;  pairs 8 R + 28 S;
 *   frames 16 V + 8 K;  bent_frames 16 V + 8 K + 4;  note_melody and / or flat_note_melody 16 F (shared).
 * The matching of pairs runs in its own launches of at most 2 GiB (bp_match_grid_*); salience and melody run their
 * own chunks. */
int64_t bp_evaluate_chunk_params(int64_t total_frames, int32_t n_files, const bp_eval_request_t* req);

/* ---- the whole path: predict() for a batch of files -------------------------------------------
 * reference: predict (basic_pitch/inference.py:431-506) minus file I/O and the MIDI object:
 * run_inference + model_output_to_notes.  Posteriorgram outputs are optional (pass NULL to keep
 * them on the device only).  `h_frame_off` [n_files+1] is always written.  bp_transcribe_host uploads the audio and
 * returns the posteriorgrams sub-batch by sub-batch, overlapped with the kernels, like bp_run_inference_host. */
int bp_transcribe_host(bp_model_t* m, const float* h_audio, const int64_t* h_sample_off, int32_t n_files,
                       const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                       int64_t* h_frame_off, bp_notes_t* notes);
int bp_transcribe_device(bp_model_t* m, const float* d_audio, const int64_t* h_sample_off, int32_t n_files,
                         const bp_decode_params_t* params, int64_t* h_frame_off, bp_notes_t* notes, void* stream);

/* ---- the two sub-steps of the decode the reference also exposes as functions --------------------------------------
 * bp_infer_onsets_host — reference: basic_pitch/note_creation.py:289-311 get_infered_onsets (n_diff = 2):
 *   out[t][f] (float64) = max(onsets, max(onsets) * frame_diff / max(frame_diff)) of one file, h_onset / h_note (T,88) f32.
 *   All-NaN when max(frame_diff) == 0, like the reference.
 * bp_pitch_bends_host — reference: note_creation.py:182-219 get_pitch_bends (n_bins_tolerance = 25): for every given
 *   note (start_frame, end_frame, pitch_midi) the per-frame pitch-bend estimates (1/3-semitone units) from the contour
 *   posteriorgram (T,264); h_bend_off[n_notes+1] receives the offsets into h_bends (BP_E_CAPACITY: "need N"). */
int bp_infer_onsets_host(bp_model_t* m, const float* h_onset, const float* h_note, int64_t n_frames, double* h_out);
int bp_pitch_bends_host(bp_model_t* m, const float* h_contour, int64_t n_frames, int32_t n_notes, const int32_t* h_start,
                        const int32_t* h_end, const int32_t* h_pitch_midi, int32_t* h_bend_off, int32_t* h_bends,
                        int64_t bend_capacity);

/* ---- introspection used by tests / profiling ----------------------------------------------------
 * Copies an internal activation of the most recent bp_forward_* call for window 0..n-1 to host.
 * which: 0 = CQT log-magnitude after normalisation+BN (n,172,309); 1 = contour conv1 output
 * (n,8,172,264); 2 = note conv1 output (n,32,172,88); 3 = onset conv1 output (n,32,172,88) — 2 and 3 exist only on
 * the FP32 path (bp_model_set_path(m, 0)) and 1 on paths 0 and 2: the tensor-core kernels reduce these activations
 * against the following convolution in their epilogues and never store them.
 * Only valid when the batch fitted in one internal chunk (n <= bp_model_chunk_windows). */
int bp_debug_activation(bp_model_t* m, int which, float* h_out, int64_t n_windows);
int64_t bp_model_chunk_windows(const bp_model_t* m);
/* Selects the arithmetic path: 0 = FP32 FFMA kernels everywhere; 1 = tensor-core kernels (wgmma, split-bf16
 * operands, FP32 accumulate) for the constant-Q projection and the three wide convolutions, each with the following
 * single-output convolution reduced in its epilogue (default); 2 = as 1 but the contour convolution stores its
 * 8-channel activations (bp_debug_activation which = 1). */
int bp_model_set_path(bp_model_t* m, int path);
/* Front-end buffers of the most recent forward call (same rule as bp_debug_activation: windows 0..n-1 of a call that
 * fitted in one chunk).  which:
 *   0 = the decimation chain x_1..x_8, float [n][stride] (bp_debug_chain_layout);
 *   1 = the raw log-magnitudes 10 log10(P + 1e-10) before normalisation, float [n][172][309]: on the tensor-core paths
 *       until bp_debug_activation(0) normalises them; otherwise only when bp_model_set_debug_frontend(m, 1) was on
 *       during the forward call;
 *   2 = the per-window min / max of the raw log-magnitudes, float [n][2];
 *   3 = the split operand of the contour / onset convs (paths 1 and 2), bf16 bits [2][chunks8][rows_stride][8] for
 *       the whole chunk (bp_debug_split_layout).
 * An id the last call did not produce is an error. */
int bp_debug_frontend(bp_model_t* m, int which, void* h_out, int64_t n_windows);
/* on != 0: every later forward call copies the raw log-magnitudes aside before normalising them (one device copy per
 * chunk, no extra kernel launch); 0 (default): the forward pass is exactly the one without this switch. */
int bp_model_set_debug_frontend(bp_model_t* m, int on);
/* Host-only: where x_o (o = 1..8) starts in one window's chain buffer (offsets[0] = -1: x_0 is the window itself), the
 * length of x_o (o = 0..8), and the floats per window. */
int bp_debug_chain_layout(int32_t* offsets, int32_t* lengths, int32_t* stride);
/* The split-operand layout of bp_debug_frontend(3): out[0] rows_stride (rows per plane and chunk of the buffer), out[1]
 * rows the last forward call wrote, out[2] lead rows, out[3] rows per window (172 frames + zero rows), out[4] chunks8
 * (8-bin chunks per row).  Row lead + b * rows_per_window + t holds frame t of window b. */
int bp_debug_split_layout(const bp_model_t* m, int32_t* out);

/* `bp_transcribe_host` for audio that is NOT packed: file i is audio[i][0 .. n_samples[i]) in ordinary (pageable) host
 * memory — what a caller holding one array per file has (reference: basic_pitch/inference.py:509-604, `predict_and_save`
 * loops `predict` over `audio_path_list`).  The library gathers the files sub-batch by sub-batch into pinned staging with
 * a few host threads, so that the gather and upload of sub-batch k+1 overlap the kernels of k; sub-batches are at most
 * two chunks of windows (four for packed input), which bounds that staging.  Everything else (the posteriorgrams
 * h_note / h_onset / h_contour, row-major [total_frames][88 | 88 | 264], any may be NULL, coming back per sub-batch;
 * h_frame_off, notes, errors) as bp_transcribe_host. */
int bp_transcribe_files_host(bp_model_t* m, const float* const* audio, const int64_t* n_samples, int32_t n_files,
                             const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                             int64_t* h_frame_off, bp_notes_t* notes);
/* Page-locked host memory for the outputs of the host entry points (cudaHostAlloc / cudaFreeHost); NULL on failure. */
void* bp_host_alloc(size_t bytes);
void bp_host_free(void* p);
/* After a BP_E_CAPACITY failure of a decode / transcribe call on this thread: the capacities that call needed
 * (0 = that one was sufficient), so that the caller can retry without parsing the error text. */
void bp_last_required(int64_t* note_capacity, int64_t* bend_capacity);

/* Audio ingest — `librosa.load(path, sr=22050, mono=True)` minus the container decode (reference:
 * basic_pitch/inference.py:239): interleaved PCM frames of `channels` channels at `sample_rate` Hz -> mono float32 at
 * 22 050 Hz.  sample_format: 0 float32, 1 int16 (/ 2^15), 2 int32 (/ 2^31; 24-bit WAV left-justified), 3 uint8
 * ((x - 128) / 128).  Channels are averaged in float32 in NumPy's order (`x.mean(axis=1, dtype=np.float32)`), so at
 * 22 050 Hz the output is the host loader's (basic_pitch_b200/audio_io.py) bit for bit; other rates go through a
 * Kaiser-windowed polyphase FIR (pass band 0.913 x Nyquist of the lower rate, 125 dB stop band) applied like
 * scipy.signal.resample_poly, each output within a per-element float32-accumulation bound of the float64 result
 * (DESIGN.md §4.4).  Rates needing more than 200 KB of staged input per 256 outputs (ratios beyond ~100:1, e.g.
 * 2 822 400 Hz) return BP_E_INVALID, as do formats outside 0..3 and channels or sample_rate below 1.  The output has
 * bp_resampled_length(n_frames, sample_rate) = ceil(n_frames * 22050 / sample_rate) samples.
 * _device: PCM and output in device memory, asynchronous on `stream` — the output can feed bp_transcribe_device directly;
 * _host: both in host memory (the PCM crosses PCIe as stored: 2 bytes per sample for 16-bit audio). */
int64_t bp_resampled_length(int64_t n_frames, int32_t sample_rate);
int bp_load_pcm_device(bp_model_t* m, const void* d_pcm, int32_t sample_format, int64_t n_frames, int32_t channels,
                       int32_t sample_rate, float* d_audio, void* stream);
int bp_load_pcm_host(bp_model_t* m, const void* h_pcm, int32_t sample_format, int64_t n_frames, int32_t channels,
                     int32_t sample_rate, float* h_audio);

/* One file of a batch as stored PCM: interleaved frames, format codes and conversions as bp_load_pcm_*. */
typedef struct bp_pcm_file {
  const void* pcm;       /* n_frames x channels samples; may be NULL when n_frames == 0 */
  int64_t n_frames;
  int32_t sample_format; /* 0 float32, 1 int16, 2 int32, 3 uint8 (a bp_pcm_source_t also takes 4 and 5) */
  int32_t channels;
  int32_t sample_rate;
  int32_t reserved;
} bp_pcm_file_t;

/* The ingest for a batch of files in one kernel launch — `librosa.load(path, sr=22050, mono=True)` minus the container
 * decode, which the reference calls once per file (basic_pitch/inference.py:239 inside predict, looped by
 * predict_and_save :509-604).  Files may differ in format, channel count and sample rate.  File i's signal has exactly
 * the bits bp_load_pcm_device gives for that file alone, wherever it sits in the batch.
 * Every file is validated before anything is enqueued: a format outside 0..3, channels or sample_rate below 1, a
 * negative length, a NULL pcm with frames, or a rate ratio beyond the limit of bp_load_pcm_device return BP_E_INVALID
 * with the file's index in bp_last_error() and leave the device untouched.  n_files == 0 is a valid empty call.
 * bp_load_pcm_files_device: files[i].pcm are device pointers aligned to their sample type; the 22 050 Hz signals are
 *   written back to back into d_audio (sum of bp_resampled_length samples) and their offsets into
 *   h_sample_off[n_files + 1] (written before the call returns); asynchronous on `stream`.  d_audio and h_sample_off
 *   feed bp_transcribe_device / bp_run_inference_device directly.
 * bp_transcribe_pcm_files_host: predict() for a batch of files given as stored PCM in ordinary (pageable) host memory —
 *   bp_transcribe_files_host with the ingest in front, on the same sub-batch pipeline: per sub-batch the library packs
 *   the files' PCM (every file starting on a 16-byte boundary) behind their descriptors in pinned staging, uploads that
 *   while the previous sub-batch computes, and one batched ingest leaves the signals on the device, where the forward
 *   pass reads them.  Each sample crosses PCIe once, as stored.  The staging (three pinned buffers, two on the device)
 *   is sized by the largest sub-batch in PCM bytes.  h_sample_off (may be NULL) receives the resampled lengths as
 *   offsets [n_files + 1]; everything else as bp_transcribe_files_host.  The same call as
 *   bp_transcribe_pcm_sources_host on in-memory sources. */
int bp_load_pcm_files_device(bp_model_t* m, const bp_pcm_file_t* files, int32_t n_files, float* d_audio,
                             int64_t* h_sample_off, void* stream);
int bp_transcribe_pcm_files_host(bp_model_t* m, const bp_pcm_file_t* files, int32_t n_files,
                                 const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                                 int64_t* h_frame_off, int64_t* h_sample_off, bp_notes_t* notes);

/* One file of a batch as stored PCM either in memory (path NULL: pcm as bp_pcm_file_t) or in a file: with `path`
 * non-NULL the n_frames x channels samples are bytes [data_offset, data_offset + size) of that file, as they lie in a
 * WAV file's data chunk (pcm.pcm is ignored), and the library reads them itself.  pcm.sample_format takes the four
 * formats of bp_pcm_file_t and two that WAV files bring: 4 packed signed 24-bit little-endian (3 bytes per sample,
 * 1-byte aligned; v / 2^23, bit for bit format 2 of v << 8) and 5 float64 (8 bytes; rounded to float32, then as
 * format 0).  Both cross PCIe as stored. */
typedef struct bp_pcm_source {
  bp_pcm_file_t pcm;
  const char* path;    /* NULL: in memory */
  int64_t data_offset; /* byte offset of the first sample in `path` (>= 0) */
} bp_pcm_source_t;

/* Host-only (no GPU needed): reads the header of each WAV file and either accepts it (accepted[i] = 1, out[i] the
 * source that reads its samples: format, channels, rate, frame count, path = paths[i] and the byte offset of the first
 * sample) or declines it (accepted[i] = 0, out[i] zeroed).  A file is accepted only when its reading is unambiguous and
 * agrees with scipy.io.wavfile.read (dtype, channels, rate, frames and sample bytes; 24-bit as scipy's int32 >> 8):
 *   - RIFF ... WAVE; chunks walked as id, little-endian size, body and a pad byte after an odd body, while the
 *     position is below the RIFF size + 8;
 *   - exactly one `fmt ` chunk before exactly one `data` chunk; other chunks anywhere are skipped;
 *   - format tag 1 (PCM; byte rate = rate x block_align), 3 (IEEE float) or 0xFFFE (EXTENSIBLE, cbSize >= 22) with the
 *     PCM or IEEE-float sub-format GUID; PCM of 8 / 16 / 24 / 32 bits -> formats 3 / 1 / 4 / 2, float of 32 / 64 bits ->
 *     formats 0 / 5; block_align = channels x bytes per sample, channels >= 1;
 *   - a sample rate the batched ingest takes;
 *   - a data size that is a multiple of block_align, with the whole data chunk inside the file.
 * Everything else is declined: RIFX, RF64 / W64, mu-law / A-law, ADPCM, 64-bit integer PCM, a missing or repeated
 * chunk, truncation, a path that does not exist or cannot be read.  BP_E_INVALID only for bad arguments (a NULL path). */
int bp_probe_wav_files(const char* const* paths, int32_t n_files, bp_pcm_source_t* out, int32_t* accepted);
/* bp_transcribe_pcm_files_host / bp_evaluate_pcm_files_host over sources: in-memory files are gathered as there, and a
 * file source is read with pread by the same gather threads straight into the pinned staging, each thread opening a
 * file once for its share of it; files are split across threads as in-memory ones are.  Every source is validated (as
 * bp_pcm_file_t, plus data_offset >= 0; a file source needs no pcm) and every length is known before any launch.  A
 * file that cannot be opened, fails to read or ends before its samples do (e.g. it shrank after the probe) returns
 * BP_E_IO with its index and path in bp_last_error(); the gather threads have ended, queued work has finished, outputs
 * are unspecified and the model works normally on its next call. */
int bp_transcribe_pcm_sources_host(bp_model_t* m, const bp_pcm_source_t* sources, int32_t n_files,
                                   const bp_decode_params_t* params, float* h_note, float* h_onset, float* h_contour,
                                   int64_t* h_frame_off, int64_t* h_sample_off, bp_notes_t* notes);
int bp_evaluate_pcm_sources_host(bp_model_t* m, const bp_pcm_source_t* sources, int32_t n_files,
                                 const bp_eval_request_t* req, float* h_note, float* h_onset, float* h_contour,
                                 int64_t* h_frame_off, int64_t* h_sample_off);
/* bp_load_pcm_files_device for in-memory sources (device pointers, aligned to their sample type: 1 byte for format 4)
 * with every source format; a source with a path is BP_E_INVALID. */
int bp_load_pcm_sources_device(bp_model_t* m, const bp_pcm_source_t* sources, int32_t n_files, float* d_audio,
                               int64_t* h_sample_off, void* stream);
/* Host-only (no GPU needed): validates the files as bp_load_pcm_files_device / bp_transcribe_pcm_files_host do and
 * returns where
 * bp_transcribe_pcm_files_host would pack them if they formed one sub-batch: file i's PCM at byte_off[i] (a multiple
 * of 16) from the first file's, byte_off[n_files] the size of the packed PCM; and sample_off[n_files + 1], the offsets
 * of their 22 050 Hz signals. */
int bp_debug_pcm_layout(const bp_pcm_file_t* files, int32_t n_files, int64_t* byte_off, int64_t* sample_off);
/* bp_debug_pcm_layout for sources, validated as bp_transcribe_pcm_sources_host validates them (formats 0..5). */
int bp_debug_pcm_sources_layout(const bp_pcm_source_t* sources, int32_t n_files, int64_t* byte_off,
                                int64_t* sample_off);

/* Batched writers (host threads, no GPU): one Standard MIDI File and / or one note-event CSV per file of a batch, straight
 * from the concatenated note arrays (times already in seconds).  Replaces, for batches, note_events_to_midi (reference:
 * basic_pitch/note_creation.py:222-271, incl. drop_overlapping_pitch_bends :274-286 when multiple_pitch_bends = 0) +
 * PrettyMIDI.write (inference.py:574-584) and save_note_events (inference.py:409-428).  File i owns notes
 * [note_off[i], note_off[i+1]); note j owns bends [bend_off[j], bend_off[j+1]) (bend_off may be NULL: no bends).
 * midi_paths / csv_paths: arrays of n_files paths (the array or single entries may be NULL = skip).  n_threads <= 0: auto.
 * A note's velocity is int(np.round(127 * amplitude)) of the float32 product, an exact integer of any size: the CSV
 * prints all its digits, the MIDI file clamps it to 0..127.  An amplitude that is NaN or whose product is +-inf (where
 * Python's int() raises) is BP_E_INVALID, before any file is written. */
int bp_write_note_files(int32_t n_files, const char* const* midi_paths, const char* const* csv_paths,
                        const int32_t* note_off, const double* start_s, const double* end_s, const int32_t* pitch_midi,
                        const float* amplitude, const int32_t* bend_off, const int32_t* bends,
                        int32_t multiple_pitch_bends, double midi_tempo, int32_t n_threads);

/* MIDI sonification of a batch of files on the GPU: for file i the float64 samples of
 * note_events_to_midi(events_i, multiple_pitch_bends).synthesize(sample_rate) with this package's additive stand-in
 * synthesiser (basic_pitch_b200/midi.py: PrettyMIDI.synthesize), which stands in for the reference's sonify_midi
 * (basic_pitch/note_creation.py:119-128, called by inference.py:586-592).  The note arrays are those of
 * bp_write_note_files (times in seconds, finite and >= 0; bend_off may be NULL).  h_sample_off[n_files + 1] is always
 * written: file i's samples are h_audio[h_sample_off[i] .. h_sample_off[i+1]), none for a file without notes.
 * h_audio == NULL is a size query (host only, no device work); otherwise `capacity` (in samples) must hold them all
 * (BP_E_CAPACITY).  sample_rate <= 0 or malformed offsets: BP_E_INVALID.  Each note is scaled by velocity / 127.0,
 * the velocity being int(np.round(127 * amplitude)) of the float32 product, unclamped and exact at any size; an
 * amplitude that is NaN or whose product is +-inf is BP_E_INVALID, with no device work.  Synchronous on the model's
 * device; the device buffers are sized per call (about 8 bytes per output sample), and a file is never split, so one
 * very long file is one unit of work.  Samples match the stand-in except for the rounding of the phase (DESIGN.md §4.4). */
int bp_sonify_notes_host(bp_model_t* m, int32_t n_files, const int32_t* note_off, const double* start_s,
                         const double* end_s, const int32_t* pitch_midi, const float* amplitude, const int32_t* bend_off,
                         const int32_t* bends, int32_t multiple_pitch_bends, int32_t sample_rate, int64_t* h_sample_off,
                         double* h_audio, int64_t capacity);

/* Host-only: the low-pass of the ingest resampler for the reduced ratio up / down (unit DC gain, before the gain `up`);
 * returns the number of taps, copies them if capacity allows.  Tests pin it against scipy.signal.firwin. */
int64_t bp_debug_resample_filter(int32_t up, int32_t down, double* taps, int64_t capacity);

/* Host-only (no GPU needed): builds the tensor-core plan (split-bf16 Toeplitz weight tiles and the per-group MMA
 * programs, csrc/tc_conv.cu) of the contour conv (which = 0, w = [8][8][3][39]), the onset conv (which = 1,
 * w = [32][8][5][5]) or the note conv (which = 2, w = [32][1][7][7]) so that tests can emulate the program on the CPU.  sizes[4] = {n_tiles, n_steps, n_uses,
 * n_groups}; pass NULL arrays to query sizes first.  tiles: n_tiles x 4096 bf16 ([plane hi/lo][k-chunk 2][n 128][8]);
 * slot_words: [2][n_steps]; group_step_off has n_groups + 1 entries, group_ft n_groups x 2.  The kernels run the
 * contour plan only; the onset and note plans pin the planner on stride-3 geometry (see bp_debug_tc_gather). */
int bp_debug_tc_plan(int which, const float* w, int32_t* sizes, uint16_t* tiles, int32_t* tile_seq, uint32_t* slot_words,
                     int32_t* group_step_off, int32_t* group_ft);

/* Host-only: the conv1 of the onset (which = 1, w = [32][8][5][5]) or note (which = 2, w = [32][1][7][7]) layer as the
 * kernel computes it, an implicit GEMM with a gathered A operand (csrc/tc_conv.cu, tc_build_b1).  sizes[4] = {K, n_ci, KH,
 * wout}; b1 (may be NULL): the two B matrices, [parity of the output bin 2][plane hi/lo][K / 8][32][8] bf16, row
 * k = 8 (dt * n_ci + ci) + j (the 8-bin-window form; the kernel's own K order is bp_debug_tc_gather_packed); starts (may
 * be NULL): [wout][n_ci] first input bin of the window of output bin f and channel ci; ranges (may be NULL): [n_ci][2]
 * the input bins [lo, hi) of each channel that hold data (zero elsewhere). */
int bp_debug_tc_gather(int which, const float* w, int32_t* sizes, uint16_t* b1, int32_t* starts, int32_t* ranges);
/* Host-only: the same B matrices in the K order the kernel runs (the onset packs its windows to 6 bins).  sizes[1] = {K};
 * b1 (may be NULL): [2][2][K / 8][32][8] bf16; kmap (may be NULL): [K][3] the (dt, ci, window bin j) of row k, all -1
 * for K padding.  Window starts and ranges are those of bp_debug_tc_gather. */
int bp_debug_tc_gather_packed(int which, const float* w, int32_t* sizes, uint16_t* b1, int32_t* kmap);

/* Host-only: the bf16 hi/lo weight tiles of the fused SECOND convolution of a tensor-core layer (csrc/tc_conv.cu, tc_build_b2):
 * which = 0 contour conv2 (w2 = [1][8][5][5], reference models.py:254-262), 1 onset conv2 ([1][33][3][3], models.py:305-313),
 * 2 note conv2 ([1][32][7][3], models.py:282-290).  sizes[5] = {n_tiles, N, time taps, accumulator columns, columns per output offset}; tiles
 * (may be NULL to query sizes): n_tiles x [plane hi/lo][k-chunk 2][n N][8] bf16. */
int bp_debug_tc_b2(int which, const float* w2, int32_t* sizes, uint16_t* tiles);

/* Host-only: the items one launch of a tensor-core conv kernel runs for a batch of n_windows on n_sms SMs (csrc/tc_conv.cu,
 * tc_schedule), which = 0 contour (fused != 0: with its conv2 fused, the forward path 1), 1 onset, 2 note.  CTA c of the
 * launch runs items c, c + grid, ...  sizes[8] = {n_items, grid, n_mtiles, whole M-tiles (items 0 .. n_full - 1),
 * group ranges of the other M-tiles, frames an M-tile finishes (ms), first frame row of the cut M-tiles (n_full * ms),
 * frequency groups}; items (may be NULL): [n_items][3] the item's M-tile and its groups [g0, g1); edges (may be NULL):
 * [2] bit b = boundary b between frequency tiles b - 1 and b is finished by edge_fix_kernel in the rows of whole M-tiles
 * (edges[0]) and in the rows of cut M-tiles (edges[1]). */
int bp_debug_tc_schedule(int which, int fused, int n_windows, int n_sms, int32_t* sizes, int32_t* items, uint32_t* edges);

/* Host-only: the row map of a tensor-core layer for n_windows windows (csrc/tc_conv.cu, tc_row_map), which = 0 contour,
 * 1 onset, 2 note.  trimmed = 0: the uniform map of whole windows (bp_forward_*); else the trimmed map the unwrapping
 * entry points run on path 1, kept[b] = the centre frames window b keeps (<= 0: none).  map (may be NULL when
 * n_windows = 0): [n_windows][3] = {base, first, rows}: input rows [base, base + rows) of the layer's row space hold
 * frames first .. first + rows - 1 of window b; info[3] = {rows of the row space, lo1, lo2}: conv1 row / output frame i
 * of a window is computed for use iff lo1 / lo2 <= i < rows - lo1 / lo2. */
int bp_debug_tc_row_map(int which, int trimmed, const int32_t* kept, int32_t n_windows, int32_t* map, int32_t* info);

/* Per-kernel device timing for the roofline line of bench.py: records CUDA events on the launching
 * stream around every launch of one kernel family (0 = contour conv 3x39, 1 = onset conv 5x5,
 * 2 = CQT projection + log-normalise, 3 = decimation chain, 4 = the remaining small convs,
 * 5 = decode (prep / candidates / sequential loops), 6 = amplitudes + pitch bends;
 * -1 = off, the default) and resets the accumulators.  bp_model_profile_read synchronises the device
 * and returns the summed interval time, the number of intervals and the windows processed. */
int bp_model_profile(bp_model_t* m, int which);
int bp_model_profile_read(bp_model_t* m, double* total_ms, int64_t* n_intervals, int64_t* n_windows);

/* Cycle accounting of the tensor-core conv kernels (tools/tc_clocks.py), available only in a library built with
 * -DBP_TC_CLOCKS (BP_E_INVALID otherwise).  Synchronises the device and copies the SM cycles summed over all warps of
 * all launches of layer `which` (0 contour, 1 onset, 2 note) since the last reset: cycles[8] = consumers waiting on a
 * weight stage, issuing / waiting for MMAs, in the epilogue, waiting on the data tile, other; producer waiting on a free
 * stage, waiting on the data tile to be released, other.  reset != 0 zeroes the sums after the copy. */
int bp_debug_tc_clocks(bp_model_t* m, int which, uint64_t* cycles, int reset);
/* Busy time of every CTA of the tensor-core conv kernels (tools/tc_balance.py), also only with -DBP_TC_CLOCKS.
 * Synchronises the device and copies ns[i] = the %globaltimer nanoseconds CTA i (blockIdx.x, i < n <= 256) spent from
 * its start to the end of its last MMA warp, summed over all launches of layer `which` since the last reset. */
int bp_debug_tc_cta_busy(bp_model_t* m, int which, uint64_t* ns, int n, int reset);

#ifdef __cplusplus
}
#endif
#endif /* BP_B200_H */
