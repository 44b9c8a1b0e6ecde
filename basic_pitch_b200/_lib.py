"""ctypes binding of the C ABI declared in include/bp_b200.h (libbp_b200.so, sm_90a).

There is no fallback of any kind: if the shared library is missing or no H100 is visible, loading or
model creation raises.  Build the library with `python -c "import __graft_entry__ as g; g.build()"`
or `make -C basic_pitch_b200/csrc`.
"""
from __future__ import annotations

import ctypes as C
import os
import pathlib
from typing import Optional

LIB_PATH = pathlib.Path(__file__).resolve().parent / "libbp_b200.so"

BP_OK = 0
BP_E_INVALID = -1
BP_E_CUDA = -2
BP_E_CAPACITY = -3
BP_E_NOMEM = -4
BP_E_IO = -5

EXPORTS = [
    "bp_version", "bp_last_error", "bp_default_decode_params", "bp_num_windows", "bp_num_frames",
    "bp_model_create", "bp_model_destroy", "bp_model_device", "bp_model_param_block", "bp_model_refresh",
    "bp_model_launch_count", "bp_forward_device", "bp_forward_host", "bp_run_inference_device",
    "bp_run_inference_host", "bp_decode_device", "bp_decode_host", "bp_transcribe_host", "bp_transcribe_device",
    "bp_infer_onsets_host", "bp_pitch_bends_host", "bp_debug_activation", "bp_model_chunk_windows", "bp_model_set_path", "bp_model_profile", "bp_model_profile_read", "bp_debug_tc_plan", "bp_debug_tc_gather", "bp_debug_tc_gather_packed", "bp_debug_tc_b2", "bp_debug_tc_schedule", "bp_debug_tc_row_map", "bp_debug_tc_clocks", "bp_debug_tc_cta_busy", "bp_transcribe_files_host", "bp_host_alloc", "bp_host_free", "bp_last_required", "bp_resampled_length", "bp_load_pcm_device", "bp_load_pcm_host", "bp_debug_resample_filter", "bp_write_note_files", "bp_sonify_notes_host", "bp_load_pcm_files_device", "bp_transcribe_pcm_files_host", "bp_debug_pcm_layout", "bp_debug_frontend", "bp_model_set_debug_frontend", "bp_debug_chain_layout", "bp_debug_split_layout", "bp_decode_grid_device", "bp_decode_grid_host", "bp_decode_grid_chunk_params", "bp_default_score_params", "bp_frame_times", "bp_score_grid_device", "bp_score_grid_host", "bp_score_notes_host", "bp_multipitch_map", "bp_score_frames_grid_device", "bp_score_frames_grid_host", "bp_score_multipitch_host", "bp_score_salience_grid_device", "bp_score_salience_grid_host", "bp_score_salience_chunk_params", "bp_match_grid_device", "bp_match_grid_host", "bp_match_notes_host", "bp_score_onset_offset_grid_device", "bp_score_onset_offset_grid_host", "bp_score_onset_offset_notes_host", "bp_melody_map", "bp_score_melody_grid_device", "bp_score_melody_grid_host", "bp_score_melody_host", "bp_score_melody_chunk_params", "bp_score_bent_frames_grid_device", "bp_score_bent_frames_grid_host", "bp_score_note_melody_grid_device", "bp_score_note_melody_grid_host", "bp_evaluate_device", "bp_evaluate_host", "bp_evaluate_audio_host", "bp_evaluate_pcm_files_host", "bp_evaluate_chunk_params", "bp_stream_create", "bp_stream_push_host", "bp_stream_end", "bp_stream_take", "bp_stream_held_frames", "bp_stream_destroy", "bp_stream_group_create", "bp_stream_group_open", "bp_stream_group_commit_offsets", "bp_stream_group_push_host", "bp_stream_group_push_frames_host", "bp_stream_group_end", "bp_stream_group_take", "bp_stream_group_held_frames", "bp_stream_group_destroy", "bp_stream_group_open_pcm", "bp_stream_group_push_pcm_host", "bp_stream_group_debug_tail", "bp_debug_pcm_stream_plan", "bp_probe_wav_files", "bp_transcribe_pcm_sources_host", "bp_evaluate_pcm_sources_host", "bp_load_pcm_sources_device", "bp_debug_pcm_sources_layout",
]  # fmt: skip


class DecodeParams(C.Structure):
    _fields_ = [
        ("onset_thresh", C.c_double),
        ("frame_thresh", C.c_double),
        ("min_note_len", C.c_int32),
        ("energy_tol", C.c_int32),
        ("infer_onsets", C.c_int32),
        ("melodia_trick", C.c_int32),
        ("include_pitch_bends", C.c_int32),
        ("min_pitch_idx", C.c_int32),
        ("max_pitch_idx", C.c_int32),
        ("reserved", C.c_int32),
    ]


class Notes(C.Structure):
    _fields_ = [
        ("note_capacity", C.c_int32),
        ("bend_capacity", C.c_int32),
        ("note_off", C.c_void_p),
        ("start_frame", C.c_void_p),
        ("end_frame", C.c_void_p),
        ("pitch_midi", C.c_void_p),
        ("amplitude", C.c_void_p),
        ("bend_off", C.c_void_p),
        ("bends", C.c_void_p),
    ]


class NoteSet(C.Structure):
    _fields_ = [
        ("note_off", C.c_void_p),
        ("onset_s", C.c_void_p),
        ("offset_s", C.c_void_p),
        ("log2_hz", C.c_void_p),
    ]


class MultipitchSet(C.Structure):
    _fields_ = [
        ("frame_off", C.c_void_p),
        ("time_s", C.c_void_p),
        ("value_off", C.c_void_p),
        ("midi", C.c_void_p),
        ("chroma", C.c_void_p),
    ]


class SalienceParams(C.Structure):
    _fields_ = [
        ("threshold", C.c_double),
        ("peak_pick", C.c_int32),
        ("bin_lo", C.c_int32),
        ("bin_hi", C.c_int32),
        ("reserved", C.c_int32),
    ]


class MelodySet(C.Structure):
    _fields_ = [
        ("frame_off", C.c_void_p),
        ("time_s", C.c_void_p),
        ("cent", C.c_void_p),
        ("voiced", C.c_void_p),
    ]


class MelodyParams(C.Structure):
    _fields_ = [
        ("threshold", C.c_double),
        ("bin_lo", C.c_int32),
        ("bin_hi", C.c_int32),
        ("guess_unvoiced", C.c_int32),
        ("reserved", C.c_int32),
    ]


class ScoreParams(C.Structure):
    _fields_ = [
        ("onset_tolerance", C.c_double),
        ("pitch_tolerance", C.c_double),
        ("offset_ratio", C.c_double),
        ("offset_min_tolerance", C.c_double),
    ]


class PcmFile(C.Structure):
    _fields_ = [
        ("pcm", C.c_void_p),
        ("n_frames", C.c_int64),
        ("sample_format", C.c_int32),
        ("channels", C.c_int32),
        ("sample_rate", C.c_int32),
        ("reserved", C.c_int32),
    ]


class PcmSource(C.Structure):
    """bp_pcm_source_t: stored PCM in memory (path None) or bytes [data_offset, ...) of a file."""

    _fields_ = [
        ("pcm", PcmFile),
        ("path", C.c_char_p),
        ("data_offset", C.c_int64),
    ]


class EvalRequest(C.Structure):
    """bp_eval_request_t: one block per metric family, a NULL output meaning "not requested"."""

    _fields_ = [
        ("params", C.c_void_p),
        ("n_params", C.c_int32),
        ("reserved0", C.c_int32),
        ("note_refs", C.c_void_p),
        ("score", C.c_void_p),
        ("est_log2_hz", C.c_void_p),
        ("notes_counts", C.c_void_p),
        ("onset_offset_counts", C.c_void_p),
        ("pair_notes", C.c_void_p),
        ("pair_match", C.c_void_p),
        ("mp_refs", C.c_void_p),
        ("window", C.c_double),
        ("est_midi", C.c_void_p),
        ("est_chroma", C.c_void_p),
        ("frames_counts", C.c_void_p),
        ("bin_midi", C.c_void_p),
        ("bin_chroma", C.c_void_p),
        ("bent_frames_counts", C.c_void_p),
        ("f0_refs", C.c_void_p),
        ("cent_tolerance", C.c_double),
        ("bin_cent", C.c_void_p),
        ("note_melody_counts", C.c_void_p),
        ("flat_note_melody_counts", C.c_void_p),
        ("salience_params", C.c_void_p),
        ("n_salience", C.c_int32),
        ("salience_gram", C.c_int32),
        ("salience_refs", C.c_void_p),
        ("salience_window", C.c_double),
        ("salience_midi", C.c_void_p),
        ("salience_chroma", C.c_void_p),
        ("salience_counts", C.c_void_p),
        ("melody_params", C.c_void_p),
        ("n_melody", C.c_int32),
        ("melody_gram", C.c_int32),
        ("melody_refs", C.c_void_p),
        ("melody_tolerance", C.c_double),
        ("melody_cent", C.c_void_p),
        ("melody_counts", C.c_void_p),
    ]


class BpError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libbp_b200 error {code}: {msg}")
        self.code = code


class BpIOError(BpError, OSError):
    """BP_E_IO: a file the library was reading could not be read (the message names it)."""


_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load libbp_b200.so (once) and declare every prototype of include/bp_b200.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.is_file():
        raise ImportError(
            f"{LIB_PATH} not found: the CUDA extension has not been built "
            "(run `make -C basic_pitch_b200/csrc`). There is no CPU fallback."
        )
    # BP_B200_LIB: load an instrumented build of the same library instead (tools/: trace / debug builds)
    lib = C.CDLL(os.environ.get("BP_B200_LIB") or str(LIB_PATH))
    vp, i32, i64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
    lib.bp_version.restype = C.c_int
    lib.bp_last_error.restype = C.c_char_p
    lib.bp_default_decode_params.argtypes = [C.POINTER(DecodeParams)]
    lib.bp_default_decode_params.restype = None
    lib.bp_num_windows.argtypes = [i64]
    lib.bp_num_windows.restype = i64
    lib.bp_num_frames.argtypes = [i64]
    lib.bp_num_frames.restype = i64
    lib.bp_model_create.argtypes = [vp, sz, C.c_int, C.POINTER(vp)]
    lib.bp_model_destroy.argtypes = [vp]
    lib.bp_model_destroy.restype = None
    lib.bp_model_device.argtypes = [vp]
    lib.bp_model_param_block.argtypes = [vp, C.POINTER(vp), C.POINTER(sz)]
    lib.bp_model_refresh.argtypes = [vp]
    lib.bp_model_launch_count.argtypes = [vp]
    lib.bp_model_launch_count.restype = i64
    lib.bp_model_chunk_windows.argtypes = [vp]
    lib.bp_model_chunk_windows.restype = i64
    lib.bp_model_set_path.argtypes = [vp, C.c_int]
    lib.bp_forward_device.argtypes = [vp, vp, i64, vp, vp, vp, vp]
    lib.bp_forward_host.argtypes = [vp, vp, i64, vp, vp, vp]
    lib.bp_run_inference_device.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp]
    lib.bp_run_inference_host.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp]
    lib.bp_decode_device.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), C.POINTER(Notes), vp]
    lib.bp_decode_host.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), C.POINTER(Notes)]
    lib.bp_decode_grid_device.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(Notes), vp]
    lib.bp_decode_grid_host.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(Notes)]
    lib.bp_decode_grid_chunk_params.argtypes = [i64, i32]
    lib.bp_decode_grid_chunk_params.restype = i64
    lib.bp_default_score_params.argtypes = [C.POINTER(ScoreParams)]
    lib.bp_default_score_params.restype = None
    lib.bp_frame_times.argtypes = [i64, vp]
    lib.bp_score_grid_device.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(NoteSet),
                                         C.POINTER(ScoreParams), vp, vp, vp]
    lib.bp_score_grid_host.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(NoteSet),
                                       C.POINTER(ScoreParams), vp, vp]
    lib.bp_score_notes_host.argtypes = [vp, C.POINTER(NoteSet), C.POINTER(NoteSet), i32, C.POINTER(ScoreParams), vp]
    lib.bp_match_grid_device.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(NoteSet),
                                         C.POINTER(ScoreParams), vp, C.POINTER(Notes), vp, vp]
    lib.bp_match_grid_host.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(NoteSet),
                                       C.POINTER(ScoreParams), vp, C.POINTER(Notes), vp]
    lib.bp_match_notes_host.argtypes = [vp, C.POINTER(NoteSet), C.POINTER(NoteSet), i32, C.POINTER(ScoreParams), vp]
    lib.bp_score_onset_offset_grid_device.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32,
                                                      C.POINTER(NoteSet), C.POINTER(ScoreParams), vp, vp, vp]
    lib.bp_score_onset_offset_grid_host.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32,
                                                    C.POINTER(NoteSet), C.POINTER(ScoreParams), vp, vp]
    lib.bp_score_onset_offset_notes_host.argtypes = [vp, C.POINTER(NoteSet), C.POINTER(NoteSet), i32,
                                                     C.POINTER(ScoreParams), vp]
    lib.bp_multipitch_map.argtypes = [vp, i64, vp, i64, vp]
    lib.bp_score_frames_grid_device.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(MultipitchSet),
                                                C.c_double, vp, vp, vp, vp]
    lib.bp_score_frames_grid_host.argtypes = [vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32, C.POINTER(MultipitchSet),
                                              C.c_double, vp, vp, vp]
    lib.bp_score_multipitch_host.argtypes = [vp, C.POINTER(MultipitchSet), C.POINTER(MultipitchSet), i32, C.c_double, vp]
    lib.bp_score_salience_grid_device.argtypes = [vp, vp, i32, vp, i32, C.POINTER(SalienceParams), i32,
                                                  C.POINTER(MultipitchSet), C.c_double, vp, vp, vp, vp]
    lib.bp_score_salience_grid_host.argtypes = [vp, vp, i32, vp, i32, C.POINTER(SalienceParams), i32,
                                                C.POINTER(MultipitchSet), C.c_double, vp, vp, vp]
    lib.bp_score_salience_chunk_params.argtypes = [i64, i64]
    lib.bp_score_salience_chunk_params.restype = i64
    lib.bp_melody_map.argtypes = [vp, i64, vp, i64, vp, vp]
    lib.bp_score_melody_grid_device.argtypes = [vp, vp, i32, vp, i32, C.POINTER(MelodyParams), i32, C.POINTER(MelodySet),
                                                C.c_double, vp, vp, vp]
    lib.bp_score_melody_grid_host.argtypes = [vp, vp, i32, vp, i32, C.POINTER(MelodyParams), i32, C.POINTER(MelodySet),
                                              C.c_double, vp, vp]
    lib.bp_score_melody_host.argtypes = [vp, C.POINTER(MelodySet), C.POINTER(MelodySet), i32, C.c_double, vp]
    lib.bp_score_melody_chunk_params.argtypes = [i64]
    lib.bp_score_melody_chunk_params.restype = i64
    lib.bp_score_bent_frames_grid_device.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32,
                                                     C.POINTER(MultipitchSet), C.c_double, vp, vp, vp, vp]
    lib.bp_score_bent_frames_grid_host.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32,
                                                   C.POINTER(MultipitchSet), C.c_double, vp, vp, vp]
    lib.bp_score_note_melody_grid_device.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32,
                                                     C.POINTER(MelodySet), C.c_double, vp, vp, vp]
    lib.bp_score_note_melody_grid_host.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(DecodeParams), i32,
                                                   C.POINTER(MelodySet), C.c_double, vp, vp]
    lib.bp_evaluate_device.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(EvalRequest), vp]
    lib.bp_evaluate_host.argtypes = [vp, vp, vp, vp, vp, i32, C.POINTER(EvalRequest)]
    lib.bp_evaluate_audio_host.argtypes = [vp, vp, vp, i32, C.POINTER(EvalRequest), vp, vp, vp, vp]
    lib.bp_evaluate_pcm_files_host.argtypes = [vp, C.POINTER(PcmFile), i32, C.POINTER(EvalRequest), vp, vp, vp, vp, vp]
    lib.bp_evaluate_chunk_params.argtypes = [i64, i32, C.POINTER(EvalRequest)]
    lib.bp_evaluate_chunk_params.restype = i64
    lib.bp_stream_create.argtypes = [vp, C.POINTER(DecodeParams), i64, C.POINTER(vp)]
    lib.bp_stream_push_host.argtypes = [vp, vp, vp, vp, i64]
    lib.bp_stream_end.argtypes = [vp]
    lib.bp_stream_take.argtypes = [vp, C.POINTER(Notes)]
    lib.bp_stream_held_frames.argtypes = [vp]
    lib.bp_stream_held_frames.restype = i64
    lib.bp_stream_destroy.argtypes = [vp]
    lib.bp_stream_destroy.restype = None
    lib.bp_stream_group_create.argtypes = [vp, C.POINTER(DecodeParams), i64, C.POINTER(vp)]
    lib.bp_stream_group_open.argtypes = [vp, vp]
    lib.bp_stream_group_commit_offsets.argtypes = [vp, i32, vp, vp, i32, vp]
    lib.bp_stream_group_push_host.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.bp_stream_group_push_frames_host.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    lib.bp_stream_group_end.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    lib.bp_stream_group_take.argtypes = [vp, i32, vp, C.POINTER(Notes)]
    lib.bp_stream_group_held_frames.argtypes = [vp, i32]
    lib.bp_stream_group_held_frames.restype = i64
    lib.bp_stream_group_destroy.argtypes = [vp]
    lib.bp_stream_group_destroy.restype = None
    lib.bp_stream_group_open_pcm.argtypes = [vp, i32, i32, i32, vp]
    lib.bp_stream_group_push_pcm_host.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.bp_stream_group_debug_tail.argtypes = [vp, i32, vp, i64, vp, vp]
    lib.bp_debug_pcm_stream_plan.argtypes = [i32, i32, i32, i32, vp, i32, vp, vp, vp, vp]
    lib.bp_transcribe_host.argtypes = [vp, vp, vp, i32, C.POINTER(DecodeParams), vp, vp, vp, vp, C.POINTER(Notes)]
    lib.bp_transcribe_device.argtypes = [vp, vp, vp, i32, C.POINTER(DecodeParams), vp, C.POINTER(Notes), vp]
    lib.bp_infer_onsets_host.argtypes = [vp, vp, vp, i64, vp]
    lib.bp_pitch_bends_host.argtypes = [vp, vp, i64, i32, vp, vp, vp, vp, vp, i64]
    lib.bp_debug_activation.argtypes = [vp, C.c_int, vp, i64]
    lib.bp_debug_frontend.argtypes = [vp, C.c_int, vp, i64]
    lib.bp_model_set_debug_frontend.argtypes = [vp, C.c_int]
    lib.bp_debug_chain_layout.argtypes = [vp, vp, vp]
    lib.bp_debug_split_layout.argtypes = [vp, vp]
    lib.bp_debug_tc_plan.argtypes = [C.c_int, vp, vp, vp, vp, vp, vp, vp]
    lib.bp_debug_tc_gather.argtypes = [C.c_int, vp, vp, vp, vp, vp]
    lib.bp_debug_tc_gather_packed.argtypes = [C.c_int, vp, vp, vp, vp]
    lib.bp_debug_tc_b2.argtypes = [C.c_int, vp, vp, vp]
    lib.bp_debug_tc_clocks.argtypes = [vp, C.c_int, vp, C.c_int]
    lib.bp_debug_tc_schedule.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.bp_debug_tc_row_map.argtypes = [C.c_int, C.c_int, vp, C.c_int32, vp, vp]
    lib.bp_debug_tc_cta_busy.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int]
    lib.bp_transcribe_files_host.argtypes = [vp, vp, vp, i32, C.POINTER(DecodeParams), vp, vp, vp, vp, C.POINTER(Notes)]
    lib.bp_host_alloc.argtypes = [sz]
    lib.bp_host_alloc.restype = vp
    lib.bp_host_free.argtypes = [vp]
    lib.bp_host_free.restype = None
    lib.bp_last_required.argtypes = [vp, vp]
    lib.bp_last_required.restype = None
    lib.bp_resampled_length.argtypes = [i64, i32]
    lib.bp_resampled_length.restype = i64
    lib.bp_load_pcm_device.argtypes = [vp, vp, i32, i64, i32, i32, vp, vp]
    lib.bp_load_pcm_host.argtypes = [vp, vp, i32, i64, i32, i32, vp]
    lib.bp_load_pcm_files_device.argtypes = [vp, C.POINTER(PcmFile), i32, vp, vp, vp]
    lib.bp_transcribe_pcm_files_host.argtypes = [vp, C.POINTER(PcmFile), i32, C.POINTER(DecodeParams), vp, vp, vp, vp, vp,
                                                 C.POINTER(Notes)]
    lib.bp_debug_pcm_layout.argtypes = [C.POINTER(PcmFile), i32, vp, vp]
    lib.bp_probe_wav_files.argtypes = [vp, i32, C.POINTER(PcmSource), vp]
    lib.bp_transcribe_pcm_sources_host.argtypes = [vp, C.POINTER(PcmSource), i32, C.POINTER(DecodeParams), vp, vp, vp, vp,
                                                   vp, C.POINTER(Notes)]
    lib.bp_evaluate_pcm_sources_host.argtypes = [vp, C.POINTER(PcmSource), i32, C.POINTER(EvalRequest), vp, vp, vp, vp, vp]
    lib.bp_load_pcm_sources_device.argtypes = [vp, C.POINTER(PcmSource), i32, vp, vp, vp]
    lib.bp_debug_pcm_sources_layout.argtypes = [C.POINTER(PcmSource), i32, vp, vp]
    lib.bp_debug_resample_filter.argtypes = [i32, i32, vp, i64]
    lib.bp_debug_resample_filter.restype = i64
    lib.bp_write_note_files.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, C.c_double, i32]
    lib.bp_sonify_notes_host.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, i64]
    lib.bp_model_profile.argtypes = [vp, C.c_int]
    lib.bp_model_profile_read.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i64), C.POINTER(i64)]
    for name in EXPORTS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("bp_version", "bp_model_device"):  # (the int64 / pointer / void returns set restype above)
            fn.errcheck = _check
    _lib = lib
    return lib


def _check(result, func, args):
    if result != BP_OK:
        msg = load().bp_last_error().decode(errors="replace")
        raise (BpIOError if result == BP_E_IO else BpError)(result, msg)
    return result
