"""Command line front end (flag-compatible with reference: basic_pitch/predict.py:34-194).

    python -m basic_pitch_b200.predict <output_dir> <audio> [<audio> ...] [options]
"""
from __future__ import annotations

import argparse
import pathlib
import traceback


def main() -> None:
    from . import ICASSP_2022_MODEL_PATH

    p = argparse.ArgumentParser(description="Predict MIDI from audio on an H100.")
    p.add_argument("output_dir", type=str, help="directory to save outputs")
    p.add_argument("audio_paths", type=str, nargs="+", help="audio file(s) to transcribe")
    p.add_argument("--model-path", type=str, default=str(ICASSP_2022_MODEL_PATH), help="packed .bpw blob or .onnx export")
    p.add_argument("--model-serialization", type=str, default=None,
                   help="accepted for compatibility (tf/coreml/tflite/onnx); this build has a single CUDA runtime")
    p.add_argument("--save-midi", action="store_true", default=True)
    p.add_argument("--sonify-midi", action="store_true")
    p.add_argument("--save-model-outputs", action="store_true")
    p.add_argument("--save-note-events", action="store_true")
    p.add_argument("--onset-threshold", type=float, default=0.5)
    p.add_argument("--frame-threshold", type=float, default=0.3)
    p.add_argument("--minimum-note-length", type=float, default=127.70)
    p.add_argument("--minimum-frequency", type=float, default=None)
    p.add_argument("--maximum-frequency", type=float, default=None)
    p.add_argument("--multiple-pitch-bends", action="store_true")
    p.add_argument("--sonification-samplerate", type=int, default=44100)
    p.add_argument("--midi-tempo", type=float, default=120)
    p.add_argument("--debug-file", default=None)
    p.add_argument("--no-melodia", default=False, action="store_true")
    args = p.parse_args()

    from .inference import Model, predict_and_save, verify_input_path, verify_output_dir

    output_dir = pathlib.Path(args.output_dir)
    verify_output_dir(output_dir)
    audio_paths = [pathlib.Path(a) for a in args.audio_paths]
    for a in audio_paths:
        verify_input_path(a)
    model = Model(args.model_path)
    try:
        predict_and_save(
            audio_paths, output_dir, args.save_midi, args.sonify_midi, args.save_model_outputs, args.save_note_events,
            model, args.onset_threshold, args.frame_threshold, args.minimum_note_length, args.minimum_frequency,
            args.maximum_frequency, args.multiple_pitch_bends, not args.no_melodia,
            pathlib.Path(args.debug_file) if args.debug_file else None, args.sonification_samplerate, args.midi_tempo,
        )
        print("\n✨ Done ✨\n")
    except IOError as e:  # the reference prints and exits normally (predict.py:188-194)
        print(e)
    except Exception:
        print("🚨 Something went wrong 😔 - see the traceback below for details.")
        print("")
        print(traceback.format_exc())


if __name__ == "__main__":
    main()
