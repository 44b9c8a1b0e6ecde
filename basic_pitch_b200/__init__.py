"""basic-pitch hot path, Hopper-native: audio -> harmonic CQT -> CNN -> note events on sm_90a.

Public names mirror the reference package root (reference: basic_pitch/__init__.py:74-95):
`FilenameSuffix`, `build_icassp_2022_model_path`, `ICASSP_2022_MODEL_PATH`.  There is exactly one
runtime here (the CUDA library in `csrc/`), so the default model file is the packed weight blob
`saved_models/icassp_2022/nmp.bpw`; `.onnx` exports of the same graph are also accepted by `Model`.
"""
import enum
import pathlib

__version__ = "0.2.0"


class FilenameSuffix(enum.Enum):
    # the reference's four containers (reference: basic_pitch/__init__.py:74-78) plus this build's blob
    tf = "nmp"
    coreml = "nmp.mlpackage"
    tflite = "nmp.tflite"
    onnx = "nmp.onnx"
    b200 = "nmp.bpw"


def build_icassp_2022_model_path(suffix: FilenameSuffix) -> pathlib.Path:
    return pathlib.Path(__file__).parent / "saved_models/icassp_2022" / suffix.value


ICASSP_2022_MODEL_PATH = build_icassp_2022_model_path(FilenameSuffix.b200)
