"""Drop-in namespace: `from basic_pitch import ICASSP_2022_MODEL_PATH`, `from basic_pitch.inference import predict`
keep working unchanged on top of the H100 implementation (package `basic_pitch_b200`).
Mirrors the public names of reference: basic_pitch/__init__.py:74-95."""
from basic_pitch_b200 import (  # noqa: F401
    ICASSP_2022_MODEL_PATH,
    FilenameSuffix,
    __version__,
    build_icassp_2022_model_path,
)

# runtime-presence flags of the reference (basic_pitch/__init__.py:23-71): none of those runtimes is used here
TF_PRESENT = CT_PRESENT = TFLITE_PRESENT = ONNX_PRESENT = False
B200_PRESENT = True
