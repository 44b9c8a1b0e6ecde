import pathlib
import sys

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def golden_dir():
    return ROOT / "tests" / "golden"


@pytest.fixture(scope="session")
def weights_np():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, weights

    return weights.load(ICASSP_2022_MODEL_PATH)
