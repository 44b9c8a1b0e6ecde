"""GPU: the melody scorers on the adversarial sets of tests/melodysets.py (csrc/score_melody.cu, the melody section of
csrc/api.cu).  For every set and two tolerances, bp_score_melody_grid_host and bp_score_melody_grid_device (on a caller
stream) agree bit for bit and equal oracle/melody_ref.counts_cents applied to the host definition of every (setting,
file); the model's tables also go through Model.score_melody_grid and the one-pass Model.evaluate, and the bent-note
set through Model.score_note_melody_grid against evaluate.note_frames_to_melody of the device decode.

tests/test_melody_edges_cpu.py shows that the sets reach the edges they are built for and that a slip in any rule
changes the expected counts."""
import ctypes as C

import numpy as np
import pytest

from tests import melodysets as ms
from tests.test_gpu_decode_edges import _kw
from tests.test_gpu_note_f0 import _mel_oracle
from tests.test_melody_edges_cpu import expected

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


def _ref_set(refs):
    """bp_melody_set_t of [(times, cents, voiced)] as given."""
    from basic_pitch_b200 import _lib

    f_off = np.cumsum([0] + [len(t) for t, _, _ in refs]).astype(np.int64)
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), dt)  # noqa: E731
    arrs = (f_off, cat([t for t, _, _ in refs], np.float64), cat([c for _, c, _ in refs], np.float64),
            cat([v for _, _, v in refs], np.int32))
    s = _lib.MelodySet()
    s.frame_off, s.time_s, s.cent, s.voiced = (a.ctypes.data for a in arrs)
    return s, arrs


def _call(model, s, tol, stream=None):
    """bp_score_melody_grid_host, or _device from a torch copy of the posteriorgrams on `stream`, on raw arguments."""
    import torch

    from basic_pitch_b200 import _lib

    W = len(s.cents)
    foff = np.cumsum([0] + [g.shape[0] for g in s.grams]).astype(np.int64)
    g_all = np.ascontiguousarray(np.concatenate(s.grams), np.float32)
    ps = (_lib.MelodyParams * len(s.params))(*[_lib.MelodyParams(thr, lo, hi, g, 0) for thr, lo, hi, g in s.params])
    refs, keep = _ref_set(s.refs)
    tab = np.ascontiguousarray(s.cents, np.float64)
    out = np.full((len(s.params), len(s.grams), 7), -1, np.int64)
    if stream is None:
        model._lib.bp_score_melody_grid_host(model.handle, g_all.ctypes.data, W, foff.ctypes.data, len(s.grams), ps,
                                             len(s.params), C.byref(refs), tol, tab.ctypes.data, out.ctypes.data)
    else:
        dev = f"cuda:{model.device}"
        d = torch.from_numpy(g_all).to(dev)
        torch.cuda.synchronize(dev)
        with torch.cuda.stream(stream):
            model._lib.bp_score_melody_grid_device(model.handle, d.data_ptr(), W, foff.ctypes.data, len(s.grams), ps,
                                                   len(s.params), C.byref(refs), tol, tab.ctypes.data,
                                                   out.ctypes.data, stream.cuda_stream)
    return out


@pytest.mark.parametrize("name", ms.NAMES)
def test_grid_sets_host_device_and_oracle(model, name):
    import torch

    s = ms.get(name)
    stream = torch.cuda.Stream(device=f"cuda:{model.device}")
    for tol in ms.TOLS:
        before = model.launch_count
        host = _call(model, s, tol)
        assert model.launch_count - before == 3  # one chunk: arg-max, hold, counts
        dev = _call(model, s, tol, stream)
        assert dev.tobytes() == host.tobytes(), (name, tol)
        np.testing.assert_array_equal(host, expected(name, tol), err_msg=f"{name} tol {tol}")
        if s.kind:
            before = model.launch_count
            got = model.score_melody_grid(s.grams, ms.hz_settings(s), s.ref_hz, kind=s.kind, cent_tolerance=tol)
            assert model.launch_count - before == 3
            assert got.tobytes() == host.tobytes(), (name, tol)
    assert host[..., 4].sum() > 0 and host[..., 3].sum() > 0  # pitches right and false alarms somewhere


def test_one_pass_melody_family_equals_the_standalone_call(model):
    s = ms.get("contour")
    hs = ms.hz_settings(s)
    notes = [np.zeros((g.shape[0], 88), np.float32) for g in s.grams]
    for tol in ms.TOLS:
        exp = model.score_melody_grid(s.grams, hs, s.ref_hz, kind="contour", cent_tolerance=tol)
        got = model.evaluate(["melody"], [dict()], grams=(notes, notes, s.grams), cent_tolerance=tol,
                             melody=dict(settings=hs, kind="contour", references=s.ref_hz))
        assert got["melody"].tobytes() == exp.tobytes(), tol


def test_bent_note_set_equals_the_oracle(model):
    from tests.test_postsets import oracle

    files, grid, refs = ms.bent()
    notes, onsets, contours = ([f[k] for f in files] for k in range(3))
    settings = [{**_kw(p), "include_pitch_bends": b} for p in grid for b in (True, False)]
    res = model.decode_grid(notes, onsets, contours, settings)
    # the device decode is the one the set was checked against (tests/test_melody_edges_cpu.py)
    for k, p in enumerate(settings[::2]):
        for i, f in enumerate(files):
            cpu = oracle(*f, grid[k])
            r = res[2 * k][i]
            assert sorted(tuple(n[:3]) for n in cpu) == sorted(zip(r["start"].tolist(), r["end"].tolist(),
                                                                   r["pitch"].tolist()))
    for tol in ms.TOLS:
        before = model.launch_count
        got = model.score_note_melody_grid(notes, onsets, contours, settings, refs, cent_tolerance=tol)
        assert model.launch_count - before == 3 + 4  # the decode's three, then roll scatter, prefix, pick + hold, counts
        np.testing.assert_array_equal(got, _mel_oracle(res, notes, refs, tol), err_msg=str(tol))
        assert got[..., 4].sum() > 0
