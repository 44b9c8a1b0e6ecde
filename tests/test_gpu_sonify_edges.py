"""GPU: the sonification (csrc/sonify.cu through note_creation.sonify_batch and bp_sonify_notes_host) on the adversarial
note sets of tests/sonifysets.py, at every rate and both values of multiple_pitch_bends.

  bound       every file of every set is within the stand-in's per-sample bound (`standin` of
              tests/test_gpu_sonify.py); the largest err / bound per set is printed
  placement   all the sets of a rate in one call, and each file alone, give the same bits
  launches    two per call; none for a size query or a call whose total is 0
  validation  an amplitude whose velocity Python cannot form (NaN, or a float32 product 127 * amplitude that is +-inf)
              is BP_E_INVALID without a launch, and the model stays usable

tests/test_sonify_edges_cpu.py shows that the sets reach the edges they are built for and that a slip in any placement
or velocity rule leaves the bound on at least one of them."""
import numpy as np
import pytest

from tests import sonifysets as ss
from tests.test_gpu_sonify import standin

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH, device=0)


def _worst(got, ev, fs, multi):
    ref, tol = standin(ev, fs, multi)
    assert got.dtype == np.float64 and got.shape == ref.shape, (got.shape, ref.shape)
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / tol)
    return float(r.max()) if r.size else 0.0


@pytest.mark.parametrize("fs", ss.RATES)
def test_every_set_is_within_the_bound(model, fs):
    from basic_pitch_b200 import note_creation as nc

    worst = {}
    for s in ss.sets(fs):
        for multi in (False, True):
            launches = model.launch_count
            got = nc.sonify_batch(s.files, fs, multi, model)
            assert model.launch_count == launches + 2, (s.name, multi)
            assert len(got) == len(s.files)
            for i, ev in enumerate(s.files):
                r = _worst(got[i], ev, fs, multi)
                assert r <= 1.0, (fs, s.name, i, multi, r)
                worst[s.name] = max(worst.get(s.name, 0.0), r)
    print(f"\n{fs} Hz, largest err / bound per set: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("fs", ss.RATES)
def test_one_call_and_each_file_alone_give_the_same_bits(model, fs):
    from basic_pitch_b200 import note_creation as nc

    files = [ev for s in ss.sets(fs) for ev in s.files]
    for multi in (False, True):
        packed = [a.copy() for a in nc.sonify_batch(files, fs, multi, model)]
        for i, ev in enumerate(files):
            if not ev and i % 50:  # the empty files of `many`: a sample of them is enough
                continue
            alone = nc.sonify_batch([ev], fs, multi, model)[0]
            assert np.array_equal(alone.view(np.uint64), packed[i].view(np.uint64)), (fs, i, multi)


def _raw_call(model, files, sr, out=None, cap=0):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200 import note_creation as nc

    noff, st, en, pitch, amp, boff, flat = nc._pack_note_events(files)
    soff = np.full(len(files) + 1, -7, np.int64)
    lib = _lib.load()
    lib.bp_sonify_notes_host(model.handle, len(files), noff.ctypes.data, st.ctypes.data, en.ctypes.data,
                             pitch.ctypes.data, amp.ctypes.data, boff.ctypes.data, flat.ctypes.data, 0, sr,
                             soff.ctypes.data, None if out is None else out.ctypes.data, cap)
    return soff


def test_launches_size_queries_and_empty_totals(model):
    from basic_pitch_b200 import note_creation as nc

    files = ss.layout(8000)[0].files
    launches = model.launch_count
    soff = _raw_call(model, files, 8000)  # size query: host only
    assert model.launch_count == launches and soff[0] == 0
    assert np.diff(soff).tolist() == [len(standin(ev, 8000, False)[0]) for ev in files]
    assert [int(x) % 256 for x in np.diff(soff)[0::4]] == [0, 1, 255]
    out = np.zeros(int(soff[-1]))
    _raw_call(model, files, 8000, out, len(out))
    assert model.launch_count == launches + 2
    for empty in ([], [[]], [[]] * 7):  # total 0: nothing to launch
        assert all(len(a) == 0 for a in nc.sonify_batch(empty, 8000, False, model))
        soff = _raw_call(model, empty, 8000, np.zeros(1), 0)
        assert soff.tolist() == [0] * (len(empty) + 1)
    assert model.launch_count == launches + 2


@pytest.mark.parametrize("amp", [np.nan, -np.nan, np.inf, -np.inf, 3e38, -3e38, np.finfo(np.float32).max])
def test_amplitudes_without_a_velocity_are_refused_without_a_launch(model, amp):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200 import note_creation as nc

    good = [(0.1, 0.5, 60, np.float32(0.5), [1, 2])]
    files = [good, [(0.2, 0.4, 61, np.float32(0.5), None), (0.3, 0.6, 62, np.float32(amp), None)]]
    launches = model.launch_count
    for sr in (8000, 44100):
        with pytest.raises(_lib.BpError) as e:
            nc.sonify_batch(files, sr, False, model)
        assert e.value.code == _lib.BP_E_INVALID
        with pytest.raises(_lib.BpError):
            _raw_call(model, files, sr)  # the size query refuses it too
    assert model.launch_count == launches
    got = nc.sonify_batch([good], 44100, True, model)[0]  # still usable
    ref, tol = standin(good, 44100, True)
    assert got.shape == ref.shape and np.all(np.abs(got - ref) <= tol)
    assert model.launch_count == launches + 2
