"""The GPU render of the MIDI sonification (csrc/sonify.cu: `note_creation.sonify_batch`, `bp_sonify_notes_host`) against
the bundled stand-in synthesiser `midi.PrettyMIDI.synthesize`, which defines it (DESIGN.md §4.4).

Everything that places a sample is exact; the phase differs by rounding only (NumPy's sequential cumsum against the
closed form per bend segment, plus ulp-level pow / sin).  `standin` returns the stand-in's samples together with the
per-sample bound of that difference; the CPU test at the end checks the cumsum bound the tolerance rests on."""
import math
from fractions import Fraction

import numpy as np
import pytest

U = 2.0**-53
RATES = (8000, 22050, 44100, 48000, 96000)


def standin(events, fs, multiple_pitch_bends):
    """-> (samples of note_events_to_midi(events, multiple_pitch_bends).synthesize(fs), per-sample tolerance).

    tol(k) = (dY(k) + max dY) / P + 2 (n(k) + 1) u, with
      dY(k)      = sum over the n(k) notes covering k of (|v| / 127) (dphi(k) + 8u),
      dphi(k)    = 2 [pi u f (k - a + 1)^2 / fs + 4u |phi(k)|]  (cumsum bound and pow / sin / product roundings, for both
                   implementations), f the note's highest frequency (its pitch bent 2 semitones up), phi the stand-in's
                   own phase (captured through `synthesize`'s `wave` argument),
      P          = the stand-in's peak before normalisation;
    the last term covers the rounding of the sum of n(k) notes and of the normalising division."""
    from basic_pitch_b200 import note_creation as nc

    mid = nc.note_events_to_midi(list(events), multiple_pitch_bends)
    phases = []

    def wave(ph):
        phases.append(ph)
        return np.sin(ph)

    ref = mid.synthesize(fs, wave=wave)
    n = len(ref)
    y, dy, cnt = np.zeros(n), np.zeros(n), np.zeros(n)
    it = iter(phases)
    for inst in mid.instruments:
        for note in inst.notes:
            a, b = int(fs * note.start), int(fs * note.end)
            if b <= a:
                continue
            ph = next(it)
            env = np.ones(b - a)
            fade = min(int(0.01 * fs), (b - a) // 2)
            if fade > 0:
                env[:fade] = np.linspace(0.0, 1.0, fade, endpoint=False)
                env[-fade:] = env[:fade][::-1]
            y[a:b] += np.sin(ph) * env * (note.velocity / 127.0)
            f = 440.0 * 2.0 ** ((note.pitch + 2 - 69) / 12.0)
            m1 = np.arange(1, b - a + 1, dtype=np.float64)
            dphi = 2.0 * (np.pi * U * f * m1 * m1 / fs + 4.0 * U * np.abs(ph))
            dy[a:b] += abs(note.velocity) / 127.0 * (dphi + 8.0 * U)
            cnt[a:b] += 1
    peak = float(np.abs(y).max()) if n else 0.0
    if peak == 0.0:
        return ref, np.zeros(n)  # all zeros, no division: exact
    return ref, (dy + dy.max()) / peak + 2.0 * (cnt + 1.0) * U


def assert_within(got, events, fs, multi, what=""):
    ref, tol = standin(events, fs, multi)
    assert got.dtype == np.float64 and got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got - ref)
    bad = np.flatnonzero(err > tol)
    assert bad.size == 0, (what, int(bad[0]), float(err[bad[0]]), float(tol[bad[0]]))


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH, device=0)


@pytest.fixture(scope="module")
def decoded(model):
    """Note events of the device decode on the synthetic clips (NoteEventLists, pitch bends included)."""
    from basic_pitch_b200 import note_creation as nc
    from basic_pitch_b200 import synth

    clips = [synth.tones_clip(3.0, seed=1), synth.random_notes_clip(10.0, seed=21), synth.dense_chords_clip(3.0, seed=7)]
    _outs, arrs, _frames = model.transcribe_arrays(clips, return_model_output=False, split_notes=False)
    events = nc.note_events_batch(arrs, len(clips))
    assert all(len(e) > 3 for e in events) and sum(len(e[i][4]) for e in events for i in range(len(e))) > 100
    return events


@pytest.mark.gpu
@pytest.mark.parametrize("multi", [False, True])
def test_decoded_notes_match_the_standin(model, decoded, multi):
    from basic_pitch_b200 import note_creation as nc

    for fs in RATES:
        got = nc.sonify_batch(decoded, fs, multi, model)
        for i, ev in enumerate(decoded):
            assert_within(got[i], ev, fs, multi, (fs, i))


def edge_files(fs):
    """Hand-made files, each exercising one rule of the stand-in at sample rate fs."""
    f32 = np.float32
    s = lambda k: k / fs  # noqa: E731  time of sample k
    return [
        [(0.1, 0.6, 60, f32(0.7), [0, 3, -3])],
        [],  # no notes: empty
        [(0.1, 0.5, 60, f32(0.0), [1, 2]), (0.3, 0.9, 64, f32(0.001), None)],  # all velocities 0: all zeros
        [(0.2, 0.2, 62, f32(0.5), [4]), (0.3, 0.3 + 0.4 / fs, 64, f32(0.5), None), (0.5, 0.9, 65, f32(0.6), None)],  # b == a
        [(s(1000.5), s(1001.5), 70, f32(0.5), None), (s(2000.5), s(2002.5), 71, f32(0.6), [2]),
         (s(3000.5), s(3003.5), 72, f32(0.7), None), (s(4000.2), s(4000.2) + 0.012, 73, f32(0.8), [1, -1]),
         (0.3, 0.314, 74, f32(0.9), None)],  # 1-3 samples, shorter than two fades
        [(s(4410), s(8820), 67, f32(0.6), [3, -3, 2, -2]), (s(8820), s(13230), 69, f32(0.5), [-1, 1])],  # bends on k / fs
        [(0.05, 0.4, 50, f32(0.8), [7, -7, 9, -12]), (0.4, 0.7, 52, f32(0.5), None)],  # ticks clipped, bend held after
        # overlapping notes of one pitch (one instrument with multiple_pitch_bends) and touching notes (one instrument
        # without): their bends bend each other
        [(0.1, 0.8, 60, f32(0.6), [1, 2, 3, 4, 5, 6]), (0.4, 1.2, 60, f32(0.5), [-6, -5, -4]), (0.8, 1.5, 64, f32(0.4), None),
         (1.5, 1.9, 55, f32(0.7), [2, 0, -2])],
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("fs", [22050, 44100])
def test_edge_cases_match_the_standin(model, fs, multi):
    from basic_pitch_b200 import note_creation as nc

    files = edge_files(fs)
    got = nc.sonify_batch(files, fs, multi, model)
    assert len(got[1]) == 0
    assert len(got[2]) > 0 and not np.any(got[2])
    for i, ev in enumerate(files):
        assert_within(got[i], ev, fs, multi, i)


@pytest.mark.gpu
def test_a_long_bent_note_stays_within_the_bound(model):
    """One 60 s note with a bend every 50 ms: the cumsum bound at its largest (~2.5e-4 rad at the end)."""
    from basic_pitch_b200 import note_creation as nc

    rng = np.random.default_rng(3)
    ev = [[(0.25, 60.25, 96, np.float32(0.8), rng.integers(-6, 7, 1200).tolist())]]
    for multi in (False, True):
        got = nc.sonify_batch(ev, 44100, multi, model)
        assert_within(got[0], ev[0], 44100, multi)


@pytest.mark.gpu
def test_output_is_deterministic_and_independent_of_batch_position(model, decoded):
    from basic_pitch_b200 import note_creation as nc

    target = decoded[1]
    others = [decoded[i % 3] for i in range(199)]
    alone = nc.sonify_batch([target], 44100, False, model)[0].copy()
    for pos in (0, 17, 199):
        batch = others[:pos] + [target] + others[pos:]
        got = nc.sonify_batch(batch, 44100, False, model)
        assert np.array_equal(got[pos].view(np.uint64), alone.view(np.uint64)), pos
    first = [a.copy() for a in nc.sonify_batch(others, 44100, True, model)]
    second = nc.sonify_batch(others, 44100, True, model)
    assert all(np.array_equal(a.view(np.uint64), b.view(np.uint64)) for a, b in zip(first, second))


@pytest.mark.gpu
def test_size_query_capacity_and_invalid_arguments(model):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200 import note_creation as nc

    files = edge_files(44100)
    noff, st, en, pitch, amp, boff, flat = nc._pack_note_events(files)
    lib = _lib.load()
    soff = np.full(len(files) + 1, -7, np.int64)

    def call(sr, out, cap):
        lib.bp_sonify_notes_host(model.handle, len(files), noff.ctypes.data, st.ctypes.data, en.ctypes.data,
                                 pitch.ctypes.data, amp.ctypes.data, boff.ctypes.data, flat.ctypes.data, 0, sr,
                                 soff.ctypes.data, out, cap)

    launches = model.launch_count
    call(44100, None, 0)  # size query: no device work
    assert model.launch_count == launches
    want = [len(standin(ev, 44100, False)[0]) for ev in files]
    assert np.diff(soff).tolist() == want and soff[0] == 0
    total = int(soff[-1])
    out = np.zeros(total, np.float64)
    with pytest.raises(_lib.BpError) as e:
        call(44100, out.ctypes.data, total - 1)
    assert e.value.code == _lib.BP_E_CAPACITY and int(soff[-1]) == total
    for sr in (0, -44100):
        with pytest.raises(_lib.BpError) as e:
            call(sr, out.ctypes.data, total)
        assert e.value.code == _lib.BP_E_INVALID
    call(44100, out.ctypes.data, total)
    assert model.launch_count == launches + 2
    got = nc.sonify_batch(files, 44100, False, model)
    assert np.array_equal(np.concatenate(got), out)


@pytest.mark.gpu
def test_predict_and_save_batch_path_sonifies_on_the_gpu(model, tmp_path):
    """predict_and_save over several files with sonify_midi=True: the batch path renders the WAVs with one
    bp_sonify_notes_host call; against the per-file path (the stand-in) the WAV headers and lengths are identical and
    the samples within the bound; MIDI, CSV and NPZ files stay byte-identical."""
    from scipy.io import wavfile

    from basic_pitch_b200 import inference as inf
    from basic_pitch_b200 import synth

    paths = []
    for i, (sr, secs) in enumerate(((22050, 3.0), (44100, 4.5), (22050, 0.7), (22050, 5.0))):
        clip = synth.random_notes_clip(secs, seed=80 + i) if i == 3 else synth.tones_clip(secs, seed=70 + i)
        if sr != 22050:
            clip = np.repeat(clip, 2)
        p = tmp_path / f"clip{i}.wav"
        wavfile.write(p, sr, (clip * 20000).astype(np.int16))
        paths.append(p)
    for multi in (False, True):
        out_b, out_s = tmp_path / f"batch{multi}", tmp_path / f"single{multi}"
        out_b.mkdir(), out_s.mkdir()
        inf.predict_and_save(paths, out_b, True, True, True, True, model, multiple_pitch_bends=multi,
                             sonification_samplerate=48000)
        for p in paths:
            inf.predict_and_save([p], out_s, True, True, True, True, model, multiple_pitch_bends=multi,
                                 sonification_samplerate=48000)
        for p in paths:
            stem = f"{p.stem}_basic_pitch"
            for ext in ("mid", "csv"):
                assert (out_b / f"{stem}.{ext}").read_bytes() == (out_s / f"{stem}.{ext}").read_bytes(), (p.name, ext)
            za = np.load(out_b / f"{stem}.npz", allow_pickle=True)["basic_pitch_model_output"].item()
            zb = np.load(out_s / f"{stem}.npz", allow_pickle=True)["basic_pitch_model_output"].item()
            for k in ("note", "onset", "contour"):
                np.testing.assert_array_equal(za[k], zb[k])
            wa, wb = (out_b / f"{stem}.wav").read_bytes(), (out_s / f"{stem}.wav").read_bytes()
            assert wa[:58] == wb[:58] and len(wa) == len(wb), p.name
            ra, rb = wavfile.read(out_b / f"{stem}.wav"), wavfile.read(out_s / f"{stem}.wav")
            assert ra[0] == rb[0] == 48000 and ra[1].dtype == np.float64 and len(ra[1]) > 48000
            _out, _midi, events = inf.predict(p, model, multiple_pitch_bends=multi)
            assert_within(ra[1], events, 48000, multi, p.name)


def test_cumsum_phase_error_stays_within_the_bound():
    """CPU: the bound the tolerance rests on.  For long constant-frequency and bent notes the stand-in's phase
    (`synthesize`'s own, captured through its `wave` argument) against the exact phase of the same frequencies
    (prefix sums in exact rational arithmetic) stays within pi u f (k + 1)^2 / fs + 4u |phi(k)| (half of dphi: one
    implementation), f the note's highest frequency."""
    from basic_pitch_b200 import midi

    fs = 96000
    rng = np.random.default_rng(5)
    for pitch, ticks in ((105, []), (93, rng.integers(-8192, 8192, 400).tolist())):
        pm = midi.PrettyMIDI()
        inst = midi.Instrument(program=4)
        inst.notes.append(midi.Note(velocity=100, pitch=pitch, start=0.5, end=40.5))
        times = np.linspace(0.5, 40.5, len(ticks)) if ticks else []
        for t, v in zip(times, ticks):
            inst.pitch_bends.append(midi.PitchBend(int(v), float(t)))
        pm.instruments.append(inst)
        phases = []
        pm.synthesize(fs, wave=lambda ph: (phases.append(ph), np.sin(ph))[1])
        phi = phases[0]
        a = int(fs * 0.5)
        n = len(phi)
        # the frequencies of the stand-in's samples: piecewise constant between the bend events
        k = np.arange(a, a + n)
        bt = np.array([float(t) for t in times])
        semis = np.full(n, float(pitch))
        if len(bt):
            j = np.searchsorted(bt, k / fs, side="right") - 1
            semis = semis + np.where(j >= 0, np.array(ticks, np.float64)[np.maximum(j, 0)] * (2.0 / 8192.0), 0.0)
        freq = 440.0 * 2.0 ** ((semis - 69.0) / 12.0)
        # exact prefix sums per constant run: S(k) = C_run + (k - k_run + 1) f_run, C_run exact (Fraction)
        starts = np.flatnonzero(np.r_[True, freq[1:] != freq[:-1]])
        lens = np.diff(np.r_[starts, n])
        exact = np.empty(n, np.longdouble)
        c = Fraction(0)
        for s0, ln in zip(starts.tolist(), lens.tolist()):
            f = freq[s0]
            num, den = c.numerator, c.denominator
            sh = max(0, num.bit_length() - 62)
            c_ld = np.longdouble(num >> sh) * np.longdouble(2) ** sh / np.longdouble(den)
            exact[s0 : s0 + ln] = c_ld + np.arange(1, ln + 1, dtype=np.longdouble) * np.longdouble(f)
            c += Fraction(f) * ln
        phi_exact = np.longdouble(2.0 * np.pi) * exact / np.longdouble(fs)
        fmax = float(freq.max())
        m1 = np.arange(1, n + 1, dtype=np.float64)
        bound = math.pi * U * fmax * m1 * m1 / fs + 4.0 * U * np.abs(phi)
        err = np.abs(phi.astype(np.longdouble) - phi_exact).astype(np.float64)
        assert np.all(err <= bound), (pitch, int(np.argmax(err / bound)), float((err / bound).max()))
        assert err.max() > 0  # the stand-in's phase is not exact: the comparison has something to bound
