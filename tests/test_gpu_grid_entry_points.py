"""GPU: the two entry points of every grid scorer (bp_decode_grid, bp_score_grid, bp_match_grid, bp_score_onset_offset_grid,
bp_score_frames_grid, bp_score_salience_grid), side by side on one small set of decode_edges.npz: _host from host
memory and _device from device memory on a caller stream give the same outputs, reject the same input with the same
message and no launch, and name the entry point the caller called when a note capacity is too small."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_decode_edges import _kw, _set

pytestmark = pytest.mark.gpu

SET = "runs"  # four files of 132 .. 185 frames, eight settings
NOTE_CAP, BEND_CAP = 200000, 4000000


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def inp(model, golden_dir):
    """Posteriorgrams on the host and on the device, settings and seeded references of every kind."""
    import torch

    from basic_pitch_b200 import evaluate

    files, grid = _set(dict(np.load(golden_dir / "decode_edges.npz")), SET)
    n = len(files)
    lens = [f[0].shape[0] for f in files]
    rng = np.random.default_rng(7)
    notes, series = [], []
    for T in lens:
        on = np.sort(rng.uniform(0.0, T * 0.0116, 12))
        iv = np.stack([on, on + rng.uniform(0.03, 0.4, 12)], 1)
        notes.append((iv, 440.0 * 2.0 ** ((rng.integers(40, 84, 12) - 69) / 12.0)))
        t = np.arange(T // 2) * 0.0232
        series.append((t, [rng.uniform(100.0, 1000.0, rng.integers(0, 4)) for _ in t]))
    host = {k: np.ascontiguousarray(np.concatenate([f[j] for f in files])) for j, k in enumerate(("note", "onset", "contour"))}
    dev = f"cuda:{model.device}"
    d = {k: torch.from_numpy(v).to(dev) for k, v in host.items()}
    torch.cuda.synchronize(dev)
    hz, midi, chroma = evaluate.salience_bins("contour")
    return dict(n=n, foff=np.cumsum([0] + lens).astype(np.int64), host=host, dev=d, stream=torch.cuda.Stream(device=dev),
                settings=[_kw(p) for p in grid], notes=notes, intervals=[iv for iv, _ in notes], series=series,
                bins=(len(hz), midi, chroma))


def _bad_notes(notes):
    out = [(iv.copy(), hz) for iv, hz in notes]
    out[1][0][0, 0] = np.nan
    return out


def _bad_series(series):
    out = list(series)
    out[2] = (-series[2][0], series[2][1])
    return out


class _Pair:
    """One grid scorer: `grams` its posteriorgram arguments; args(model, inp, bad) the arguments after them (minus the
    stream), the output arrays and what keeps them alive.  bad is None, "ref" or "setting"; `bad_msg` what each names."""

    def __init__(self, name, grams, args, bad_msg, notes=False):
        self.name, self.grams, self.args, self.bad_msg, self.notes = name, grams, args, bad_msg, notes

    def call(self, model, inp, entry, rest):
        import torch

        fn = getattr(model._lib, f"{self.name}_{entry}")
        if entry == "host":
            return fn(model.handle, *[inp["host"][g].ctypes.data for g in self.grams], *rest)
        with torch.cuda.stream(inp["stream"]):
            return fn(model.handle, *[inp["dev"][g].data_ptr() for g in self.grams], *rest, inp["stream"].cuda_stream)


def _decode_params(model, inp, bad):
    settings = inp["settings"][:3]
    if bad == "setting":
        settings = [settings[0], {**settings[1], "energy_tol": 0}, settings[2]]
    return model._grid_params(settings), len(settings)


def _notes_out(model, inp, n_params, note_cap=NOTE_CAP):
    nt, arrs = model._alloc_notes(inp["n"] * n_params, note_cap, BEND_CAP)
    return nt, arrs


def _decode_args(model, inp, bad, note_cap=NOTE_CAP):
    ps, P = _decode_params(model, inp, bad)
    nt, arrs = _notes_out(model, inp, P, note_cap)
    return [inp["foff"].ctypes.data, inp["n"], ps, P, C.byref(nt)], {"notes": arrs}, (ps, nt)


def _note_refs(model, inp, bad):
    return model._note_set(_bad_notes(inp["notes"]) if bad == "ref" else inp["notes"], "references")


def _score_args(model, inp, bad):
    from basic_pitch_b200 import evaluate

    ps, P = _decode_params(model, inp, bad)
    refs, keep = _note_refs(model, inp, bad)
    sp = model._score_params({})
    counts = np.full((P, inp["n"], 4), -1, np.int64)
    return ([inp["foff"].ctypes.data, inp["n"], ps, P, C.byref(refs), C.byref(sp), evaluate.EST_LOG2_HZ.ctypes.data,
             counts.ctypes.data], {"counts": counts}, (ps, refs, keep, sp))


def _match_args(model, inp, bad, note_cap=NOTE_CAP):
    from basic_pitch_b200 import evaluate

    ps, P = _decode_params(model, inp, bad)
    refs, keep = _note_refs(model, inp, bad)
    sp = model._score_params({})
    nt, arrs = _notes_out(model, inp, P, note_cap)
    match = np.full((P, 2, int(keep[0][-1])), -2, np.int32)
    return ([inp["foff"].ctypes.data, inp["n"], ps, P, C.byref(refs), C.byref(sp), evaluate.EST_LOG2_HZ.ctypes.data,
             C.byref(nt), match.ctypes.data], {"notes": arrs, "match": match}, (ps, refs, keep, sp, nt))


def _onset_offset_args(model, inp, bad):
    ps, P = _decode_params(model, inp, bad)
    ivs = [iv for iv, _ in _bad_notes(inp["notes"])] if bad == "ref" else inp["intervals"]
    refs, keep = model._note_set([(iv, np.ones(len(iv))) for iv in ivs], "references")
    refs.log2_hz = None
    sp = model._score_params({})
    counts = np.full((P, inp["n"], 4), -1, np.int64)
    return ([inp["foff"].ctypes.data, inp["n"], ps, P, C.byref(refs), C.byref(sp), None, counts.ctypes.data],
            {"counts": counts}, (ps, refs, keep, sp))


def _mp_refs(model, inp, bad):
    return model._multipitch_set(_bad_series(inp["series"]) if bad == "ref" else inp["series"], "references")


def _frames_args(model, inp, bad):
    from basic_pitch_b200 import evaluate

    ps, P = _decode_params(model, inp, bad)
    refs, keep = _mp_refs(model, inp, bad)
    counts = np.full((P, inp["n"], 7), -1, np.int64)
    return ([inp["foff"].ctypes.data, inp["n"], ps, P, C.byref(refs), 0.5, evaluate.EST_MIDI.ctypes.data,
             evaluate.EST_CHROMA.ctypes.data, counts.ctypes.data], {"counts": counts}, (ps, refs, keep))


def _salience_args(model, inp, bad):
    settings = [dict(threshold=0.3), dict(threshold=0.5, peak_picking=False), dict(threshold=0.2, minimum_frequency=200.0)]
    ps = model._salience_params(settings, "contour")
    if bad == "setting":
        ps[1].threshold = 0.0
    refs, keep = _mp_refs(model, inp, bad)
    width, midi, chroma = inp["bins"]
    counts = np.full((len(settings), inp["n"], 7), -1, np.int64)
    return ([width, inp["foff"].ctypes.data, inp["n"], ps, len(settings), C.byref(refs), 0.5, midi.ctypes.data,
             chroma.ctypes.data, counts.ctypes.data], {"counts": counts}, (ps, refs, keep, midi, chroma))


PAIRS = [
    _Pair("bp_decode_grid", ("note", "onset", "contour"), _decode_args, {"setting": "decode params[1]"}, notes=True),
    _Pair("bp_score_grid", ("note", "onset"), _score_args,
          {"setting": "decode params[1]", "ref": "references file 1 note 0: non-finite time"}),
    _Pair("bp_match_grid", ("note", "onset"), _match_args,
          {"setting": "decode params[1]", "ref": "references file 1 note 0: non-finite time"}, notes=True),
    _Pair("bp_score_onset_offset_grid", ("note", "onset"), _onset_offset_args,
          {"setting": "decode params[1]", "ref": "references file 1 note 0: non-finite time"}),
    _Pair("bp_score_frames_grid", ("note", "onset"), _frames_args,
          {"setting": "decode params[1]", "ref": "references file 2 frame 1: time < 0"}),
    _Pair("bp_score_salience_grid", ("contour",), _salience_args,
          {"setting": "salience params[1]", "ref": "references file 2 frame 1: time < 0"}),
]
IDS = [p.name for p in PAIRS]


def _used_notes(arrs):
    """The filled part of a call's note arrays."""
    n = int(arrs["note_off"][-1])
    return {"note_off": arrs["note_off"], "bend_off": arrs["bend_off"][: n + 1],
            "bends": arrs["bends"][: int(arrs["bend_off"][n])],
            **{k: arrs[k][:n] for k in ("start", "end", "pitch", "amp")}}  # fmt: skip


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_host_and_device_give_the_same_outputs(model, inp, pair):
    """(a) The same counts, and for the note-returning pairs the same note arrays and matchings, from host memory and
    from device memory on a non-default stream."""
    got = {}
    for entry in ("host", "device"):
        rest, out, keep = pair.args(model, inp, None)
        pair.call(model, inp, entry, rest)
        got[entry] = out
    for key, h in got["host"].items():
        d = got["device"][key]
        if key == "notes":
            h, d = _used_notes(h), _used_notes(d)
            assert int(h["note_off"][-1]) > 0, pair.name
            for k in h:
                np.testing.assert_array_equal(h[k], d[k], err_msg=f"{pair.name}: {k}")
        else:
            assert (h >= -1).all(), f"{pair.name}: {key} not written"
            np.testing.assert_array_equal(h, d, err_msg=f"{pair.name}: {key}")
    if "counts" in got["host"]:
        assert got["host"]["counts"][..., :2].sum() > 0, pair.name


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_invalid_input_is_rejected_alike_without_a_launch(model, inp, pair):
    """(b) An invalid reference and an invalid setting: both entry points fail with BP_E_INVALID and the same message,
    up to the name of the entry point (which a reference's message starts with), and launch nothing."""
    from basic_pitch_b200 import _lib

    for bad, what in pair.bad_msg.items():
        msgs = {}
        for entry in ("host", "device"):
            rest, out, keep = pair.args(model, inp, bad)
            before = model.launch_count
            with pytest.raises(_lib.BpError) as e:
                pair.call(model, inp, entry, rest)
            assert e.value.code == _lib.BP_E_INVALID, str(e.value)
            assert model.launch_count == before, f"{pair.name}_{entry}: {bad}"
            msg = str(e.value).split(": ", 1)[1]
            assert what in msg, msg
            if bad == "ref":
                assert msg.startswith(f"{pair.name}_{entry}: "), msg
            msgs[entry] = msg.replace(f"{pair.name}_{entry}", pair.name)
        assert msgs["host"] == msgs["device"], msgs


@pytest.mark.parametrize("pair", [p for p in PAIRS if p.notes], ids=[p.name for p in PAIRS if p.notes])
def test_note_capacity_error_names_the_entry_point_called(model, inp, pair):
    """(c) A note capacity of one: both entry points fail with BP_E_CAPACITY and a message naming themselves, and
    bp_last_required reports the same need after either."""
    from basic_pitch_b200 import _lib

    need = {}
    for entry in ("device", "host"):
        rest, out, keep = pair.args(model, inp, None, note_cap=1)
        with pytest.raises(_lib.BpError) as e:
            pair.call(model, inp, entry, rest)
        assert e.value.code == _lib.BP_E_CAPACITY, str(e.value)
        assert f"{pair.name}_{entry}: note_capacity too small" in str(e.value), str(e.value)
        a, b = C.c_int64(0), C.c_int64(0)
        model._lib.bp_last_required(C.byref(a), C.byref(b))
        need[entry] = a.value
    assert need["host"] == need["device"] > 1, need
