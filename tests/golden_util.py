"""Helpers to read the fixtures written by oracle/make_golden.py."""
import numpy as np


def dequant(q):
    return q.astype(np.float32) / np.float32(65535.0)


def case_params(z, name):
    p = z[f"{name}/params"]
    return dict(
        onset_thresh=float(p[0]),
        frame_thresh=float(p[1]),
        min_note_len=int(p[2]),
        infer_onsets=bool(p[3]),
        melodia_trick=bool(p[4]),
        min_freq=None if p[5] < 0 else float(p[5]),
        max_freq=None if p[6] < 0 else float(p[6]),
    )


def case_expected(z, name):
    return {k: z[f"{name}/{k}"] for k in ("frames", "start", "end", "pitch", "amp", "bend_flat", "bend_off", "bend_has")}


def events_to_arrays(frames_notes_with_bends, events):
    """Convert decode output lists to the fixture array layout."""
    n = len(events)
    fr = np.array([[a, b, p] for a, b, p, _amp, _bd in frames_notes_with_bends], dtype=np.int32).reshape(-1, 3)
    flat, off = [], [0]
    for e in events:
        if e[4] is not None:
            flat.extend(int(v) for v in e[4])
        off.append(len(flat))
    return {
        "frames": fr,
        "start": np.array([e[0] for e in events], dtype=np.float64).reshape(n),
        "end": np.array([e[1] for e in events], dtype=np.float64).reshape(n),
        "pitch": np.array([e[2] for e in events], dtype=np.int32).reshape(n),
        "amp": np.array([e[3] for e in events], dtype=np.float32).reshape(n),
        "bend_flat": np.array(flat, dtype=np.int32),
        "bend_off": np.array(off, dtype=np.int32),
    }


def assert_events_equal(got, exp, amp_atol=0.0, ctx=""):
    assert got["frames"].shape == exp["frames"].shape, f"{ctx}: {got['frames'].shape[0]} notes, expected {exp['frames'].shape[0]}"
    np.testing.assert_array_equal(got["frames"], exp["frames"], err_msg=f"{ctx}: (start,end,pitch) frames")
    np.testing.assert_array_equal(got["pitch"], exp["pitch"], err_msg=f"{ctx}: pitch")
    np.testing.assert_array_equal(got["start"], exp["start"], err_msg=f"{ctx}: start times")
    np.testing.assert_array_equal(got["end"], exp["end"], err_msg=f"{ctx}: end times")
    np.testing.assert_array_equal(got["bend_off"], exp["bend_off"], err_msg=f"{ctx}: bend offsets")
    np.testing.assert_array_equal(got["bend_flat"], exp["bend_flat"], err_msg=f"{ctx}: pitch bends")
    if amp_atol == 0.0:
        np.testing.assert_array_equal(got["amp"], exp["amp"], err_msg=f"{ctx}: amplitude")
    else:
        np.testing.assert_allclose(got["amp"], exp["amp"], rtol=0, atol=amp_atol, err_msg=f"{ctx}: amplitude")


def edges_case(z, key):
    """The reference's notes for one set and parameter set of decode_edges.npz (`key` = "<set>/p<j>"), concatenated over
    the set's files: int32 start / end / pitch, float32 amp, int32 bends, the bend offsets (every note has end - start
    bends) and the per-file note offsets."""
    start, end, pitch = (z[f"{key}/{k}"].astype(np.int32) for k in ("start", "end", "pitch"))
    return {
        "start": start, "end": end, "pitch": pitch, "amp": z[f"{key}/amp"], "bends": z[f"{key}/bend_flat"].astype(np.int32),
        "bend_off": np.concatenate([[0], np.cumsum(end - start)]).astype(np.int32), "note_off": z[f"{key}/note_off"],
    }  # fmt: skip
