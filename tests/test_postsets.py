"""CPU: the adversarial posteriorgram sets of tests/postsets.py reach what they are built for (liveness), and the decode
comparison they feed has teeth: NumPy mutants of the decode, each a one-line slip a kernel could make, disagree with
oracle/decode_ref.py on at least one case.

Both rest on `decode`, a pick-by-pick restatement of the reference decode (reference: basic_pitch/note_creation.py
:182-219, :289-511) that can record what each step saw and can be mutated.  Unmutated it equals decode_ref exactly."""
import numpy as np
import pytest

from oracle import decode_ref
from tests import postsets

BLOCK = postsets.BLOCK


def decode(note, onset, contour, p, mut=(), trace=None):
    """[(start, end, pitch, amp, bends)] of one file.  `mut`: names of slips to make (see MUTANTS); `trace`: a dict
    that receives the melodia picks and every scan."""
    n_t = note.shape[0]
    if n_t == 0:
        return []
    frames, onsets = np.array(note), np.array(onset)
    lo, hi = p["lo_col"], p["hi_col"]
    for m in (frames, onsets):
        m[:, :lo] = 0
        m[:, hi:] = 0
    with np.errstate(all="ignore"):
        if p["infer_onsets"]:
            onsets = decode_ref.infer_onsets(onsets, frames)
        pk = decode_ref.strict_time_peaks(onsets)
        cand_t, cand_f = np.where(np.where(pk, onsets, 0.0) >= p["onset_thresh"])
    tol, thr, mnl = p["energy_tol"], p["frame_thresh"], p["min_note_len"]
    stop = tol - 1 if "run_one_short" in mut else tol
    E = frames.astype(np.float64)
    scans = [] if trace is None else trace.setdefault("scans", [])
    picks = [] if trace is None else trace.setdefault("picks", [])

    def wipe(t0, t1, f):
        E[t0:t1, max(f - 1, 0) : f + 2] = 0

    def scan(i, step, f, wiping):
        start, quiet = i, 0
        while (i < n_t - 1 if step > 0 else i > 0) and quiet < stop:
            quiet = quiet + 1 if E[i, f] < thr else 0
            if wiping:
                wipe(i, i + 1, f)
            i += step
        if trace is not None:
            scans.append((start, step, i, quiet, tol))
        return i, quiet

    notes = []
    for t0, f in zip(cand_t[::-1], cand_f[::-1]):
        t0, f = int(t0), int(f)
        if t0 >= n_t - 1:
            continue
        i, quiet = scan(t0 + 1, 1, f, False)
        i -= quiet
        if i - t0 <= mnl:
            continue
        wipe(t0, i, f)
        notes.append((t0, i, f))
    while p["melodia_trick"] and E.max() > thr:
        top = E.max()
        cells = np.argwhere(E == top)  # (t, f) in the order np.argmax walks: frame, then pitch
        if "tie_highest_frame" in mut:
            tm, f = cells[cells[:, 0] == cells[:, 0].max()][0]
        elif "tie_highest_pitch" in mut:
            tm, f = cells[cells[:, 0] == cells[0, 0]][-1]
        else:
            tm, f = cells[0]
        tm, f = int(tm), int(f)
        E[tm, f] = 0
        i, q = scan(tm + 1, 1, f, True)
        t_end = i - 1 - q
        i, q = scan(tm - 1, -1, f, True)
        t_start = i + 1 + q
        picks.append(dict(tm=tm, f=f, v=top, ties=cells, note=(t_start, t_end)))
        if t_end - t_start > mnl:
            notes.append((t_start, t_end, f))

    win = decode_ref.gaussian_window(51, 5.0)
    out = []
    for a, b, f in notes:
        col = frames[a:b, f]
        if "amp_sequential" in mut:
            s = np.float32(0)
            for v in col:
                s = np.float32(s + v)
            amp = np.float32(s / np.float32(len(col)))
        elif "amp_float64" in mut:
            amp = np.float32(np.mean(col.astype(np.float64)))
        else:
            amp = np.mean(col)
        c = 3 * f
        top_bin = decode_ref.N_CONTOUR_BINS - (1 if "gauss_top_one_off" in mut else 0)
        lo_b, hi_b = max(c - 25, 0), min(top_bin, c + 26)
        w = win[max(0, 25 - c) : max(0, 25 - c) + hi_b - lo_b]
        sub = contour[a:b, lo_b:hi_b] * w
        if "bend_last_index" in mut:
            idx = sub.shape[1] - 1 - np.argmax(sub[:, ::-1], axis=1)
        else:
            idx = np.argmax(sub, axis=1)
        out.append((a, b, f + 21, amp, [int(x) for x in idx - (25 - max(0, 25 - c))]))
    return out


def oracle(note, onset, contour, p):
    if note.shape[0] == 0:
        return []
    with np.errstate(all="ignore"):
        wb, _ = decode_ref.model_output_to_note_events(
            {"note": np.array(note), "onset": np.array(onset), "contour": contour}, p["onset_thresh"], p["frame_thresh"],
            p["infer_onsets"], p["min_note_len"], melodia_trick=p["melodia_trick"], energy_tol=p["energy_tol"],
            lo_col=p["lo_col"], hi_col=p["hi_col"])  # fmt: skip
    return [(a, b, pitch, amp, [int(x) for x in bends]) for a, b, pitch, amp, bends in wb]


def same(x, y):
    """Bit-level equality of two note lists (amplitudes compared as float32 bytes)."""
    return len(x) == len(y) and all(
        a[:3] == b[:3] and np.float32(a[3]).tobytes() == np.float32(b[3]).tobytes() and a[4] == b[4] for a, b in zip(x, y))


# a few cases per set that the restatement is checked on (the whole grids run in tests/test_oracle_golden.py)
CHECKED = {"lengths": [1, 3], "ties": [0, 1, 5], "runs": [1, 3, 4, 5, 6], "crowded": [0, 1], "long_notes": [0, 1, 2],
           "pitch_edges": [0, 1, 2], "nan_file": [0, 1, 2]}  # fmt: skip


@pytest.mark.parametrize("name", postsets.NAMES)
def test_restatement_equals_decode_ref(name):
    files, grid = postsets.get(name)
    for j in CHECKED[name]:
        for i, f in enumerate(files):
            assert same(decode(*f, grid[j]), oracle(*f, grid[j])), f"{name}/p{j} file {i}"


def _liveness_ties():
    (f, f_long), grid = postsets.get("ties")
    reached = set()
    for j in (1, 3, 5):
        tr = {}
        notes = decode(*f, grid[j], trace=tr)
        picks = tr["picks"]
        n_t = f[0].shape[0]
        for k, pk in enumerate(picks):
            tm, col, ties = pk["tm"], pk["f"], pk["ties"]
            others = ties[(ties[:, 0] != tm) | (ties[:, 1] != col)]
            for t, g in others:
                if t // BLOCK != tm // BLOCK and abs(int(t) - tm) == 1:
                    reached.add("tie across a block boundary (t, t + 1)")
                if g == col and t // BLOCK != tm // BLOCK:
                    reached.add("tie in another block of the picked column")
                if t == tm and abs(int(g) - col) == 1:
                    reached.add("same-frame tie, adjacent column")
                if t == tm and abs(int(g) - col) > 1:
                    reached.add("same-frame tie, distant column")
            if len(others) and tm == 0:
                reached.add("tie, pick at t = 0")
            if len(others) and (tm == n_t - 1 or (others[:, 0] == n_t - 1).any()):
                reached.add("tie at t = T - 1")
            if k + 1 < len(picks):
                a, b = pk["note"][0] - grid[j]["energy_tol"], pk["note"][1] + grid[j]["energy_tol"]
                nx = picks[k + 1]
                touched = abs(nx["f"] - col) <= 1 and max(a, 0) // BLOCK <= nx["tm"] // BLOCK <= min(b, n_t - 1) // BLOCK
                reached.add("next maximum in a block the note touched" if touched else
                            "next maximum in a block the note did not touch")
        for a, b, _p, _amp, _bd in notes:
            if (b - 1) // BLOCK - a // BLOCK >= 2:
                reached.add("note spanning three or more blocks")
    tr = {}
    decode(*f_long, grid[0], trace=tr)
    for pk in tr["picks"]:
        if any(g == pk["f"] and abs(int(t) // BLOCK - pk["tm"] // BLOCK) == 32 for t, g in pk["ties"]):
            reached.add("tie 32 blocks apart in the picked column")
    return reached


def _liveness_runs():
    files, grid = postsets.get("runs")
    reached = set()
    for j, p in enumerate(grid):
        if p["energy_tol"] <= 32:
            continue
        for f in files:
            tr = {}
            decode(*f, p, trace=tr)
            for start, step, i, quiet, tol in tr["scans"]:
                if quiet < tol:
                    continue
                first = (i - quiet - start) * step if step > 0 else (start - (i + quiet))
                last = first + quiet - 1
                if first // 32 != last // 32:
                    reached.add(f"quiet run of {tol} frames across a 32-frame boundary of the scan ({'fwd' if step > 0 else 'bwd'})")
                if first in postsets.RUN_OFFSETS:
                    reached.add(f"run ending a note at offset {first} ({'fwd' if step > 0 else 'bwd'})")
    return reached


def test_ties_reach_their_targets():
    reached = _liveness_ties()
    print("ties:", sorted(reached))
    assert reached >= {
        "tie across a block boundary (t, t + 1)", "tie in another block of the picked column", "same-frame tie, adjacent column",
        "same-frame tie, distant column", "tie, pick at t = 0", "tie at t = T - 1", "next maximum in a block the note touched",
        "next maximum in a block the note did not touch", "note spanning three or more blocks",
        "tie 32 blocks apart in the picked column",
    }  # fmt: skip


def test_runs_reach_their_targets():
    reached = _liveness_runs()
    print("runs:", sorted(reached))
    for d in ("fwd", "bwd"):
        assert any(r.startswith("quiet run") and r.endswith(f"({d})") for r in reached), d
        for o in postsets.RUN_OFFSETS:
            assert f"run ending a note at offset {o} ({d})" in reached
    files, grid = postsets.get("runs")
    ends = set()
    for f in files:
        n_t = f[0].shape[0]
        for a, b, *_ in oracle(*f, grid[1]):
            ends |= {("end", n_t - b)} | {("start", a if a <= 1 else n_t - a)}
    edge = {("end", 1), ("end", 2), ("start", 1), ("start", 2)}  # ends at T - 1 / T - 2, starts at 1 / T - 2
    print("runs: notes at the file edges", sorted(edge & ends))
    assert edge <= ends


def test_crowded_needs_more_than_the_first_slot_allowance():
    files, grid = postsets.get("crowded")
    n_t = files[1][0].shape[0]
    counts = [len(oracle(*files[1], p)) for p in grid]
    print(f"crowded: {counts} notes in the middle file, first allowance {8 * n_t + 64}")
    assert sum(c > 8 * n_t + 64 for c in counts) >= 2


def test_long_notes_cover_every_length():
    (f,), grid = postsets.get("long_notes")
    lengths = {b - a for a, b, *_ in oracle(*f, grid[0])}
    print("long_notes: lengths", sorted(lengths))
    assert set(postsets.LONG_LENGTHS) <= lengths
    assert {b - a for a, b, *_ in oracle(*f, grid[1])} >= {ln - 1 for ln in postsets.LONG_LENGTHS if ln > 1}


def test_pitch_edges_have_tied_bends_at_both_clipped_ends():
    (f,), grid = postsets.get("pitch_edges")
    contour = f[2]
    win = decode_ref.gaussian_window(51, 5.0)
    tied = set()
    for a, b, pitch, *_ in oracle(*f, grid[0]):
        c = 3 * (pitch - 21)
        lo, hi = max(c - 25, 0), min(264, c + 26)
        sub = contour[a:b, lo:hi] * win[max(0, 25 - c) : max(0, 25 - c) + hi - lo]
        if ((sub == sub.max(axis=1, keepdims=True)).sum(axis=1) > 1).any():
            tied.add(pitch)
        if pitch == 108:
            assert (np.argmax(sub, axis=1) == sub.shape[1] - 1).any()  # the maximum on bin 263
    print("pitch_edges: pitches with a tied bend", sorted(tied))
    assert {21, 108} <= tied and set(postsets.EDGE_PITCHES) == {p for *_, p in postsets.edge_notes()}
    assert (contour < 0).any() and (contour > 1).any()


def test_lengths_and_nan_file_reach_their_targets():
    files, grid = postsets.get("lengths")
    ts = [f[0].shape[0] for f in files]
    assert sorted(ts) == sorted(postsets.LENGTHS) and ts != sorted(ts)
    assert grid[0]["onset_thresh"] <= 0 and grid[1]["onset_thresh"] < 0
    # a note from the candidate at t = 0 of a file whose first 32-cell word holds the previous file's last cells
    base, shared = 0, 0
    for f in files:
        if base * 88 % 32 and any(a == 0 for a, *_ in oracle(*f, grid[0])):
            shared += 1
        base += f[0].shape[0]
    print(f"lengths: {shared} files with a note at t = 0 in a shared candidate word")
    assert shared >= 5
    files, _ = postsets.get("nan_file")
    with np.errstate(all="ignore"):
        inf = [decode_ref.infer_onsets(f[1], f[0]) for f in files]
    assert np.isnan(inf[1]).all() and not np.isnan(inf[0]).any() and not np.isnan(inf[2]).any()
    assert files[3][1].max() == 0 and files[4][1].max() > 0


MUTANTS = {  # slip -> cases (set, parameter set) it is tried on
    "tie_highest_frame": [("ties", 1), ("ties", 5)],
    "tie_highest_pitch": [("ties", 1), ("ties", 5)],
    "run_one_short": [("runs", 3), ("runs", 4)],
    "amp_sequential": [("long_notes", 0)],
    "amp_float64": [("long_notes", 0)],
    "bend_last_index": [("pitch_edges", 0)],
    "gauss_top_one_off": [("pitch_edges", 0)],
}


@pytest.mark.parametrize("mut", sorted(MUTANTS))
def test_mutants_are_caught(mut):
    """Each slip changes the decode of at least one case of the sets (what a kernel making it would be caught on)."""
    caught = []
    for name, j in MUTANTS[mut]:
        files, grid = postsets.get(name)
        for i, f in enumerate(files):
            if not same(decode(*f, grid[j], mut=(mut,)), oracle(*f, grid[j])):
                caught.append(f"{name}/p{j} file {i}")
    print(f"{mut}: caught on {caught}")
    assert caught, mut
