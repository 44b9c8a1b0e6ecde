"""GPU: the unwrapping entry points run the tensor-core convs on the trimmed row maps (tc_row_map, csrc/tc_conv.cu:
only the frames the kept centre frames depend on), bp_forward_* on the uniform ones (whole windows).  Every kept
posteriorgram value must be bit-identical between the two, for files whose last window keeps every class of frame
count (none, 1, 13, 126 and others), for calls of more than one chunk of windows, under every synthetic weight set,
and with forward and unwrapping calls interleaved on one model (the trimmed calls write the note conv's operand where
the uniform layout keeps zero rows)."""
import numpy as np
import pytest

from oracle import host_ref
from tests import weightsets
from tests.test_gpu_weightsets import blob_paths, models  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu

HOP, LEAD, KEEP = 36164, 3840, 142
POSTS = ("note", "onset", "contour")


def _geometry(n):
    """(windows, frames) of a file of n samples (bp_num_windows / bp_num_frames)"""
    return (n + LEAD + HOP - 1) // HOP, int(n / HOP * KEEP) if n > 0 else 0


def _length(full, r):
    """a file length whose last window (index `full`) keeps r frames (r <= 0: none)"""
    n0 = max(1, int((KEEP * full + r) * HOP / KEEP) - 2 * HOP // KEEP)
    for n in range(n0, n0 + 4 * HOP):
        nw, nf = _geometry(n)
        if nw == full + 1 and nf - full * KEEP == r:
            return n
    raise AssertionError((full, r))


def _clips(seed, spec):
    rng = np.random.default_rng(seed)
    out = []
    for full, r in spec:
        n = _length(full, r)
        t = np.arange(n) / 22050.0
        f = rng.uniform(80.0, 2000.0, 3)
        x = sum(0.3 * np.sin(2 * np.pi * fk * t) for fk in f) + 0.05 * rng.standard_normal(n)
        out.append((x * (t < n / 22050.0 * rng.uniform(0.5, 1.0))).astype(np.float32))
    return out


# (windows before the last, frames the last keeps): every last-window class, on files of 1 .. 7 windows.  A last
# window keeps -15 .. 126 frames (it starts less than one hop before the end); the others keep 142.
SPEC = [(0, 1), (0, 13), (0, 126), (1, 126), (1, -15), (1, -1), (1, 0), (2, 1), (3, 13), (6, 125), (6, 13), (4, 77),
        (5, 126), (2, 100), (0, 60)]


def _forward_unwrapped(model, clips):
    """bp_forward_* on the windowed files (uniform row maps), unwrapped on the host"""
    wins = [host_ref.window_audio(c) for c in clips]
    raw = model.predict(np.concatenate(wins))
    out, w0 = [], 0
    for c, w in zip(clips, wins):
        out.append({k: host_ref.unwrap(raw[k][w0 : w0 + len(w)], len(c)) for k in POSTS})
        w0 += len(w)
    return out


def _assert_bits(got, exp, label):
    for i, (g, e) in enumerate(zip(got, exp)):
        for k in POSTS:
            assert g[k].shape == e[k].shape, (label, i, k, g[k].shape, e[k].shape)
            bad = np.argwhere(g[k].view(np.uint32) != e[k].view(np.uint32))
            assert not len(bad), f"{label}: file {i} {k}: {len(bad)} values differ, first at frame / bin {bad[0].tolist()}"


@pytest.mark.parametrize("wset", weightsets.NAMES)
def test_trimmed_rows_match_whole_windows(models, wset):  # noqa: F811
    model = models[wset]
    model.set_path(1)
    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    clips = _clips(1, SPEC)
    classes = sorted({_geometry(len(c))[1] - (_geometry(len(c))[0] - 1) * KEEP for c in clips})
    print(f"{wset}: {len(clips)} files, {sum(_geometry(len(c))[0] for c in clips)} windows; last-window frames {classes}")
    ref = _forward_unwrapped(model, clips)
    before = model.predict(np.concatenate([host_ref.window_audio(c) for c in clips[:3]]))
    _assert_bits(model.run_inference_arrays(clips), ref, f"{wset} run_inference")
    # forward after a trimmed call: the uniform note conv must see its zero rows again
    after = model.predict(np.concatenate([host_ref.window_audio(c) for c in clips[:3]]))
    for k in POSTS:
        assert np.array_equal(before[k].view(np.uint32), after[k].view(np.uint32)), (wset, k)
    outs, res, _ = model.transcribe_arrays(clips)
    _assert_bits(outs, ref, f"{wset} transcribe")
    exp = model.decode_arrays([r["note"] for r in ref], [r["onset"] for r in ref], [r["contour"] for r in ref])
    for i, (g, e) in enumerate(zip(res, exp)):
        for k in e:
            assert np.array_equal(g[k], e[k]), (wset, i, k)
    # more than one chunk of windows in one call: the row maps start again at every chunk
    many = _clips(2, [(6, 125), (5, 13), (4, 1), (6, 126)] * (chunk // 24 + 2))
    assert sum(_geometry(len(c))[0] for c in many) > chunk
    _assert_bits(model.run_inference_arrays(many), _forward_unwrapped(model, many), f"{wset} {len(many)} files")
