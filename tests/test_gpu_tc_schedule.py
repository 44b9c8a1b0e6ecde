"""GPU: a frame's posteriorgram values do not depend on the items the tensor-core convs cut a batch into (tc_schedule,
csrc/tc_conv.cu).  Batch sizes are chosen from the library's own schedules (bp_debug_tc_schedule) so that every
schedule class of every launch is reached on this device: whole M-tiles only, cut M-tiles only, or both, with every
set of group ranges the planner picks for the cut ones (the boundaries edge_fix_kernel finishes move with them).  Three
distinct windows tiled to each size must give bit-identical posteriorgrams at every size and position, on forward
paths 1 (contour conv2 fused) and 2, under the trained and the dense weights, and match the oracle once."""
import numpy as np
import pytest

from tests.test_gpu_weightsets import POSTS, _check_forward, blob_paths, models, windows  # noqa: F401 (fixtures)
from tests.test_tc_schedule import schedule

pytestmark = pytest.mark.gpu

LAUNCHES = {"contour (fused, path 1)": (0, 1), "contour (path 2)": (0, 0), "onset": (1, 1), "note": (2, 1)}


def schedule_class(which, fused, n_windows, n_sms):
    s, items, _ = schedule(which, fused, n_windows, n_sms)
    tail = tuple(sorted({(int(g0), int(g1)) for _mt, g0, g1 in items[s["n_full"]:]}))
    return s["n_full"] > 0, tail


def sweep_sizes(chunk, n_sms):
    """batch sizes (<= one chunk) that reach every schedule class of every launch, greedy; and the classes per launch"""
    classes = {k: {} for k in LAUNCHES}
    for n in range(1, chunk + 1):
        for k, (which, fused) in LAUNCHES.items():
            classes[k].setdefault(schedule_class(which, fused, n, n_sms), set()).add(n)
    need = {(k, c) for k in LAUNCHES for c in classes[k]}
    sizes = []
    while need:
        best = max(range(1, chunk + 1), key=lambda n: (sum(n in classes[k][c] for k, c in need), -n))
        sizes.append(best)
        need -= {(k, c) for k, c in need if best in classes[k][c]}
    return sorted(sizes), classes


@pytest.mark.parametrize("wset", ["trained", "dense"])
def test_every_schedule_gives_bit_identical_windows(models, windows, wset):  # noqa: F811
    import torch

    model = models[wset]
    n_sms = torch.cuda.get_device_properties(model.device).multi_processor_count
    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    sizes, classes = sweep_sizes(chunk, n_sms)
    print(f"{n_sms} SMs, chunk {chunk}: {len(sizes)} batch sizes {sizes}; schedule classes per launch "
          + ", ".join(f"{k}: {len(v)}" for k, v in classes.items()))
    for k, (which, fused) in LAUNCHES.items():
        assert {schedule_class(which, fused, n, n_sms) for n in sizes} == set(classes[k]), k
    base = windows[[0, 1, 8]]  # two music windows and the click at sample 20 000
    for path in (1, 2):
        ref = _check_forward(model, wset, base, path, "sched", label=" (3 distinct windows)")
        model.set_path(path)
        try:
            for n in sizes:
                x = np.ascontiguousarray(np.tile(np.roll(base, n % 3, axis=0), (-(-n // 3), 1))[:n])
                got = model.predict(x)
                for i in range(n):
                    j = (i - n % 3) % 3
                    for k in POSTS:
                        if not np.array_equal(got[k][i], ref[k][j]):
                            d = float(np.abs(got[k][i] - ref[k][j]).max())
                            pytest.fail(f"{wset} path {path}: batch of {n}, window {i} (= distinct window {j}): {k} differs by {d:.3e}")
        finally:
            model.set_path(1)
