import glob
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
for p in (ROOT, os.path.join(ROOT, "oracle"), GOLDEN):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def _cuda_device_count():
    try:
        from rayopt_b200 import _lib
        return _lib.load().rtx_device_count()
    except Exception:
        return 0


def pytest_collection_modifyitems(config, items):
    """`gpu` tests are skipped (not errored) on a box without a CUDA device or
    without the built library, so that a CPU-only run reports the oracle /
    host-logic results cleanly"""
    if not any("gpu" in item.keywords for item in items):
        return
    if _cuda_device_count() >= 1:
        return
    skip = pytest.mark.skip(reason="no CUDA device / librtx.so (the engine has no CPU fallback)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def golden_names():
    return sorted(os.path.basename(p)[:-4]
                  for p in glob.glob(os.path.join(GOLDEN, "*.npz")))


def load_golden(name):
    d = np.load(os.path.join(GOLDEN, name + ".npz"))
    case = {k: d[k] for k in d.files}
    case["clip"] = bool(case["clip"])
    case["rot0"] = case["rot0"] if case["rot0"].size else None
    case["meta"] = json.loads(str(case["meta"]))
    case["name"] = name
    case["rotated"] = bool((case["table"]["flags"] & 1).any()
                           or case["rot0"] is not None)
    return case


def load_systems():
    from rayopt_b200.surface_table import table_from_json
    with open(os.path.join(GOLDEN, "systems.json")) as f:
        raw = json.load(f)
    for ent in raw.values():
        ent["tables"] = [table_from_json(t) for t in ent["tables"]]
    return raw


def assert_parity(got, want, rtol, what="", scale_floor=1.0, global_scale=False):
    """The comparator of SURVEY 8(d): identical NaN mask and
    |a-b| <= rtol*max(|b|, scale) with scale = max finite |b| of the array
    row (per surface) for lengths, 1 for direction cosines."""
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), "%s: NaN mask differs at %d entries" % (
        what, np.count_nonzero(gn != wn))
    fin = ~wn
    if not fin.any():
        return 0.0
    # per-surface scale (axis 0 = surface)
    absw = np.where(fin, np.abs(want), 0.0)
    scale = absw.reshape(absw.shape[0], -1).max(1)
    if global_scale:      # one scale for the whole trace (the lens's size)
        scale = np.full_like(scale, scale.max())
    scale = np.maximum(scale, scale_floor).reshape((-1,) + (1,)*(want.ndim - 1))
    with np.errstate(invalid="ignore"):
        err = np.where(fin, np.abs(got - want)/np.maximum(np.abs(want), scale), 0.0)
    worst = float(err.max())
    assert worst <= rtol, "%s: rel err %.3e > %.1e" % (what, worst, rtol)
    return worst


@pytest.fixture(scope="session")
def systems():
    return load_systems()
