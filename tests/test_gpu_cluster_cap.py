"""The cap on resident clusters of the clustered FP64 store kernel: by default
at most MAX_STORE_CLUSTERS (6) clusters of 16 CTAs run, RTX_MAX_CLUSTERS
overrides it, and the number of clusters changes which CTA stores which tile
but not one stored byte.  Needs a GPU: `pytest -m gpu`."""
import numpy as np
import pytest

from conftest import load_systems

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5


def _engine(monkeypatch, max_clusters):
    from rayopt_b200.engine import Engine
    if max_clusters is None:
        monkeypatch.delenv("RTX_MAX_CLUSTERS", raising=False)
    else:
        monkeypatch.setenv("RTX_MAX_CLUSTERS", str(max_clusters))
    return Engine(0)


def _trace(eng, ent, n, ld, li=0):
    table = ent["tables"][li]
    S = len(table)
    aim = ent["aim"][li][3]
    y0, u0 = eng.aim_infinite_device(aim["field"], aim["z"], aim["p"], ent["object_angle"],
                                     nrays=int(n*1.01) + 1000)
    out = [eng.empty((S, ld, 3)) for _ in range(3)] + [eng.empty((S, ld))]
    for a in out:
        eng.memset(a, SENTINEL)
    eng.trace_device(table, y0, u0, *out, N=n, ld=ld, clip=True)
    eng.sync()
    assert eng.last_launch_config() == (2, 2, 16, 1, 16)
    ctas = eng.last_launch_ctas()
    host = [a.download() for a in out]
    for a in out + [y0, u0]:
        a.free()
    return ctas, host


@pytest.mark.parametrize("n, ld, li", [(2_000_017, 2_000_064, 1), (1_600_000, 1_600_000 + 5*64, 0)])
def test_capped_launch_stores_the_same_bytes(monkeypatch, n, ld, li):
    ent = load_systems()["double_gauss"]
    eng = _engine(monkeypatch, None)
    try:
        ctas, got = _trace(eng, ent, n, ld, li)
    finally:
        eng.close()
    assert ctas % 16 == 0 and 16 <= ctas <= 6*16, ctas
    for cap in (0, 3):  # all clusters that fit; fewer than the default
        e = _engine(monkeypatch, cap)
        try:
            c, want = _trace(e, ent, n, ld, li)
        finally:
            e.close()
        assert c % 16 == 0 and (c >= ctas if cap == 0 else c == 3*16), (cap, c)
        for a, b, w in zip(got, want, "yuit"):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), \
                "cap %d, %s: %d words differ" % (cap, w, np.count_nonzero(a.view(np.uint64) != b.view(np.uint64)))
