"""Host-side logic of rayopt_b200.opds: the (mm, rm) Analysis.opds takes from
the last height with rays, the rtx_opd record's radius rule and frame
change, and argument checks that come before any device work."""
import types

import numpy as np
import pytest

from rayopt_b200.lazy import opd_spec
from rayopt_b200.opd import opds, scales


def height(max_abs, ee, dx):
    return dict(max_abs=max_abs, ee=np.asarray(ee, float), dx=dx)


def test_scales_from_the_last_height_with_rays():
    a = height(.5, [.2, .6, .95, 1.], .25)
    b = height(2., [.1, .3, .5, .91, 1.], .5)
    # Analysis walks the heights in reverse: the last one with rays sets both
    assert scales([a, None, b]) == (2., 3*1.5*.5)
    assert scales([a, b, None]) == (2., 3*1.5*.5)
    assert scales([a, None, None]) == (.5, 2*1.5*.25)
    assert scales([None, None]) == (None, None)
    assert scales([]) == (None, None)
    # np.searchsorted(ee, .9): the first bin whose cumulative energy reaches .9
    assert scales([height(1., [.9, 1.], 1.)]) == (1., 0.)


class FakeSystem(list):
    """the attributes opd_spec reads of a rayopt System"""


def fake_system(telecentric, distance=-80., finite=False, rotated=False):
    s = FakeSystem(types.SimpleNamespace(rotated=False) for _ in range(4))
    s[2] = types.SimpleNamespace(rotated=rotated,
                                 rot_normal=np.array([[0., -1, 0], [1, 0, 0], [0, 0, 1]]))
    s.image = types.SimpleNamespace(pupil=types.SimpleNamespace(telecentric=telecentric,
                                                                distance=distance))
    s.object = types.SimpleNamespace(finite=finite)
    return s


@pytest.mark.parametrize("telecentric", [False, True])
@pytest.mark.parametrize("rotated", [False, True])
def test_opd_spec_radius_and_frame(telecentric, rotated):
    s = fake_system(telecentric, rotated=rotated)
    track = np.array([0., 10., 35., 95.])
    origins = np.array([[0., 0, 0], [0, 0, 10], [0, 1, 35], [0, 2, 95]])
    y0, u0, yi = np.array([0., 1, 0]), np.array([0., 0, 1]), np.array([.1, .2, 0])
    spec = opd_spec(s, track, origins, 2, 3, 1.0, 1.5, y0, u0, yi)
    assert spec["radius"] == (95. - 35. if telecentric else 80.)
    assert opd_spec(s, track, origins, 2, 3, 1.0, 1.5, y0, u0, yi, radius=7.)["radius"] == 7.
    Ra = s[2].rot_normal if rotated else np.eye(3)
    assert np.array_equal(spec["M"], Ra @ np.eye(3).T)
    assert np.array_equal(spec["d"], (origins[2] - origins[3]) - yi)
    assert spec["n0"] == 1. and spec["n_after"] == 1.5 and spec["infinite"]
    assert spec["y0_ref"] is y0 and spec["u0_ref"] is u0


def test_opds_refuses_before_device_work():
    with pytest.raises(ValueError, match="triangulation"):
        opds(None, triangulation="gpu")
