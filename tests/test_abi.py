"""CPU-side checks of the C-ABI library: it loads without a GPU and exports
every symbol include/rtx.h declares; argument errors are reported, and there
is no CPU fallback."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from rayopt_b200 import _lib, build
from rayopt_b200.surface_table import SURFACE_DTYPE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_header_symbols_all_exported(lib):
    text = open(os.path.join(ROOT, "include", "rtx.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    declared = set(re.findall(r"\b(rtx_[a-z0-9_]+)\s*\(", text))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    raw = C.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), name


def test_abi_version_matches_header_and_layout(lib):
    """version 3: the library reports the version include/rtx.h declares"""
    text = open(os.path.join(ROOT, "include", "rtx.h")).read()
    declared = int(re.search(r"#define\s+RTX_ABI_VERSION\s+(\d+)", text).group(1))
    assert lib.rtx_abi_version() == declared == 3
    assert lib.rtx_sizeof_surface() == SURFACE_DTYPE.itemsize
    from rayopt_b200.engine import OPD_DTYPE
    from rayopt_b200.rays import aim_dtype
    assert lib.rtx_sizeof_opd() == OPD_DTYPE.itemsize       # struct rtx_opd
    assert lib.rtx_sizeof_aim() == aim_dtype().itemsize     # struct rtx_aim


def test_selftest_math2_refuses_bad_arguments(lib):
    """the primitives' self-test entry point checks its arguments before any
    device work (ABI version 3)"""
    a = np.ones(4)
    p = a.ctypes.data_as(C.c_void_p)
    assert lib.rtx_selftest_math2(None, 4, p, p, p, p) == -1         # RTX_E_BADARG
    assert lib.rtx_abi_version() == 3


def test_strerror(lib):
    assert b"bad argument" in lib.rtx_strerror(-1)
    assert lib.rtx_strerror(0) == b"ok"


def test_surface_finalize_matches_packer(lib):
    """the C helper and the Python packer agree on the derived members"""
    from rayopt_b200.surface_table import pack_element

    class E:
        offset = (0, 0, 2.)
        rotated = False
        curvature = 1/21.25
        conic = -.3
        aspherics = [0, 2e-6, -1e-8]
        radius = 6.5

        def get_n_mu(self, n0, l):
            return 1.62, n0/1.62
    t = np.zeros(1, SURFACE_DTYPE)
    pack_element(t[0], E(), 1.0003, 587e-9)
    t2 = t.copy()
    for k in ("kc2", "radius2", "muf", "sgn", "mu2m1", "dasph"):
        t2[k] = -7
    r = np.array([6.5])
    assert lib.rtx_surface_finalize(t2.ctypes.data_as(C.c_void_p), 1,
                                    r.ctypes.data_as(C.c_void_p)) == 0
    for k in ("kc2", "radius2", "muf", "sgn", "mu2m1", "dasph"):
        np.testing.assert_allclose(t2[k], t[k], rtol=1e-15)


@pytest.mark.skipif(_lib.load().rtx_device_count() > 0 if os.path.exists(_lib.LIB_PATH) else False,
                    reason="GPU present")
def test_no_cpu_fallback():
    """without a GPU the engine refuses to trace"""
    from rayopt_b200.engine import Engine
    with pytest.raises(_lib.RtxError):
        Engine(0)


def test_cpu_reference_arm_harness():
    """oracle/cpu_bench.py (the bench's reference arm): persistent worker
    processes, whole-workload sharding, both kinds -- a tiny run on two
    processes returns a consistent record"""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import cpu_bench
    kinds = ["port"] + (["reference"] if cpu_bench.reference_available() else [])
    for kind in kinds:
        r = cpu_bench.run("double_gauss", (0., .7), procs=2, steps=2, warmup=2, kind=kind,
                          rays_total=4001, warm_rays=100)
        assert r["kind"] == kind and r["cores"] == 2 and r["rays_per_proc"] == 2001
        assert r["surfaces"] == 12 and r["wavelengths"] == 3 and len(r["seconds"]) == 2
        assert r["ray_surfaces_per_step"] == 2*2001*3*12
        assert abs(r["value"] - r["ray_surfaces_per_step"]*2/sum(r["seconds"])) < 1e-6*r["value"]
