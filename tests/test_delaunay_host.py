"""The device triangulation's step bodies (rtx_delaunay.cuh) run sequentially
on the CPU (tests/delaunay_host.cu, built here with nvcc into a temporary
directory) and checked by the exact checker: the topology of splits, 2 -> 4
splits, ghost flips, pointer repair, relocation and duplicates without a GPU."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.spatial import Delaunay

import delaunay_oracle as dto
from test_gpu_delaunay import (degenerate_sets, disc, exit_pupil, first_copies, triples,
                               with_extreme_copies)

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    out = str(tmp_path_factory.mktemp("dt") / "libdthost.so")
    subprocess.run([nvcc, "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                    "-gencode", "arch=compute_90a,code=sm_90a", "-o", out,
                    os.path.join(HERE, "delaunay_host.cu")], check=True)
    lib = C.CDLL(out)
    lib.dt_host.argtypes = [C.c_longlong, C.c_void_p, C.POINTER(C.c_longlong), C.c_void_p,
                            C.c_void_p, C.c_void_p]
    return lib


def run(lib, p):
    p = np.ascontiguousarray(p, np.float64)
    m = len(p)
    s, nb, tr = np.zeros((2*m, 3), np.int32), np.zeros((2*m, 3), np.int32), np.zeros((2*m, 3, 2))
    T = C.c_longlong()
    rc = lib.dt_host(m, p.ctypes.data, C.byref(T), s.ctypes.data, nb.ctypes.data, tr.ctypes.data)
    if rc:
        return rc
    return s[:T.value], nb[:T.value], tr[:T.value]


SETS = degenerate_sets()


@pytest.mark.parametrize("name", list(SETS))
def test_degenerate_sets_on_host(host_lib, name):
    p = SETS[name]
    s, nb, tr = run(host_lib, p)
    dto.check(p, s, nb, ccw=True)
    assert not np.isnan(tr).any()
    # exact duplicates: the lowest index is the vertex
    assert set(np.unique(s).tolist()) == first_copies(p), name
    dev_q, ref_q = dto.cocircular_differences(p, s, Delaunay(p).simplices)
    cs, cr = dto.canonical(p, s), dto.canonical(p, Delaunay(p).simplices)
    assert triples(cs) - triples(cr) <= dev_q
    assert triples(cr) - triples(cs) <= ref_q


@pytest.mark.parametrize("m", [3, 4, 5, 100, 3000])
def test_general_position_on_host(host_lib, m):
    p = with_extreme_copies(disc(m, m))
    s, nb, _ = run(host_lib, p)
    dto.check(p, s, nb, ccw=True)
    assert set(np.unique(s).tolist()) == first_copies(p)
    q = disc(m, m)
    assert triples(run(host_lib, q)[0]) == triples(Delaunay(q).simplices)


@pytest.mark.parametrize("name", ["psf_cooke_f07", "psf_double_gauss_f07"])
def test_exit_pupils_on_host(host_lib, name):
    p, _ = exit_pupil(name)
    s, nb, _ = run(host_lib, p)
    assert triples(s) == triples(Delaunay(p).simplices)
    dto.check(p, s, nb, ccw=True)


def test_refusals_on_host(host_lib):
    k = np.arange(20.)
    assert run(host_lib, np.stack([k, 2*k + 1], -1)) == -1          # all collinear
    q = disc(20, 1)
    q[3, 0] = np.nan
    assert run(host_lib, q) == -1
