"""The kernel the library picks changes the speed of a trace, never its numbers.

For one set of probe rays per system, every kernel configuration and every
front end stores bit-identical y, u, i, t for every probe ray, in each mode
(RTX_EXACT, fast FP64, FP32).  The reference result of a system and mode is
the per-thread store kernel at N = the probe count (`canon`); it is itself
checked against the numpy oracle once.  Every case also asserts, through
Engine.last_launch_config(), that the launch landed in the configuration it
targets, so that a moved threshold cannot quietly turn the matrix into
repeats of one kernel.

Bundles larger than the probe set are the probe rays tiled on the device:
ray j*P + k is probe k, so tile boundaries and the ragged tail are compared
too, one surface row at a time.

Systems: Cooke with even aspheres aimed at fields 0 and 0.7, the Newton
edge goldens, seeded random systems with tilted surfaces and aspheres of up
to 10 coefficients (beyond the 4 the Newton loop keeps in registers),
Double-Gauss and the zoom as analytic controls, and 256 thin plates whose
FP64 table forces the shared-memory step-down.  Needs a GPU: `pytest -m gpu`.
"""
import os

import numpy as np
import pytest

import np_oracle
from conftest import assert_parity, load_golden, load_systems
from rayopt_b200.engine import DeviceArray
from rayopt_b200.rays import aim_infinite, disc
from rayopt_b200.surface_table import SURFACE_DTYPE

pytestmark = pytest.mark.gpu

DIRECT, WARP, CTA = 0, 1, 2                     # store paths (rtx_last_launch_config)
R1W8 = (1, WARP, 8, 2, 1)
PER_RAY = (1, DIRECT, 8, 1, 1)
MODES = {"exact": (np.float64, True), "fast": (np.float64, False), "fp32": (np.float32, False)}
# the instantiated tuning space (rtx.cu KERNELS), forced through RTX_* in a fresh engine
FORCED = {
    "r1w8": (R1W8, 1), "r2w8": ((2, WARP, 8, 2, 1), 1), "r2c16": ((2, CTA, 16, 1, 1), 1),
    "r1c16": ((1, CTA, 16, 1, 1), 1), "r2c32": ((2, CTA, 32, 1, 1), 1),
    "r2c8": ((2, CTA, 8, 1, 1), 1), "r2w16": ((2, WARP, 16, 2, 1), 1),
    "r4c16": ((4, CTA, 16, 1, 1), 1), "r4w16": ((4, WARP, 16, 1, 1), 1),
    "cluster16": ((2, CTA, 16, 1, 16), 1),
    "r2w8_free": ((2, WARP, 8, 2, 1), 0), "r2w16_free": ((2, WARP, 16, 2, 1), 0),
}
FP32_ONLY, FP64_ONLY = ("r4c16", "r4w16"), ("cluster16",)   # (FP32 clusters are not instantiated)
NEWTON = ["cooke_asph", "newton_edge_clip0", "newton_edge_clip1", "cooke_asph_f07_clip",
          "rand_asph0", "rand_asph1", "rand_asph2"]
ANALYTIC = ["double_gauss", "zoom"]
MIN_FORCED = 40_017      # tuned engines take the one-ray kernel up to 32 768 rays


# ---- seeded random systems (the generator of test_gpu_random_systems.py, with
# aspheres of up to RTX_MAX_ASPH coefficients and at least one tilted surface)
def euler(a, b, c):
    ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
    rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
    return rx @ ry @ rz


def random_table(rng, S):
    t = np.zeros(S, SURFACE_DTYPE)
    n0 = 1.0
    for j in range(S):
        r = t[j]
        r["offset"] = (0, 0, rng.uniform(.5, 6.))
        r["rot"] = np.eye(3).reshape(9)
        flags = 0
        if j == 2 or rng.random() < .3:
            r["offset"][:2] = rng.normal(0, .05, 2)
            r["rot"] = euler(*rng.normal(0, .03, 3)).reshape(9)
            flags |= 1
        kind = "asph" if j in (0, 1) else rng.choice(["sphere", "conic", "plane", "asph"])
        c = 0. if kind == "plane" else rng.choice([-1, 1])/rng.uniform(8., 200.)
        k = rng.uniform(-1.5, .8) if kind in ("conic", "asph") and rng.random() < .7 else 0.
        r["c"], r["k"] = c, k
        r["kc2"] = (1 + k)*c**2
        radius = rng.uniform(3., 6.)
        r["radius2"] = radius**2 if rng.random() < .8 else np.inf
        u = rng.random()
        if u < .08:
            n, mu = n0, -1.                        # mirror
        elif u < .16:
            n, mu = n0, 1.                         # no material
        else:
            n = rng.choice([1.0, rng.uniform(1.4, 1.9)]) if n0 > 1 else rng.uniform(1.4, 1.9)
            mu = n0/n
        r["mu"], r["muf"], r["sgn"], r["mu2m1"] = mu, abs(mu), np.sign(mu), mu**2 - 1
        r["n0"], r["n"] = n0, n
        n0 = n
        r["n_asph"] = -1
        if kind == "asph":
            # surface 0: 5..10 coefficients (the loop over the table's
            # coefficients); elsewhere 1..10
            na = int(rng.integers(5, 11)) if j == 0 else int(rng.integers(1, 11))
            a = rng.normal(0, 1, na)*10.0**(-3 - 2*np.arange(na))
            r["n_asph"] = na
            r["asph"][:na] = a
            r["dasph"][:na] = [2*(i + 1)*a[i] for i in range(na)]
        if kind != "plane" and rng.random() < .05:
            flags |= 2                             # alternate intersection
        r["flags"] = flags
    return t


def random_rays(rng, n):
    y = np.c_[rng.normal(0, 1.2, (n, 2)), np.zeros(n)]
    u = rng.normal(0, .08, (n, 2))
    return y, np.c_[u, np.sqrt(1 - np.square(u).sum(1))]


def plates(S=256):
    """thin plane-parallel plates: a 92 KB FP64 table"""
    big = np.zeros(S, SURFACE_DTYPE)
    big["rot"] = np.eye(3).reshape(9)
    big["offset"][:, 2] = .01
    big["radius2"] = np.inf
    big["n_asph"] = -1
    nn = np.where(np.arange(S) % 2 == 0, 1.5, 1.0)
    n0 = np.r_[1.0, nn[:-1]]
    big["n0"], big["n"] = n0, nn
    big["mu"] = n0/nn
    big["muf"], big["sgn"], big["mu2m1"] = np.abs(big["mu"]), np.sign(big["mu"]), big["mu"]**2 - 1
    return big


def _make_system(name, systems):
    """dict: tables (one per wavelength), rot0, clip, probe rays y0, u0 (float64),
    newton (>= 25 % Newton surfaces), bit (exact mode is bit-identical to the
    oracle), exact_rtol, fp32 (None: no FP32 oracle check; 'edge': mask-aware)"""
    d = dict(rot0=None, bit=False, exact_rtol=1e-12, fp32="plain")
    # (fp32 "edge": goldens built on Newton's limit of convergence, where the
    # float32 NaN mask legitimately depends on the last bit)
    if name in ("cooke_asph", "double_gauss", "zoom"):
        ent = systems[name]
        n = {"cooke_asph": 100_000, "double_gauss": 50_000, "zoom": 25_000}[name]
        ys, us = zip(*[aim_infinite(a["field"], disc(n, 40 + fi), a["z"], a["p"],
                                    ent["object_angle"])
                       for fi, a in ((0, ent["aim"][0][0]), (3, ent["aim"][0][3]))])
        d.update(tables=ent["tables"], clip=True, y0=np.concatenate(ys), u0=np.concatenate(us),
                 newton=name == "cooke_asph", bit=name != "cooke_asph")
    elif name.startswith("rand_asph"):
        rng = np.random.default_rng(3000 + int(name[-1]))
        table = random_table(rng, int(rng.integers(4, 9)))
        y0, u0 = random_rays(rng, 30_000)
        # exact mode: 1e-10, as test_gpu_random_systems allows on every ray of a
        # random tilted system; FP32 on random systems is checked there, on
        # well-conditioned rays only
        d.update(tables=[table], clip=bool(int(name[-1]) % 2), y0=y0, u0=u0, newton=True,
                 rot0=euler(.01, -.02, .015) if name.endswith("0") else None,
                 exact_rtol=1e-10, fp32=None)
    elif name == "plates256":
        rng = np.random.default_rng(5)
        u = rng.normal(0, .1, (2048, 2))
        d.update(tables=[plates()], clip=False, y0=np.c_[rng.normal(0, 1, (2048, 2)),
                                                          np.zeros(2048)],
                 u0=np.c_[u, np.sqrt(1 - np.square(u).sum(1))], newton=False, bit=True)
    else:
        c = load_golden(name)
        d.update(tables=[c["table"]], rot0=c["rot0"], clip=c["clip"], y0=c["y0"], u0=c["u0"],
                 newton=True, fp32="edge" if name.startswith("newton_edge") else "plain")
    return d


@pytest.fixture(scope="module")
def sysdb():
    systems = load_systems()
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _make_system(name, systems)
        return cache[name]
    return get


@pytest.fixture(scope="module")
def eng():
    from rayopt_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def forced():
    """engines pinned to one configuration each (RTX_* are read by rtx_init)"""
    from rayopt_b200.engine import Engine
    engines = {}

    def get(cfg_name):
        if cfg_name not in engines:
            (rpt, store, warps, nbuf, cluster), lock = FORCED[cfg_name]
            env = dict(RTX_RPT=rpt, RTX_STORE=store, RTX_WARPS=warps, RTX_NBUF=nbuf,
                       RTX_CLUSTER=cluster, RTX_LOCK=lock)
            saved = {k: os.environ.get(k) for k in env}
            try:
                os.environ.update({k: str(v) for k, v in env.items()})
                engines[cfg_name] = Engine(0)
            finally:
                for k, v in saved.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return engines[cfg_name]
    yield get
    for e in engines.values():
        e.close()


@pytest.fixture(scope="module")
def canon(eng, sysdb):
    """(system, mode, wavelength) -> host y, u, i, t (S, P, k) of the probe rays
    from the per-thread store kernel"""
    cache = {}

    def get(name, mode, li=0):
        key = (name, mode, li)
        if key not in cache:
            s = sysdb(name)
            dtype, exact = MODES[mode]
            table = s["tables"][li]
            P, S = len(s["y0"]), len(table)
            dy, du = eng.to_device(s["y0"], dtype), eng.to_device(s["u0"], dtype)
            out = _outputs(eng, S, P, dtype)
            eng.trace_device(table, dy, du, *out, N=P, ld=P, clip=s["clip"], rot0=s["rot0"],
                             exact=exact, direct=True)
            eng.sync()
            assert eng.last_launch_config() == PER_RAY
            cache[key] = [a.download() for a in out]
            for a in out + [dy, du]:
                a.free()
        return cache[key]
    return get


# ---- helpers --------------------------------------------------------------
def _view(a, byte_off, shape):
    """a DeviceArray aliasing `a` from byte `byte_off` (no copy, not owned)"""
    v = object.__new__(DeviceArray)
    v.engine, v.dtype, v.shape = a.engine, a.dtype, tuple(shape)
    v.nbytes = int(np.prod(v.shape))*a.dtype.itemsize
    v.ptr = a.ptr + byte_off
    v.free = lambda: None
    v._parent = a
    return v


def _outputs(e, rows, ld, dtype, offset=0):
    """Y, U, I (rows, ld, 3), T (rows, ld); `offset` > 0: outputs that start
    `offset` bytes into their allocation (not 16-byte aligned)"""
    out = []
    for k in (3, 3, 3, 1):
        shape = (rows, ld, k) if k == 3 else (rows, ld)
        if offset:
            base = e.empty((int(np.prod(shape)) + 16//np.dtype(dtype).itemsize,), dtype)
            out.append(_view(base, offset, shape))
            out[-1].free = base.free
        else:
            out.append(e.empty(shape, dtype))
    return out


def _tiled(e, s, dtype, N):
    """device y0, u0 of N rays: the probe rays repeated (ray j*P + k = probe k)"""
    P, isz = len(s["y0"]), np.dtype(dtype).itemsize
    res = []
    for h in (s["y0"], s["u0"]):
        probe = e.to_device(h, dtype)
        d = e.empty((N, 3), dtype)
        for j in range(0, N, P):
            n = min(P, N - j)
            _view(d, j*3*isz, (n, 3)).copy_from(probe, n*3*isz)
        e.sync()
        probe.free()
        res.append(d)
    return res


def _host_tiled(s, N):
    k = np.arange(N) % len(s["y0"])
    return s["y0"][k], s["u0"][k]


def _bad(a, b):
    """(n,) rays whose stored bits differ (NaN == NaN whatever its payload)"""
    u = np.uint64 if a.dtype == np.float64 else np.uint32
    d = (a.view(u) != b.view(u)) & ~(np.isnan(a) & np.isnan(b))
    return d.reshape(len(a), -1).any(1)


class Mismatch:
    """probe rays whose result differs from the reference, over all tiles,
    rows and arrays"""

    def __init__(self, P):
        self.bad = np.zeros(P, bool)
        self.where = []

    def row(self, got, want, what):
        """got (N, k) of one surface row, want (P, k): every tile of got"""
        P = len(want)
        for j in range(0, len(got), P):
            n = min(P, len(got) - j)
            b = _bad(got[j:j + n], want[:n])
            if b.any() and len(self.where) < 4:
                self.where.append("%s ray %d" % (what, j + int(np.flatnonzero(b)[0])))
            self.bad[:n] |= b

    def check(self, label):
        nb = int(self.bad.sum())
        assert nb == 0, "%s: %d of %d probe rays differ from the per-thread store kernel (%s)" % (
            label, nb, len(self.bad), ", ".join(self.where))


def _compare_device(e, out, want, N, keep_last, label):
    """device outputs (rows, ld, k) against the reference rows, row by row"""
    e.sync()
    m = Mismatch(want[0].shape[1])
    S = want[0].shape[0]
    for a, w, nm in zip(out, want, "yuit"):
        for r in range(a.shape[0]):
            s = S - 1 if keep_last else r
            m.row(a.rows(r).download()[0][:N], w[s], "%s[%d]" % (nm, s))
    m.check(label)


def _compare_host(got, want, keep_last, label):
    m = Mismatch(want[0].shape[1])
    S = want[0].shape[0]
    for a, w, nm in zip(got, want, "yuit"):
        for r in range(a.shape[0]):
            s = S - 1 if keep_last else r
            m.row(a[r], w[s], "%s[%d]" % (nm, s))
    m.check(label)


def _trace_device(e, s, mode, N, ld, li=0, keep_last=False, offset=0, rpt=0):
    """trace N tiled probe rays on `e`; returns (outputs, launch config)"""
    dtype, exact = MODES[mode]
    table = s["tables"][li]
    dy, du = _tiled(e, s, dtype, N)
    out = _outputs(e, 1 if keep_last else len(table), ld, dtype, offset)
    e.trace_device(table, dy, du, *out, N=N, ld=ld, clip=s["clip"], rot0=s["rot0"],
                   exact=exact, keep_last=keep_last, rpt=rpt)
    e.sync()
    cfg = e.last_launch_config()
    dy.free(), du.free()
    return out, cfg


def _free(arrays):
    for a in arrays:
        a.free()


def _up(n, m):
    return -(-n//m)*m


# ---- the reference result against the oracle ------------------------------
def _fp32_err(a, b):
    """SURVEY 8(d) comparator (test_fp32_vs_reference_golden) on the entries
    finite in both: (max error, NaN-mask flips)"""
    a = np.asarray(a, np.float64)
    flips = int((np.isnan(a) != np.isnan(b)).sum())
    fin = ~np.isnan(a) & ~np.isnan(b)
    absb = np.where(np.isnan(b), 0, np.abs(b))
    scale = np.maximum(absb.reshape(len(b), -1).max(1), 1.0).reshape((-1,) + (1,)*(b.ndim - 1))
    with np.errstate(invalid="ignore"):
        e = np.where(fin, np.abs(a - b)/np.maximum(np.abs(np.where(fin, b, 1)), scale), 0)
    return float(e.max()), flips


@pytest.mark.parametrize("name,mode", [
    pytest.param(n, m, id="%s-%s" % (n, m)) for n in NEWTON + ANALYTIC + ["plates256"]
    for m in MODES
    # FP32 on random tilted systems is checked on well-conditioned rays only,
    # in test_gpu_random_systems
    if not (n.startswith("rand") and m == "fp32")])
def test_reference_vs_oracle(sysdb, canon, name, mode):
    """exact: bit-identical on unrotated analytic systems, else 1e-12 (1e-10
    on random tilted systems); fast: 1e-10 with the oracle's NaN mask; FP32:
    the per-surface comparator at 1e-5 or 1.5 x what float32 numpy reaches"""
    s = sysdb(name)
    got = canon(name, mode)
    table = s["tables"][0]
    want = np_oracle.trace(table, s["y0"], s["u0"], clip=s["clip"], rot0=s["rot0"])
    if mode == "exact":
        for a, b, w in zip(got, want, "yuit"):
            if s["bit"]:
                assert np.array_equal(a, b, equal_nan=True), "%s exact %s" % (name, w)
            else:
                assert_parity(a, b, s["exact_rtol"], "%s exact %s" % (name, w))
    elif mode == "fast":
        for a, b, w in zip(got, want, "yuit"):
            assert_parity(a, b, 1e-10, "%s fast %s" % (name, w))
    else:
        f32 =np_oracle.trace(table, s["y0"], s["u0"], clip=s["clip"], rot0=s["rot0"],
                              dtype=np.float32)
        for a, o, b, w in zip(got, f32, want, "yuit"):
            err, flips = _fp32_err(a, b)
            err_np, flips_np = _fp32_err(o, b)
            # rays within float32 of an aperture edge or of Newton's limit may flip
            assert flips <= max(flips_np, 1e-3*b.size if s["fp32"] == "plain" else
                                3*len(table)), (name, w, flips, flips_np)
            assert err <= max(1e-5 if s["fp32"] == "plain" else 2e-5, 1.5*err_np), (
                name, w, err, err_np)


# ---- every instantiated configuration --------------------------------------
def _forced_cases():
    for mode in MODES:
        for cfg in FORCED:
            if cfg in (FP64_ONLY if mode == "fp32" else FP32_ONLY):
                continue
            for name in NEWTON + ANALYTIC:
                yield pytest.param(name, mode, cfg, id="%s-%s-%s" % (name, mode, cfg))


@pytest.mark.parametrize("name,mode,cfg", list(_forced_cases()))
def test_forced_configuration(sysdb, canon, forced, name, mode, cfg):
    """each kernel of the tuning space, pinned through RTX_* in its own engine"""
    s = sysdb(name)
    e = forced(cfg)
    P = len(s["y0"])
    N = max(P, MIN_FORCED)
    out, got_cfg = _trace_device(e, s, mode, N, _up(N, 128))
    try:
        assert got_cfg == FORCED[cfg][0], (cfg, got_cfg)
        _compare_device(e, out, canon(name, mode), N, False, "%s %s %s" % (name, mode, cfg))
    finally:
        _free(out)


# ---- the library's own choice on each side of every size threshold ---------
def _by_size(dtype, newton, N):
    """the default configuration of an untuned engine (rtx.cu choose_trace_cfg) for
    aligned outputs with a pitch that is a multiple of 128"""
    if N <= 150_000:
        return R1W8
    if dtype == np.float32:
        if newton:
            return (4, WARP, 16, 1, 1)
        return (2, CTA, 8, 1, 1) if 500_000 < N <= 2_500_000 else (4, CTA, 16, 1, 1)
    if newton:
        return (2, WARP, 16, 2, 1)
    return (1, CTA, 16, 1, 1) if N <= 1_500_000 else (2, CTA, 16, 1, 16)


SIZES64 = [32_768, 32_769, 150_000, 150_001, 1_500_000, 1_500_001]
SIZES32 = [32_768, 32_769, 150_000, 150_001, 500_000, 500_001, 2_500_000, 2_500_001]


def _size_cases():
    for mode in MODES:
        for N in (SIZES32 if mode == "fp32" else SIZES64):
            for name in ("cooke_asph", "double_gauss"):
                yield pytest.param(name, mode, N, id="%s-%s-N%d" % (name, mode, N))


@pytest.mark.parametrize("name,mode,N", list(_size_cases()))
def test_default_choice_by_size(eng, sysdb, canon, name, mode, N):
    s = sysdb(name)
    out, cfg = _trace_device(eng, s, mode, N, _up(N, 128))
    try:
        assert cfg == _by_size(MODES[mode][0], s["newton"], N), cfg
        _compare_device(eng, out, canon(name, mode), N, False, "%s %s N=%d" % (name, mode, N))
    finally:
        _free(out)


# ---- pitch, alignment, keep-LAST, long tables, explicit RPT ----------------
# (name, mode, N, pitch, output offset in elements, keep_last, rpt, expected)
LAYOUTS = {
    "fp32_analytic_ld64": ("double_gauss", "fp32", 200_000, 128*1563 + 64, 0, False, 0,
                           (2, CTA, 32, 1, 1)),
    "fp32_analytic_ld32": ("double_gauss", "fp32", 200_000, 64*3125 + 32, 0, False, 0, R1W8),
    "fp32_newton_ld64": ("cooke_asph", "fp32", 200_000, 128*1563 + 64, 0, False, 0,
                         (2, WARP, 8, 2, 1)),
    "fp32_newton_ld32": ("cooke_asph", "fp32", 200_000, 64*3125 + 32, 0, False, 0, R1W8),
    "fp64_newton_ld32": ("cooke_asph", "fast", 200_000, 64*3125 + 32, 0, False, 0, R1W8),
    "fp64_cluster_ld64": ("double_gauss", "fast", 1_600_000, 128*12500 + 64, 0, False, 0,
                          (2, CTA, 16, 1, 16)),
    "fp64_cluster_ld32": ("double_gauss", "fast", 1_600_000, 64*25000 + 32, 0, False, 0, R1W8),
    "fp64_unaligned": ("cooke_asph", "fast", 200_001, 200_064, 1, False, 0, PER_RAY),
    "fp32_unaligned": ("double_gauss", "fp32", 200_001, 200_064, 1, False, 0, PER_RAY),
    "exact_unaligned": ("double_gauss", "exact", 200_001, 200_064, 1, False, 0, PER_RAY),
    "fp64_odd_pitch": ("rand_asph1", "fast", 200_001, 200_001, 0, False, 0, PER_RAY),
    "fp64_last_newton": ("cooke_asph", "fast", 200_003, 200_064, 0, True, 0,
                         (2, WARP, 16, 2, 1)),
    "fp64_last_analytic": ("double_gauss", "fast", 200_003, 200_064, 0, True, 0,
                           (2, WARP, 16, 2, 1)),
    "exact_last": ("cooke_asph", "exact", 200_003, 200_064, 0, True, 0, (2, WARP, 16, 2, 1)),
    "fp32_last": ("rand_asph0", "fp32", 200_003, 200_064, 0, True, 0, (4, WARP, 16, 1, 1)),
    # 256 FP64 plates: the keep-LAST kernel's staging does not fit next to the
    # 92 KB table; the launch steps down to the one-ray per-warp kernel
    "plates_last_smem": ("plates256", "fast", 200_003, 200_064, 0, True, 0, R1W8),
    "plates_mid": ("plates256", "fast", 200_003, 200_064, 0, False, 0, (1, CTA, 16, 1, 1)),
    "plates_fp32": ("plates256", "fp32", 200_003, 200_064, 0, False, 0, (4, CTA, 16, 1, 1)),
    # explicit RPT requests at every size
    "rpt2_small": ("cooke_asph", "fast", 20_011, 20_096, 0, False, 2, (2, WARP, 8, 2, 1)),
    "rpt2_mid": ("newton_edge_clip1", "fast", 100_000, 100_032, 0, False, 2,
                 (2, WARP, 8, 2, 1)),
    "rpt2_exact": ("cooke_asph_f07_clip", "exact", 100_000, 100_032, 0, False, 2,
                   (2, WARP, 8, 2, 1)),
    "rpt2_fp32": ("rand_asph2", "fp32", 100_000, 100_032, 0, False, 2, (2, WARP, 8, 2, 1)),
    "rpt1_large": ("cooke_asph", "fast", 400_000, 400_000, 0, False, 1, R1W8),
    "rpt2_ld32": ("cooke_asph", "fast", 100_000, 64*1562 + 32, 0, False, 2, R1W8),
}


@pytest.mark.parametrize("case", LAYOUTS)
def test_layout(eng, sysdb, canon, case):
    name, mode, N, ld, off, keep_last, rpt, want_cfg = LAYOUTS[case]
    s = sysdb(name)
    isz = np.dtype(MODES[mode][0]).itemsize
    out, cfg = _trace_device(eng, s, mode, N, ld, keep_last=keep_last, offset=off*isz, rpt=rpt)
    try:
        assert cfg == want_cfg, cfg
        _compare_device(eng, out, canon(name, mode), N, keep_last, case)
    finally:
        _free(out)


# ---- front ends ------------------------------------------------------------
def _chunk(S, dtype):
    """rays per chunk of rtx_trace_host's pipeline (rtx.cu trace_host)"""
    isz = np.dtype(dtype).itemsize
    return max(((256 << 20)//(S*10*isz + 6*isz))//128*128, 4096)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["cooke_asph", "rand_asph0", "double_gauss"])
def test_host_paths(eng, sysdb, canon, name, mode, monkeypatch):
    """rtx_trace_host: zero-copy (a handful of rays), the DMA small path (with
    and without RTX_NO_ZERO_COPY) and a pipeline of three chunks on a ring of
    two chunk buffers whose last chunk is ragged (and small enough for the
    one-ray kernel, while the full chunks take the bundle-size kernel)"""
    s = sysdb(name)
    dtype, exact = MODES[mode]
    table = s["tables"][0]
    want = canon(name, mode)
    kw = dict(clip=s["clip"], rot0=s["rot0"], dtype=dtype, exact=exact)
    y0, u0 = s["y0"], s["u0"]
    for n, env in ((7, None), (7, "1"), (1000, None)):
        if env:
            monkeypatch.setenv("RTX_NO_ZERO_COPY", env)
        got = eng.trace(table, y0[:n], u0[:n], **kw)
        monkeypatch.delenv("RTX_NO_ZERO_COPY", raising=False)
        assert eng.last_launch_config() == PER_RAY
        _compare_host(got, want, False, "%s %s host n=%d" % (name, mode, n))
    C = _chunk(len(table), dtype)
    N = 2*C + 100_017
    y, u = _host_tiled(s, N)
    got = eng.trace(table, y, u, **kw)
    assert eng.last_launch_config() == R1W8        # the ragged last chunk
    _compare_host(got, want, False, "%s %s host chunked N=%d" % (name, mode, N))
    del got
    got = eng.trace(table, y, u, keep_last=True, **kw)
    _compare_host(got, want, True, "%s %s host chunked keep-LAST" % (name, mode))


# (name, mode, ragged sizes of the bundles, keep_last, expected)
BATCHES = {
    "fp64_cta": ("double_gauss", "fast", [200_003, 145_679, 40_001], False, (1, CTA, 16, 1, 1)),
    "fp64_newton": ("cooke_asph", "fast", [200_003, 145_679, 40_001], False,
                    (2, WARP, 16, 2, 1)),
    "exact": ("cooke_asph", "exact", [200_003, 150_001, 1_001], False, (2, WARP, 16, 2, 1)),
    "exact_analytic": ("double_gauss", "exact", [200_003, 150_001, 1_001], False,
                       (1, CTA, 16, 1, 1)),
    "fp32_rpt4": ("double_gauss", "fp32", [200_003, 145_679, 40_001], False,
                  (4, CTA, 16, 1, 1)),
    "fp32_newton": ("cooke_asph", "fp32", [200_003, 145_679, 40_001], False,
                    (4, WARP, 16, 1, 1)),
    "last": ("cooke_asph", "fast", [200_003, 145_679, 40_001], True, (2, WARP, 16, 2, 1)),
    "last_fp32": ("double_gauss", "fp32", [200_003, 145_679, 40_001], True,
                  (4, WARP, 16, 1, 1)),
    "small": ("cooke_asph", "fast", [60_001, 33_333, 77], False, R1W8),
    # a single bundle is eligible for the clustered kernel
    "one_bundle_cluster": ("double_gauss", "fast", [1_500_032], False, (2, CTA, 16, 1, 16)),
}


@pytest.mark.parametrize("case", BATCHES)
def test_batched_launch(eng, sysdb, canon, case):
    """rtx_trace_batch: one launch over ragged bundles of the three wavelengths"""
    name, mode, Ns, keep_last, want_cfg = BATCHES[case]
    s = sysdb(name)
    dtype, exact = MODES[mode]
    nl = len(s["tables"])
    ld = _up(max(Ns), 128)
    rows = 1 if keep_last else len(s["tables"][0])
    ins = [_tiled(eng, s, dtype, n) for n in Ns]
    outs = [_outputs(eng, rows, ld, dtype) for _ in Ns]
    tabs = [s["tables"][b % nl] for b in range(len(Ns))]
    try:
        eng.trace_device_batch(tabs, [a[0] for a in ins], [a[1] for a in ins],
                               *[[o[k] for o in outs] for k in range(4)], Ns=Ns, ld=ld,
                               clip=s["clip"], keep_last=keep_last, rot0=s["rot0"], exact=exact)
        eng.sync()
        assert eng.last_launch_config() == want_cfg
        for b, (n, o) in enumerate(zip(Ns, outs)):
            _compare_device(eng, o, canon(name, mode, b % nl), n, keep_last,
                            "%s bundle %d" % (case, b))
    finally:
        for a in ins + outs:
            _free(a)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["cooke_asph", "double_gauss"])
def test_trace_bundles(eng, sysdb, canon, name, mode):
    """rtx_trace_batch_host: 11 small ragged bundles (two launches of up to 8),
    then 3 bundles whose results exceed the 64 MB staging budget (one
    chunked host trace per bundle), all arrays and keep-LAST"""
    s = sysdb(name)
    dtype, exact = MODES[mode]
    nl = len(s["tables"])
    for Ns in ([200 + 97*b for b in range(11)], [100_000, 77_777, 100_001]):
        tabs = [s["tables"][b % nl] for b in range(len(Ns))]
        rays = [_host_tiled(s, n) for n in Ns]
        for keep_last in (False, True):
            got = eng.trace_bundles(tabs, [r[0] for r in rays], [r[1] for r in rays],
                                    clip=s["clip"], keep_last=keep_last, rot0=s["rot0"],
                                    dtype=dtype, exact=exact)
            for b, g in enumerate(got):
                _compare_host(g, canon(name, mode, b % nl), keep_last,
                              "%s %s bundle %d of %d keep_last=%s" % (name, mode, b, len(Ns),
                                                                      keep_last))


# (name, mode, N, destination offset, expected)
GATHERS = {
    "fp64_analytic": ("double_gauss", "fast", 200_000, 64, (1, CTA, 16, 1, 1)),
    "fp64_newton": ("cooke_asph", "fast", 200_000, 64, (2, WARP, 16, 2, 1)),
    "exact": ("cooke_asph", "exact", 200_000, 64, (2, WARP, 16, 2, 1)),
    # 200 000 is not a multiple of 128: the four-ray kernels step down
    "fp32_analytic": ("double_gauss", "fp32", 200_000, 64, (2, CTA, 32, 1, 1)),
    "fp32_newton": ("cooke_asph", "fp32", 200_000, 64, (2, WARP, 8, 2, 1)),
    "ragged": ("cooke_asph", "fast", 200_001, 64, PER_RAY),
    "small": ("rand_asph2", "fast", 40_000, 0, R1W8),
    # the size takes the clustered kernel's configuration; a gather keeps it unclustered
    "fp64_cluster_size": ("double_gauss", "fast", 1_500_032, 64, (2, CTA, 16, 1, 1)),
}


@pytest.mark.parametrize("case", GATHERS)
def test_gather_local(eng, sysdb, canon, case):
    """rtx_trace_gather into a local buffer: the last surface's y and i at a
    ray offset"""
    name, mode, N, off, want_cfg = GATHERS[case]
    s = sysdb(name)
    dtype, exact = MODES[mode]
    dy, du = _tiled(eng, s, dtype, N)
    Y, I = eng.empty((off + N, 3), dtype), eng.empty((off + N, 3), dtype)
    try:
        eng.trace_gather(s["tables"][0], dy, du, [Y.ptr], off, N=N, clip=s["clip"],
                         rot0=s["rot0"], exact=exact, dst_i_ptrs=[I.ptr])
        eng.sync()
        assert eng.last_launch_config() == want_cfg
        want = canon(name, mode)
        m = Mismatch(want[0].shape[1])
        m.row(Y.download()[off:], want[0][-1], "y")
        m.row(I.download()[off:], want[2][-1], "i")
        m.check(case)
    finally:
        _free([dy, du, Y, I])
