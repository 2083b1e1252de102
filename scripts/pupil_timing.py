#!/usr/bin/env python
"""Times of the direct-sum diffraction PSF (rtx_pupil_sum,
rtx_pupil_intensity, rayopt_b200.psfs), in one run.

    python scripts/pupil_timing.py [--reps 5] [--out FILE]

Kernel sweep: N in {1e4, 1e5, 1e6} synthetic exit-pupil rays (NA 0.2, about
a wave of aberration), grids 128^2, 256^2 and 512^2 at an eighth of the Airy
radius, K in {1, 5} planes.  For each it prints the median and range over
`reps` calls (after one warm-up) of the rtx_pupil_sum device time (CUDA
events, both kernels), the complex terms (ray x pixel x plane) per second,
and the share of the data-sheet FP64 tensor-core rate of the H100 SXM, 67
TFLOP/s, that 8 flops per term would be -- a data-sheet figure, not one
reached.  The intensity pass is timed on the largest grid.

Phasor share: scripts/pupil_phasor_share.cu, built with nvcc into a
temporary directory, times the sum kernel against the same kernel with the
products left out (1e5 and 1e6 rays, 256^2 and 512^2, K = 1 and 5).

End to end: rayopt_b200.psfs (one wavelength, three fields, 128^2 pixels)
against rayopt_b200.opds' FFT PSF at the same ray count on the Cooke triplet
(the reference's System, staged under oracle/_ref), host clock, after a
warm-up.  It prints the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)

FP64_TC_DATASHEET = 67e12     # H100 SXM, FP64 tensor core, FLOP/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(v):
    return statistics.median(v), (min(v), max(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from rayopt_b200.engine import Engine, pupil_spec
    eng = Engine(0)
    rows = []
    print("# card: %s" % card())
    lam, R = 5e-4, 50.
    pitch = .61*lam/.2/8
    for N in (10**4, 10**5, 10**6):
        rng = np.random.default_rng(N)
        r, th = 10*np.sqrt(rng.random(N)), 2*np.pi*rng.random(N)
        x, y = r*np.cos(th), r*np.sin(th)
        P = np.stack([x, y, -np.sqrt(R*R - x*x - y*y)], -1)
        A = 100 + 3e-4*(r/10)**4
        dA, dP = eng.to_device(A), eng.to_device(P)
        for n in (128, 256, 512):
            for K in (1, 5):
                spec = pupil_spec(np.linspace(-.02, .02, K), (n, n), -(n//2)*pitch, pitch,
                                  -(n//2)*pitch, pitch, 100., lam, 1/lam, R)
                U = eng.empty((K, n, n), np.complex128)
                eng.memset(U)
                eng.pupil_sum(dA, dP, spec, U)
                ms = []
                for _ in range(a.reps):
                    eng.pupil_sum(dA, dP, spec, U)
                    ms.append(eng.last_kernel_ms())
                med, rng_ = stats(ms)
                terms = N*n*n*K
                row = dict(N=N, grid=n, K=K, sum_ms=med, sum_ms_range=rng_,
                           terms_per_s=terms/(med*1e-3),
                           tc_share=8*terms/(med*1e-3)/FP64_TC_DATASHEET)
                if N == 10**6 and n == 512:
                    psf = eng.empty((K, n, n))
                    eng.memset(psf)
                    eng.pupil_intensity(spec, U, psf, 1e-12)
                    im = []
                    for _ in range(a.reps):
                        eng.pupil_intensity(spec, U, psf, 1e-12)
                        im.append(eng.last_kernel_ms())
                    row["intensity_ms"] = stats(im)[0]
                    psf.free()
                U.free()
                rows.append(row)
                print(json.dumps(row))
        dA.free(), dP.free()
    # the phasor generation alone against the whole kernel
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "pupil_phasor_share")
        from rayopt_b200.build import nvcc
        subprocess.run([nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-o", exe, os.path.join(ROOT, "scripts", "pupil_phasor_share.cu")],
                       check=True)
        for line in subprocess.run([exe], capture_output=True, text=True,
                                   check=True).stdout.splitlines():
            row = json.loads(line)
            rows.append(row)
            print(json.dumps(row))
    # end to end on the Cooke triplet
    import ref_shim
    if ref_shim.available():
        import yaml
        import systems_yaml
        from rayopt_b200 import opds, psfs
        Rf = ref_shim.load()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            s = Rf.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
            s.update()
            s.paraxial.refocus()
            for nrays in (10**4, 10**5):
                t = {}
                for name, f in (("psfs", lambda: psfs(s, nrays=nrays, wavelengths=s.wavelengths[:1],
                                                       engine=eng)),
                                ("opds", lambda: opds(s, nrays=nrays, engine=eng))):
                    f()
                    v = []
                    for _ in range(max(a.reps//2, 2)):
                        t0 = time.perf_counter()
                        f()
                        eng.sync()
                        v.append(time.perf_counter() - t0)
                    t[name] = statistics.median(v)
                row = dict(e2e="cooke, 3 fields, 1 wavelength", nrays=nrays, psfs_s=t["psfs"],
                           opds_s=t["opds"])
                rows.append(row)
                print(json.dumps(row))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(card=card(), rows=rows), fh, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
