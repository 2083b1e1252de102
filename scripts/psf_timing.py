#!/usr/bin/env python
"""Stage times of the diffraction PSF (GeometricTrace.psf, rayopt/
geometric_trace.py:133-169) on the device path and the host path, in one run.

    python scripts/psf_timing.py [--nrays 1e4 1e5 1e6] [--reps 3] [--out FILE]

Workload: Cooke triplet at field 0.7, hexapolar bundle, resident trace
(ResidentTrace), resample 4, pad 4.  Needs the reference's System (its tree
staged by build() under oracle/_ref) and an H100.

Device path: the per-ray OPD (rtx_trace_opd, download of x, y, t), the host
Delaunay triangulation with its barycentric transforms, rtx_grid_linear (uploads + kernel; CUDA events give
the kernel), the same triangulation on the device (rtx_delaunay: the call with
the upload of the points, its kernels by CUDA events, and whether its
triangles are scipy's; not part of the total), rtx_psf (pupil, cuFFT, |.|^2, stats; CUDA events) and the
download of the PSF.  Host path: griddata's evaluation on the SAME
triangulation (LinearNDInterpolator) and the padded numpy fft2 + |.|^2.  The
two PSFs are compared in the same run.

Encircled energy and MTF (Analysis.opds, rayopt/analysis.py:330-346) of the
device's PSF about its centroid: on the device rtx_psf_profiles (the call, its
kernels by CUDA events and the PSF bytes read over that time), on the host the
fftshift, polar_sum, line sums and the two 1-d inverse FFTs of the downloaded
PSF (whose download is the device path's download row).  Every shape is warmed once; the
median and the range of --reps repetitions are printed (host path at 1e6 rays:
one repetition).
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nrays", type=float, nargs="+", default=[1e4, 1e5, 1e6])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    import yaml
    from scipy.interpolate import LinearNDInterpolator
    from scipy.spatial import Delaunay
    import profile_oracle
    import psf_oracle
    import ref_shim
    import systems_yaml
    from rayopt_b200 import ResidentTrace
    from rayopt_b200.engine import Engine
    R = ref_shim.load()
    eng = Engine(0)
    info = card()
    print("card: %s (name, power limit)" % info)
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS["cooke"]))
    s.update()
    s.paraxial.refocus()
    g = ResidentTrace(s, engine=eng)
    rows = []
    for nr in a.nrays:
        g.rays_point((0, .7), nrays=int(nr), distribution="hexapolar", clip=False)
        radius = s[-1].distance
        wl = g.l/s.scale

        def device():
            st = {}
            t0 = time.perf_counter()
            x, y, t = g.opd_rays(radius=radius)
            t1 = time.perf_counter()
            ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(t)
            x, y, t = x[ok], y[ok], t[ok]
            n = int(4*g.nrays**.5)
            xs, ys, gh = psf_oracle.grid(n, np.fabs((x, y)).max())
            pts = np.stack([x, y], axis=-1)
            tri = Delaunay(pts)
            tri.transform                   # computed lazily by scipy: part of the triangulation
            t2 = time.perf_counter()
            o = eng.grid_linear(pts, t, tri, n, gh, download=False)
            t3 = time.perf_counter()
            st["regrid_kernel_ms"] = eng.last_kernel_ms()
            out, raw = eng.psf(o, 4)
            t4 = time.perf_counter()
            st["psf_kernels_ms"] = eng.last_kernel_ms()
            # encircled-energy bins and line sums about the centroid, as
            # ResidentMixin.psf_profiles takes them
            f = psf_oracle.frequencies(xs, 4*n, wl, radius)
            ps = eng.psf_stats(raw, f)
            cp, cq, fs = ps["cp"], ps["cq"], np.fft.fftshift(f)
            dx = (fs[1] - cp) - (fs[0] - cp)
            center = (2*n + cp/dx, 2*n + cq/dx)
            t5 = time.perf_counter()
            prof = eng.psf_profiles(out, center)
            t6 = time.perf_counter()
            st["profiles_kernels_ms"] = ms = eng.last_kernel_ms()
            st["profiles_read_GBps"] = out.nbytes/ms/1e6
            psf = out.download()
            t7 = time.perf_counter()
            o.free()
            out.free()
            # the same triangulation on the device (rtx_delaunay): upload of
            # the points and the synchronous call; CUDA events give its kernels
            t8 = time.perf_counter()
            dpts = eng.to_device(pts)
            dtri = eng.delaunay(dpts)
            t9 = time.perf_counter()
            st["dev_triangulation_kernels_ms"] = eng.last_kernel_ms()
            st["dev_triangulation_call_s"] = t9 - t8
            simp = dtri.download()[0]
            dtri.free()
            dpts.free()
            st["dev_triangulation_same"] = float(
                {tuple(sorted(r)) for r in simp.tolist()} == {tuple(sorted(r)) for r in tri.simplices.tolist()})
            st.update(opd_rays_s=t1 - t0, triangulation_s=t2 - t1, regrid_call_s=t3 - t2,
                      psf_call_s=t4 - t3, profiles_call_s=t6 - t5, download_s=t7 - t6,
                      total_s=t7 - t0 - (t6 - t5))
            return st, (x, y, t, tri, xs, ys, n, center, prof), psf

        def host_profiles(psf, center):
            """Analysis.opds's reduction of the downloaded PSF"""
            t0 = time.perf_counter()
            s = np.fft.fftshift(psf)
            t1 = time.perf_counter()
            bins = profile_oracle.polar_sum_azimuthal(s, center)
            t2 = time.perf_counter()
            lsf = [np.fft.ifftshift(s.sum(i)) for i in range(2)]
            t3 = time.perf_counter()
            mtf = [np.absolute(np.fft.ifft(v*s.size**.5)) for v in lsf]
            t4 = time.perf_counter()
            return dict(prof_fftshift_s=t1 - t0, prof_polar_sum_s=t2 - t1,
                        prof_line_sums_s=t3 - t2, prof_ifft_s=t4 - t3,
                        prof_host_total_s=t4 - t0), (bins, *lsf)

        def host(data):
            x, y, t, tri, xs, ys, n = data[:7]
            t0 = time.perf_counter()
            o = LinearNDInterpolator(tri, t, fill_value=np.nan)(xs, ys)
            t1 = time.perf_counter()
            _, _, psf = psf_oracle.psf(xs, o, 4, wl, radius)
            t2 = time.perf_counter()
            return dict(griddata_eval_s=t1 - t0, fft2_s=t2 - t1), psf

        device()                                          # warm this shape
        dev = [device() for _ in range(a.reps)]
        data, psf_d = dev[-1][1], dev[-1][2]
        hreps = 1 if nr >= 1e6 else a.reps
        hst = [host(data) for _ in range(hreps)]
        psf_h = hst[-1][1]
        err = float(np.abs(psf_d - psf_h).max()/psf_h.max())
        # the host's profile path on the device's PSF (its download is timed
        # on the device side); one run at 1e6 rays
        hprof = [host_profiles(psf_d, data[7]) for _ in range(hreps)]
        perr = max(float(np.abs(np.cumsum(a) - np.cumsum(b)).max())
                   for a, b in zip(data[8], hprof[-1][1]))
        hst = [(dict(h[0], **hp[0]), h[1]) for h, hp in zip(hst, hprof)]
        row = dict(nrays=g.nrays, n=data[6], padded=4*data[6], rel_err_vs_host=err,
                   profiles_cumsum_err_vs_host=perr, host_reps=hreps, card=info)
        for key in dev[0][0]:
            v = [d[0][key] for d in dev]
            row[key] = (statistics.median(v), min(v), max(v))
        for key in hst[0][0]:
            v = [h[0][key] for h in hst]
            row[key] = (statistics.median(v), min(v), max(v))
        rows.append(row)
        print(json.dumps(row))
        del psf_d, psf_h, dev, hst, data
    g.free()
    eng.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
