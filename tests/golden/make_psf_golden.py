#!/usr/bin/env python
"""Generate tests/golden/vs_reference/psf_*.npz FROM THE LIVE REFERENCE.

Needs the reference tree (oracle/ref_shim.py: $RAYOPT_REFERENCE or oracle/_ref):

    python tests/golden/make_psf_golden.py

Per case the reference's own GeometricTrace traces a hexapolar bundle and
computes its diffraction PSF (rayopt/geometric_trace.py:101-169, pad 4,
resample 4, radius = system[-1].distance as psf() uses).  Stored: the
per-ray exit-pupil coordinates and OPD (x, y, t) = opd(resample=False), the
regridded OPD o = opd(resample=4) on the axis gh (xs = gh[:, None], ys =
gh[None, :]), the PSF and its frequency axis f (p = f[:, None], q = f[None,
:]), and what the device needs to recompute them: nrays, the wavelength in
system units (l/scale) and the radius.  Nothing here comes from the oracle or
the CUDA engine.
"""
import json
import os
import sys
import warnings

import numpy as np
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, HERE)

import ref_shim  # noqa: E402
import systems_yaml  # noqa: E402

warnings.simplefilter("ignore")
np.seterr(all="ignore")
R = ref_shim.load()

# (case, system, field, nrays): about 270 rays keep a case under 1 MB
CASES = [("psf_cooke_f0", "cooke", 0., 300), ("psf_cooke_f07", "cooke", .7, 300),
         ("psf_double_gauss_f07", "double_gauss", .7, 300), ("psf_mirror", "mirror", 0., 300)]


def build(name):
    s = R.System(**yaml.safe_load(systems_yaml.SYSTEMS[name]))
    s.update()
    s.paraxial.refocus()
    return s


def main():
    os.makedirs(os.path.join(HERE, "vs_reference"), exist_ok=True)
    for case, name, field, nrays in CASES:
        s = build(name)
        g = R.GeometricTrace(s)
        g.rays_point((0, field), nrays=nrays, distribution="hexapolar", clip=False)
        radius = s[-1].distance
        x, y, t = g.opd(resample=False, radius=radius)
        xs, ys, o = g.opd(resample=4, radius=radius)
        p, q, psf = g.psf(pad=4, resample=4)
        assert np.array_equal(xs, np.broadcast_to(xs[:, :1], xs.shape))
        assert np.array_equal(ys, np.broadcast_to(ys[:1], ys.shape))
        assert np.array_equal(p, np.broadcast_to(p[:, :1], p.shape))
        out = dict(x=x, y=y, t=t, gh=xs[:, 0].copy(), o=o, f=p[:, 0].copy(), psf=psf,
                   nrays=np.array(g.y.shape[1]), wavelength=np.array(g.l/s.scale),
                   radius=np.array(radius), ref=np.array(g.ref),
                   meta=np.array(json.dumps(dict(system=name, field=field, pad=4, resample=4))))
        path = os.path.join(HERE, "vs_reference", case + ".npz")
        np.savez_compressed(path, **out)
        print("%-22s N=%4d n=%3d psf=%s finite=%d  %6.1f kB" % (
            case, g.y.shape[1], o.shape[0], psf.shape, np.isfinite(o).sum(),
            os.path.getsize(path)/1e3))


if __name__ == "__main__":
    main()
