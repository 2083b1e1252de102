"""rayopt_b200 -- H100-native engine for rayopt's geometric propagate loop.

Hot path only: ``GeometricTrace.propagate`` / ``System.propagate``
(rayopt/geometric_trace.py:72-80, rayopt/system.py:459-464) as one hand-written
CUDA (sm_90a) launch behind a C ABI (include/rtx.h).  No PyTorch, no CPU
fallback: importing works anywhere, tracing needs librtx.so and a GPU.
"""
from .surface_table import (SURFACE_DTYPE, PackedSystem, pack_system,  # noqa: F401
                            pack_element, table_from_json, table_to_json)
from .geometric_trace import (GeometricTrace, PropagateMixin, bind,  # noqa: F401
                              system_propagate, install, propagate_many)
from .engine import Engine, DeviceArray, default_engine  # noqa: F401
from . import elements  # noqa: F401
from .lazy import LazyRows, ResidentMixin, ResidentTrace  # noqa: F401
from ._lib import RtxError  # noqa: F401
from .spot import spots  # noqa: F401
from .opd import opds  # noqa: F401
from .mtf import geometric_mtf  # noqa: F401
from .psf import psfs  # noqa: F401
from .tolerance import (tolerance, tolerance_mtf, tolerance_wavefront,  # noqa: F401
                        perturbed_tables, sensitivity_deltas, monte_carlo_deltas,
                        record_tangents)
from .zernike import tolerance_zernike, zernike  # noqa: F401
from .optimize import (spot_jacobian, optimize_spot, wavefront_jacobian,  # noqa: F401
                       optimize_wavefront, mtf_jacobian, optimize_mtf)

__version__ = "0.2.0"
