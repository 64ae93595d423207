"""parcels_b200 -- Lagrangian particle advection on the H100 behind the Parcels v4 API.

``ParticleSet.execute([AdvectionRK4 | AdvectionRK4_3D | ...], dt=, runtime=|endtime=)`` runs the
whole per-particle time loop in hand-written sm_90a CUDA (``csrc/engine.cu``) through the C-ABI
``include/parcels_b200.h`` (ctypes).  There is no CPU implementation in this package.
"""

from . import kernels

__version__ = "0.1.0"
from .install import install, uninstall
from .fieldset import EARTH_RADIUS, Field, FieldSet, SphericalMesh, VectorField, XGrid
from .kernels import (
    AdvectionDiffusionEM,
    AdvectionDiffusionM1,
    AdvectionEE,
    AdvectionRK2,
    AdvectionRK2_3D,
    AdvectionRK4,
    AdvectionRK4_3D,
    AdvectionRK45,
    DeleteParticle,
    DiffusionUniformKh,
)
from .particle import Particle, ParticleClass, Variable
from .particlefile import ParticleFile, read_particlefile
from .particleset import Kernel, ParticleSet
from .statuscodes import (
    KernelWarning,
    ParticleSetWarning,
    FieldInterpolationError,
    FieldOutOfBoundError,
    FieldOutOfBoundSurfaceError,
    GeneralError,
    GridSearchingError,
    OutsideTimeInterval,
    StatusCode,
)

__all__ = [
    "AdvectionDiffusionEM", "AdvectionDiffusionM1", "AdvectionEE", "AdvectionRK2", "AdvectionRK2_3D", "AdvectionRK4", "AdvectionRK4_3D", "AdvectionRK45", "DeleteParticle",
    "DiffusionUniformKh", "Field", "FieldInterpolationError", "FieldOutOfBoundError", "FieldOutOfBoundSurfaceError",
    "FieldSet", "GeneralError", "GridSearchingError", "Kernel", "KernelWarning", "OutsideTimeInterval", "ParticleSetWarning", "Particle", "ParticleClass", "ParticleFile", "ParticleSet", "Variable", "read_particlefile", "StatusCode",
    "EARTH_RADIUS", "SphericalMesh", "VectorField", "XGrid", "kernels", "install", "uninstall",
]  # fmt: skip
