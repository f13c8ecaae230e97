"""dmosopt_b200 -- H100-native surrogate-generation hot path for dmosopt.

Plugin import paths (dmosopt resolves them with ``config.import_object_by_path``):

    optimizer_name         = "dmosopt_b200.NSGA2" | "dmosopt_b200.AGEMOEA" | "dmosopt_b200.SMPSO" | "dmosopt_b200.CMAES" | "dmosopt_b200.TRS"
    surrogate_method_name  = "dmosopt_b200.GPR_Matern" | "dmosopt_b200.GPR_RBF"

``dmosopt_b200.install()`` additionally routes the controller-side helpers that dmosopt calls on its own modules
(resample / get_best duplicates + sort, per-generation termination hypervolume) to the same kernels.

Importing the package does not touch CUDA; the first numerical call loads
``libdmosopt_b200.so`` and creates the context, and fails loudly when either
is unavailable (there is no CPU fallback).
"""

from .MOEA import MOEA as MOEABase  # noqa: F401
from .MOEA import Struct  # noqa: F401
from .NSGA2 import NSGA2  # noqa: F401
from .model import GPR_Matern, GPR_RBF, Model  # noqa: F401

from .AGEMOEA import AGEMOEA  # noqa: F401
from .CMAES import CMAES  # noqa: F401
from .SMPSO import SMPSO  # noqa: F401
from .TRS import TRS  # noqa: F401


def install(package="dmosopt"):
    """Route the reference controller's own hot helpers (resample duplicates / crowding, get_best, termination
    hypervolume, dda_ens) to the GPU library: see dmosopt_b200/patch.py.  Opt-in; nothing is patched on import."""
    from . import patch

    return patch.install(package)


def uninstall():
    from . import patch

    patch.uninstall()


__version__ = "0.1.0"
