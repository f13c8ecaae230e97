"""dmosopt_b200 -- H100-native surrogate-generation hot path for dmosopt.

Plugin import paths (dmosopt resolves them with ``config.import_object_by_path``):

    optimizer_name         = "dmosopt_b200.NSGA2" | "dmosopt_b200.AGEMOEA" | "dmosopt_b200.SMPSO" | "dmosopt_b200.CMAES" | "dmosopt_b200.TRS"
    surrogate_method_name  = "dmosopt_b200.GPR_Matern" | "dmosopt_b200.GPR_RBF"
                             | "dmosopt_b200.SVGP_Matern" | "dmosopt_b200.VGP_Matern" | "dmosopt_b200.SIV_Matern"
                             | "dmosopt_b200.SPV_Matern" | "dmosopt_b200.CRV_Matern"
    surrogate_custom_training = "dmosopt_b200.feasibility.train_with_feasibility"   (a GPU logistic feasibility model)

``dmosopt_b200.install()`` additionally routes the controller-side helpers that dmosopt calls on its own modules
(resample / get_best duplicates + sort, per-generation termination hypervolume, the epsilon-nondominated archive of
epsilon_get_best) to the same kernels; ``install(resident_epoch=True)`` also runs eligible surrogate epochs
(``dmosopt_b200.MOASMO.optimize``: NSGA2 or SMPSO with one of the GPU surrogates) on the resident generation step.
``dmosopt_b200.MOEA.EpsilonSort`` and ``dmosopt_b200.MOASMO.epsilon_get_best`` are the GPU archive's own mirrors of the
reference's.

Importing the package does not touch CUDA; the first numerical call loads
``libdmosopt_b200.so`` and creates the context, and fails loudly when either
is unavailable (there is no CPU fallback).
"""

from .MOEA import MOEA as MOEABase  # noqa: F401
from .MOEA import Struct  # noqa: F401
from .NSGA2 import NSGA2  # noqa: F401
from .model import GPR_Matern, GPR_RBF, Model  # noqa: F401
from .model_gpflow import CRV_Matern, SIV_Matern, SPV_Matern, SVGP_Matern, VGP_Matern  # noqa: F401

from .AGEMOEA import AGEMOEA  # noqa: F401
from .CMAES import CMAES  # noqa: F401
from .SMPSO import SMPSO  # noqa: F401
from .TRS import TRS  # noqa: F401
from .feasibility import LogisticFeasibilityModel, train_with_feasibility  # noqa: F401


def install(package="dmosopt", resident_epoch=False):
    """Route the reference controller's own hot helpers (resample duplicates / crowding, get_best, termination
    hypervolume, dda_ens, EpsilonSort) to the GPU library; with ``resident_epoch=True``, also run eligible surrogate
    epochs of ``MOASMO.optimize`` (NSGA2 or SMPSO with a GPU surrogate) on the resident generation step: see
    dmosopt_b200/patch.py.  Opt-in; nothing is
    patched on import."""
    from . import patch

    return patch.install(package, resident_epoch=resident_epoch)


def uninstall():
    from . import patch

    patch.uninstall()


__version__ = "0.1.0"
