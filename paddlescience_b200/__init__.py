"""paddlescience_b200 — H100-native PINN PDE-residual engine behind the PaddleScience API.

The package mirrors the part of ``ppsci`` that lies on the hot path named in BASELINE.json
(SURVEY.md §8): ``arch.MLP``, ``arch.DeepONet``, ``equation.PDE`` (+ Laplace/Poisson/NavierStokes/Biharmonic/
AllenCahn/Helmholtz), ``autodiff.{jacobian,hessian}``, ``constraint.{Interior,Boundary,
Supervised}Constraint``, ``geometry.{Interval,Rectangle,Cuboid,Hypercube}``, the three array
datasets, ``loss.MSELoss`` / ``loss.mtl.Sum``, ``optimizer.Adam`` + LR schedules,
``solver.Solver`` and the evaluation side of it (``validate.{Geometry,Supervised}Validator``, ``metric.*``).  All arithmetic of that path runs in hand-written sm_90a CUDA behind the
C-ABI in ``include/ppsci_b200.h``; there is no CPU fallback."""
from . import arch, autodiff, constraint, data, equation, geometry, loss, metric, optimizer, solver, utils, validate  # noqa: F401
from .utils import logger  # noqa: F401
from .utils.symbolic import lambdify  # noqa: F401

__version__ = "0.1.0"
__all__ = ["arch", "autodiff", "constraint", "data", "equation", "geometry", "loss", "metric", "optimizer", "solver", "utils", "validate",
           "logger", "lambdify"]
