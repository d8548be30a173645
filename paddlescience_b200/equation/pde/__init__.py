from .allen_cahn import AllenCahn
from .base import PDE
from .biharmonic import Biharmonic
from .heat_exchanger import HeatExchanger
from .helmholtz import Helmholtz
from .laplace import Laplace
from .navier_stokes import NavierStokes
from .poisson import Poisson
from .viv import Vibration

__all__ = ["PDE", "AllenCahn", "Biharmonic", "HeatExchanger", "Helmholtz", "Laplace", "NavierStokes", "Poisson", "Vibration"]
