from .base import Constraint
from .boundary_constraint import BoundaryConstraint
from .initial_constraint import InitialConstraint
from .interior_constraint import InteriorConstraint
from .supervised_constraint import SupervisedConstraint

__all__ = ["Constraint", "BoundaryConstraint", "InitialConstraint", "InteriorConstraint", "SupervisedConstraint"]
