"""``PointCloud`` (reference: ppsci/geometry/pointcloud.py:27-316): a geometry that is a given set of points, e.g. the
collocation points of the NSFNet examples.

Sampling picks rows of the given arrays: ``random_points`` / ``random_boundary_points`` draw without replacement from
numpy's global stream (``np.random.choice``, as the reference), ``uniform_points`` takes the first n rows.  A point
cloud has no signed distance function, so ``sample_interior`` produces no ``sdf`` column.

Where the reference tests an optional array for truth (``if self.boundary:``, which raises for any array of more than
one element) this class tests ``is not None``, and ``translate`` offsets each boundary column by its own entry."""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np

from ..utils import misc
from . import geometry


class PointCloud(geometry.Geometry):
    """Interior points ``{key: [N, 1] array}`` over ``coord_keys``, optional boundary points and their normals
    (``{f"{key}_normal": [M, 1] array}``).  The bounding box is that of the interior points, the diameter infinite.

    >>> import numpy as np
    >>> import ppsci
    >>> geom = ppsci.geometry.PointCloud({"x": np.linspace(0, 2, 5, dtype="float32").reshape((-1, 1))}, ("x",))
    >>> np.random.seed(0)
    >>> geom.random_points(2)
    array([[1.],
           [0.]], dtype=float32)
    """

    def __init__(self, interior: Dict[str, np.ndarray], coord_keys: Tuple[str, ...],
                 boundary: Optional[Dict[str, np.ndarray]] = None,
                 boundary_normal: Optional[Dict[str, np.ndarray]] = None):
        self.interior = misc.convert_to_array(interior, coord_keys)
        self.len = self.interior.shape[0]
        self.boundary = None if boundary is None else misc.convert_to_array(boundary, coord_keys)
        self.normal = None
        if boundary_normal is not None:
            self.normal = misc.convert_to_array(boundary_normal, tuple(f"{key}_normal" for key in coord_keys))
            if self.boundary is None or list(self.normal.shape) != list(self.boundary.shape):
                raise ValueError(f"boundary's shape({None if self.boundary is None else self.boundary.shape}) must "
                                 f"equal to normal's shape({self.normal.shape})")
        self.input_keys = tuple(coord_keys)
        super().__init__(len(coord_keys), (np.amin(self.interior, axis=0), np.amax(self.interior, axis=0)), np.inf)

    @property
    def dim_keys(self):
        return self.input_keys

    @staticmethod
    def _among(x: np.ndarray, points: np.ndarray) -> np.ndarray:
        """Whether each row of x is one of ``points`` (componentwise ``np.isclose``, atol 1e-6)."""
        return np.isclose(x[:, None, :] - points[None, :, :], 0, atol=1e-6).all(axis=2).any(axis=1)

    def is_inside(self, x: np.ndarray) -> np.ndarray:
        """Whether each row of x is an interior point (a boundary point counts only if it is also one)."""
        return self._among(x, self.interior)

    def on_boundary(self, x: np.ndarray) -> np.ndarray:
        if self.boundary is None:
            raise ValueError("self.boundary must be initialized when call 'on_boundary' function")
        return self._among(x, self.boundary)

    def translate(self, translation: np.ndarray) -> "PointCloud":
        """Offset column i of the interior and boundary points by ``translation[i]``, in place."""
        for i, offset in enumerate(translation):
            self.interior[:, i] += offset
            if self.boundary is not None:
                self.boundary[:, i] += offset
        return self

    def scale(self, scale: np.ndarray) -> "PointCloud":
        """Scale column i of the interior points, boundary points and normals by ``scale[i]``, in place."""
        for i, factor in enumerate(scale):
            self.interior[:, i] *= factor
            if self.boundary is not None:
                self.boundary[:, i] *= factor
            if self.normal is not None:
                self.normal[:, i] *= factor
        return self

    def uniform_boundary_points(self, n: int):
        raise NotImplementedError("PointCloud do not have 'uniform_boundary_points' method")

    def random_boundary_points(self, n: int, random: str = "pseudo") -> np.ndarray:
        if self.boundary is None:
            raise ValueError("boundary points can't be empty when call 'random_boundary_points' method")
        if n > len(self.boundary):
            raise ValueError(f"number of sample points({n}) can't be more than that in boundary({len(self.boundary)})")
        return self.boundary[np.random.choice(len(self.boundary), size=n, replace=False)]

    def random_points(self, n: int, random: str = "pseudo") -> np.ndarray:
        if n > len(self.interior):
            raise ValueError(f"number of sample points({n}) can't be more than that in points({len(self.interior)})")
        return self.interior[np.random.choice(len(self.interior), size=n, replace=False)]

    def uniform_points(self, n: int, boundary: bool = True) -> np.ndarray:
        """The first n interior points."""
        return self.interior[:n]

    def union(self, other):
        raise NotImplementedError("Union operation for PointCloud is not supported yet.")

    __or__ = union

    def difference(self, other):
        raise NotImplementedError("Subtraction operation for PointCloud is not supported yet.")

    __sub__ = difference

    def intersection(self, other):
        raise NotImplementedError("Intersection operation for PointCloud is not supported yet.")

    __and__ = intersection

    def __str__(self) -> str:
        return ", ".join([self.__class__.__name__, f"num_points = {len(self.interior)}", f"ndim = {self.ndim}",
                          f"bbox = {self.bbox}", f"dim_keys = {self.dim_keys}"])
