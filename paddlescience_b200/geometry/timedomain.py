"""``TimeDomain`` and ``TimeXGeometry`` (reference: ppsci/geometry/timedomain.py:39-793): a time interval, and its
product with a space geometry whose points are (t, *space).

With ``timestamps`` (or ``time_step``) every sampler is time-major: the space points are drawn once and repeated for
each time after t0 (``timestamps[1:]``), so that the interior and the boundary leave out the initial time; the points
at t0 come from ``sample_initial_interior``.  Random draws consume numpy's global stream in the reference's order, so a
seeded sample matches its algorithm point for point."""
from __future__ import annotations

import itertools
from typing import Callable, Dict, Optional, Tuple

import numpy as np

from ..utils import misc
from . import geometry
from .geometry_1d import Interval
from .sampler import DEFAULT_DTYPE


class TimeDomain(Interval):
    """The time interval [t0, t1], optionally with a step or explicit timestamps (t0 included).

    >>> import ppsci
    >>> ppsci.geometry.TimeDomain(0, 1).on_initial([0, 0.01, 0.126, 0.2, 0.3])
    array([ True, False, False, False, False])
    """

    def __init__(self, t0: float, t1: float, time_step: Optional[float] = None,
                 timestamps: Optional[Tuple[float, ...]] = None):
        super().__init__(t0, t1)
        self.t0, self.t1 = t0, t1
        self.time_step = time_step
        self.timestamps = None if timestamps is None else np.array(timestamps, dtype=DEFAULT_DTYPE).reshape([-1])
        self.num_timestamps = None
        if time_step is not None:
            if time_step <= 0:
                raise ValueError(f"time_step({time_step}) must be larger than 0.")
            self.num_timestamps = int(np.ceil((t1 - t0) / time_step)) + 1
        elif timestamps is not None:
            self.num_timestamps = len(self.timestamps)

    def on_initial(self, t) -> np.ndarray:
        """Whether each time is t0 (``np.isclose``), flattened."""
        return np.isclose(t, self.t0).flatten()


def _tile_time(t: np.ndarray, x: np.ndarray, n: int) -> np.ndarray:
    """[(t_i, x_j)] time-major (every x for t_0, then every x for t_1, ...), cut to the first n rows."""
    t = np.asarray(t, dtype=DEFAULT_DTYPE).reshape([-1])
    tx = np.hstack((np.repeat(t, len(x)).reshape([-1, 1]), np.tile(x, (len(t), 1)))).astype(DEFAULT_DTYPE)
    return tx[:n] if len(tx) > n else tx


class TimeXGeometry(geometry.Geometry):
    """(t, *space) points of ``timedomain`` x ``geometry``; ``dim_keys`` is ``("t", *geometry.dim_keys)``.

    A ``criteria`` of ``sample_interior`` / ``sample_boundary`` / ``sample_initial_interior`` takes t as its first
    argument, e.g. ``lambda t, x, y: np.isclose(y, 0.05)``.  Where the space points are drawn before the times are
    attached (the random samplers), it is first called with t = None to filter them, as in the reference."""

    def __init__(self, timedomain: TimeDomain, geometry: geometry.Geometry):
        self.timedomain = timedomain
        self.geometry = geometry
        self.ndim = geometry.ndim + timedomain.ndim

    @property
    def dim_keys(self):
        return ("t",) + tuple(self.geometry.dim_keys)

    def on_boundary(self, x):
        return self.geometry.on_boundary(x[:, 1:])

    def on_initial(self, x):
        return self.timedomain.on_initial(x[:, :1])

    def boundary_normal(self, x):
        # column 0 carries t through, as in the reference (timedomain.py:130-133)
        return np.hstack((x[:, :1], self.geometry.boundary_normal(x[:, 1:])))

    # ---- the times after t0 that the interior and boundary samplers repeat the space points over ----
    def _step_times(self, boundary: bool = False) -> np.ndarray:
        """t0 < t <= t1 by the time step (also t0 when ``boundary``), or ``timestamps[1:]``."""
        td = self.timedomain
        if td.time_step is not None:
            nt = int(np.ceil(td.diam / td.time_step))
            return np.linspace(td.t1, td.t0, num=nt, endpoint=boundary, dtype=DEFAULT_DTYPE)[::-1]
        return td.timestamps[1:]

    def _space_points(self, nx: int, draw: Callable[[], np.ndarray], criteria, what: str) -> np.ndarray:
        """nx space points from repeated draws, filtered by criteria(None, *space) (reference loop and truncation)."""
        x = np.empty((nx, self.geometry.ndim), dtype=DEFAULT_DTYPE)
        filled, tries, hits = 0, 0, 0
        while filled < nx:
            pts = draw()
            if criteria is not None:
                pts = pts[criteria(None, *np.split(pts, self.geometry.ndim, axis=1)).flatten()]
            pts = pts[: nx - filled]
            x[filled: filled + len(pts)] = pts
            filled += len(pts)
            tries += 1
            hits += 1 if len(pts) > 0 else 0
            if tries >= 1000 and hits == 0:
                raise ValueError(f"Sample {what} points failed, please check correctness of geometry and given criteria.")
        return x

    def _require_times(self):
        if self.timedomain.time_step is None and self.timedomain.timestamps is None:
            raise ValueError("Either time_step or timestamps must be provided.")

    def uniform_points(self, n: int, boundary: bool = True) -> np.ndarray:
        """About n evenly spaced (t, x) points: ``timestamps[1:]`` (or the step's times after t0) x the space grid;
        without either, a time grid and a space grid sized by the space box's volume over the time span."""
        td = self.timedomain
        timed = td.time_step is not None or td.timestamps is not None
        if timed:
            nt = len(self._step_times())
            nx = int(np.ceil(n / nt))
        else:
            nx = int(np.ceil((n * np.prod(self.geometry.bbox[1] - self.geometry.bbox[0]) / td.diam) ** 0.5))
            nt = int(np.ceil(n / nx))
        x = self.geometry.uniform_points(nx, boundary=boundary)
        if not timed and boundary:
            t = td.uniform_points(nt, boundary=True)
        elif td.time_step is not None:
            t = self._step_times(boundary)
        else:
            t = td.timestamps[1:]
        return _tile_time(t, x, n)

    def random_points(self, n: int, random: str = "pseudo", criteria: Optional[Callable] = None) -> np.ndarray:
        """Random space points, drawn once and repeated over the times after t0 (time-major)."""
        self._require_times()
        t = self._step_times()
        nx = int(np.ceil(n / len(t)))
        x = self._space_points(nx, lambda: self.geometry.random_points(nx, random), criteria, "interior")
        return _tile_time(t, x, n)

    def uniform_boundary_points(self, n: int, criteria: Optional[Callable] = None) -> np.ndarray:
        """Evenly spaced space-boundary points x evenly spaced times after t0, sized by the boundary's area over the
        time span."""
        if self.geometry.ndim == 1:
            nx = 2
        else:
            side = np.asarray(self.geometry.bbox[1] - self.geometry.bbox[0]).reshape([-1])
            s = 2 * sum(a * b for a, b in itertools.combinations(side, 2))
            nx = int((n * s / self.timedomain.diam) ** 0.5)
        nt = int(np.ceil(n / nx))
        x = self._space_points(nx, lambda: self.geometry.uniform_boundary_points(nx), criteria, "boundary")
        td = self.timedomain
        t = np.linspace(td.t1, td.t0, num=nt, endpoint=False, dtype=DEFAULT_DTYPE)[::-1]
        return _tile_time(t, x, n)

    def random_boundary_points(self, n: int, random: str = "pseudo", criteria: Optional[Callable] = None) -> np.ndarray:
        """Random space-boundary points, drawn once and repeated over the times after t0 (time-major)."""
        self._require_times()
        t = self._step_times()
        nx = int(np.ceil(n / len(t)))
        x = self._space_points(nx, lambda: self.geometry.random_boundary_points(nx, random), criteria, "boundary")
        return _tile_time(t, x, n)

    def uniform_initial_points(self, n: int) -> np.ndarray:
        """n points at t0 from the space geometry's even grid."""
        x = self.geometry.uniform_points(n, True)[:n]
        return np.hstack((np.full([len(x), 1], self.timedomain.t0, dtype=DEFAULT_DTYPE), x)).astype(DEFAULT_DTYPE)

    def random_initial_points(self, n: int, random: str = "pseudo") -> np.ndarray:
        """n random points at t0."""
        x = self.geometry.random_points(n, random=random)
        return np.hstack((np.full([n, 1], self.timedomain.t0, dtype=DEFAULT_DTYPE), x)).astype(DEFAULT_DTYPE)

    # ---- named-column samplers: criteria(t, *space) on the drawn points, as Geometry's ----
    def sample_interior(self, n: int, random: str = "pseudo", criteria: Optional[Callable] = None,
                        evenly: bool = False, compute_sdf_derivatives: bool = False) -> Dict[str, np.ndarray]:
        draw = (lambda: self.uniform_points(n)) if evenly else (lambda: self.random_points(n, random, criteria))
        return misc.convert_to_dict(self._collect(n, draw, criteria, 1000, "interior"), self.dim_keys)

    def sample_boundary(self, n: int, random: str = "pseudo", criteria: Optional[Callable] = None,
                        evenly: bool = False) -> Dict[str, np.ndarray]:
        draw = (lambda: self.uniform_boundary_points(n)) if evenly else (
            lambda: self.random_boundary_points(n, random, criteria))
        x = self._collect(n, draw, criteria, 10000, "boundary")
        normal = self.boundary_normal(x)
        return {**misc.convert_to_dict(x, self.dim_keys),
                **misc.convert_to_dict(normal, tuple(f"normal_{k}" for k in self.dim_keys))}

    def sample_initial_interior(self, n: int, random: str = "pseudo", criteria: Optional[Callable] = None,
                                evenly: bool = False, compute_sdf_derivatives: bool = False) -> Dict[str, np.ndarray]:
        """n points at t0, filtered by criteria(t, *space); with the space geometry's signed distance (``sdf``, and
        ``sdf__<key>`` with ``compute_sdf_derivatives``) where it has one."""
        draw = (lambda: self.uniform_initial_points(n)) if evenly else (lambda: self.random_initial_points(n, random))
        x = self._collect(n, draw, criteria, 1000, "initial interior")
        extra = {}
        if hasattr(self.geometry, "sdf_func"):
            extra["sdf"] = -self.geometry.sdf_func(x[:, 1:])
            if compute_sdf_derivatives:
                d = -self.geometry.sdf_derivatives(x[:, 1:])
                extra.update(misc.convert_to_dict(d, tuple(f"sdf__{k}" for k in self.geometry.dim_keys)))
        return {**misc.convert_to_dict(x, self.dim_keys), **extra}

    def __str__(self) -> str:
        return ", ".join([self.__class__.__name__, f"ndim = {self.ndim}",
                          f"bbox = (time){self.timedomain.bbox} x (space){self.geometry.bbox}",
                          f"diam = (time){self.timedomain.diam} x (space){self.geometry.diam}",
                          f"dim_keys = {self.dim_keys}"])
