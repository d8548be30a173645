from .geometry import Geometry
from .geometry_1d import Interval
from .geometry_2d import Rectangle
from .geometry_3d import Cuboid
from .geometry_nd import Hypercube
from .pointcloud import PointCloud
from .timedomain import TimeDomain, TimeXGeometry

__all__ = ["Geometry", "Interval", "Rectangle", "Cuboid", "Hypercube", "PointCloud", "TimeDomain", "TimeXGeometry", "build_geometry"]


def build_geometry(cfg):
    """ppsci/geometry/__init__.py — build geometries from a list of single-key dicts."""
    if cfg is None:
        return None
    geoms = {}
    for item in cfg:
        name = next(iter(item.keys()))
        kw = dict(item[name])
        cls = next(iter(kw.keys()))
        geoms[name] = globals()[cls](**kw[cls])
    return geoms
