from .pde import PDE, AllenCahn, Biharmonic, HeatExchanger, Helmholtz, Laplace, NavierStokes, Poisson, Vibration

__all__ = ["PDE", "AllenCahn", "Biharmonic", "HeatExchanger", "Helmholtz", "Laplace", "NavierStokes", "Poisson", "Vibration", "build_equation"]


def build_equation(cfg):
    """ppsci/equation/__init__.py — build equations from a list of single-key dicts."""
    if cfg is None:
        return None
    eqs = {}
    for item in cfg:
        cls = next(iter(item.keys()))
        kw = dict(item[cls])
        name = kw.pop("name", cls)
        eqs[name] = globals()[cls](**kw)
    return eqs
