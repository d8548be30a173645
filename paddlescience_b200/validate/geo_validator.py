"""``GeometryValidator`` (reference: ppsci/validate/geo_validator.py:35-165): evaluation points sampled once inside a
geometry, labels from numbers / sympy / callables, unit weights."""
from __future__ import annotations

from typing import Any, Callable, Dict, Optional, Union

import numpy as np

from ..constraint import base as cbase
from ..data import dataset
from . import base


class GeometryValidator(base.Validator):
    """Same arguments as the reference (geo_validator.py:72-85).  On a ``TimeXGeometry`` with timestamps (or a time
    step), ``total_size`` is split evenly over the times: the points after t0, time-major, and with ``with_initial``
    also ``total_size / num_timestamps`` points at t0 in front of them (geo_validator.py:94-130).  Random times
    raise ``NotImplementedError``, as in the reference."""

    def __init__(
        self,
        output_expr: Dict[str, Callable],
        label_dict: Dict[str, Union[float, Callable]],
        geom,
        dataloader_cfg: Dict[str, Any],
        loss,
        random: str = "pseudo",
        criteria: Optional[Callable] = None,
        evenly: bool = False,
        metric: Optional[Dict[str, Any]] = None,
        with_initial: bool = False,
        name: Optional[str] = None,
    ):
        self.output_expr = output_expr
        self.label_dict = label_dict
        self.input_keys = geom.dim_keys
        self.output_keys = tuple(label_dict.keys())
        self.num_timestamps = 1
        nx = dataloader_cfg["total_size"]
        if hasattr(geom, "timedomain"):
            nts = geom.timedomain.num_timestamps
            if nts is None:
                raise NotImplementedError("TimeXGeometry with random timestamp not implemented yet.")
            self.num_timestamps = nts if with_initial else nts - 1
            if nx % self.num_timestamps != 0:
                raise ValueError(f"total_size {nx} is not a multiple of the {self.num_timestamps} timestamps")
            nx //= self.num_timestamps
            inputs = geom.sample_interior(nx * (nts - 1), random, criteria, evenly)
            if with_initial:
                initial = geom.sample_initial_interior(nx, random, criteria, evenly)
                inputs = {key: np.vstack((initial[key], inputs[key])) for key in inputs}
        else:
            inputs = geom.sample_interior(nx, random, criteria, evenly)
        like = next(iter(inputs.values()))
        label = cbase.materialize(label_dict, inputs, geom.dim_keys, like)
        weight = {key: np.ones_like(next(iter(label.values()))) for key in label}
        dataloader_cfg = dict(dataloader_cfg)
        ds_cfg = dataloader_cfg["dataset"]
        ds_cfg = {"name": ds_cfg} if isinstance(ds_cfg, str) else dict(ds_cfg)
        ds_cfg.update({"input": inputs, "label": label, "weight": weight})
        dataloader_cfg["dataset"] = ds_cfg
        super().__init__(dataset.build_dataset(ds_cfg), dataloader_cfg, loss, metric, name)
