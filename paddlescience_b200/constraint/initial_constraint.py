"""``InitialConstraint`` (reference: ppsci/constraint/initial_constraint.py:37-172)."""
from __future__ import annotations

from typing import Any, Callable, Dict, Optional, Union

from ..data import dataset
from . import base


class InitialConstraint(base.Constraint):
    """Constraint on points sampled once at the initial time t0 of a ``TimeXGeometry``
    (``geom.sample_initial_interior``; ``criteria`` takes t first).  Same arguments as the reference
    (initial_constraint.py:90-103).  It trains through the fused path like any other constraint."""

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
        weight_dict: Optional[Dict[str, Union[Callable, float]]] = None,
        compute_sdf_derivatives: bool = False,
        name: str = "IC",
    ):
        self.label_dict = label_dict
        self.input_keys = geom.dim_keys
        self.output_keys = tuple(label_dict.keys())
        self.output_expr = {k: v for k, v in output_expr.items() if k in self.output_keys}
        if isinstance(criteria, str):
            criteria = eval(criteria)
        dataloader_cfg = dict(dataloader_cfg)
        n = dataloader_cfg["batch_size"] * dataloader_cfg["iters_per_epoch"]
        inputs = geom.sample_initial_interior(n, random, criteria, evenly, compute_sdf_derivatives)
        if "area" in inputs:
            inputs["area"] *= dataloader_cfg["iters_per_epoch"]
        like = next(iter(inputs.values()))
        label = base.materialize(label_dict, inputs, geom.dim_keys, like)
        weight = base.materialize_weights(weight_dict, label, inputs, geom.dim_keys)
        ds_cfg = dataloader_cfg["dataset"]
        ds_cfg = {"name": ds_cfg} if isinstance(ds_cfg, str) else dict(ds_cfg)
        ds_cfg.update({"input": inputs, "label": label, "weight": weight})
        dataloader_cfg["dataset"] = ds_cfg
        super().__init__(dataset.build_dataset(ds_cfg), dataloader_cfg, loss, name)
