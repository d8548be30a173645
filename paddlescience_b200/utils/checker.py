"""``ppsci.utils.run_check`` (reference: ppsci/utils/checker.py:34-117): a two-epoch Navier-Stokes smoke training plus
one evaluation through the public API — here it exercises the native library end to end (fused residual / loss / weight-
gradient call, fused Adam, forward-only evaluation).  Needs an H100: the engine has no CPU fallback."""
from __future__ import annotations

import traceback

from . import logger

__all__ = ["run_check"]


def run_check() -> bool:
    """Returns True when the demo trains and evaluates; problems are logged like the reference does."""
    import ppsci

    try:
        ppsci.utils.set_random_seed(42)
        model = ppsci.arch.MLP(("x", "y"), ("u", "v", "p"), 3, 16, "tanh")
        equation = {"NavierStokes": ppsci.equation.NavierStokes(0.01, 1.0, 2, False)}
        geom = {"rect": ppsci.geometry.Rectangle((-0.05, -0.05), (0.05, 0.05))}
        iters_per_epoch = 5
        train_dataloader_cfg = {"dataset": "IterableNamedArrayDataset", "iters_per_epoch": iters_per_epoch}
        npoint_pde = 8 ** 2
        pde_constraint = ppsci.constraint.InteriorConstraint(
            equation["NavierStokes"].equations, {"continuity": 0, "momentum_x": 0, "momentum_y": 0}, geom["rect"],
            {**train_dataloader_cfg, "batch_size": npoint_pde}, ppsci.loss.MSELoss("sum"), evenly=True,
            weight_dict={"continuity": 0.0001, "momentum_x": 0.0001, "momentum_y": 0.0001}, name="EQ")
        constraint = {pde_constraint.name: pde_constraint}
        residual_validator = ppsci.validate.GeometryValidator(
            equation["NavierStokes"].equations, {"continuity": 0, "momentum_x": 0, "momentum_y": 0}, geom["rect"],
            {"dataset": "NamedArrayDataset", "total_size": 8 ** 2, "batch_size": 32, "sampler": {"name": "BatchSampler"}},
            ppsci.loss.MSELoss("sum"), evenly=True, metric={"MSE": ppsci.metric.MSE(False)}, name="Residual")
        validator = {residual_validator.name: residual_validator}
        epochs = 2
        optimizer = ppsci.optimizer.Adam(0.001)(model)
        solver = ppsci.solver.Solver(model, constraint, None, optimizer, None, epochs, iters_per_epoch, equation=equation,
                                     validator=validator)
        solver.train()
        solver.eval(epochs)
    except Exception as e:  # noqa: BLE001 — the reference reports any failure the same way
        traceback.print_exc()
        logger.error(f"the H100-native ppsci engine meets some problem with \n {repr(e)} \nplease check that the native "
                     "library is built (python -c 'import __graft_entry__ as g; g.build()') and an H100 is visible.")
        return False
    logger.message("ppsci (H100-native engine) is installed successfully.")
    return True
