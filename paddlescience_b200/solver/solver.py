"""``Solver`` — orchestration with the reference's constructor and public methods
(ppsci/solver/solver.py:62-1116), hosting the H100-native hot loop.

Kept: ``Solver(model, constraint, output_dir, optimizer, lr_scheduler, epochs, iters_per_epoch,
update_freq, save_freq, log_freq, ..., equation, geom, validator, ...)``, ``train()``, ``eval()``,
``predict()``, checkpoint save/resume.  Out of scope (SURVEY.md §2 rows 12/17/18): export/ONNX,
VisualDL/WandB writers, AMP.  ``to_static=True`` records the training iteration as a CUDA graph
(solver/graph_step.py) instead of tracing a static program."""
from __future__ import annotations

import os
from typing import Any, Dict, Optional

import numpy as np
import torch

from ..loss import mtl
from ..utils import expression, logger, misc, save_load
from . import train as train_mod


class Solver:
    def __init__(
        self,
        model,
        constraint: Optional[Dict[str, Any]] = None,
        output_dir: Optional[str] = "./output/",
        optimizer=None,
        lr_scheduler=None,
        epochs: int = 5,
        iters_per_epoch: int = 20,
        update_freq: int = 1,
        save_freq: int = 0,
        log_freq: int = 10,
        eval_during_train: bool = False,
        start_eval_epoch: int = 1,
        eval_freq: int = 1,
        seed: int = 42,
        use_vdl: bool = False,
        use_wandb: bool = False,
        use_tbd: bool = False,
        wandb_config=None,
        device: str = "gpu",
        equation: Optional[Dict[str, Any]] = None,
        geom: Optional[Dict[str, Any]] = None,
        validator: Optional[Dict[str, Any]] = None,
        visualizer: Optional[Dict[str, Any]] = None,
        use_amp: bool = False,
        amp_level: str = "O1",
        pretrained_model_path: Optional[str] = None,
        checkpoint_path: Optional[str] = None,
        compute_metric_by_batch: bool = False,
        eval_with_no_grad: bool = False,
        to_static: bool = False,
        loss_aggregator=None,
        *,
        cfg=None,
    ):
        if use_amp:
            raise NotImplementedError("AMP is not supported: the jet kernels compute in fp32 (3xTF32 on tensor cores) or fp64")
        self.model = model
        self.constraint = constraint or {}
        self.output_dir = output_dir
        self.optimizer = optimizer
        self.lr_scheduler = lr_scheduler
        self.epochs, self.iters_per_epoch = epochs, iters_per_epoch
        self.update_freq, self.save_freq, self.log_freq = update_freq, save_freq, log_freq
        self.eval_during_train, self.start_eval_epoch, self.eval_freq = eval_during_train, start_eval_epoch, eval_freq
        self.seed = seed
        self.equation, self.geom, self.validator, self.visualizer = equation, geom, validator, visualizer
        self.compute_metric_by_batch = compute_metric_by_batch
        self.eval_with_no_grad = eval_with_no_grad
        self.global_step = 0
        self.to_static = bool(to_static)
        self._graph_step = None  # GraphedTrainStep, created by the first training iteration when to_static is set
        self.max_steps = self.epochs * self.iters_per_epoch
        self.train_output_info: Dict[str, misc.AverageMeter] = {}
        self.train_time_info = {"reader_cost": misc.AverageMeter("reader_cost", ".5f", postfix="s"),
                                "batch_cost": misc.AverageMeter("batch_cost", ".5f", postfix="s")}
        self.eval_output_info: Dict[str, misc.AverageMeter] = {}
        self.last_loss = float("nan")
        self.best_metric = {"metric": float("inf"), "epoch": 0}
        self.benchmark_flag = bool(os.getenv("BENCHMARK_ROOT", None))
        self.nvtx_flag = bool(os.getenv("NVTX", None))

        # device / distributed (one process per GPU, launched by torchrun; solver.py:247-310)
        import torch.distributed as dist

        self.rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        self.world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        if device in ("gpu", "cuda") and torch.cuda.is_available():
            local = int(os.environ.get("LOCAL_RANK", "0"))
            self.device = torch.device("cuda", local if local < torch.cuda.device_count() else 0)
            # the native library allocates / launches on the CURRENT device (plan_create: cudaGetDevice + cudaMalloc)
            torch.cuda.set_device(self.device)
            self.model.to(self.device)
            for eq in (self.equation or {}).values():  # learnable equation scalars live beside the model (paddle creates them there)
                for q in getattr(eq, "learnable_parameters", ()):
                    q.data = q.data.to(self.device)
                    if q.grad is not None:
                        q.grad = q.grad.to(self.device)
        else:
            self.device = torch.device("cpu")  # construction / host logic only; train() raises
        for cst in self.constraint.values():
            ds = getattr(getattr(cst.data_loader, "loader", None), "ds", None) or getattr(cst.data_loader, "loader", None)
            if hasattr(ds, "to") and self.device.type == "cuda":
                ds.to(self.device)  # IterableNamedArrayDataset keeps its full batch device-resident

        if pretrained_model_path is not None:
            save_load.load_pretrain(self.model, pretrained_model_path, self.equation)
        if checkpoint_path is not None:
            self.best_metric.update(save_load.load_checkpoint(checkpoint_path, self.model, self.optimizer, self.equation) or {})

        if self.world_size > 1 and hasattr(self.model, "flat"):
            # Paddle's DataParallel broadcasts rank 0's parameters at wrap time (solver.py:299-310); ranks seeded
            # differently would otherwise train diverging replicas without any error
            dist.broadcast(self.model.flat.data, src=0)
            for eq in (self.equation or {}).values():  # the equations are wrapped the same way (paddle.DataParallel around every equation with learnable parameters, like the model)
                for q in getattr(eq, "learnable_parameters", ()):
                    dist.broadcast(q.data, src=0)

        self.forward_helper = expression.ExpressionSolver()
        self.forward_helper.nvtx_flag = self.nvtx_flag
        self.loss_aggregator = loss_aggregator or mtl.Sum()
        if type(self.loss_aggregator).__name__ not in ("Sum", "PCGrad", "GradNorm", "NTK", "Relobralo", "AGDA"):
            raise NotImplementedError("loss aggregators supported by the adjoint kernels: Sum (one fused call); PCGrad, "
                                      "GradNorm, NTK, Relobralo, AGDA (one call per loss term)")
        if getattr(self.loss_aggregator, "needs_per_key_grads", False) and getattr(self.loss_aggregator, "model", None) is None:
            self.loss_aggregator.model = self.model  # Relobralo(num_losses) has no model argument in the reference
        # compile every constraint's expressions now (solver.py:496-535 does its sympy conversion here)
        for cst in ([] if hasattr(self.model, "fused_train_forward") else self.constraint.values()):
            sample_keys = None
            ds = getattr(cst.data_loader, "loader", None)
            ds = getattr(ds, "ds", ds)
            if hasattr(ds, "input"):
                sample_keys = {k: None for k in ds.input}
            self.forward_helper.compiled_for(self.model, cst, sample_keys)
        logger.info(f"Using {self.world_size} process(es), device {self.device}")

    # ------------------------------------------------------------------------------------------
    def train(self):
        if self.device.type != "cuda":
            raise RuntimeError("Solver.train needs a CUDA (H100) device: the engine has no CPU fallback")
        if self.optimizer is None:
            raise ValueError("Solver.train needs an optimizer")
        start_epoch = self.best_metric["epoch"] + 1
        self.global_step = (start_epoch - 1) * self.iters_per_epoch
        for epoch_id in range(start_epoch, self.epochs + 1):
            if getattr(self.optimizer, "is_lbfgs", False):
                train_mod.train_LBFGS_epoch_func(self, epoch_id, self.log_freq)
            else:
                train_mod.train_epoch_func(self, epoch_id, self.log_freq)
            if self.lr_scheduler is not None and self.lr_scheduler.by_epoch:
                self.lr_scheduler.step()
            # evaluation during training (solver.py:577-607): keep the best model by the target metric
            if self.eval_during_train and self.validator and epoch_id % self.eval_freq == 0 and epoch_id >= self.start_eval_epoch:
                cur_metric, _ = self.eval(epoch_id)
                if cur_metric < self.best_metric["metric"]:
                    self.best_metric.update({"metric": cur_metric, "epoch": epoch_id})
                    if self.output_dir:
                        save_load.save_checkpoint(self.model, self.optimizer, dict(self.best_metric), self.output_dir,
                                                  "best_model", self.equation)
                logger.info(f"[Eval][Epoch {epoch_id}][best metric: {self.best_metric['metric']}]")
            if self.save_freq > 0 and epoch_id % self.save_freq == 0:
                save_load.save_checkpoint(self.model, self.optimizer, {"metric": self.last_loss, "epoch": epoch_id},
                                          self.output_dir, f"epoch_{epoch_id}", self.equation)
            if self.output_dir and self.save_freq > 0:
                save_load.save_checkpoint(self.model, self.optimizer, {"metric": self.last_loss, "epoch": epoch_id},
                                          self.output_dir, "latest", self.equation, print_log=(epoch_id == self.epochs))
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)

    @torch.no_grad()
    def predict(self, input_dict: Dict[str, Any], expr_dict: Optional[Dict[str, Any]] = None, batch_size: Optional[int] = 64,
                no_grad: bool = True, return_numpy: bool = False):
        """Batched forward of the model (+ expressions) — solver.py:729-872 without the DP gather."""
        if self.device.type != "cuda":
            raise RuntimeError("Solver.predict needs a CUDA (H100) device: the engine has no CPU fallback")
        n = len(next(iter(input_dict.values())))
        bs = n if batch_size is None else batch_size
        chunks: Dict[str, list] = {}
        for s in range(0, n, bs):
            batch = {k: torch.as_tensor(np.asarray(v[s: s + bs]) if not torch.is_tensor(v) else v[s: s + bs]).to(
                self.device, self.model.dtype) for k, v in input_dict.items()}
            out = self.forward_helper.visu_forward(expr_dict, batch, self.model)
            for k, v in out.items():
                chunks.setdefault(k, []).append(v)
        res = {k: torch.cat(v, dim=0) for k, v in chunks.items()}
        return {k: v.cpu().numpy() for k, v in res.items()} if return_numpy else res

    @torch.no_grad()
    def eval(self, epoch_id: int = 0):
        """Evaluate every validator; returns (mean target metric, metric dict)."""
        if not self.validator:
            raise ValueError("Solver.eval needs validators")
        from ..validate import evaluate

        return evaluate(self, epoch_id)
