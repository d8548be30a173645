"""One training iteration recorded as a CUDA graph and replayed (``Solver(to_static=True)``).

The reference's ``to_static=True`` (ppsci/solver/solver.py:487, 907-937) hands the forward to a tracing compiler so that
small problems stop paying the per-operator host overhead.  On the H100 the same goal needs no compiler: the iteration is
already a fixed launch train (input packing, the fused residual / adjoint kernels behind
``ppsci_b200_residual_loss_fwd_bwd``, loss aggregation, ``ppsci_b200_adam_step_dev``), so it is captured once per batch
signature and replayed with one ``cudaGraphLaunch`` per step.  Everything that changes from step to step lives in device
memory: the batch (copied into the graph's static input buffers), and the optimizer scalars {lr, bias corrections,
gradient scale} in a 4-double device buffer refreshed from a ring of pinned host slots.

Restrictions (anything else falls back to the eager iteration with a one-line reason): one process (no data-parallel
all-reduce inside the graph), ``update_freq == 1``, Adam, the ``Sum`` loss aggregator."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

_RING = 64


def _flatten(dicts) -> Tuple[list, tuple]:
    """-> ([(i, key, tensor)], signature) over a tuple of {key: tensor | float | None} (None entries allowed)."""
    items, sig = [], []
    for i, d in enumerate(dicts):
        if d is None:
            sig.append((i, None))
            continue
        for k in d:
            v = d[k]
            if torch.is_tensor(v):
                items.append((i, k, v))
                sig.append((i, k, tuple(v.shape), str(v.dtype)))
            else:
                sig.append((i, k, "const", None if v is None else float(v)))
    return items, tuple(sig)


class GraphedTrainStep:
    """``step(input_dicts, label_dicts, weight_dicts) -> (total_loss, losses_constraint)``; the returned tensors are the
    graph's static outputs (overwritten by the next replay — read them before stepping again)."""

    WARMUP = 2  # eager iterations before the capture (workspaces, plans and cuBLAS-free lazy state get created there)

    def __init__(self, solver):
        self.solver = solver
        self._entries: Dict[tuple, dict] = {}
        self.replays = 0
        self.always_copy = False  # True: re-copy every batch tensor each step even when it is the unmodified same object

    # -- eligibility ------------------------------------------------------------------------------------------------
    def unsupported_reason(self) -> Optional[str]:
        s = self.solver
        dev = s.model.flat.device
        if dev.type != "cuda":
            return "parameters are not on a CUDA device"
        if s.world_size > 1:
            return "data parallel (the gradient all-reduce stays outside the graph)"
        if s.update_freq != 1:
            return "update_freq > 1"
        if not hasattr(s.optimizer, "step_dev"):
            return f"{type(s.optimizer).__name__} has no graph-replayable step"
        if type(s.loss_aggregator).__name__ != "Sum":
            return f"loss aggregator {type(s.loss_aggregator).__name__}"
        if getattr(s.loss_aggregator, "needs_per_key_grads", False):
            return "per-term gradients"
        for c in s.constraint.values():  # not validated under capture: stay eager
            if type(getattr(c, "loss", None)).__name__ == "CausalMSELoss":
                return "CausalMSELoss (two native calls with device-side weight arithmetic between them)"
        if getattr(s.optimizer, "grad_clip", None) is not None:
            return "gradient clipping"
        return None

    # -- the iteration body (runs eagerly during warm-up, once under capture) ------------------------------------------
    def _body(self, input_dicts, label_dicts, weight_dicts, hyper_dev):
        s = self.solver
        losses_all, losses_constraint = s.forward_helper.train_forward(
            tuple(c.output_expr for c in s.constraint.values()), input_dicts, s.model, s.constraint, label_dicts,
            weight_dicts)[:2]
        total = s.loss_aggregator(losses_all, s.global_step).loss
        s.optimizer.step_dev(hyper_dev, zero_grads=True)
        return total, losses_constraint

    def _push_hyper(self, e):
        """Next ring slot <- this step's optimizer scalars; async H2D into the device buffer the graph reads."""
        slot = e["slot"] = (e["slot"] + 1) % _RING
        ev = e["events"][slot]
        if ev is not None:
            ev.synchronize()  # the copy that last read this pinned slot has run (no-op unless the host is 64 steps ahead)
        vals = self.solver.optimizer.advance()
        host = e["ring"][slot]
        host[0], host[1], host[2], host[3] = vals
        e["hyper"].copy_(host, non_blocking=True)
        ev = e["events"][slot] = ev if ev is not None else torch.cuda.Event()
        ev.record()

    def _new_entry(self, dev):
        return {"n": 0, "graph": None, "slot": -1, "events": [None] * _RING,
                "ring": torch.zeros(_RING, 4, dtype=torch.float64).pin_memory(),
                "hyper": torch.zeros(4, dtype=torch.float64, device=dev)}

    def __call__(self, input_dicts, label_dicts, weight_dicts):
        s = self.solver
        model = s.model
        dev, dtype = model.flat.device, model.flat.dtype
        s.optimizer.grad_scale = 1.0
        groups = (tuple(input_dicts), tuple(label_dicts), tuple(weight_dicts))
        flat: List[list] = []
        sig = []
        for g in groups:
            items, sg = _flatten(g)
            flat.append(items)
            sig.append(sg)
        sig = tuple(sig)
        e = self._entries.get(sig)
        if e is None:
            e = self._entries[sig] = self._new_entry(dev)
        if e["graph"] is None and e["n"] < self.WARMUP:
            e["n"] += 1
            self._push_hyper(e)
            ins = [self._device_dicts(g, dev, dtype) for g in groups]
            return self._body(ins[0], ins[1], ins[2], e["hyper"])
        if e["graph"] is None:
            # static copies of the batch: the graph reads these addresses on every replay
            statics = []
            for g in groups:
                sg = []
                for d in g:
                    if d is None:
                        sg.append(None)
                        continue
                    sd = {}
                    for k, v in d.items():
                        if torch.is_tensor(v):
                            sd[k] = torch.empty(v.shape, dtype=dtype if v.is_floating_point() else v.dtype, device=dev)
                            sd[k].copy_(v)
                        else:
                            sd[k] = v
                    sg.append(sd)
                statics.append(tuple(sg))
            e["statics"] = statics
            if model.flat.grad is None:
                model.flat.grad = torch.zeros_like(model.flat.data)
            torch.cuda.synchronize(dev)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                e["out"] = self._body(statics[0], statics[1], statics[2], e["hyper"])
            e["graph"] = graph
            e["src"] = None
        # refresh the static batch (skipped for tensors that are the very objects, unmodified, copied last time)
        src = e.get("src") or {}
        new_src = {}
        for gi, items in enumerate(flat):
            for (i, k, v) in items:
                tag = (id(v), v._version, v.data_ptr())
                key = (gi, i, k)
                if self.always_copy or src.get(key) != tag:
                    e["statics"][gi][i][k].copy_(v, non_blocking=True)
                new_src[key] = tag
        e["src"] = new_src
        e["keep"] = flat  # the ids above stay unique while the tensors are alive
        self._push_hyper(e)
        e["graph"].replay()
        self.replays += 1
        return e["out"]

    @staticmethod
    def _device_dicts(group, dev, dtype):
        out = []
        for d in group:
            if d is None:
                out.append(None)
                continue
            dd = {}
            for k, v in d.items():
                if torch.is_tensor(v):
                    if v.device != dev:
                        v = v.to(dev, non_blocking=True)
                    if v.is_floating_point() and v.dtype != dtype:
                        v = v.to(dtype)
                dd[k] = v
            out.append(dd)
        return tuple(out)
