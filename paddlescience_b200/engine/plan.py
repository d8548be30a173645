"""Plan objects: a compiled constraint bound to the native library.

``ResidualPlan`` is what ``ExpressionSolver.train_forward`` (reference:
ppsci/utils/expression.py:60-131) dispatches to in this framework: one C-ABI call evaluates
network jets, residuals, MSE and (optionally) the weight gradient for one constraint.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence

import torch

from . import binding as B
from .compiler import CompiledResidual


def _dtype_id(dtype: torch.dtype) -> int:
    if dtype == torch.float32:
        return B.F32
    if dtype == torch.float64:
        return B.F64
    raise TypeError(f"unsupported dtype {dtype}: the engine computes in float32 or float64")


def _col(t: torch.Tensor, n: int, dtype: torch.dtype, device, what: str) -> torch.Tensor:
    if t.dtype != dtype:
        raise TypeError(f"{what}: dtype {t.dtype} does not match the plan dtype {dtype}")
    if t.device != device:
        raise ValueError(f"{what}: tensor is on {t.device}, parameters are on {device}")
    if t.numel() != n:
        raise ValueError(f"{what}: expected {n} values, got shape {tuple(t.shape)}")
    return t.contiguous()


class ResidualPlan:
    def __init__(
        self,
        compiled: CompiledResidual,
        dtype: torch.dtype = torch.float32,
        reductions: Optional[Sequence[str]] = None,
        loss_weights: Optional[Sequence[float]] = None,
        chunk_points: int = 0,
        backend: int = 0,
        library: Optional[B.Library] = None,
    ):
        self.lib = library or B.get_library()
        self.compiled = compiled
        self.dtype = dtype
        net = compiled.net
        n_res = len(compiled.res_reg)
        if len(net.input_keys) > B.MAX_IN:
            raise NotImplementedError(f"more than {B.MAX_IN} network inputs")
        if len(net.widths) - 1 > B.MAX_LAYERS:
            raise NotImplementedError(f"more than {B.MAX_LAYERS} linear layers")
        if n_res > B.MAX_RES:
            raise NotImplementedError(f"more than {B.MAX_RES} residuals per constraint")
        if net.act.lower() not in B.ACT_IDS:
            raise NotImplementedError(f"activation {net.act!r} has no jet kernel (supported: {sorted(B.ACT_IDS)})")
        s = B.PlanSpec()
        s.dtype = _dtype_id(dtype)
        s.n_in = len(net.input_keys)
        s.n_feat = net.widths[0]
        self.dense_in = bool(getattr(net, "dense_in", False))
        s.dense_in = 1 if self.dense_in else 0
        if not self.dense_in:
            omega_param = getattr(net, "feat_omega_param", None) or [-1] * s.n_feat
            for f in range(s.n_feat):
                s.feat_src[f] = net.feat_src[f]
                s.feat_kind[f] = net.feat_kind[f]
                s.feat_omega[f] = net.feat_omega[f]
                s.feat_omega_param[f] = omega_param[f]  # trainable frequency index (read from params), or -1
            s.n_omega = int(getattr(net, "n_omega", 0) or 0)
        s.n_layers = len(net.widths) - 1
        for i, w in enumerate(net.widths):
            s.widths[i] = w
        s.act = B.ACT_IDS[net.act.lower()]
        act_first = getattr(net, "act_first", None)
        if act_first is not None and act_first.lower() not in B.ACT_IDS:
            raise NotImplementedError(f"activation {act_first!r} has no jet kernel (supported: {sorted(B.ACT_IDS)})")
        s.act_first = B.ACT_IDS[act_first.lower()] if act_first is not None else -1
        s.gated = int(getattr(net, "gated", 0) or 0)  # 1 ModifiedMLP, 2 PirateNet (embeddings + gates [+ adaptive residuals])
        s.n_dir = len(compiled.dirs)
        for d, dr in enumerate(compiled.dirs):
            s.dir_order[d] = dr.order
            for i, v in enumerate(dr.vec):
                s.dir_vec[d][i] = float(v)
        s.n_aux = len(compiled.aux_keys)
        if s.n_aux > B.MAX_IN:
            raise NotImplementedError(f"more than {B.MAX_IN} auxiliary columns / learnable parameters")
        # learnable equation parameters: one scalar for all points + dLoss/dparameter accumulated by the head kernel
        self.param_keys = list(getattr(compiled, "param_keys", []) or [])
        for i, k in enumerate(compiled.aux_keys):
            s.aux_bcast[i] = 1 if k in self.param_keys else 0
        s.n_pgrad = len(getattr(compiled, "pgrad_res", []) or [])
        for g in range(s.n_pgrad):
            s.pgrad_res[g] = compiled.pgrad_res[g]
            s.pgrad_aux[g] = compiled.pgrad_aux[g]
            s.pgrad_reg[g] = compiled.pgrad_reg[g]
        self._param_grad = None  # fp64 [n_aux] device buffer the head kernel accumulates dLoss/dparameter into
        self.two_phase_launches = 0  # kernels launched by values_fwd_keep / values_bwd_kept calls so far (bench instrumentation)
        s.n_reg = compiled.n_reg
        s.n_ops = len(compiled.prog)
        flat = [x for op in compiled.prog for x in op]
        self._prog = (C.c_int32 * max(1, len(flat)))(*flat)
        self._consts = (C.c_double * max(1, len(compiled.consts)))(*compiled.consts)
        self._gres = (C.c_int32 * max(1, len(compiled.grad_res)))(*compiled.grad_res)
        self._gin = (C.c_int32 * max(1, len(compiled.grad_in)))(*compiled.grad_in)
        self._greg = (C.c_int32 * max(1, len(compiled.grad_reg)))(*compiled.grad_reg)
        s.prog = C.cast(self._prog, C.POINTER(C.c_int32))
        s.n_consts = len(compiled.consts)
        s.consts = C.cast(self._consts, C.POINTER(C.c_double))
        s.n_res = n_res
        for k in range(n_res):
            s.res_reg[k] = compiled.res_reg[k]
            red = (reductions[k] if reductions else "mean")
            if red not in ("mean", "sum"):
                raise ValueError(f"reduction should be 'mean' or 'sum', but got {red}")
            s.reduction[k] = B.REDUCE_MEAN if red == "mean" else B.REDUCE_SUM
            s.loss_weight[k] = float(loss_weights[k]) if loss_weights else 1.0
        s.n_grad = len(compiled.grad_res)
        s.grad_res = C.cast(self._gres, C.POINTER(C.c_int32))
        s.grad_in = C.cast(self._gin, C.POINTER(C.c_int32))
        s.grad_reg = C.cast(self._greg, C.POINTER(C.c_int32))
        s.chunk_points = int(chunk_points)
        if int(backend) == 0 and os.environ.get("PPSCI_B200_BACKEND"):
            backend = int(os.environ["PPSCI_B200_BACKEND"])  # 1 = force SIMT kernels, 2 = require the wgmma kernels
        s.backend = int(backend)
        self.spec = s
        handle = C.c_void_p()
        self.lib.check(self.lib.lib.ppsci_b200_plan_create(C.byref(s), C.byref(handle)), "plan_create")
        self.handle = handle
        self.n_params = int(self.lib.lib.ppsci_b200_plan_param_count(handle))
        self.channels = int(self.lib.lib.ppsci_b200_plan_channels(handle))
        self.n_res = n_res
        self.n_out = net.widths[-1]
        self._ws: Optional[torch.Tensor] = None
        self._loss: Optional[torch.Tensor] = None

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.lib.ppsci_b200_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ------------------------------------------------------------------------------------
    @property
    def uses_tcgen05(self) -> bool:
        return bool(self.lib.lib.ppsci_b200_plan_uses_tcgen05(self.handle))

    @property
    def last_launches(self) -> int:
        return int(self.lib.lib.ppsci_b200_plan_last_launches(self.handle))

    PROFILE_CLASSES = ("fwd_gemm", "head", "dw_gemm", "dx_gemm", "misc", "thin_fwd", "thin_dx", "thin_dw")

    def set_profile(self, on: bool):
        self.lib.check(self.lib.lib.ppsci_b200_plan_set_profile(self.handle, 1 if on else 0), "set_profile")

    def get_profile(self):
        ms = (C.c_double * 8)()
        cnt = (C.c_int64 * 8)()
        self.lib.check(self.lib.lib.ppsci_b200_plan_get_profile(self.handle, ms, cnt), "get_profile")
        return {k: {"ms": ms[i], "launches": int(cnt[i])} for i, k in enumerate(self.PROFILE_CLASSES)}

    def _workspace(self, n: int, device) -> torch.Tensor:
        need = int(self.lib.lib.ppsci_b200_plan_workspace_bytes(self.handle, n))
        if self._ws is None or self._ws.numel() < need + 256 or self._ws.device != device:
            self._ws = torch.empty(need + 256, dtype=torch.uint8, device=device)
        return self._ws

    @staticmethod
    def _aligned(ws: torch.Tensor):
        p = ws.data_ptr()
        off = (-p) % 256
        return p + off, ws.numel() - off

    def _stream(self, device) -> int:
        if device.type == "cuda":
            return torch.cuda.current_stream(device).cuda_stream
        return 0

    def _aux_tensors(self, inputs, aux_keys, n: int, device):
        """Auxiliary data columns ([n] values) and learnable parameters (ONE value of the plan's dtype on the device)."""
        out = []
        for k in aux_keys:
            if k in self.param_keys:
                t = inputs[k]
                if t.numel() != 1:
                    raise ValueError(f"learnable parameter '{k}' must be a scalar, got shape {tuple(t.shape)}")
                t = t.detach().reshape(1)
                if t.dtype != self.dtype or t.device != device:
                    t = t.to(device=device, dtype=self.dtype)
                out.append(t.contiguous())
            else:
                out.append(_col(inputs[k], n, self.dtype, device, f"aux '{k}'"))
        return out

    def param_grad_buffer(self, device) -> Optional[torch.Tensor]:
        """fp64 [n_aux] device buffer registered with the plan: entry i ACCUMULATES dLoss/d(aux key i) for the learnable
        parameters over every loss_fwd_bwd call until the caller zeroes it (None if the plan has none)."""
        if not self.param_keys:
            return None
        if self._param_grad is None or self._param_grad.device != device:
            self._param_grad = torch.zeros(len(self.compiled.aux_keys), dtype=torch.float64, device=device)
            for i, k in enumerate(self.compiled.aux_keys):
                if k in self.param_keys:
                    rc = self.lib.lib.ppsci_b200_plan_set_aux_grad(self.handle, i, self._param_grad.data_ptr() + 8 * i)
                    self.lib.check(rc, "plan_set_aux_grad")
        return self._param_grad

    def _ptr_array(self, tensors: Sequence[Optional[torch.Tensor]], length: int):
        arr = (C.c_void_p * max(1, length))()
        for i, t in enumerate(tensors):
            arr[i] = t.data_ptr() if t is not None else None
        return arr

    def loss_fwd_bwd(
        self,
        inputs: Dict[str, torch.Tensor],
        params: torch.Tensor,
        grads: Optional[torch.Tensor],
        labels: Optional[Dict[str, torch.Tensor]] = None,
        weights: Optional[Dict[str, torch.Tensor]] = None,
        label_consts: Optional[Dict[str, float]] = None,
        n_norm: Optional[int] = None,
        residual_out: Optional[Dict[str, torch.Tensor]] = None,
    ) -> torch.Tensor:
        """Returns a tensor [n_res] of per-residual losses (device resident; no host sync)."""
        cr = self.compiled
        net = cr.net
        device = params.device
        first = inputs[net.input_keys[0]]
        n = first.numel()
        keep = []  # keep contiguous copies alive for the duration of the call
        xs = [_col(inputs[k], n, self.dtype, device, f"input '{k}'") for k in net.input_keys]
        auxs = self._aux_tensors(inputs, cr.aux_keys, n, device)
        labs: List[Optional[torch.Tensor]] = []
        wts: List[Optional[torch.Tensor]] = []
        lconst = (C.c_double * B.MAX_RES)()
        for k, name in enumerate(cr.names):
            lt = labels.get(name) if labels else None
            labs.append(_col(lt, n, self.dtype, device, f"label '{name}'") if lt is not None else None)
            lconst[k] = float(label_consts.get(name, 0.0)) if label_consts else 0.0
            wt = weights.get(name) if weights else None
            wts.append(_col(wt, n, self.dtype, device, f"weight '{name}'") if wt is not None else None)
        res = [None] * self.n_res
        if residual_out:
            for k, name in enumerate(cr.names):
                if name in residual_out:
                    res[k] = _col(residual_out[name], n, self.dtype, device, f"residual_out '{name}'")
                    if res[k].data_ptr() != residual_out[name].data_ptr():
                        raise ValueError("residual_out tensors must be contiguous")
        keep += xs + auxs + labs + wts
        if params.dtype != self.dtype or params.numel() != self.n_params or not params.is_contiguous():
            raise ValueError(f"params must be a contiguous {self.dtype} tensor with {self.n_params} elements")
        if grads is not None and (grads.dtype != self.dtype or grads.numel() != self.n_params or not grads.is_contiguous()
                                  or grads.device != device):
            raise ValueError("grads must match params in dtype/size/device and be contiguous")
        if self._loss is None or self._loss.device != device:
            self._loss = torch.zeros(B.MAX_RES, dtype=self.dtype, device=device)
        if grads is not None:
            self.param_grad_buffer(device)
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        rc = self.lib.lib.ppsci_b200_residual_loss_fwd_bwd(
            self.handle,
            self._ptr_array(xs, len(xs)),
            self._ptr_array(auxs, len(auxs)),
            self._ptr_array(labs, self.n_res),
            lconst,
            self._ptr_array(wts, self.n_res),
            n,
            int(n_norm if n_norm is not None else n),
            params.data_ptr(),
            grads.data_ptr() if grads is not None else None,
            self._loss.data_ptr(),
            self._ptr_array(res, self.n_res),
            wptr,
            wbytes,
            self._stream(device),
        )
        self.lib.check(rc, "residual_loss_fwd_bwd")
        del keep
        return self._loss[: self.n_res]

    def _inputs(self, inputs: Dict[str, torch.Tensor], device):
        """(n_points, [input tensors in column order]); a dense-input net takes ONE row-major [N, n_feat] matrix."""
        net = self.compiled.net
        if self.dense_in:
            m = inputs[net.input_keys[0]]
            if m.dim() != 2 or m.shape[1] != net.widths[0]:
                raise ValueError(f"input '{net.input_keys[0]}' must be [N, {net.widths[0]}], got {tuple(m.shape)}")
            if m.device != device:
                raise ValueError(f"input '{net.input_keys[0]}': tensor is on {m.device}, parameters are on {device}")
            return int(m.shape[0]), [m.to(self.dtype).contiguous()]
        n = inputs[net.input_keys[0]].numel()
        return n, [_col(inputs[k], n, self.dtype, device, f"input '{k}'") for k in net.input_keys]

    def values_fwd_bwd(self, inputs: Dict[str, torch.Tensor], params: torch.Tensor, grads: torch.Tensor, ybar: torch.Tensor):
        """Forward of the network values + adjoint for caller-supplied output adjoints ``ybar`` [N, n_out]
        (dL/dy); accumulates dL/d(params) into ``grads`` (``ppsci_b200_values_fwd_bwd``)."""
        cr = self.compiled
        device = params.device
        n, xs = self._inputs(inputs, device)
        auxs = self._aux_tensors(inputs, cr.aux_keys, n, device)
        if ybar.shape != (n, self.n_out) or ybar.dtype != self.dtype or ybar.device != device:
            raise ValueError(f"ybar must be [{n}, {self.n_out}] {self.dtype} on {device}")
        if grads.dtype != params.dtype or grads.numel() != params.numel() or grads.device != device or not grads.is_contiguous():
            raise ValueError("grads must match params in dtype/size/device and be contiguous")
        yb = ybar.contiguous()
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        rc = self.lib.lib.ppsci_b200_values_fwd_bwd(
            self.handle, self._ptr_array(xs, len(xs)), self._ptr_array(auxs, len(auxs)), n, params.data_ptr(),
            grads.data_ptr(), yb.data_ptr(), wptr, wbytes, self._stream(device))
        self.lib.check(rc, "values_fwd_bwd")

    @property
    def chunk_points(self) -> int:
        return int(self.lib.lib.ppsci_b200_plan_chunk_points(self.handle))

    def values_fwd_keep(self, inputs: Dict[str, torch.Tensor], params: torch.Tensor) -> torch.Tensor:
        """Forward of the network values with the adjoint's stash kept in this plan's workspace; returns y [N, n_out].
        At most ``chunk_points`` points (``ppsci_b200_values_fwd_keep``); follow with ``values_bwd_kept``."""
        device = params.device
        n, xs = self._inputs(inputs, device)
        auxs = self._aux_tensors(inputs, self.compiled.aux_keys, n, device)
        y = torch.empty((n, self.n_out), dtype=self.dtype, device=device)
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        self._kept = (xs, auxs, n)  # the same input buffers must be handed to the adjoint call
        rc = self.lib.lib.ppsci_b200_values_fwd_keep(self.handle, self._ptr_array(xs, len(xs)), self._ptr_array(auxs, len(auxs)), n,
                                                     params.data_ptr(), y.data_ptr(), wptr, wbytes, self._stream(device))
        self.lib.check(rc, "values_fwd_keep")
        self.two_phase_launches += self.last_launches
        return y

    def values_fwd_keep_inplace(self, inputs: Dict[str, torch.Tensor], params: torch.Tensor):
        """``values_fwd_keep`` without the output copy: returns (y, ybar) VIEWS [N, n_out] into this plan's workspace (the
        network outputs, and the buffer the caller's head writes the output adjoints into before ``values_bwd_kept``).
        Needs n_out % 4 == 0 (row pitch = n_out); otherwise use ``values_fwd_keep``."""
        if self.n_out % 4:
            raise ValueError("in-place outputs need n_out to be a multiple of 4")
        device = params.device
        n, xs = self._inputs(inputs, device)
        auxs = self._aux_tensors(inputs, self.compiled.aux_keys, n, device)
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        self._kept = (xs, auxs, n)
        rc = self.lib.lib.ppsci_b200_values_fwd_keep(self.handle, self._ptr_array(xs, len(xs)), self._ptr_array(auxs, len(auxs)), n,
                                                     params.data_ptr(), None, wptr, wbytes, self._stream(device))
        self.lib.check(rc, "values_fwd_keep")
        self.two_phase_launches += self.last_launches
        base = wptr - ws.data_ptr()
        es = 8 if self.dtype == torch.float64 else 4
        views = []
        for code in (len(self.compiled.net.widths) - 1, 300):  # output jets Y, output adjoints Ybar
            off = int(self.lib.lib.ppsci_b200_plan_stash_offset(self.handle, n, code))
            if off < 0:
                raise RuntimeError("plan_stash_offset failed")
            views.append(ws[base + off: base + off + n * self.n_out * es].view(self.dtype).view(n, self.n_out))
        return views[0], views[1]

    def values_bwd_kept(self, params: torch.Tensor, grads: torch.Tensor, ybar: torch.Tensor):
        """Adjoint of the most recent ``values_fwd_keep`` (its forward is NOT recomputed); accumulates into ``grads``."""
        xs, auxs, n = self._kept
        device = params.device
        if ybar.shape != (n, self.n_out) or ybar.dtype != self.dtype or ybar.device != device:
            raise ValueError(f"ybar must be [{n}, {self.n_out}] {self.dtype} on {device}")
        yb = ybar.contiguous()
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        rc = self.lib.lib.ppsci_b200_values_bwd_kept(self.handle, self._ptr_array(xs, len(xs)), self._ptr_array(auxs, len(auxs)), n,
                                                     params.data_ptr(), grads.data_ptr(), yb.data_ptr(), wptr, wbytes,
                                                     self._stream(device))
        self.lib.check(rc, "values_bwd_kept")
        self.two_phase_launches += self.last_launches
        self._kept = None

    def jets_fwd_keep(self, inputs: Dict[str, torch.Tensor], params: torch.Tensor):
        """Forward with the adjoint's stash kept (``ppsci_b200_jets_fwd_keep``, any number of jet channels, at most
        ``chunk_points`` points); the output jets stay in this plan's workspace.  Returns (address of the output jets,
        address of their adjoints, row pitch, plane stride): both [C][N][pitch] planes, the adjoints to be written by the
        caller before ``jets_bwd_kept``."""
        device = params.device
        n, xs = self._inputs(inputs, device)
        auxs = self._aux_tensors(inputs, self.compiled.aux_keys, n, device)
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        self._kept = (xs, auxs, n)
        rc = self.lib.lib.ppsci_b200_jets_fwd_keep(self.handle, self._ptr_array(xs, len(xs)), self._ptr_array(auxs, len(auxs)),
                                                   n, params.data_ptr(), wptr, wbytes, self._stream(device))
        self.lib.check(rc, "jets_fwd_keep")
        offs = [int(self.lib.lib.ppsci_b200_plan_stash_offset(self.handle, n, code))
                for code in (len(self.compiled.net.widths) - 1, 300)]
        if min(offs) < 0:
            raise RuntimeError("plan_stash_offset failed")
        ld = (self.n_out + 3) // 4 * 4
        return wptr + offs[0], wptr + offs[1], ld, n * ld

    def jets_bwd_kept(self, params: torch.Tensor, grads: torch.Tensor):
        """Adjoint of the most recent ``jets_fwd_keep`` from the output-jet adjoints the caller left in the workspace;
        accumulates into ``grads``."""
        xs, auxs, n = self._kept
        device = params.device
        if grads.dtype != params.dtype or grads.numel() != params.numel() or grads.device != device or not grads.is_contiguous():
            raise ValueError("grads must match params in dtype/size/device and be contiguous")
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        rc = self.lib.lib.ppsci_b200_jets_bwd_kept(self.handle, self._ptr_array(xs, len(xs)), self._ptr_array(auxs, len(auxs)),
                                                   n, params.data_ptr(), grads.data_ptr(), wptr, wbytes, self._stream(device))
        self.lib.check(rc, "jets_bwd_kept")
        self._kept = None

    def forward(
        self,
        inputs: Dict[str, torch.Tensor],
        params: torch.Tensor,
        want_jets: bool = False,
        want_residuals: bool = True,
    ):
        """Forward only.  Returns (jets [C, N, n_out] or None, {name: residual [N,1]})."""
        cr = self.compiled
        net = cr.net
        device = params.device
        n, xs = self._inputs(inputs, device)
        auxs = self._aux_tensors(inputs, cr.aux_keys, n, device)
        jets = torch.empty((self.channels, n, self.n_out), dtype=self.dtype, device=device) if want_jets else None
        res_t = [torch.empty((n, 1), dtype=self.dtype, device=device) for _ in range(self.n_res)] if want_residuals else []
        ws = self._workspace(n, device)
        wptr, wbytes = self._aligned(ws)
        rc = self.lib.lib.ppsci_b200_residual_fwd(
            self.handle,
            self._ptr_array(xs, len(xs)),
            self._ptr_array(auxs, len(auxs)),
            n,
            params.data_ptr(),
            jets.data_ptr() if jets is not None else None,
            self._ptr_array(res_t, self.n_res) if want_residuals else None,
            wptr,
            wbytes,
            self._stream(device),
        )
        self.lib.check(rc, "residual_fwd")
        return jets, {name: res_t[k] for k, name in enumerate(cr.names)} if want_residuals else {}
