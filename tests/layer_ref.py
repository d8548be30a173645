"""Test helper: an fp64 reference of one linear layer's kernels, evaluated on the exact inputs those kernels read.

After a fused call the plan's workspace still holds the pre-activation jets Z_l of every hidden layer, the output jets
Y, the output adjoints Ybar and the two Zbar ping-pong buffers, which after the adjoint hold Zbar_1 and Zbar_2
(``ppsci_b200_plan_stash_offset``, codes l, n_layers, 300, 301 and 302).  From them each of a layer's three GEMM-shaped
kernels can be recomputed in fp64 on the fp32 values it read, so that a comparison measures that kernel's error alone:

* forward of layer l:  Z_l = act_jets(Z_{l-1}) W_l (+ b_l on channel 0);
* dx through layer l:  Zbar_{l-1} = the vector-Jacobian product of Z_{l-1} -> act_jets(Z_{l-1}) with cotangent
  Zbar_l W_l^T;
* weight gradient:     dW_l = sum over channels and points of act_jets(Z_{l-1})^T Zbar_l,  db_l = sum_p Zbar_l[0].

The activation jets are derived here independently of the kernels' closed-form coefficients: s_k = sigma^(k)(z0) / k!
by nested autograd on the oracle's activation, then the truncated power series  sum_k s_k delta(t)^k  with
delta(t) = sum_j z_j t^j  per Taylor direction.

Errors of the GEMM-shaped outputs (forward, dW, db) are componentwise: max |out - ref| / ref_abs, where ref_abs is the
same contraction carried out on absolute values (|A| |W| + |b|, ...).  The absolute twin of the activation jets uses
|s_k| + (k + 1) |z0| |s_{k+1}| (the change of s_k under a relative perturbation of its argument, so that an fp32
evaluation of sin(30 z) at large z is not mistaken for a GEMM error) and |z_j| in the series.  Divided by 2^-24 this
is the error in units of the fp32 rounding of each output's own terms: insensitive to cancellation, and a single wrong
element shows.  The dx error is taken per output channel plane, normalised by that plane's largest |ref|.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from oracle import ppsci_oracle as O
from paddlescience_b200.engine.compiler import compile_residuals
from paddlescience_b200.engine.plan import ResidualPlan
from tests.cases import _ac_exprs, _biharm_exprs, _value_exprs, make_net

U32 = 2.0 ** -24  # unit roundoff of fp32

CODE_YBAR = 300  # ppsci_b200_plan_stash_offset: output adjoints
CODE_ZBAR0 = 301  # ... and the two Zbar ping-pong buffers (302 the second)


def stash_views(plan, n: int) -> Dict[str, torch.Tensor]:
    """Views [C, n, width] into ``plan``'s workspace after its most recent call, which took ``n`` points:
    "Z<l>" for every hidden layer, "Y", "Ybar", and "Zbar1" / "Zbar2" for the hidden adjoints that survive the call
    (Zbar_l was last written to buffer (L-1-l) mod 2).  Needs n <= plan.chunk_points (one workspace chunk)."""
    if n > plan.chunk_points:
        raise ValueError(f"{n} points span more than one workspace chunk ({plan.chunk_points} points)")
    ws = plan._ws
    wptr, _ = plan._aligned(ws)
    base = wptr - ws.data_ptr()
    es = 8 if plan.dtype == torch.float64 else 4
    C = plan.channels
    widths = plan.compiled.net.widths
    L = len(widths) - 1

    def view(code: int, width: int) -> torch.Tensor:
        off = int(plan.lib.lib.ppsci_b200_plan_stash_offset(plan.handle, n, code))
        if off < 0:
            raise RuntimeError(f"plan_stash_offset({code}) failed")
        ld = (width + 3) // 4 * 4
        raw = ws[base + off: base + off + C * n * ld * es]
        return raw.view(plan.dtype).view(C, n, ld)[:, :, :width]

    out = {f"Z{l}": view(l, widths[l]) for l in range(1, L)}
    out["Y"] = view(L, widths[L])
    out["Ybar"] = view(CODE_YBAR, widths[L])
    for l in (1, 2):
        if l < L:
            out[f"Zbar{l}"] = view(CODE_ZBAR0 + (L - 1 - l) % 2, widths[l])
    return out


def param_blocks(widths: Sequence[int]) -> List[Tuple[slice, slice, Tuple[int, int]]]:
    """(W_l slice, b_l slice, (fan-in, fan-out)) of the flat [W_1 (in, out) | b_1 | W_2 | b_2 | ...] vector, l = 1.."""
    out, off = [], 0
    for l in range(1, len(widths)):
        k, m = widths[l - 1], widths[l]
        out.append((slice(off, off + k * m), slice(off + k * m, off + k * m + m), (k, m)))
        off += k * m + m
    return out


def act_coefs(name: str, z0: torch.Tensor, kmax: int) -> List[torch.Tensor]:
    """[s_0 .. s_kmax], s_k = sigma^(k)(z0) / k!, by nested autograd on the oracle's activation.  Differentiable with
    respect to z0 when z0 requires grad (the dx reference differentiates through them)."""
    f = O.get_activation(name)
    x = z0 if z0.requires_grad else z0.detach().requires_grad_(True)
    g = f(x)
    s = [g]
    for k in range(1, kmax + 1):
        nxt = None
        if g.requires_grad:  # piecewise-linear activations: the derivative is a constant without a graph
            (nxt,) = torch.autograd.grad(g.sum(), x, create_graph=True, allow_unused=True)
        g = nxt if nxt is not None else torch.zeros_like(x)
        s.append(g / math.factorial(k))
    if not z0.requires_grad:
        s = [v.detach() for v in s]
    return s


def _directions(compiled) -> List[Tuple[int, List[int]]]:
    """(order, [channel of coefficient 1 .. order]) per Taylor direction; channel 0 is shared by all of them."""
    return [(d.order, [compiled.channel_of(i, k) for k in range(1, d.order + 1)]) for i, d in enumerate(compiled.dirs)]


def _series(s: Sequence[torch.Tensor], z: Sequence[torch.Tensor], order: int) -> List[torch.Tensor]:
    """Coefficients 1..order of sum_k s_k delta(t)^k, delta(t) = sum_j z[j-1] t^j (truncated at t^order)."""
    delta = [None] + list(z)  # delta[m]: coefficient of t^m (no constant term)
    power = delta  # delta^k
    out = [s[1] * delta[m] for m in range(1, order + 1)]
    for k in range(2, order + 1):
        # delta^k has no term below t^k
        power = [None] * k + [sum(power[i] * delta[m - i] for i in range(k - 1, m)) for m in range(k, order + 1)]
        for m in range(k, order + 1):
            out[m - 1] = out[m - 1] + s[k] * power[m]
    return out


def act_jets(name: str, Z: torch.Tensor, compiled, absolute: bool = False) -> torch.Tensor:
    """Activation jets [C, n, w] of pre-activation jets Z [C, n, w] (fp64); ``absolute``: their absolute twin."""
    dirs = _directions(compiled)
    kmax = max([o for o, _ in dirs], default=0)
    z0 = Z[0]
    if absolute:
        s = act_coefs(name, z0.detach(), kmax + 1)
        s = [s[k].abs() + (k + 1) * z0.abs() * s[k + 1].abs() for k in range(kmax + 1)]
    else:
        s = act_coefs(name, z0, kmax)
    planes = [None] * Z.shape[0]
    planes[0] = s[0]
    for order, chans in dirs:
        z = [Z[c].abs() if absolute else Z[c] for c in chans]
        for c, y in zip(chans, _series(s, z, order)):
            planes[c] = y
    return torch.stack(planes)


def _cw_err(out: torch.Tensor, ref: torch.Tensor, ref_abs: torch.Tensor) -> float:
    """max |out - ref| / ref_abs; an element with ref_abs == 0 must be exact."""
    d = (out.double() - ref).abs()
    r = torch.where(ref_abs > 0, d / ref_abs.clamp_min(1e-300), torch.where(d > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def layer_errors(compiled, act: Optional[str], A_in: torch.Tensor, W: torch.Tensor, b: torch.Tensor, *,
                 out: Optional[torch.Tensor] = None, zbar: Optional[torch.Tensor] = None,
                 zbar_prev: Optional[torch.Tensor] = None, dw: Optional[torch.Tensor] = None,
                 db: Optional[torch.Tensor] = None, seed: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                 block: int = 8192) -> Dict[str, float]:
    """Errors of the kernels of one linear layer l against the fp64 reference on the engine's own inputs.

    compiled   the plan's CompiledResidual (Taylor directions, channel map)
    act        activation applied to A_in (the activation of layer l - 1's output); None: A_in is the dense first
               layer's operand, a [n, K] matrix used as is (one channel)
    A_in       Z_{l-1} [C, n, K] as the engine stored it
    W, b       the layer's parameters, [K, N] and [N]
    out        the engine's Z_l (or Y) [C, n, N]                      -> "fwd"
    zbar       the engine's Zbar_l (or Ybar) [C, n, N]: the input of the dx and dW
    zbar_prev  the engine's Zbar_{l-1} [C, n, K]                      -> "dx" (needs zbar)
    dw, db     the engine's gradient blocks [K, N] and [N]            -> "dw", "db" (need zbar)
    seed       (dW_0, db_0): the gradient the call accumulated onto; dw / db must then be the whole blocks, and
               |seed| joins ref_abs (the rounding of the accumulation)
    Returns raw relative errors (divide by U32 for units of the fp32 rounding)."""
    dev = A_in.device
    W64, b64 = W.double().to(dev), b.double().to(dev)
    Wa, ba = W64.abs(), b64.abs()
    n = A_in.shape[-2]
    K, N = W64.shape
    res: Dict[str, float] = {}
    want_dx = zbar_prev is not None
    dW = torch.zeros(K, N, dtype=torch.float64, device=dev) if dw is not None else None
    dWa = torch.zeros_like(dW) if dw is not None else None
    dx_num = dx_den = None
    fwd_err = 0.0
    for p0 in range(0, n, block):
        sl = slice(p0, min(n, p0 + block))
        if act is None:
            Z = None
            A = A_in[sl].double().unsqueeze(0)
            Aa = A.abs()
        else:
            Z = A_in[:, sl].double().detach().requires_grad_(want_dx)
            A = act_jets(act, Z, compiled)
            Aa = act_jets(act, Z.detach(), compiled, absolute=True)
        if out is not None:
            ref = A.detach() @ W64
            ref[0] += b64
            ref_abs = Aa @ Wa
            ref_abs[0] += ba
            fwd_err = max(fwd_err, _cw_err(out[:, sl], ref, ref_abs))
        if zbar is None:
            continue
        zb = zbar[:, sl].double()
        if dW is not None:
            dW += A.detach().flatten(0, 1).T @ zb.flatten(0, 1)
            dWa += Aa.flatten(0, 1).T @ zb.abs().flatten(0, 1)
        if want_dx:
            (g,) = torch.autograd.grad(A, Z, grad_outputs=zb @ W64.T)
            e = (zbar_prev[:, sl].double() - g).abs().flatten(1).amax(1)
            m = g.abs().flatten(1).amax(1)
            dx_num = e if dx_num is None else torch.maximum(dx_num, e)
            dx_den = m if dx_den is None else torch.maximum(dx_den, m)
    if out is not None:
        res["fwd"] = fwd_err
    if want_dx:
        res["dx"] = float((dx_num / dx_den.clamp_min(1e-300)).max())
    if dw is not None:
        s_w = seed[0].double().to(dev) if seed is not None else 0.0
        ra = dWa + (s_w.abs() if seed is not None else 0.0)
        res["dw"] = _cw_err(dw.double() - s_w, dW, ra)
    if db is not None:
        zb0 = zbar[0].double()
        s_b = seed[1].double().to(dev) if seed is not None else 0.0
        ra = zb0.abs().sum(0) + (s_b.abs() if seed is not None else 0.0)
        res["db"] = _cw_err(db.double() - s_b, zb0.sum(0), ra)
    return res


def check_layer(plan, views: Dict[str, torch.Tensor], params: torch.Tensor, grads: torch.Tensor, l: int, kinds,
                seed: Optional[torch.Tensor] = None, x_dense: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """``layer_errors`` for layer l of an ungated plan after a call (``views`` from ``stash_views``): kinds among
    "fwd" (Z_l, or Y for the output layer), "dx" (Zbar_{l-1}) and "dw" (dW_l and db_l of ``grads``, which
    accumulated onto ``seed`` if given).  Layer 1 only as a dense first layer, whose operand ``x_dense`` is the
    caller's [n, n_feat] matrix."""
    net = plan.compiled.net
    L = len(net.widths) - 1
    w_sl, b_sl, (K, N) = param_blocks(net.widths)[l - 1]
    kw = {}
    if "fwd" in kinds:
        kw["out"] = views[f"Z{l}"] if l < L else views["Y"]
    if "dx" in kinds or "dw" in kinds:
        kw["zbar"] = views[f"Zbar{l}"] if l < L else views["Ybar"]
    if "dx" in kinds:
        kw["zbar_prev"] = views[f"Zbar{l - 1}"]
    if "dw" in kinds:
        kw["dw"] = grads[w_sl].view(K, N)
        kw["db"] = grads[b_sl]
        if seed is not None:
            kw["seed"] = (seed[w_sl].view(K, N), seed[b_sl])
    if l == 1:
        return layer_errors(plan.compiled, None, x_dense, params[w_sl].view(K, N), params[b_sl], **kw)
    act = net.act_first if (l == 2 and net.act_first) else net.act  # the activation of layer l - 1's output
    return layer_errors(plan.compiled, act, views[f"Z{l - 1}"], params[w_sl].view(K, N), params[b_sl], **kw)


# One equation per compile-time jet layout of the kernels: (input keys, output keys, residual expressions, C, input
# ranges, random labels).  Channels C = 1 + the sum of the Taylor directions' orders.
def _ns2():
    return O.navier_stokes_expr(0.01, 1.0, 2, False)


def _ns3():
    return O.navier_stokes_expr(0.05, 1.0, 3, False)


def layouts():
    return {
        "LayV": dict(in_keys=("x", "y"), out_keys=("u", "v"), exprs=_value_exprs, C=1, labels_rand=True),
        "Lay12": dict(in_keys=("t", "x"), out_keys=("u",), exprs=_ac_exprs, C=4, ranges={"x": (-1, 1)}),
        "Lay22": dict(in_keys=("x", "y"), out_keys=("u", "v", "p"), exprs=_ns2, C=5),
        "Lay222": dict(in_keys=("x", "y", "z"), out_keys=("u", "v", "w", "p"), exprs=_ns3, C=7),
        "Lay4444": dict(in_keys=("x", "y"), out_keys=("u",), exprs=_biharm_exprs, C=17, ranges={"x": (0, 2), "y": (0, 3)}),
    }


def run_fused(layout: str, hidden: Sequence[int], n: int, *, dtype=torch.float32, act: str = "tanh",
              act_first: Optional[str] = None, backend: int = 2, library=None, device="cuda:0", seed: int = 0,
              grads0: Optional[torch.Tensor] = None):
    """One fused loss_fwd_bwd of an MLP with the given hidden widths on the layout's equation (seeded inputs and
    parameters; ``grads0``: the gradient buffer's initial value, zero by default).  Returns (plan, params, grads, views)."""
    spec = layouts()[layout]
    torch.manual_seed(seed)
    net = make_net(spec["in_keys"], spec["out_keys"], hidden, act)
    net.act_first = act_first
    cr = compile_residuals(net, spec["exprs"]())
    assert cr.channels == spec["C"], (layout, cr.channels)
    nres = len(cr.names)
    plan = ResidualPlan(cr, dtype, ["mean"] * nres, [1.0 + 0.5 * k for k in range(nres)], backend=backend,
                        library=library)
    params = O.xavier_uniform_params(net.widths, 1, torch.float64)
    params = (params + 0.1 * torch.randn_like(params)).to(dtype)
    inputs = {}
    for k in spec["in_keys"]:
        lo, hi = spec.get("ranges", {}).get(k, (0, 1))
        inputs[k] = (torch.rand(n, 1, dtype=torch.float64) * (hi - lo) + lo).to(dtype)
    labels = {k: (torch.randn(n, 1, dtype=torch.float64).to(dtype) if spec.get("labels_rand") else
                  torch.zeros(n, 1, dtype=dtype)) for k in cr.names}
    dev = torch.device(device)
    params = params.to(dev)
    grads = grads0.clone().to(dev) if grads0 is not None else torch.zeros_like(params)
    plan.loss_fwd_bwd({k: v.to(dev) for k, v in inputs.items()}, params, grads,
                      labels={k: v.to(dev) for k, v in labels.items()})
    return plan, params, grads, stash_views(plan, n)
