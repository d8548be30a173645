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

import sympy as sp
import torch

from oracle import ppsci_oracle as O
from paddlescience_b200.engine.compiler import compile_residuals
from paddlescience_b200.engine.plan import ResidualPlan
from tests.cases import _ac_exprs, _biharm_exprs, _value_exprs, make_net

U32 = 2.0 ** -24  # unit roundoff of fp32

CODE_YBAR = 300  # ppsci_b200_plan_stash_offset: output adjoints
CODE_ZBAR0 = 301  # ... and the two Zbar ping-pong buffers (302 the second)


def last_chunk(plan, n: int) -> Tuple[int, int]:
    """(first point, points) of the last workspace chunk of a call over ``n`` points."""
    ch = plan.chunk_points
    x_off = (n - 1) // ch * ch
    return x_off, n - x_off


def stash_views(plan, n: int, last: bool = False,
                extra: Optional[Dict[str, Tuple[int, int]]] = None) -> Dict[str, torch.Tensor]:
    """Views [C, n, width] into ``plan``'s workspace after its most recent call, which took ``n`` points:
    "Z<l>" for every hidden layer, "Y", "Ybar", and "Zbar1" / "Zbar2" for the hidden adjoints that survive the call
    (Zbar_l was last written to buffer (L-1-l) mod 2).  Needs n <= plan.chunk_points (one workspace chunk), unless
    ``last``: then the views cover the points of the call's last chunk (``last_chunk``), which the workspace still
    holds; their weight gradients are sums over every chunk and cannot be checked from them.  ``extra``: {name:
    (stash code, width)} of more planes to view."""
    if n > plan.chunk_points and not last:
        raise ValueError(f"{n} points span more than one workspace chunk ({plan.chunk_points} points)")
    n_pts = last_chunk(plan, n)[1] if last else n
    n = min(n, plan.chunk_points)  # points per plane of the workspace
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
        return raw.view(plan.dtype).view(C, n, ld)[:, :n_pts, :width]

    out = {f"Z{l}": view(l, widths[l]) for l in range(1, L)}
    out["Y"] = view(L, widths[L])
    out["Ybar"] = view(CODE_YBAR, widths[L])
    for l in (1, 2):
        if l < L:
            out[f"Zbar{l}"] = view(CODE_ZBAR0 + (L - 1 - l) % 2, widths[l])
    for name, (code, width) in (extra or {}).items():
        out[name] = view(code, width)
    return out


def param_blocks(widths: Sequence[int]) -> List[Tuple[slice, slice, Tuple[int, int]]]:
    """(W_l slice, b_l slice, (fan-in, fan-out)) of the flat [W_1 (in, out) | b_1 | W_2 | b_2 | ...] vector, l = 1.."""
    out, off = [], 0
    for l in range(1, len(widths)):
        k, m = widths[l - 1], widths[l]
        out.append((slice(off, off + k * m), slice(off + k * m, off + k * m + m), (k, m)))
        off += k * m + m
    return out


def act_fn(name: str, beta: Optional[torch.Tensor] = None):
    """The activation as a function of z: the oracle's, or for the two with a trainable parameter (stan: tanh(z)
    (1 + beta z), swish_b: z sigmoid(beta z); ppsci/arch/activation.py:28-58) the same with ``beta`` broadcast
    against z (one value per unit, or a scalar)."""
    if name == "stan":
        return lambda x: torch.tanh(x) * (1 + beta * x)
    if name == "swish_b":
        return lambda x: x * torch.sigmoid(beta * x)
    return O.get_activation(name)


def act_coefs(name, z0: torch.Tensor, kmax: int, beta: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
    """[s_0 .. s_kmax], s_k = sigma^(k)(z0) / k!, by nested autograd on the oracle's activation (``name``, or a
    callable of z).  Differentiable with respect to z0 when z0 requires grad (the dx reference differentiates through
    them), and with respect to ``beta`` when it does."""
    f = name if callable(name) else act_fn(name, beta)
    x = z0 if z0.requires_grad else z0.detach().requires_grad_(True)
    g = f(x)
    s = [g]
    for k in range(1, kmax + 1):
        nxt = None
        if g.requires_grad:  # piecewise-linear activations: the derivative is a constant without a graph
            (nxt,) = torch.autograd.grad(g.sum(), x, create_graph=True, allow_unused=True)
        g = nxt if nxt is not None else torch.zeros_like(x)
        s.append(g / math.factorial(k))
    if not z0.requires_grad and not (beta is not None and beta.requires_grad):
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


def act_jets(name, Z: torch.Tensor, compiled, absolute: bool = False,
             beta: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Activation jets [C, n, w] of pre-activation jets Z [C, n, w] (fp64); ``absolute``: their absolute twin;
    ``beta``: the activation's trainable parameter."""
    dirs = _directions(compiled)
    kmax = max([o for o, _ in dirs], default=0)
    z0 = Z[0]
    if absolute:
        b = beta.detach() if beta is not None else None
        s = act_coefs(name, z0.detach(), kmax + 1, b)
        s = [s[k].abs() + (k + 1) * z0.abs() * s[k + 1].abs() for k in range(kmax + 1)]
    else:
        s = act_coefs(name, z0, kmax, beta)
    planes = [None] * Z.shape[0]
    planes[0] = s[0]
    for order, chans in dirs:
        z = [Z[c].abs() if absolute else Z[c] for c in chans]
        for c, y in zip(chans, _series(s, z, order)):
            planes[c] = y
    return torch.stack(planes)


def _g_deriv(kind: int, theta: torch.Tensor, j: int) -> torch.Tensor:
    """j-th derivative of cos (kind 1) or sin (kind 2) at theta."""
    ph = j + (1 if kind == 1 else 0)  # cos = sin(. + pi/2)
    return [torch.sin, torch.cos, lambda t: -torch.sin(t), lambda t: -torch.cos(t)][ph % 4](theta)


def seed_jets(compiled, X: torch.Tensor, omega: torch.Tensor, absolute: bool = False) -> torch.Tensor:
    """The first layer's operand: jets [C, n, n_feat] (fp64) of the period-embedded input features along the compiled
    Taylor directions.  X [n_in, n] holds the raw inputs, ``omega`` [n_feat] the frequency each feature reads (may
    require grad).  Coefficient k of g(omega (x + t v)), g = cos / sin, is omega^k v^k g^(k)(omega x) / k!; an
    identity feature has x on the value channel and v on coefficient 1 of each direction.  ``absolute``: the twin
    |c_k| (k + 1) + |omega x| |g^(k+1)| |omega v|^k / k! (rounding of omega x and of the powers)."""
    net = compiled.net
    C = compiled.channels
    X = X.double()
    n = X.shape[1]
    planes = [[None] * net.widths[0] for _ in range(C)]
    dirs = [(d.vec, d.order, compiled.channel_of(i, 1)) for i, d in enumerate(compiled.dirs)]
    zero = torch.zeros(n, dtype=torch.float64, device=X.device)
    for f in range(net.widths[0]):
        src, kind = net.feat_src[f], net.feat_kind[f]
        x = X[src]
        if kind == 0:
            planes[0][f] = x.abs() if absolute else x
            for vec, order, c1 in dirs:
                v = float(vec[src])
                planes[c1][f] = zero + (abs(v) if absolute else v)
                for k in range(2, order + 1):
                    planes[c1 + k - 1][f] = zero
            continue
        w = omega[f]
        th = w * x
        planes[0][f] = (_g_deriv(kind, th, 0).abs() + th.abs() * _g_deriv(kind, th, 1).abs()) if absolute else \
            _g_deriv(kind, th, 0)
        for vec, order, c1 in dirs:
            h = w * float(vec[src])
            for k in range(1, order + 1):
                if absolute:
                    y = (_g_deriv(kind, th, k).abs() * (k + 1) + th.abs() * _g_deriv(kind, th, k + 1).abs()) * \
                        abs(float(h)) ** k / math.factorial(k)
                else:
                    y = _g_deriv(kind, th, k) * h ** k / math.factorial(k)
                planes[c1 + k - 1][f] = y
    return torch.stack([torch.stack(p, dim=1) for p in planes])


def dseed_abs(compiled, X: torch.Tensor, omega: torch.Tensor) -> torch.Tensor:
    """Componentwise bound twin of d seed_jets / d omega (per feature): the product rule's terms in absolute value,
    each with the rounding of its argument, as seed_jets' twin has."""
    net = compiled.net
    X = X.double()
    out = torch.zeros(compiled.channels, X.shape[1], net.widths[0], dtype=torch.float64, device=X.device)
    dirs = [(d.vec, d.order, compiled.channel_of(i, 1)) for i, d in enumerate(compiled.dirs)]
    for f in range(net.widths[0]):
        src, kind = net.feat_src[f], net.feat_kind[f]
        if kind == 0:
            continue
        w = float(omega[f])
        x = X[src]
        th = w * x
        ga = lambda j: _g_deriv(kind, th, j).abs()  # noqa: E731
        out[0, :, f] = x.abs() * (2 * ga(1) + th.abs() * ga(2))
        for vec, order, c1 in dirs:
            v = abs(float(vec[src]))
            h = abs(w) * v
            for k in range(1, order + 1):
                t1 = x.abs() * h ** k * (ga(k + 1) * (k + 2) + th.abs() * ga(k + 2))
                t2 = k * abs(w) ** (k - 1) * v ** k * (ga(k) * (k + 2) + th.abs() * ga(k + 1))
                out[c1 + k - 1, :, f] = (t1 + t2) / math.factorial(k)
    return out


def _cw_err(out: torch.Tensor, ref: torch.Tensor, ref_abs: torch.Tensor) -> float:
    """max |out - ref| / ref_abs; an element with ref_abs == 0 must be exact."""
    d = (out.double() - ref).abs()
    r = torch.where(ref_abs > 0, d / ref_abs.clamp_min(1e-300), torch.where(d > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def layer_errors(compiled, act: Optional[str], A_in: torch.Tensor, W: torch.Tensor, b: torch.Tensor, *,
                 out: Optional[torch.Tensor] = None, zbar: Optional[torch.Tensor] = None,
                 zbar_prev: Optional[torch.Tensor] = None, dw: Optional[torch.Tensor] = None,
                 db: Optional[torch.Tensor] = None, seed: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                 A_abs: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None,
                 block: int = 8192) -> Dict[str, float]:
    """Errors of the kernels of one linear layer l against the fp64 reference on the engine's own inputs.

    compiled   the plan's CompiledResidual (Taylor directions, channel map)
    act        activation applied to A_in (the activation of layer l - 1's output); None: A_in is the dense first
               layer's operand, a [n, K] matrix used as is (one channel), or with ``A_abs`` the operand's jets
    A_in       Z_{l-1} [C, n, K] as the engine stored it
    A_abs      with act None: A_in is an fp64 operand [C, n, K] (the seeds' jets) and A_abs its absolute twin
    beta       the activation's trainable parameter (per unit [K], or a scalar)
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
        if act is None and A_abs is not None:
            Z = None
            A, Aa = A_in[:, sl].double(), A_abs[:, sl]
        elif act is None:
            Z = None
            A = A_in[sl].double().unsqueeze(0)
            Aa = A.abs()
        else:
            Z = A_in[:, sl].double().detach().requires_grad_(want_dx)
            A = act_jets(act, Z, compiled, beta=beta)
            Aa = act_jets(act, Z.detach(), compiled, absolute=True, beta=beta)
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


def actp_offsets(net) -> Dict[int, Tuple[int, int]]:
    """{hidden layer l: (offset, count)} of the trainable activation parameters in the flat vector of an ungated MLP:
    behind the linear layers, one per unit (stan) or per layer (swish_b), then the n_omega frequencies."""
    off = sum(sl.stop - sl.start for blk in param_blocks(net.widths) for sl in blk[:2])
    out = {}
    for l in range(1, len(net.widths) - 1):
        a = net.act_first if (l == 1 and net.act_first) else net.act
        if a in ("stan", "swish_b"):
            cnt = net.widths[l] if a == "stan" else 1
            out[l] = (off, cnt)
            off += cnt
    return out


def omega_offset(net) -> int:
    """Offset of the n_omega trainable frequencies: the last entries of the flat vector."""
    return net.n_params - (net.n_omega or 0)


def feature_omegas(plan, params: torch.Tensor) -> torch.Tensor:
    """[n_feat] frequency each feature reads, as the kernels do: the trainable entry of ``params``, or the fixed
    frequency rounded to the plan's dtype."""
    net = plan.compiled.net
    idx = net.feat_omega_param or [-1] * net.widths[0]
    o0 = omega_offset(net)
    fixed = torch.tensor(net.feat_omega, dtype=plan.dtype).double().to(params.device)
    return torch.stack([params[o0 + j].double() if j >= 0 else fixed[f] for f, j in enumerate(idx)])


def _beta(plan, params: torch.Tensor, l: int) -> Optional[torch.Tensor]:
    """The trainable parameter of hidden layer l's activation, shaped to broadcast against [n, width]."""
    ap = actp_offsets(plan.compiled.net).get(l)
    if ap is None:
        return None
    return params[ap[0]: ap[0] + ap[1]].double()


def check_layer(plan, views: Dict[str, torch.Tensor], params: torch.Tensor, grads: torch.Tensor, l: int, kinds,
                seed: Optional[torch.Tensor] = None, x_dense: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """``layer_errors`` for layer l of an ungated plan after a call (``views`` from ``stash_views``): kinds among
    "fwd" (Z_l, or Y for the output layer), "dx" (Zbar_{l-1}) and "dw" (dW_l and db_l of ``grads``, which
    accumulated onto ``seed`` if given).  Layer 1 as a dense first layer, whose operand ``x_dense`` is the caller's
    [n, n_feat] matrix, or from the input seeds, whose raw inputs ``run_fused`` leaves in views["X"]."""
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
    W, b = params[w_sl].view(K, N), params[b_sl]
    if l == 1 and x_dense is not None:
        return layer_errors(plan.compiled, None, x_dense, W, b, **kw)
    if l == 1:
        om = feature_omegas(plan, params)
        A = seed_jets(plan.compiled, views["X"], om)
        return layer_errors(plan.compiled, None, A, W, b, A_abs=seed_jets(plan.compiled, views["X"], om, True), **kw)
    act = net.act_first if (l == 2 and net.act_first) else net.act  # the activation of layer l - 1's output
    return layer_errors(plan.compiled, act, views[f"Z{l - 1}"], W, b, beta=_beta(plan, params, l - 1), **kw)


def omega_errors(plan, views: Dict[str, torch.Tensor], params: torch.Tensor, grads: torch.Tensor,
                 seed: Optional[torch.Tensor] = None,
                 consumers: Optional[Sequence[Tuple[torch.Tensor, torch.Tensor]]] = None) -> float:
    """dLoss/d omega of the trainable frequencies against fp64 autograd through omega of ``seed_jets``, contracted
    with the engine's Zbar_1 W_1^T:  sum_{c,p,f} d seed_c[p][f] / d omega_j  (Zbar_1 W_1^T)[c][p][f].  Componentwise:
    the error over the same contraction on absolute values (``dseed_abs`` |Zbar_1| |W_1|^T) plus |seed|.
    ``consumers``: the (Zbar, W) pairs of every GEMM that read the seeds, when there are more than layer 1's."""
    net = plan.compiled.net
    if consumers is None:
        w_sl, _, (K, N) = param_blocks(net.widths)[0]
        consumers = [(views["Zbar1"], params[w_sl].view(K, N))]
    om_f = feature_omegas(plan, params).detach()
    idx = net.feat_omega_param
    o0 = omega_offset(net)
    om = params[o0: o0 + net.n_omega].double().detach().requires_grad_(True)
    om_feat = torch.stack([om[j] if j >= 0 else om_f[f] for f, j in enumerate(idx)])
    A = seed_jets(plan.compiled, views["X"], om_feat)
    D = sum(zb.double() @ W.double().T for zb, W in consumers)
    Da = sum(zb.double().abs() @ W.double().abs().T for zb, W in consumers)
    (ref,) = torch.autograd.grad((A * D).sum(), om)
    per_feat = (dseed_abs(plan.compiled, views["X"], om_f) * Da).sum((0, 1))
    bound = torch.zeros_like(ref)
    for f, j in enumerate(idx):
        if j >= 0:
            bound[j] += per_feat[f]
    got = grads[o0: o0 + net.n_omega].double()
    if seed is not None:
        s = seed[o0: o0 + net.n_omega].double()
        got, bound = got - s, bound + s.abs()
    return _cw_err(got, ref, bound)


def beta_errors(plan, views: Dict[str, torch.Tensor], params: torch.Tensor, grads: torch.Tensor, l: int,
                seed: Optional[torch.Tensor] = None) -> float:
    """dLoss/d beta of hidden layer l's activation (stan: per unit, swish_b: per layer), which the dx epilogue of
    layer l + 1 reduces, against fp64 autograd through beta of ``act_jets`` contracted with the engine's
    Zbar_{l+1} W_{l+1}^T.  Componentwise: over the absolute twin of the jets of d act / d beta contracted with
    |Zbar_{l+1}| |W_{l+1}|^T, plus |seed|."""
    net = plan.compiled.net
    L = len(net.widths) - 1
    off, cnt = actp_offsets(net)[l]
    w_sl, _, (K, N) = param_blocks(net.widths)[l]
    W = params[w_sl].view(K, N).double()
    zb = (views[f"Zbar{l + 1}"] if l + 1 < L else views["Ybar"]).double()
    Z = views[f"Z{l}"].double()
    act = net.act_first if (l == 1 and net.act_first) else net.act
    beta = params[off: off + cnt].double().detach().requires_grad_(True)
    A = act_jets(act, Z, plan.compiled, beta=beta)
    (ref,) = torch.autograd.grad((A * (zb @ W.T)).sum(), beta)
    # d act / d beta elementwise, as a function of z (the double-backward of a full-shape beta)
    b_full = beta.detach().expand(Z.shape[1], Z.shape[2]).clone().requires_grad_(True)

    def dact(x):
        (d,) = torch.autograd.grad(act_fn(act, b_full)(x).sum(), b_full, create_graph=True)
        return d

    Da = act_jets(dact, Z.detach(), plan.compiled, absolute=True)
    bound = (Da * (zb.abs() @ W.abs().T)).sum((0, 1))
    if cnt == 1:
        bound = bound.sum().reshape(1)
    got = grads[off: off + cnt].double()
    if seed is not None:
        s = seed[off: off + cnt].double()
        got, bound = got - s, bound + s.abs()
    return _cw_err(got, ref.detach(), bound)


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


def _sym(names):
    return sp.symbols(names)


def _one_dir(order):
    def exprs():
        x = sp.Symbol("x")
        u = sp.Function("u")(x)
        return {"r": u.diff(x, order) + u * u - sp.sin(x)}
    return exprs


def _div2():
    x, y = _sym("x y")
    u, v = sp.Function("u")(x, y), sp.Function("v")(x, y)
    return {"div": u.diff(x) + v.diff(y), "adv": u * v.diff(x) - y}


def _div3():
    x, y, z = _sym("x y z")
    u = sp.Function("u")(x, y, z)
    return {"r": u.diff(x) + u.diff(y) * u + u.diff(z) - x * z}


def _heat3():
    t, x, y, z = _sym("t x y z")
    u = sp.Function("u")(t, x, y, z)
    return {"heat": u.diff(t) - 0.1 * (u.diff(x, 2) + u.diff(y, 2) + u.diff(z, 2)) + u ** 2}


def _five_inputs():
    x, y, z, s_, t = _sym("x y z s t")
    u = sp.Function("u")(x, y, z, s_, t)
    return {"r": u.diff(x, 2) + u.diff(y) + u.diff(t) * u - z * s_}


def _biharm3(extra_order):
    def exprs():
        x, y, z, w = _sym("x y z w")
        ins = (x, y, z, w) if extra_order else (x, y, z)
        u = sp.Function("u")(*ins)
        r = u.diff(x, 4) + u.diff(y, 4) + u.diff(z, 4) + 2 * u.diff(x, 2, y, 2) + 2 * u.diff(y, 2, z, 2) - sp.sin(x)
        if extra_order:
            r = r + u.diff(w, extra_order)
        return {"bh": r}
    return exprs


def runtime_layouts():
    """Equations whose compiled jet layout is none of the compile-time ones: the CUDA-core and generic thin kernels
    serve them through the run-time layout, at channel counts that do not divide 128 and up to C = 32 (TP = 4,
    PT = 1).  Keyed by the directions' orders."""
    return {
        "O1": dict(in_keys=("x",), out_keys=("u",), exprs=_one_dir(1), C=2),
        "O2": dict(in_keys=("x",), out_keys=("u",), exprs=_one_dir(2), C=3),
        "O3": dict(in_keys=("x",), out_keys=("u",), exprs=_one_dir(3), C=4),
        "O4": dict(in_keys=("x",), out_keys=("u",), exprs=_one_dir(4), C=5),
        "O11": dict(in_keys=("x", "y"), out_keys=("u", "v"), exprs=_div2, C=3),
        "O111": dict(in_keys=("x", "y", "z"), out_keys=("u",), exprs=_div3, C=4),
        "O1222": dict(in_keys=("t", "x", "y", "z"), out_keys=("u",), exprs=_heat3, C=8),
        "O211": dict(in_keys=("x", "y", "z", "s", "t"), out_keys=("u",), exprs=_five_inputs, C=5),
        "O4x7": dict(in_keys=("x", "y", "z"), out_keys=("u",), exprs=_biharm3(0), C=29),
        "O4x7_3": dict(in_keys=("x", "y", "z", "w"), out_keys=("u",), exprs=_biharm3(3), C=32),
    }


def all_layouts():
    return {**layouts(), **runtime_layouts()}


def run_fused(layout: str, hidden: Sequence[int], n: int, *, dtype=torch.float32, act: str = "tanh",
              act_first: Optional[str] = None, backend: int = 2, library=None, device="cuda:0", seed: int = 0,
              grads0: Optional[torch.Tensor] = None, periods: Optional[Dict[str, Tuple[float, bool]]] = None,
              chunk_points: int = 0, out_keys: Optional[Sequence[str]] = None):
    """One fused loss_fwd_bwd of an MLP with the given hidden widths on the layout's equation (seeded inputs and
    parameters; ``grads0``: the gradient buffer's initial value, zero by default).  ``periods``: {input key: (period,
    trainable)} embeds that input as cos / sin features (PeriodEmbedding), trainable frequencies 1.1 times their
    initial value; ``out_keys``: more network outputs than the equation reads (the output layer's width);
    ``chunk_points``: the plan's workspace chunk (the views then cover the last chunk).  Returns (plan, params, grads,
    views), views["X"] the raw inputs [n_in, n] of the viewed points."""
    spec = all_layouts()[layout]
    torch.manual_seed(seed)
    net = make_net(spec["in_keys"], tuple(out_keys or spec["out_keys"]), hidden, act, periods)
    net.act_first = act_first
    if periods and any(t for _, t in periods.values()):
        keys = [k for k, (_, t) in periods.items() if t]
        net.feat_omega_param = [keys.index(net.input_keys[s]) if (kind and net.input_keys[s] in keys) else -1
                                for s, kind in zip(net.feat_src, net.feat_kind)]
        net.n_omega = len(keys)
    exprs = spec["exprs"]()
    syms = sp.symbols(spec["in_keys"])
    for k in net.output_keys[len(spec["out_keys"]):]:  # outputs the equation does not read: one value residual each
        exprs[f"val_{k}"] = sp.Function(k)(*syms)
    cr = compile_residuals(net, exprs)
    assert cr.channels == spec["C"], (layout, cr.channels)
    nres = len(cr.names)
    plan = ResidualPlan(cr, dtype, ["mean"] * nres, [1.0 + 0.5 * k for k in range(nres)], backend=backend,
                        library=library, chunk_points=chunk_points)
    params = O.xavier_uniform_params(net.widths, 1, torch.float64)
    params = params + 0.1 * torch.randn_like(params)
    extra = [1.0 + 0.1 * torch.randn(cnt, dtype=torch.float64) for _, cnt in actp_offsets(net).values()]
    if net.n_omega:
        keys = [k for k, (_, t) in periods.items() if t]
        extra.append(torch.tensor([1.1 * 2 * math.pi / periods[k][0] for k in keys], dtype=torch.float64))
    params = torch.cat([params] + extra).to(dtype)
    assert params.numel() == plan.n_params, (params.numel(), plan.n_params)
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
    last = n > plan.chunk_points
    plan.views_last_chunk = last  # the views cover the last of several chunks: no weight gradients (all_errors)
    views = stash_views(plan, n, last=last)
    x_off, n_last = last_chunk(plan, n) if last else (0, n)
    views["X"] = torch.stack([inputs[k].view(-1)[x_off: x_off + n_last] for k in spec["in_keys"]]).to(dev)
    return plan, params, grads, views


def all_errors(plan, params: torch.Tensor, grads: torch.Tensor, views: Dict[str, torch.Tensor],
               seed: Optional[torch.Tensor] = None, chunked: Optional[bool] = None) -> Dict[str, float]:
    """Every check of an ungated plan with L = 3 linear layers after one call, keyed "<pass><layer>" (fwd1, dw1,
    db1, fwd2, dx2, dw2, db2, fwd3, dx3, dw3, db3), "omega" and "beta<l>"; ``chunked``: the views cover the last of
    several chunks (forward and dx only; by default as ``run_fused`` left them).  Raw relative errors."""
    if chunked is None:
        chunked = getattr(plan, "views_last_chunk", False)
    L = len(plan.compiled.net.widths) - 1
    assert L == 3, "Zbar_1 survives the call beside Zbar_2 only for L = 3"
    e = {}
    for l in range(1, L + 1):
        kinds = {"fwd"} | ({"dx"} if l >= 2 else set()) | (set() if chunked else {"dw"})
        for k, v in check_layer(plan, views, params, grads, l, kinds, seed=seed).items():
            e[f"{k}{l}"] = v
    if chunked:
        return e
    if plan.compiled.net.n_omega:
        e["omega"] = omega_errors(plan, views, params, grads, seed=seed)
    for l in actp_offsets(plan.compiled.net):
        e[f"beta{l}"] = beta_errors(plan, views, params, grads, l, seed=seed)
    return e


THIN_LAYS = {(2, 2), (1, 2), (2, 2, 2), ()}  # ThinLays of jet_layout.cuh, by the directions' orders
THIN_MAXF, THIN_MAXM, THIN_MAXCM = 8, 8, 64  # kernels_simt.cuh


def thin_kernels(plan, env: Optional[Dict[str, str]] = None) -> Dict[str, str]:
    """The kernels that run the first layer's forward / weight gradient / dLoss/d omega and the last layer's forward /
    backward of an ungated MLP plan, restating engine.cu: thin_first / thin_last / thin_vec of plan_create and the
    N % 4, K % 4 and m <= 4 conditions at the launch sites.  ``env``: PPSCI_B200_NO_THIN / NO_THINV as set at
    plan creation."""
    env = env or {}
    net = plan.compiled.net
    w = net.widths
    L = len(w) - 1
    C = plan.channels
    thin_on = "PPSCI_B200_NO_THIN" not in env
    first = thin_on and L >= 2 and w[0] <= THIN_MAXF
    last = thin_on and L >= 2 and w[L] <= THIN_MAXM and C * w[L] <= THIN_MAXCM and net.act not in ("stan", "swish_b")
    vec = plan.dtype == torch.float32 and tuple(d.order for d in plan.compiled.dirs) in THIN_LAYS and \
        "PPSCI_B200_NO_THINV" not in env
    out = {}
    if first:
        v = vec and w[1] % 4 == 0
        out["first_fwd"] = "k_first_fwd_v" if v else "k_first_fwd"
        out["first_dw"] = "k_first_dw_v" if v else "k_first_dw"
        if net.n_omega:
            out["omega"] = out["first_dw"] + "<OMEGA>"
    else:
        out["first_fwd"], out["first_dw"] = "k_gemm_fwd", "k_gemm_dw"
        if net.n_omega:
            out["omega"] = "k_omega_grad"
    if last:
        v = vec and w[L - 1] % 4 == 0 and w[L] <= 4
        out["last_fwd"] = "k_last_fwd_v" if v else "k_last_fwd"
        out["last_bwd"] = "k_last_bwd_v" if v else "k_last_bwd"
    else:
        out["last_fwd"], out["last_bwd"] = "k_gemm_fwd", "k_gemm_dx+k_gemm_dw"
    return out


# the three implementations of a thin first / last layer: by default, without the vectorised kernels, on the tile GEMMs
THIN_MODES = {"default": {}, "no_thinv": {"PPSCI_B200_NO_THINV": "1"}, "no_thin": {"PPSCI_B200_NO_THIN": "1"}}
